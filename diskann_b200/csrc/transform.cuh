// transform.cuh — the host-side transform object behind dab_transform_* (transform_kernels.cu) and the launch the
// MinMax entry points of minmax_kernels.cu run in front of the quantizer.
#pragma once

#include <vector>

#include "dab_common.cuh"

// PaddingHadamard / DoubleHadamard (diskann-quantization/src/algorithms/transforms): validated parts, host memory only
struct dab_transform {
    int kind = 0;
    uint32_t input_dim = 0;   // len(signs0)
    uint32_t inner_dim = 0;   // padded_dim / len(signs1): the length of the vector the Hadamard transforms run on
    uint32_t output_dim = 0;  // len(subsample), or inner_dim
    std::vector<uint32_t> signs0, signs1;  // 0 or 0x8000_0000: the sign flip is an xor of the float's bits
    std::vector<uint32_t> subsample;       // sorted indices into the inner vector
    bool subsampled = false;
};

namespace dab {

// The largest inner dimension: one vector has to fit the shared memory of a warp.
constexpr uint32_t kMaxTransformDim = 32768;

// transform_into for the n rows of d_src [n][input_dim] into d_dst [n][output_dim] (both device memory), on the current
// device and the legacy stream.  d_first_nan (may be NULL): atomicMin of the index of every row whose *input* holds a
// NaN.  Uploads the sign and subsample tables for the call and frees them before returning.
cudaError_t transform_rows(const dab_transform* t, const float* d_src, uint64_t n, float* d_dst, unsigned long long* d_first_nan);

// The sign and subsample tables of `t` as the kernel reads them, in one buffer: signs0, signs1, subsample
std::vector<uint32_t> transform_tables(const dab_transform* t);
// transform_rows with the tables already resident (d_tables: transform_tables(t) in device memory), queued on `stream`
cudaError_t transform_launch(const dab_transform* t, const uint32_t* d_tables, const float* d_src, uint64_t n, float* d_dst,
                             unsigned long long* d_first_nan, cudaStream_t stream);

}  // namespace dab
