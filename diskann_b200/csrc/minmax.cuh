// minmax.cuh — the MinMax compressor (minmax_compress_kernel, minmax_kernels.cu) as the other translation units launch
// it: the standalone entry points and the MinMax store of an index (minmax_index.cu).
#pragma once

#include "dab_common.cuh"

namespace dab {

// bytes of MinMaxCompensation {dim u32, b, n, a, norm_squared} in front of the codes of a canonical-front row
constexpr int kMmMeta = 20;

struct MinMaxCompressParams {
    float grid_scale;
    uint32_t dim;
    int nbits;
    const float* vectors;  // [n][dim]
    uint64_t n;
    uint8_t* rows;         // [n][row_bytes]
    uint32_t row_bytes;
    uint32_t srow_stride;  // bytes between the staged output rows of a warp (an odd number of words: conflict-free)
    float* loss;           // [n] or NULL
    unsigned long long* first_nan;
    uint32_t warp_smem;    // tile + staged rows
};

// MinMaxCompressParams for dim-long vectors and the CTA shape of minmax_compress_kernel; false if the staging buffers
// of one warp do not fit shared memory
bool mm_compress_setup(float grid_scale, uint32_t dim, int nbits, uint64_t n, MinMaxCompressParams& p, int& warps, size_t& smem);

// minmax_compress_kernel on `stream`, on the current device; p.vectors, p.rows, p.loss and p.first_nan (atomicMin of
// the index of every row whose input holds a NaN) are device pointers
cudaError_t mm_compress_launch(const MinMaxCompressParams& p, int warps, size_t smem, cudaStream_t stream = 0);

}  // namespace dab
