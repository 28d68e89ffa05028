// transform.cpp — CPU restatement of the Hadamard transforms in front of the quantizers (test infrastructure only).
//
// diskann-quantization/src/algorithms/hadamard.rs and algorithms/transforms/{padding_hadamard.rs, double_hadamard.rs}.
// hadamard_transform dispatches to the x86-64-v3 implementation (V4 retargets to V3), whose order differs from the
// scalar recursion: below 64 elements it is plain radix-2 recursion, from 64 up it recurses to 64-element blocks and
// runs micro_kernel_64 (hadamard.rs:248-371) on each.  Both orders are restated; the scalar one only so that tests can
// show that the two round differently.  Signs are 0/1 bytes (the flatbuffer's bool form of the 0 / 0x8000_0000 words).
//
// Built on its own into liboracle_transform.so (oracle/transform.mk).
// C ABI (declared here, bound by tests/test_minmax_transforms.py):
//   void  orc_hadamard_8(float* out);                             HADAMARD_8, row-major [8][8]
//   int   orc_hadamard(float* x, size_t len, int scalar_order);   in place; 1 if len is not a power of two
//   int   orc_padding_hadamard(...), orc_double_hadamard(...)      transform_into for one vector; 1 on bad dims
//   int   orc_transform_full_query_meta(...)                       CompressInto<&[f32], FullQueryMut> with a transform
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

// hadamard.rs:232-241
const float kH8[8][8] = {
    {1, 1, 1, 1, 1, 1, 1, 1},     {1, -1, 1, -1, 1, -1, 1, -1}, {1, 1, -1, -1, 1, 1, -1, -1}, {1, -1, -1, 1, 1, -1, -1, 1},
    {1, 1, 1, 1, -1, -1, -1, -1}, {1, -1, 1, -1, -1, 1, -1, 1}, {1, 1, -1, -1, -1, -1, 1, 1}, {1, -1, -1, 1, -1, 1, 1, -1},
};

inline void butterfly(float* x, size_t half) {  // hadamard.rs:171-176 / 220-225
    for (size_t i = 0; i < half; ++i) {
        const float l = x[i], r = x[i + half];
        x[i] = l + r;
        x[half + i] = l - r;
    }
}

void recurse_scalar(float* x, size_t len) {  // HadamardTransformRecursive for Scalar (hadamard.rs:154-178)
    if (len == 2) {
        butterfly(x, 1);
        return;
    }
    recurse_scalar(x, len / 2);
    recurse_scalar(x + len / 2, len / 2);
    butterfly(x, len / 2);
}

// micro_kernel_64 (hadamard.rs:248-371): eight 8-point transforms d0..d7 as FMA chains over HADAMARD_8 starting from
// +0.0, inputs j = 0..7 in order; then the e / f combination and the stores of :362-369.
void micro_kernel_64(float* x) {
    float d[8][8];
    for (int k = 0; k < 8; ++k)
        for (int l = 0; l < 8; ++l) {
            float acc = 0.0f;
            for (int j = 0; j < 8; ++j) acc = std::fmaf(x[8 * k + j], kH8[j][l], acc);
            d[k][l] = acc;
        }
    for (int l = 0; l < 8; ++l) {
        const float e0 = d[0][l] + d[1][l], e1 = d[0][l] - d[1][l];
        const float e2 = d[2][l] + d[3][l], e3 = d[2][l] - d[3][l];
        const float e4 = d[4][l] + d[5][l], e5 = d[4][l] - d[5][l];
        const float e6 = d[6][l] + d[7][l], e7 = d[6][l] - d[7][l];
        const float f0 = e0 + e2, f1 = e1 + e3, f2 = e0 - e2, f3 = e1 - e3;
        const float f4 = e4 + e6, f5 = e5 + e7, f6 = e4 - e6, f7 = e5 - e7;
        x[l] = f0 + f4;
        x[8 + l] = f1 + f5;
        x[16 + l] = f2 + f6;
        x[24 + l] = f3 + f7;
        x[32 + l] = f0 - f4;
        x[40 + l] = f1 - f5;
        x[48 + l] = f2 - f6;
        x[56 + l] = f3 - f7;
    }
}

void recurse_v3(float* x, size_t len) {  // HadamardTransformRecursive for V3 (hadamard.rs:194-227)
    if (len == 64) {
        micro_kernel_64(x);
    } else if (len == 2) {
        butterfly(x, 1);
    } else {
        recurse_v3(x, len / 2);
        recurse_v3(x + len / 2, len / 2);
        butterfly(x, len / 2);
    }
}

bool pow2(size_t n) { return n != 0 && (n & (n - 1)) == 0; }

int hadamard(float* x, size_t len, bool scalar_order) {  // HadamardTransformOuter (hadamard.rs:116-136)
    if (!pow2(len)) return 1;
    if (len == 1) return 0;
    if (scalar_order) recurse_scalar(x, len);
    else recurse_v3(x, len);
    const float m = 1.0f / std::sqrt((float)len);
    for (size_t i = 0; i < len; ++i) x[i] *= m;
    return 0;
}

inline float flip(float v, uint8_t sign) {
    uint32_t b;
    memcpy(&b, &v, 4);
    b ^= sign ? 0x80000000u : 0u;
    memcpy(&v, &b, 4);
    return v;
}

// the subsampled tail of both transform_into functions: tmp[i] * sqrt(len / n_sub) for the sorted indices
void gather(const std::vector<float>& tmp, const uint32_t* subsample, size_t n_sub, float* dst) {
    const float rescale = std::sqrt((float)tmp.size() / (float)n_sub);
    for (size_t i = 0; i < n_sub; ++i) dst[i] = tmp[subsample[i]] * rescale;
}

}  // namespace

extern "C" {

void orc_hadamard_8(float* out) { memcpy(out, kH8, sizeof(kH8)); }

int orc_hadamard(float* x, size_t len, int scalar_order) { return hadamard(x, len, scalar_order != 0); }

// PaddingHadamard::transform_into (padding_hadamard.rs:204-273): sign xor, zero pad to padded_dim, transform, then
// either the whole vector or the rescaled subsample (subsample == NULL: none).  dst has n_sub or padded_dim values.
int orc_padding_hadamard(const uint8_t* signs, size_t input_dim, size_t padded_dim, const uint32_t* subsample, size_t n_sub,
                         const float* src, float* dst) {
    if (input_dim > padded_dim || !pow2(padded_dim)) return 1;
    std::vector<float> tmp(padded_dim, 0.0f);
    for (size_t i = 0; i < input_dim; ++i) tmp[i] = flip(src[i], signs[i]);
    hadamard(tmp.data(), padded_dim, false);
    if (subsample) gather(tmp, subsample, n_sub, dst);
    else memcpy(dst, tmp.data(), padded_dim * 4);
    return 0;
}

// DoubleHadamard::transform_into (double_hadamard.rs:238-287): tmp[intermediate] = sign-flipped, zero-padded input;
// H on tmp[..split] (split = the largest power of two <= intermediate), xor signs1 over all of tmp, H on
// tmp[intermediate - split..] — both over the whole vector when intermediate is a power of two, as the code does —
// then tmp or its rescaled subsample.
int orc_double_hadamard(const uint8_t* signs0, size_t input_dim, const uint8_t* signs1, size_t intermediate,
                        const uint32_t* subsample, size_t n_sub, const float* src, float* dst) {
    if (input_dim == 0 || input_dim > intermediate) return 1;
    std::vector<float> tmp(intermediate, 0.0f);
    for (size_t i = 0; i < input_dim; ++i) tmp[i] = flip(src[i], signs0[i]);
    size_t split = 1;
    while (split * 2 <= intermediate) split *= 2;
    hadamard(tmp.data(), split, false);
    for (size_t i = 0; i < intermediate; ++i) tmp[i] = flip(tmp[i], signs1[i]);
    hadamard(tmp.data() + (intermediate - split), split, false);
    if (subsample) gather(tmp, subsample, n_sub, dst);
    else memcpy(dst, tmp.data(), intermediate * 4);
    return 0;
}

// CompressInto<&[f32], FullQueryMut> (minmax/quantizer.rs:393-415) for a transform: the NaN check runs on the input,
// before the transform; the query is the transformed vector, meta = its sequential sums {sum, norm_squared}.
// `transformed` has already been produced by one of the two functions above.  Returns 1 on NaN input.
int orc_transform_full_query_meta(const float* input, size_t input_dim, const float* transformed, size_t output_dim,
                                  float* sum_out, float* norm_squared_out) {
    for (size_t i = 0; i < input_dim; ++i)
        if (input[i] != input[i]) return 1;
    float ns = -0.0f, s = -0.0f;  // <f32 as Sum>::sum folds from -0.0
    for (size_t i = 0; i < output_dim; ++i) ns = ns + transformed[i] * transformed[i];
    for (size_t i = 0; i < output_dim; ++i) s = s + transformed[i];
    *sum_out = s;
    *norm_squared_out = ns;
    return 0;
}

}  // extern "C"
