// Tables and coordinate arithmetic shared by the STN kernels: the inference pair of glue.cu (k_stn_params,
// k_stn_sample), the part-crop targets of iuv_train.cu and the training pair of stn_train.cu.
#pragma once
#include <math.h>

namespace danet {

// utils/smpl_utlis.py:13-17,29-53 (structure tables used by iuv_estimator.py:176-184,262-301); `static`: every
// translation unit that includes this holds its own copy in its own module
static __constant__ int c_parents0[24] = {0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21};
static __constant__ int c_children1[24] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 10, 11, 15, 16, 17, 15, 18, 19, 20, 21, 22, 23, 22, 23};
// smpl2dp_part as 25-bit masks over DensePose part ids
static __constant__ unsigned c_part_mask[24] = {
    (1u << 1) | (1u << 2), (1u << 8) | (1u << 10), (1u << 7) | (1u << 9), (1u << 1) | (1u << 2),
    (1u << 8) | (1u << 10) | (1u << 12) | (1u << 14), (1u << 7) | (1u << 9) | (1u << 11) | (1u << 13),
    (1u << 1) | (1u << 2), (1u << 12) | (1u << 14) | (1u << 5), (1u << 11) | (1u << 13) | (1u << 6),
    (1u << 1) | (1u << 2), (1u << 12) | (1u << 14) | (1u << 5), (1u << 11) | (1u << 13) | (1u << 6),
    (1u << 1) | (1u << 2) | (1u << 23) | (1u << 24), (1u << 15) | (1u << 17), (1u << 16) | (1u << 18),
    (1u << 23) | (1u << 24), (1u << 15) | (1u << 17), (1u << 16) | (1u << 18),
    (1u << 15) | (1u << 17) | (1u << 19) | (1u << 21), (1u << 16) | (1u << 18) | (1u << 20) | (1u << 22),
    (1u << 19) | (1u << 21) | (1u << 4), (1u << 20) | (1u << 22) | (1u << 3),
    (1u << 19) | (1u << 21) | (1u << 4), (1u << 20) | (1u << 22) | (1u << 3)};

// torch.argmax semantics: first maximal value; NaN counts as maximal
__device__ __forceinline__ int argmax_first(const float* v, int n) {
    int best = 0; float bv = v[0];
    for (int c = 1; c < n; ++c) {
        const float x = v[c];
        if ((x > bv) || (x != x && bv == bv)) { bv = x; best = c; }
    }
    return best;
}
// the same over n values `stride` floats apart
__device__ __forceinline__ int argmax_first(const float* v, int n, size_t stride) {
    int best = 0; float bv = v[0];
    for (int c = 1; c < n; ++c) {
        const float x = v[(size_t)c * stride];
        if ((x > bv) || (x != x && bv == bv)) { bv = x; best = c; }
    }
    return best;
}

// fp32 product and sum rounded on their own: the device never contracts them into a fused multiply-add, so a host
// restatement (which has no FMA either) sees the same values
__host__ __device__ inline float rn_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline float rn_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// base grid coordinate i of affine_grid, rounded like torch's: linspace(-1, 1, S) (start + i*step on the first half,
// end - (S-1-i)*step on the second), times (S-1)/S when align_corners is off (AffineGridGenerator.cpp)
__host__ __device__ inline float affine_base(int i, int S, int align) {
    const float step = 2.f / (float)(S - 1);
    float v = i < S / 2 ? rn_add(-1.f, rn_mul(step, (float)i)) : rn_add(1.f, -rn_mul(step, (float)(S - 1 - i)));
    if (!align) v = rn_mul(v, (float)(S - 1)) / (float)S;
    return v;
}

// grid coordinate in [-1, 1] -> source pixel coordinate (torch grid_sampler_compute_source_index, no padding clip)
__host__ __device__ inline float grid_unnormalize(float g, int S, int align) {
    return align ? rn_mul(rn_mul(rn_add(g, 1.f), 0.5f), (float)(S - 1))
                 : rn_mul(rn_add(rn_mul(rn_add(g, 1.f), (float)S), -1.f), 0.5f);
}

}  // namespace danet
