// Training targets for sm_90a: the camera translation of estimate_translation solved on the device, the merge of the
// SPIN fits with the ground truth, and the key-point, camera and 229-wide regression targets of one training step.
// Replaces utils/geometry.py:94-157 (estimate_translation / estimate_translation_np: a D2H copy, one numpy
// least-squares problem per image in a Python loop, an H2D copy), train/trainer.py:157-212 (boolean-mask merges,
// the target key points and the renderer camera) and models/danet/danet.py:159-162 (`target`).  Nothing here
// synchronises with the host, so a training step's target preparation can be captured in one CUDA graph.
//   k_estimate_translation  one warp per image: the translation only (danet_estimate_translation)
//   k_fit_merge             thread per image: beta clamp, ground-truth merge, valid_fit / has_iuv
//   k_train_targets         one warp per image: the translation, target_cam, target_smpl_kps and `target`
//
// The translation (estimate_translation_np) in the reference's arithmetic: the weight sqrt(conf) is rounded to fp32
// (np.sqrt of a float32 array), everything after it is fp64 (F, O and the centre are float64 and numpy upcasts).
// For joint j, with w its fp32 weight, the two weighted rows of Q and c are
//   x row  w * [F, 0, O - x_j]   c = w * ((x_j - O) * Z_j - F * X_j)      (the y row likewise, with Y_j)
// Lane j < 24 holds joint 25 + j's share of the 6 entries of A = Q^T Q and the 3 of b = Q^T c (its x row's product
// plus its y row's), and a fixed-order xor-shuffle tree sums them in double: every lane ends with the same bits, the
// row of an image depends on nothing else in the batch, and the result is bit-for-bit repeatable.  Every lane then
// solves A t = b by LU with partial pivoting (LAPACK gesv's choice: the first row of largest |pivot| wins ties), so no
// broadcast is needed, and t is rounded once to fp32.  The products and sums use the _rn intrinsics (no FMA
// contraction), so the host build (DANET_TARGETS_HOST_CHECK) gives the device's bits.
// One deliberate difference: numpy raises LinAlgError on an exactly zero pivot (every confidence 0, in exact
// arithmetic); the device cannot raise without a host synchronisation, so that image's translation is NaN.
#include "common.cuh"

namespace danet {

constexpr int kCamJ0 = 25;        // estimate_translation uses joints 25:49 (the ground-truth joints)
constexpr int kCamJ = 24;
constexpr int kJoints49 = 49;
constexpr int kTargetWarps = 4;   // images per CTA (one warp each)

__host__ __device__ __forceinline__ double ct_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ double ct_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ double ct_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ __forceinline__ double ct_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
__host__ __device__ __forceinline__ float ct_sqrtf(float a) {
#ifdef __CUDA_ARCH__
    return __fsqrt_rn(a);
#else
    return sqrtf(a);
#endif
}

// One joint's share of A = Q^T Q and b = Q^T c: t = {A00, A01, A02, A11, A12, A22, b0, b1, b2}.  (X, Y, Z) is the 3-D
// joint, (x, y) its 2-D key point in pixels, conf its confidence; F the focal length and O the image centre.
__host__ __device__ __forceinline__ void cam_t_terms(float X, float Y, float Z, float x, float y, float conf, double F,
                                                     double O, double* t) {
    const double w = (double)ct_sqrtf(conf);
    const double q[2][3] = {{ct_mul(w, F), ct_mul(w, 0.0), ct_mul(w, ct_sub(O, x))},
                            {ct_mul(w, 0.0), ct_mul(w, F), ct_mul(w, ct_sub(O, y))}};
    const double c[2] = {ct_mul(w, ct_sub(ct_mul(ct_sub(x, O), Z), ct_mul(F, X))),
                         ct_mul(w, ct_sub(ct_mul(ct_sub(y, O), Z), ct_mul(F, Y)))};
    const int ri[6] = {0, 0, 0, 1, 1, 2}, ci[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; ++e)
        t[e] = ct_add(ct_mul(q[0][ri[e]], q[0][ci[e]]), ct_mul(q[1][ri[e]], q[1][ci[e]]));
#pragma unroll
    for (int k = 0; k < 3; ++k) t[6 + k] = ct_add(ct_mul(q[0][k], c[0]), ct_mul(q[1][k], c[1]));
}

// Solve A t = b (t = the 9 sums of cam_t_terms) like LAPACK gesv: LU with partial pivoting, the first row of largest
// |pivot| winning ties; an exactly zero pivot (numpy's LinAlgError) gives NaN.  The callers round the fp64 solution
// once to fp32.  Every loop is unrolled and the row swap is a select, so the system stays in registers.
__host__ __device__ __forceinline__ void cam_t_solve(const double* t, double* out) {
    double a[3][3] = {{t[0], t[1], t[2]}, {t[1], t[3], t[4]}, {t[2], t[4], t[5]}};
    double r[3] = {t[6], t[7], t[8]};
    bool singular = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        int p = k;
        double best = fabs(a[k][k]);
#pragma unroll
        for (int i = k + 1; i < 3; ++i)
            if (fabs(a[i][k]) > best) { best = fabs(a[i][k]); p = i; }
        singular |= best == 0.0;
#pragma unroll
        for (int i = k + 1; i < 3; ++i) {
            if (p == i) {
#pragma unroll
                for (int j = 0; j < 3; ++j) { const double s = a[k][j]; a[k][j] = a[i][j]; a[i][j] = s; }
                const double s = r[k]; r[k] = r[i]; r[i] = s;
            }
        }
#pragma unroll
        for (int i = k + 1; i < 3; ++i) {
            const double l = ct_div(a[i][k], a[k][k]);
#pragma unroll
            for (int j = k + 1; j < 3; ++j) a[i][j] = ct_sub(a[i][j], ct_mul(l, a[k][j]));
            r[i] = ct_sub(r[i], ct_mul(l, r[k]));
        }
    }
    const double x2 = ct_div(r[2], a[2][2]);
    const double x1 = ct_div(ct_sub(r[1], ct_mul(a[1][2], x2)), a[1][1]);
    const double x0 = ct_div(ct_sub(ct_sub(r[0], ct_mul(a[0][1], x1)), ct_mul(a[0][2], x2)), a[0][0]);
    const double nan_ = nan("");
    out[0] = singular ? nan_ : x0; out[1] = singular ? nan_ : x1; out[2] = singular ? nan_ : x2;
}

// The 2-D key point of one joint in pixels: as given, or de-normalised from [-1, 1] like trainer.py:168-169
// (0.5 * img_res * (k + 1), in fp32).
__host__ __device__ __forceinline__ float kp_pixels(float k, bool normalised, float half_res) {
#ifdef __CUDA_ARCH__
    return normalised ? __fmul_rn(half_res, __fadd_rn(k, 1.0f)) : k;
#else
    return normalised ? half_res * (k + 1.0f) : k;
#endif
}

// The xor-shuffle tree of the warp (the host build restates it): v[lane] += v[lane ^ o] for o = 16, 8, 4, 2, 1.
__device__ __forceinline__ void cam_t_warp_sum(double* t) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int e = 0; e < 9; ++e) t[e] = __dadd_rn(t[e], __shfl_xor_sync(0xffffffffu, t[e], o));
}

// The translation of one image: S49 / kp49 its [49,3] joints and key points (x, y, confidence); every lane returns it.
__device__ __forceinline__ void cam_t_warp(const float* __restrict__ S49, const float* __restrict__ kp49, bool normalised,
                                           float half_res, double F, double O, int lane, float* out) {
    double t[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (lane < kCamJ) {
        const float* s = S49 + (kCamJ0 + lane) * 3;
        const float* k = kp49 + (kCamJ0 + lane) * 3;
        cam_t_terms(s[0], s[1], s[2], kp_pixels(k[0], normalised, half_res), kp_pixels(k[1], normalised, half_res), k[2],
                    F, O, t);
    }
    cam_t_warp_sum(t);
    double x[3];
    cam_t_solve(t, x);
    out[0] = (float)x[0]; out[1] = (float)x[1]; out[2] = (float)x[2];
}

__global__ void __launch_bounds__(kTargetWarps * 32)
k_estimate_translation(int B, const float* __restrict__ S, const float* __restrict__ kp, double F, double O,
                       float* __restrict__ trans) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * kTargetWarps + warp;
    if (b >= B) return;                                  // whole warps leave together
    float t[3];
    cam_t_warp(S + (size_t)b * kJoints49 * 3, kp + (size_t)b * kJoints49 * 3, false, 0.0f, F, O, lane, t);
    if (lane < 3) trans[(size_t)b * 3 + lane] = lane == 0 ? t[0] : (lane == 1 ? t[1] : t[2]);
}

// trainer.py:157-161 and :177-191.  A fit row is zeroed when any |beta| > 3 (NaN is not > 3); the clamp comes before the
// merge, so a ground-truth beta above 3 survives.  valid_fit = has_smpl (| fit_valid), has_iuv = iuv_annotated & valid_fit.
__global__ void k_fit_merge(int B, const float* __restrict__ fit_pose, const float* __restrict__ fit_betas,
                            const float* __restrict__ gt_pose, const float* __restrict__ gt_betas,
                            const uint8_t* __restrict__ has_smpl, const uint8_t* __restrict__ fit_valid,
                            const uint8_t* __restrict__ iuv_annotated, float* __restrict__ opt_pose,
                            float* __restrict__ opt_betas, uint8_t* __restrict__ valid_fit, uint8_t* __restrict__ has_iuv) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    bool extreme = false;
    for (int l = 0; l < 10; ++l) extreme |= fabsf(fit_betas[(size_t)b * 10 + l]) > 3.0f;
    const bool gt = has_smpl[b] != 0;
    for (int k = 0; k < 72; ++k) opt_pose[(size_t)b * 72 + k] = gt ? gt_pose[(size_t)b * 72 + k] : fit_pose[(size_t)b * 72 + k];
    for (int l = 0; l < 10; ++l)
        opt_betas[(size_t)b * 10 + l] = gt ? gt_betas[(size_t)b * 10 + l] : (extreme ? 0.0f : fit_betas[(size_t)b * 10 + l]);
    const bool vf = gt || (fit_valid && fit_valid[b] != 0);
    valid_fit[b] = vf ? 1 : 0;
    has_iuv[b] = (vf && iuv_annotated[b] != 0) ? 1 : 0;
}

// trainer.py:163-212 after the SMPL forward of the merged fits, and danet.py:159-162.  Lane j < 24 owns joint j.
__global__ void __launch_bounds__(kTargetWarps * 32)
k_train_targets(int B, const float* __restrict__ opt_joints, const float* __restrict__ smpl_joints,
                const float* __restrict__ keypoints, const float* __restrict__ opt_pose, const float* __restrict__ opt_betas,
                const uint8_t* __restrict__ has_iuv, const uint8_t* __restrict__ has_dp, const float* __restrict__ smpl_2dkps,
                double F, int img_res, float* __restrict__ opt_cam_t, float* __restrict__ target_cam,
                float* __restrict__ target_smpl_kps, float* __restrict__ target) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * kTargetWarps + warp;
    if (b >= B) return;
    const float half_res = (float)(0.5 * img_res);
    float t[3];
    cam_t_warp(opt_joints + (size_t)b * kJoints49 * 3, keypoints + (size_t)b * kJoints49 * 3, true, half_res, F,
               img_res / 2.0, lane, t);
    // gt_camera = [2 f / img_res / t_z, t_x, t_y] (trainer.py:208-211): torch evaluates `scalar / tensor` as
    // reciprocal(tensor) * scalar
    const float cam0 = __fmul_rn(__frcp_rn(t[2]), (float)(2.0 * F / img_res));
    float* tg = target + (size_t)b * 229;
    if (lane < 3) {
        const float tl = lane == 0 ? t[0] : (lane == 1 ? t[1] : t[2]);
        const float cl = lane == 0 ? cam0 : (lane == 1 ? t[0] : t[1]);
        opt_cam_t[(size_t)b * 3 + lane] = tl;
        target_cam[(size_t)b * 3 + lane] = cl;
        tg[lane] = cl;
    }
    if (lane < 10) tg[3 + lane] = opt_betas[(size_t)b * 10 + lane];
    if (lane >= kCamJ) return;
    // target_smpl_kps (trainer.py:194-204): smpl_joints projected with R = I, t = opt_cam_t, centre img_res / 2,
    // normalised to [-1, 1]; confidence 1 where has_iuv == 1; the row is smpl_2dkps where has_dp == 1
    float* kp = target_smpl_kps + ((size_t)b * kCamJ + lane) * 3;
    if (has_dp[b] == 1) {
        const float* s = smpl_2dkps + ((size_t)b * kCamJ + lane) * 3;
        kp[0] = s[0]; kp[1] = s[1]; kp[2] = s[2];
    } else {
        const float* p = smpl_joints + ((size_t)b * kCamJ + lane) * 3;
        const float eye[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};
        const float ctr[2] = {half_res, half_res};
        float uv[2];
        persp_point(eye, t, (float)F, ctr, p[0], p[1], p[2], uv);
        kp[0] = __fsub_rn(__fdiv_rn(uv[0], half_res), 1.0f);
        kp[1] = __fsub_rn(__fdiv_rn(uv[1], half_res), 1.0f);
        kp[2] = has_iuv[b] == 1 ? 1.0f : 0.0f;
    }
    // target = cat(target_cam, opt_betas, batch_rodrigues(opt_pose)) with the quaternion Rodrigues (danet.py:159-161)
    float R[9];
    rodrigues_quat(opt_pose + (size_t)b * 72 + lane * 3, R);
#pragma unroll
    for (int e = 0; e < 9; ++e) tg[13 + lane * 9 + e] = R[e];
}

}  // namespace danet

using namespace danet;

extern "C" int danet_estimate_translation(int32_t B, const float* S, const float* joints_2d, double focal_length,
                                          double img_size, float* trans, danet_stream_t stream) {
    DANET_CHECK(B >= 0, "danet_estimate_translation: negative batch (B=%d)", B);
    if (B == 0) return 0;
    DANET_CHECK(S && joints_2d && trans, "danet_estimate_translation: null pointer");
    k_estimate_translation<<<cdiv(B, kTargetWarps), kTargetWarps * 32, 0, (cudaStream_t)stream>>>(
        B, S, joints_2d, focal_length, img_size / 2.0, trans);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_fit_merge(int32_t B, const float* fit_pose, const float* fit_betas, const float* gt_pose,
                               const float* gt_betas, const uint8_t* has_smpl, const uint8_t* fit_valid,
                               const uint8_t* iuv_annotated, float* opt_pose, float* opt_betas, uint8_t* valid_fit,
                               uint8_t* has_iuv, danet_stream_t stream) {
    DANET_CHECK(B >= 0, "danet_fit_merge: negative batch (B=%d)", B);
    if (B == 0) return 0;
    DANET_CHECK(fit_pose && fit_betas && gt_pose && gt_betas && has_smpl && iuv_annotated && opt_pose && opt_betas &&
                valid_fit && has_iuv, "danet_fit_merge: null pointer");
    k_fit_merge<<<cdiv(B, 128), 128, 0, (cudaStream_t)stream>>>(B, fit_pose, fit_betas, gt_pose, gt_betas, has_smpl,
                                                                fit_valid, iuv_annotated, opt_pose, opt_betas, valid_fit,
                                                                has_iuv);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_train_targets(int32_t B, const float* opt_joints, const float* smpl_joints, const float* keypoints,
                                   const float* opt_pose, const float* opt_betas, const uint8_t* has_iuv,
                                   const uint8_t* has_dp, const float* smpl_2dkps, double focal_length, int32_t img_res,
                                   float* opt_cam_t, float* target_cam, float* target_smpl_kps, float* target,
                                   danet_stream_t stream) {
    DANET_CHECK(B >= 0 && img_res > 0, "danet_train_targets: bad sizes (B=%d, img_res=%d)", B, img_res);
    if (B == 0) return 0;
    DANET_CHECK(opt_joints && smpl_joints && keypoints && opt_pose && opt_betas && has_iuv && has_dp && smpl_2dkps &&
                opt_cam_t && target_cam && target_smpl_kps && target, "danet_train_targets: null pointer");
    k_train_targets<<<cdiv(B, kTargetWarps), kTargetWarps * 32, 0, (cudaStream_t)stream>>>(
        B, opt_joints, smpl_joints, keypoints, opt_pose, opt_betas, has_iuv, has_dp, smpl_2dkps, focal_length, img_res,
        opt_cam_t, target_cam, target_smpl_kps, target);
    DANET_LAUNCH_CHECK();
    return 0;
}

#ifdef DANET_TARGETS_HOST_CHECK
// The per-image arithmetic of k_estimate_translation / k_train_targets walked on the host: the same terms, the warp's
// xor tree over 32 lanes (lanes 24..31 hold zeros), the same solve.  `normalised` de-normalises the key points first.
// trans64 (may be NULL) receives the fp64 solution before its rounding to fp32.
extern "C" int danet_test_estimate_translation_host(int32_t B, const float* S, const float* kp, int32_t normalised,
                                                    double focal_length, double img_size, float* trans, double* trans64) {
    const double O = img_size / 2.0;
    const float half_res = (float)(0.5 * img_size);
    for (int b = 0; b < B; ++b) {
        double v[32][9] = {};
        for (int j = 0; j < kCamJ; ++j) {
            const float* s = S + ((size_t)b * kJoints49 + kCamJ0 + j) * 3;
            const float* k = kp + ((size_t)b * kJoints49 + kCamJ0 + j) * 3;
            cam_t_terms(s[0], s[1], s[2], kp_pixels(k[0], normalised != 0, half_res),
                        kp_pixels(k[1], normalised != 0, half_res), k[2], focal_length, O, v[j]);
        }
        for (int o = 16; o > 0; o >>= 1) {
            double nv[32][9];
            for (int l = 0; l < 32; ++l)
                for (int e = 0; e < 9; ++e) nv[l][e] = ct_add(v[l][e], v[l ^ o][e]);
            for (int l = 0; l < 32; ++l)
                for (int e = 0; e < 9; ++e) v[l][e] = nv[l][e];
        }
        double x[3];
        cam_t_solve(v[0], x);
        for (int k = 0; k < 3; ++k) {
            trans[(size_t)b * 3 + k] = (float)x[k];
            if (trans64) trans64[(size_t)b * 3 + k] = x[k];
        }
    }
    return 0;
}
#endif
