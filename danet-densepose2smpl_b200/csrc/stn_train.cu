// The STN part crops and their thetas in training mode, on fp32 NCHW tensors (models/danet/iuv_estimator.py):
//
//   part_crops   :193-204  24x F.affine_grid(theta.detach(), xd.size()) + F.grid_sample(xd, grid), cat on dim 1;
//                          forward and the backward w.r.t. xd (theta is a constant, as in the reference)
//   part_thetas  :137-140,172-191,262-301  soft-argmax centres, centre jitter, part visibility and affine_para with
//                          its two scale jitters; the noise is an input (the caller draws it), nothing is differentiable
//
// The sampler is separable: theta = [[s_x, 0, c_x], [0, s_y, c_y]] (the form affine_para builds); the off-diagonal
// entries are not read.  Along each axis the crop pixel p samples the source coordinate ix(p) = unnormalize(s * base(p)
// + c), every product and sum rounded on its own (crop_coord), and taps the pixels floor(ix) and floor(ix) + 1 with
// weights 1 - t and t.  The 2-D weight is w_x * w_y.
//
// The backward is a gather: one thread per (image, input pixel, 4 channels).  Per part and axis, crop_candidates bounds
// the crop pixels whose tap can touch the input pixel (an interval from ix ~ s p + k, widened by the coordinate's
// rounding bound and one pixel); each candidate's tap is recomputed with the forward's own crop_tap and kept only if
// it lands there.  So the gradient is the exact adjoint of the forward as executed, summed in double in (part, py, px)
// order.  No float atomics and no host synchronisation: results repeat bit for bit and the calls can be captured in a
// CUDA graph.  crop_coord, crop_tap and crop_candidates are __host__ __device__: the CPU suite compiles them with
// DANET_STN_HOST_CHECK and checks that the gather visits exactly the forward's (crop pixel, input pixel, weight) triples.
#include "common.cuh"
#include "stn_common.cuh"
#ifdef DANET_STN_HOST_CHECK
#include <vector>
#endif

namespace danet {
namespace stn {

constexpr int kThreads = 256;
constexpr int kFwdCh = 8;                        // channels per forward thread (the taps are computed once for them)
constexpr int kBwdCh = 4;                        // channels per backward thread
constexpr int kNoTap = -2;                       // tap origin of a sample that reads nothing along its axis

// source pixel coordinate of crop pixel p along one axis (scale s, centre c)
__host__ __device__ inline float crop_coord(int p, int S, float s, float c, int align) {
    return grid_unnormalize(rn_add(rn_mul(s, affine_base(p, S, align)), c), S, align);
}

// the pixels floor(ix) (weight w0 = 1 - t) and floor(ix) + 1 (weight w1 = t).  A coordinate whose floor lies outside
// (-2, S) -- or is NaN / infinite -- touches no pixel: i0 = kNoTap, checked before the int conversion
struct Tap { int i0; float w0, w1; };
__host__ __device__ inline Tap crop_tap(int p, int S, float s, float c, int align) {
    const float ix = crop_coord(p, S, s, c, align);
    const float f = floorf(ix);
    Tap t;
    if (!(f > -2.f && f < (float)S)) { t.i0 = kNoTap; t.w0 = t.w1 = 0.f; return t; }
    t.i0 = (int)f;
    t.w1 = rn_add(ix, -f);
    t.w0 = rn_add(1.f, -t.w1);
    return t;
}

// weight with which the tap touches input pixel q (0 <= q < S), false when it does not
__host__ __device__ inline bool tap_hits(const Tap& t, int q, float* w) {
    if (t.i0 == q) { *w = t.w0; return true; }
    if (t.i0 + 1 == q) { *w = t.w1; return true; }
    return false;
}

__host__ __device__ inline float crop_weight(float wx, float wy) { return rn_mul(wx, wy); }

// Inclusive range [lo, hi] of the crop pixels whose tap can touch input pixel q (empty when lo > hi).  Without
// rounding, ix(p) = s p + k and p touches q iff q - 1 <= ix(p) < q + 1.  The fp32 coordinate is within
// 2^-20 S (|s| + |c| + 1) of s p + k (16x the bound of its roundings), so the interval is widened by that over |s|
// pixels, and by one more.  Scale 0 samples one point: every crop pixel is a candidate.  A non-finite theta samples
// nothing.  The bounds are clamped in double before the int conversion.
__host__ __device__ inline void crop_candidates(int q, int S, float s, float c, int align, int* lo, int* hi) {
    *lo = 0; *hi = -1;
    const double sd = s, cd = c;
    if (!isfinite(sd) || !isfinite(cd)) return;
    if (sd == 0.0) { *hi = S - 1; return; }
    const double k = align ? (cd + 1.0 - sd) * (double)(S - 1) * 0.5 : (sd * (double)(1 - S) + (cd + 1.0) * (double)S - 1.0) * 0.5;
    const double err = ldexp((double)S * (fabs(sd) + fabs(cd) + 1.0), -20);
    double a = ((double)q - 1.0 - k - err) / sd, b = ((double)q + 1.0 - k + err) / sd;
    if (sd < 0.0) { const double t = a; a = b; b = t; }
    a = fmax(floor(a) - 1.0, 0.0);
    b = fmin(ceil(b) + 1.0, (double)(S - 1));
    if (a > b) return;
    *lo = (int)a; *hi = (int)b;
}

// Every (crop pixel, weight) of one part that samples input pixel (xx, yy), in (py, px) order.  th = the part's
// theta [2][3]; the kernel's gather and the host check walk the same code.
template <class Fn>
__host__ __device__ inline void gather_part(int S, int align, const float* th, int xx, int yy, Fn&& fn) {
    int xlo, xhi, ylo, yhi;
    crop_candidates(xx, S, th[0], th[2], align, &xlo, &xhi);
    crop_candidates(yy, S, th[4], th[5], align, &ylo, &yhi);
    for (int py = ylo; py <= yhi; ++py) {
        float wy;
        if (!tap_hits(crop_tap(py, S, th[4], th[5], align), yy, &wy)) continue;
        for (int px = xlo; px <= xhi; ++px) {
            float wx;
            if (tap_hits(crop_tap(px, S, th[0], th[2], align), xx, &wx)) fn(py, px, crop_weight(wx, wy));
        }
    }
}

// bilinear footprint of crop pixel (px, py): origin (x0, y0) and the weights nw, ne, sw, se.  An axis without a tap
// puts its origin at kNoTap, so all four corners fall outside the map.
struct Foot { int x0, y0; float w[4]; };
__host__ __device__ inline Foot crop_foot(int S, int align, const float* th, int px, int py) {
    const Tap tx = crop_tap(px, S, th[0], th[2], align), ty = crop_tap(py, S, th[4], th[5], align);
    Foot f;
    f.x0 = tx.i0; f.y0 = ty.i0;
    f.w[0] = crop_weight(tx.w0, ty.w0); f.w[1] = crop_weight(tx.w1, ty.w0);
    f.w[2] = crop_weight(tx.w0, ty.w1); f.w[3] = crop_weight(tx.w1, ty.w1);
    return f;
}

// grid (crop pixel tiles, B * 24, channel chunks of kFwdCh); out [B][24][C][S][S]
__global__ void __launch_bounds__(kThreads)
k_part_crops_fwd(int S, int C, const float* __restrict__ xd, const float* __restrict__ theta, int align, float* __restrict__ out) {
    const int HW = S * S;
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= HW) return;
    const int bp = blockIdx.y, b = bp / 24;
    float th[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) th[k] = __ldg(theta + (size_t)bp * 6 + k);
    const Foot f = crop_foot(S, align, th, p % S, p / S);
    int off[4];
    bool ok[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xx = f.x0 + (k & 1), yy = f.y0 + (k >> 1);
        ok[k] = xx >= 0 && xx < S && yy >= 0 && yy < S;
        off[k] = ok[k] ? yy * S + xx : 0;
    }
    const int c0 = blockIdx.z * kFwdCh, c1 = min(c0 + kFwdCh, C);
    for (int c = c0; c < c1; ++c) {
        const float* x = xd + ((size_t)b * C + c) * HW;
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (ok[k]) acc = fmaf(f.w[k], __ldg(x + off[k]), acc);
        out[((size_t)bp * C + c) * HW + p] = acc;
    }
}

// grid (input pixel tiles, B, channel chunks of kBwdCh); dcrops [B][24][C][S][S] -> dxd [B][C][S][S]
__global__ void __launch_bounds__(kThreads)
k_part_crops_bwd(int S, int C, const float* __restrict__ dcrops, const float* __restrict__ theta, int align,
                 float* __restrict__ dxd) {
    __shared__ float s_th[24 * 6];
    const int b = blockIdx.y;
    for (int k = threadIdx.x; k < 24 * 6; k += kThreads) s_th[k] = __ldg(theta + (size_t)b * 24 * 6 + k);
    __syncthreads();
    const int HW = S * S;
    const int q = blockIdx.x * kThreads + threadIdx.x;
    if (q >= HW) return;
    const int c0 = blockIdx.z * kBwdCh, nc = min(kBwdCh, C - c0);
    double acc[kBwdCh];
#pragma unroll
    for (int k = 0; k < kBwdCh; ++k) acc[k] = 0.0;
    for (int i = 0; i < 24; ++i) {
        const float* g = dcrops + (((size_t)b * 24 + i) * C + c0) * HW;
        gather_part(S, align, s_th + i * 6, q % S, q / S, [&](int py, int px, float w) {
            const float* gp = g + py * S + px;
#pragma unroll
            for (int k = 0; k < kBwdCh; ++k)
                if (k < nc) acc[k] += (double)w * (double)__ldg(gp + (size_t)k * HW);
        });
    }
#pragma unroll
    for (int k = 0; k < kBwdCh; ++k)
        if (k < nc) dxd[((size_t)b * C + c0 + k) * HW + q] = (float)acc[k];
}

// ------------------------------------------------------------------------------------------------
// part_thetas: one CTA per image
// ------------------------------------------------------------------------------------------------
struct ThetaArgs {
    int Sh, Si, align;
    const float* hm; const float* index; const float* ratio; const float* offset;
    const float* center_noise; const float* scale_noise;
    float vis_score, center_jitter, scale_jitter;
    int B;
    float* centers; float* theta;
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// 1[argmax over the 25 index channels of pixel (xx, yy) lies in part i's DensePose set]
__device__ inline float part_indicator(const ThetaArgs& a, const float* idx, int i, int xx, int yy) {
    const size_t HW = (size_t)a.Si * a.Si, q = (size_t)yy * a.Si + xx;
    float v[25];
#pragma unroll
    for (int c = 0; c < 25; ++c) v[c] = __ldg(idx + c * HW + q);
    return ((c_part_mask[i] >> argmax_first(v, 25)) & 1u) ? 1.f : 0.f;
}

// grid_sample (bilinear, zeros) of the part indicator at the centre (gx, gy)
__device__ inline float part_score(const ThetaArgs& a, const float* idx, int i, float gx, float gy) {
    const int S = a.Si;
    const float ix = grid_unnormalize(gx, S, a.align), iy = grid_unnormalize(gy, S, a.align);
    const float fx = floorf(ix), fy = floorf(iy);
    if (!(fx > -2.f && fx < (float)S && fy > -2.f && fy < (float)S)) return 0.f;
    const int x0 = (int)fx, y0 = (int)fy;
    const float tx = ix - fx, ty = iy - fy;
    float acc = 0.f;
    for (int k = 0; k < 4; ++k) {
        const int xx = x0 + (k & 1), yy = y0 + (k >> 1);
        if (xx < 0 || xx >= S || yy < 0 || yy >= S) continue;
        const float w = rn_mul((k & 1) ? tx : 1.f - tx, (k >> 1) ? ty : 1.f - ty);
        acc = rn_add(acc, rn_mul(part_indicator(a, idx, i, xx, yy), w));
    }
    return acc;
}

__device__ __forceinline__ float jitter(float v, float amount, float r) {   // v * (1 + amount * (r - 0.5))
    return rn_mul(v, rn_add(1.f, rn_mul(amount, rn_add(r, -0.5f))));
}

__global__ void __launch_bounds__(kThreads) k_part_thetas(const ThetaArgs a) {
    __shared__ float s_c[24][2];
    const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = a.Sh, HW = S * S;
    // soft-argmax of 10 * hm per joint, one warp per joint: max, then sums of e, e x and e y in double
    for (int j = warp; j < 24; j += kThreads / 32) {
        const float* h = a.hm + ((size_t)b * 24 + j) * HW;
        float m = -INFINITY;
        for (int p = lane; p < HW; p += 32) m = fmaxf(m, rn_mul(10.f, __ldg(h + p)));
        m = warp_max(m);
        double se = 0.0, sx = 0.0, sy = 0.0;
        for (int p = lane; p < HW; p += 32) {
            const double e = (double)expf(rn_add(rn_mul(10.f, __ldg(h + p)), -m));
            se += e; sx += e * (double)(p % S); sy += e * (double)(p / S);
        }
        se = warp_sum_d(se); sx = warp_sum_d(sx); sy = warp_sum_d(sy);
        if (lane == 0) {
            // / (0.5 S) - 1, then the centre jitter (iuv_estimator.py:137-140,172-173)
            float cx = rn_add((float)(sx / se) / (0.5f * (float)S), -1.f);
            float cy = rn_add((float)(sy / se) / (0.5f * (float)S), -1.f);
            if (a.center_noise) {
                const float* r = a.center_noise + ((size_t)b * 24 + j) * 2;
                cx = rn_add(cx, rn_mul(a.center_jitter, rn_add(__ldg(r), -0.5f)));
                cy = rn_add(cy, rn_mul(a.center_jitter, rn_add(__ldg(r + 1), -0.5f)));
            }
            s_c[j][0] = cx; s_c[j][1] = cy;
        }
    }
    __syncthreads();
    if (threadIdx.x >= 24) return;
    const int i = threadIdx.x;
    // affine_para (iuv_estimator.py:262-301) on the jittered centres
    float xmin = s_c[0][0], xmax = xmin, ymin = s_c[0][1], ymax = ymin;
    for (int j = 1; j < 24; ++j) {
        xmin = fminf(xmin, s_c[j][0]); xmax = fmaxf(xmax, s_c[j][0]);
        ymin = fminf(ymin, s_c[j][1]); ymax = fmaxf(ymax, s_c[j][1]);
    }
    const float scale_box = fmaxf(rn_add(xmax, -xmin), rn_add(ymax, -ymin)) / 2.f;
    float scale = scale_box;
    if (i != 0) {
        const int pi = c_parents0[i], ci = c_children1[i];
        const float dcx = rn_add(s_c[ci][0], -s_c[i][0]), dcy = rn_add(s_c[ci][1], -s_c[i][1]);
        const float dpx = rn_add(s_c[pi][0], -s_c[i][0]), dpy = rn_add(s_c[pi][1], -s_c[i][1]);
        const float sc = sqrtf(rn_add(rn_mul(dcx, dcx), rn_mul(dcy, dcy))) / 2.f;
        const float sp = sqrtf(rn_add(rn_mul(dpx, dpx), rn_mul(dpy, dpy))) / 2.f;
        scale = rn_mul(2.f, fmaxf(sc, sp));
    }
    scale = rn_mul(scale, fmaxf(__ldg(a.ratio + i), 0.f));
    scale = rn_add(scale, fmaxf(__ldg(a.offset + i), 0.f));
    const float* r = a.scale_noise ? a.scale_noise + (size_t)i * 2 * a.B + b : nullptr;      // [24][2][B]
    if (r) scale = jitter(scale, a.scale_jitter, __ldg(r));
    if (i != 0 && a.vis_score > 0.f &&
        part_score(a, a.index + (size_t)b * 25 * a.Si * a.Si, i, s_c[i][0], s_c[i][1]) < a.vis_score)
        scale = rn_mul(0.8f, scale_box);
    if (r) scale = jitter(scale, a.scale_jitter, __ldg(r + a.B));
    float* c = a.centers + ((size_t)b * 24 + i) * 2;
    c[0] = s_c[i][0]; c[1] = s_c[i][1];
    float* t = a.theta + ((size_t)b * 24 + i) * 6;
    t[0] = scale; t[1] = 0.f; t[2] = s_c[i][0];
    t[3] = 0.f; t[4] = scale; t[5] = s_c[i][1];
}

}  // namespace stn
}  // namespace danet

using namespace danet;

static bool crops_shape_ok(int32_t B, int32_t C, int32_t S) {
    // grid y = B * 24 (forward) and B (backward), grid z = the channel chunks of both kernels: at most 65535 each
    return B >= 1 && C >= 1 && S >= 2 && S <= 4096 && (long long)B * 24 * C * S * S < (1LL << 31) &&
           (long long)B * 24 <= 65535 && cdiv(C, stn::kBwdCh) <= 65535 && cdiv(C, stn::kFwdCh) <= 65535;
}

extern "C" int danet_part_crops_forward(int32_t B, int32_t C, int32_t S, const float* xd, const float* theta,
                                        int32_t align_corners, float* crops, danet_stream_t stream) {
    DANET_CHECK(crops_shape_ok(B, C, S), "danet_part_crops_forward: bad sizes B=%d C=%d S=%d", B, C, S);
    DANET_CHECK(xd && theta && crops, "danet_part_crops_forward: xd, theta and crops must be non-null");
    const dim3 grid(cdiv(S * S, stn::kThreads), B * 24, cdiv(C, stn::kFwdCh));
    stn::k_part_crops_fwd<<<grid, stn::kThreads, 0, (cudaStream_t)stream>>>(S, C, xd, theta, align_corners ? 1 : 0, crops);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_part_crops_backward(int32_t B, int32_t C, int32_t S, const float* dcrops, const float* theta,
                                         int32_t align_corners, float* dxd, danet_stream_t stream) {
    DANET_CHECK(crops_shape_ok(B, C, S), "danet_part_crops_backward: bad sizes B=%d C=%d S=%d", B, C, S);
    DANET_CHECK(dcrops && theta && dxd, "danet_part_crops_backward: dcrops, theta and dxd must be non-null");
    const dim3 grid(cdiv(S * S, stn::kThreads), B, cdiv(C, stn::kBwdCh));
    stn::k_part_crops_bwd<<<grid, stn::kThreads, 0, (cudaStream_t)stream>>>(S, C, dcrops, theta, align_corners ? 1 : 0, dxd);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_part_thetas(int32_t B, int32_t Sh, int32_t Si, const float* hm, const float* index_pred,
                                 const float* learned_ratio, const float* learned_offset, float vis_score,
                                 const float* center_noise, float center_jitter, const float* scale_noise, float scale_jitter,
                                 int32_t align_corners, float* centers, float* theta, danet_stream_t stream) {
    DANET_CHECK(B >= 1 && B <= 65535 && Sh >= 1 && Si >= 2 && (long long)Sh * Sh * 24 * B < (1LL << 31) &&
                (long long)Si * Si * 25 * B < (1LL << 31), "danet_part_thetas: bad sizes B=%d Sh=%d Si=%d", B, Sh, Si);
    DANET_CHECK(hm && learned_ratio && learned_offset && centers && theta,
                "danet_part_thetas: hm, learned_ratio, learned_offset, centers and theta must be non-null");
    DANET_CHECK(index_pred || !(vis_score > 0.f), "danet_part_thetas: vis_score > 0 needs index_pred");
    stn::ThetaArgs a;
    a.Sh = Sh; a.Si = Si; a.align = align_corners ? 1 : 0;
    a.hm = hm; a.index = index_pred; a.ratio = learned_ratio; a.offset = learned_offset;
    a.center_noise = center_noise; a.scale_noise = scale_noise;
    a.vis_score = vis_score; a.center_jitter = center_jitter; a.scale_jitter = scale_jitter;
    a.B = B; a.centers = centers; a.theta = theta;
    stn::k_part_thetas<<<B, stn::kThreads, 0, (cudaStream_t)stream>>>(a);
    DANET_LAUNCH_CHECK();
    return 0;
}

#ifdef DANET_STN_HOST_CHECK
// Test-only (never part of libdanet_b200.so: the flag is set by the CPU tests alone): the forward's and the gather's
// (py, px, yy, xx, weight) records of one part on the host, through the kernels' own functions.  Returns the count,
// or -1 past cap.
extern "C" int64_t danet_test_crop_forward_pairs(int32_t S, int32_t align, const float* th, int32_t* rec, float* w,
                                                 int64_t cap) {
    int64_t n = 0;
    for (int py = 0; py < S; ++py)
        for (int px = 0; px < S; ++px) {
            const stn::Foot f = stn::crop_foot(S, align, th, px, py);
            for (int k = 0; k < 4; ++k) {
                const int xx = f.x0 + (k & 1), yy = f.y0 + (k >> 1);
                if (xx < 0 || xx >= S || yy < 0 || yy >= S) continue;
                if (n >= cap) return -1;
                rec[4 * n] = py; rec[4 * n + 1] = px; rec[4 * n + 2] = yy; rec[4 * n + 3] = xx; w[n] = f.w[k];
                ++n;
            }
        }
    return n;
}

extern "C" int64_t danet_test_crop_gather_pairs(int32_t S, int32_t align, const float* th, int32_t* rec, float* w,
                                                int64_t cap) {
    int64_t n = 0;
    bool over = false;
    for (int yy = 0; yy < S; ++yy)
        for (int xx = 0; xx < S; ++xx)
            stn::gather_part(S, align, th, xx, yy, [&](int py, int px, float wt) {
                if (n >= cap) { over = true; return; }
                rec[4 * n] = py; rec[4 * n + 1] = px; rec[4 * n + 2] = yy; rec[4 * n + 3] = xx; w[n] = wt;
                ++n;
            });
    return over ? -1 : n;
}

extern "C" void danet_test_crop_candidates(int32_t S, int32_t align, float s, float c, int32_t q, int32_t* lo, int32_t* hi) {
    stn::crop_candidates(q, S, s, c, align, lo, hi);
}

extern "C" float danet_test_crop_coord(int32_t S, int32_t align, float s, float c, int32_t p) {
    return stn::crop_coord(p, S, s, c, align);
}
#endif
