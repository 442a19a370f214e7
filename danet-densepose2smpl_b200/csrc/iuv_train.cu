// Training-step supervision of the IUV branch beyond the dense maps (csrc/losses.cu): the sparse DensePose-point
// losses, the STN key-point losses and the part-crop IUV targets.  Forward and backward of each loss in one pass.
//
//   dp_uvia_losses    models/danet/iuv_estimator.py:343-419 (called from :106-121)
//   stn_kps_losses    iuv_estimator.py:137-171, utils/keypoints.py:268-331 (generate_heatmap), :334-394 (soft-argmax)
//   part_iuv_targets  iuv_estimator.py:217-230 + part_iuv_simp :422-445 (forward only; the reference detaches them)
//
// Loss sums: fp32 per thread and block, block partials to the workspace, one finishing block adds them in double in a
// fixed order -- bit-for-bit repeatable, no float atomics.  The per-point / per-pixel arithmetic is __host__ __device__
// so that the DANET_LOSSES_HOST_CHECK build walks it on the CPU against the reference-generated golden.
#include "common.cuh"
#include "stn_common.cuh"
#include "loss_common.cuh"

namespace danet {

#ifdef __CUDA_ARCH__
#define DANET_LDG(p) __ldg(p)
// coordinate arithmetic rounded step by step like torch's (no fused multiply-add: the truncations below see the
// same fp32 values as the reference's)
#define RN_MUL(a, b) __fmul_rn(a, b)
#define RN_ADD(a, b) __fadd_rn(a, b)
#else
#define DANET_LDG(p) (*(p))
#define RN_MUL(a, b) ((a) * (b))
#define RN_ADD(a, b) ((a) + (b))
#endif

__host__ __device__ inline float sl1(float d) { const float a = fabsf(d); return a < 1.f ? 0.5f * d * d : a - 0.5f; }

// bilinear footprint of one sample point: north-west corner and the four weights (nw, ne, sw, se).  Points whose
// corners are all outside the map (or NaN coordinates) get x0 = y0 = -2: nothing is read or written for them.
struct Foot { int x0, y0; float w[4]; };
__host__ __device__ inline Foot make_foot(float ix, float iy, int S) {
    Foot f;
    const float fx = floorf(ix), fy = floorf(iy);
    if (!(fx > -2.f && fx < (float)S && fy > -2.f && fy < (float)S)) {
        f.x0 = f.y0 = -2; f.w[0] = f.w[1] = f.w[2] = f.w[3] = 0.f;
        return f;
    }
    f.x0 = (int)fx; f.y0 = (int)fy;
    const float tx = ix - fx, ty = iy - fy;
    f.w[0] = (1.f - tx) * (1.f - ty); f.w[1] = tx * (1.f - ty); f.w[2] = (1.f - tx) * ty; f.w[3] = tx * ty;
    return f;
}
// zeros-padded bilinear sample of one [S,S] plane
__host__ __device__ inline float foot_sample(const float* plane, int S, const Foot& f) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xx = f.x0 + (k & 1), yy = f.y0 + (k >> 1);
        if (xx >= 0 && xx < S && yy >= 0 && yy < S) acc += DANET_LDG(plane + yy * S + xx) * f.w[k];
    }
    return acc;
}
// weight with which the sample point covers pixel (px, py); 0 outside its footprint
__host__ __device__ inline float foot_weight(const Foot& f, int px, int py) {
    const int dx = px - f.x0, dy = py - f.y0;
    return ((unsigned)dx <= 1u && (unsigned)dy <= 1u) ? f.w[dy * 2 + dx] : 0.f;
}

// ---------------------------------------------------------------------------------------------------------------------
// dp_uvia_losses
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kDpC = 25;                       // NUM_PATCHES + 1 channels of the U / V / index heads
constexpr int kDpThreads = 256;
constexpr int kDpMaxPts = 256;

struct DpArgs {
    int N, S, Cann, P, align;
    const float *u, *v, *idx, *ann;            // [N,25,S,S] x3, [N,Cann,S,S]
    const float *X, *Y, *I, *Up, *Vp, *Wp, *A; // [N,P] x3, [N,25,P] x3 (patch-major), [N,S*S]
    const uint8_t* has;
    float pw, part_w, index_w;
    float *gu, *gv, *gidx, *gann;
};

// footprint of point p of image n (iuv_estimator.py:381-384: grid = (X - S/2) * 2/S)
__host__ __device__ inline Foot dp_foot(const DpArgs& a, int n, int p) {
    const size_t o = (size_t)n * a.P + p;
    const float hs = 0.5f * (float)a.S, sc = 2.f / (float)a.S;
    const float gx = RN_MUL(RN_ADD(a.X[o], -hs), sc), gy = RN_MUL(RN_ADD(a.Y[o], -hs), sc);
    return make_foot(grid_unnormalize(gx, a.S, a.align), grid_unnormalize(gy, a.S, a.align), a.S);
}
// the point's class label: int64 of the float label (truncation toward zero); -1 if outside [0, 25)
__host__ __device__ inline int dp_label(float l, int C) { return (l > -1.f && l < (float)C) ? (int)l : -1; }

// Loss term of point p of image n for map m (0 = U, 1 = V, 2 = index), un-normalised, and d(weighted loss)/d(sample)
// per channel into coef[c] (c < 25).  U / V: w * SL1(w * (u - U)) summed over the 25 patches (the point's patch-major
// targets / weights, iuv_estimator.py:364-377,413-417).  Index: cross-entropy of the 25 sampled logits (:408-411),
// gradient already divided by the number of points `npts`.
__host__ __device__ inline float dp_point_map(const DpArgs& a, int n, int p, int m, const Foot& f, float npts, float* coef) {
    const size_t HW = (size_t)a.S * a.S;
    if (m < 2) {
        const float* pred = (m == 0 ? a.u : a.v) + (size_t)n * kDpC * HW;
        const float* tgt = (m == 0 ? a.Up : a.Vp) + (size_t)n * kDpC * a.P + p;
        const float* wt = a.Wp + (size_t)n * kDpC * a.P + p;
        float l = 0.f;
        for (int c = 0; c < kDpC; ++c) {
            const float w = DANET_LDG(wt + (size_t)c * a.P);
            const float d = w * (foot_sample(pred + c * HW, a.S, f) - DANET_LDG(tgt + (size_t)c * a.P));
            l += w * sl1(d);
            coef[c] = a.pw * w * w * sl1_grad(d);
        }
        return l;
    }
    const float* pred = a.idx + (size_t)n * kDpC * HW;
    const int lab = dp_label(a.I[(size_t)n * a.P + p], kDpC);
    float mx = -INFINITY, s = 0.f, xt = 0.f;
    for (int c = 0; c < kDpC; ++c) {
        const float x = foot_sample(pred + c * HW, a.S, f);
        coef[c] = x;
        if (c == lab) xt = x;
        lse_step(x, mx, s);
    }
    if (lab < 0) {                           // rejected by the Python layer; the kernel just contributes nothing
        for (int c = 0; c < kDpC; ++c) coef[c] = 0.f;
        return 0.f;
    }
    const float inv = 1.f / s, sc = a.part_w / npts;
    for (int c = 0; c < kDpC; ++c) coef[c] = (expf(coef[c] - mx) * inv - (c == lab ? 1.f : 0.f)) * sc;
    return mx + logf(s) - xt;
}

// d loss / d pred of map m at pixel (px, py), all 25 channels: the grid_sample backward as a gather -- the
// contributions of the points whose footprint covers the pixel, in point order.  coef [P][25], feet [P].
__host__ __device__ inline void dp_pixel_grad(const DpArgs& a, int n, int m, int pix, const Foot* feet, const float* coef,
                                              float* g) {
    const int px = pix % a.S, py = pix / a.S;
    float acc[kDpC];
#pragma unroll
    for (int c = 0; c < kDpC; ++c) acc[c] = 0.f;
    for (int p = 0; p < a.P; ++p) {
        const float w = foot_weight(feet[p], px, py);
        if (w != 0.f) {
#pragma unroll
            for (int c = 0; c < kDpC; ++c) acc[c] += w * coef[p * kDpC + c];
        }
    }
    const size_t HW = (size_t)a.S * a.S;
    float* gp = g + (size_t)n * kDpC * HW + pix;
#pragma unroll
    for (int c = 0; c < kDpC; ++c) gp[c * HW] = acc[c];
}

// cross-entropy of the annotation logits at one pixel against its label (iuv_estimator.py:400-405); gradient scaled
// by `scale` (INDEX_WEIGHTS / pixels).  Out-of-range labels contribute nothing.
__host__ __device__ inline float dp_pixel_ann(const DpArgs& a, int n, int pix, float scale, bool on) {
    const size_t HW = (size_t)a.S * a.S;
    const float* x = a.ann + (size_t)n * a.Cann * HW + pix;
    const int lab = on ? dp_label(a.A[(size_t)n * HW + pix], a.Cann) : -1;
    float mx = -INFINITY, s = 0.f, xt = 0.f;
    if (lab >= 0)
        for (int c = 0; c < a.Cann; ++c) {
            const float xv = DANET_LDG(x + c * HW);
            if (c == lab) xt = xv;
            lse_step(xv, mx, s);
        }
    if (a.gann) {
        float* g = a.gann + (size_t)n * a.Cann * HW + pix;
        const float inv = lab >= 0 ? 1.f / s : 0.f;
        for (int c = 0; c < a.Cann; ++c)
            g[c * HW] = lab >= 0 ? (expf(DANET_LDG(x + c * HW) - mx) * inv - (c == lab ? 1.f : 0.f)) * scale : 0.f;
    }
    return lab >= 0 ? mx + logf(s) - xt : 0.f;
}

__device__ inline int count_selected(const uint8_t* has, int N) {
    int n = 0;
    for (int base = 0; base < N; base += blockDim.x) {
        const int i = base + (int)threadIdx.x;
        n += __syncthreads_count(i < N && (has == nullptr || has[i] != 0));
    }
    return n;
}

// fixed-order block sum of a float4 (kDpThreads threads); result valid in thread 0
__device__ inline float4 block_sum4(float4 t, float4* sm) {
    t.x = warp_sum(t.x); t.y = warp_sum(t.y); t.z = warp_sum(t.z); t.w = warp_sum(t.w);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sm[w] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
        t = sm[0];
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i) { t.x += sm[i].x; t.y += sm[i].y; t.z += sm[i].z; t.w += sm[i].w; }
    }
    return t;
}

// grid (pixel tiles, images).  Every CTA recomputes its image's per-point terms in shared memory (cheap: P x 25
// bilinear samples per map) and gathers the gradient of its pixel tile; tile 0 alone contributes the point-loss sums.
__global__ void __launch_bounds__(kDpThreads) k_dp_uvia_losses(const DpArgs a, float4* partial) {
    __shared__ Foot s_feet[kDpMaxPts];
    __shared__ float s_coef[kDpMaxPts * kDpC];
    __shared__ float4 s_red[kDpThreads / 32];
    const int n = blockIdx.y, tile = blockIdx.x, tid = threadIdx.x;
    const int HW = a.S * a.S;
    const int pix = tile * kDpThreads + tid;
    const int nsel = count_selected(a.has, a.N);
    const bool on = nsel > 0 && (a.has == nullptr || a.has[n] != 0);
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!on) {                                                  // deselected image: zero gradients, no loss
        if (pix < HW) {
            for (int m = 0; m < 3; ++m) {
                float* g = m == 0 ? a.gu : (m == 1 ? a.gv : a.gidx);
                if (g) for (int c = 0; c < kDpC; ++c) g[((size_t)n * kDpC + c) * HW + pix] = 0.f;
            }
            if (a.gann) for (int c = 0; c < a.Cann; ++c) a.gann[((size_t)n * a.Cann + c) * HW + pix] = 0.f;
        }
    } else {
        for (int p = tid; p < a.P; p += kDpThreads) s_feet[p] = dp_foot(a, n, p);
        __syncthreads();
        const float npts = (float)nsel * (float)a.P;
        for (int m = 0; m < 3; ++m) {
            float* g = m == 0 ? a.gu : (m == 1 ? a.gv : a.gidx);
            if (!g && tile != 0) continue;                      // uniform across the CTA
            float lm = 0.f;
            for (int p = tid; p < a.P; p += kDpThreads) lm += dp_point_map(a, n, p, m, s_feet[p], npts, s_coef + p * kDpC);
            if (tile == 0) { if (m == 0) t.x = lm; else if (m == 1) t.y = lm; else t.z = lm; }
            __syncthreads();
            if (g && pix < HW) dp_pixel_grad(a, n, m, pix, s_feet, s_coef, g);
            __syncthreads();
        }
        if (pix < HW) t.w = dp_pixel_ann(a, n, pix, a.index_w / ((float)nsel * (float)HW), true);
    }
    t = block_sum4(t, s_red);
    if (tid == 0) partial[(size_t)n * gridDim.x + tile] = t;
}

__global__ void __launch_bounds__(256) k_dp_finish(const float4* partial, int nblocks, const uint8_t* has, int N, int P,
                                                   int HW, float pw, float part_w, float index_w, float* losses) {
    __shared__ double sm[4][256];
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < nblocks; i += 256) {
        const float4 t = partial[i];
        s[0] += t.x; s[1] += t.y; s[2] += t.z; s[3] += t.w;
    }
    for (int k = 0; k < 4; ++k) sm[k][threadIdx.x] = s[k];
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) for (int k = 0; k < 4; ++k) sm[k][threadIdx.x] += sm[k][threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int nsel = 0;
        for (int i = 0; i < N; ++i) nsel += (has == nullptr || has[i] != 0) ? 1 : 0;
        const bool any = nsel > 0;
        losses[0] = any ? (float)(sm[0][0] * (double)pw) : 0.f;
        losses[1] = any ? (float)(sm[1][0] * (double)pw) : 0.f;
        losses[2] = any ? (float)(sm[2][0] * (double)part_w / ((double)nsel * P)) : 0.f;
        losses[3] = any ? (float)(sm[3][0] * (double)index_w / ((double)nsel * HW)) : 0.f;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// stn_kps_losses
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kStnKThreads = 256;

// the Gaussian target of utils/keypoints.py:268-331 for one joint (sigma 1, 7 x 7 window): centre and whether any
// part of the window is on the map.  k = 0.5 * gt + 0.5, mu = int(k * S + 0.5) with Python's int (truncation).
struct HmWin { int mx, my; bool on; };
__host__ __device__ inline HmWin hm_window(float gx, float gy, int S) {
    HmWin w;
    const float kx = RN_ADD(RN_MUL(gx, 0.5f), 0.5f), ky = RN_ADD(RN_MUL(gy, 0.5f), 0.5f);
    const float tx = RN_ADD(RN_MUL(kx, (float)S), 0.5f), ty = RN_ADD(RN_MUL(ky, (float)S), 0.5f);
    const float lim = 1073741824.f;                       // far outside any map: the window is skipped
    w.on = tx > -lim && tx < lim && ty > -lim && ty < lim;
    w.mx = w.on ? (int)tx : 0; w.my = w.on ? (int)ty : 0;
    w.on = w.on && !(w.mx - 3 >= S || w.my - 3 >= S || w.mx + 4 < 0 || w.my + 4 < 0);
    return w;
}
__host__ __device__ inline float hm_target(const HmWin& w, int x, int y) {
    const int dx = x - w.mx, dy = y - w.my;
    if (!w.on || dx < -3 || dx > 3 || dy < -3 || dy > 3) return 0.f;
    return expf(-(float)(dx * dx + dy * dy) / 2.f);
}

// the heat-map loss term of one pixel (un-normalised) and the gradients d loss_roi / d hm and d loss_stnhm / d hm.
// cx / cy: soft-argmax in pixel units; gcx / gcy: d loss_roi / d centre (in [-1, 1] units); ghm: hm_weight / (B*J*S^2).
struct StnPix { float l, g_roi, g_hm; };
__host__ __device__ inline StnPix stn_pixel(float h, float e_over_se, int x, int y, int S, float cx, float cy, float gcx,
                                            float gcy, const HmWin& w, float ghm, bool hm_on) {
    StnPix r;
    r.l = 0.f; r.g_hm = 0.f;
    r.g_roi = 10.f * e_over_se * (gcx * ((float)x - cx) + gcy * ((float)y - cy)) / (0.5f * (float)S);
    if (hm_on) {
        const float d = h - hm_target(w, x, y);
        r.l = sl1(d);
        r.g_hm = ghm * sl1_grad(d);
    }
    return r;
}
// one buffer for both gradients when the caller passes the same pointer twice: their sum
__host__ __device__ inline void stn_store(float* groi, float* ghm, size_t e, const StnPix& r) {
    if (groi == ghm) { if (groi) groi[e] = r.g_roi + r.g_hm; return; }
    if (groi) groi[e] = r.g_roi;
    if (ghm) ghm[e] = r.g_hm;
}
// the loss_roi term of one joint and d loss_roi / d centre, given the soft-argmax centre in [-1, 1] units
__host__ __device__ inline float stn_roi(float c_x, float c_y, const float* kp, int cols, float kps_weight, int B,
                                         float* gcx, float* gcy) {
    *gcx = *gcy = 0.f;
    if (cols < 3 || kps_weight == 0.f) return 0.f;
    const float w = kp[2];
    if (w == 0.f) return 0.f;                            // iuv_estimator.py:162-164
    const float dx = c_x - kp[0], dy = c_y - kp[1], s = kps_weight / (float)B * w;
    *gcx = s * sl1_grad(dx); *gcy = s * sl1_grad(dy);
    return w * (sl1(dx) + sl1(dy));
}

// one CTA per (image, joint): three passes over the joint's S^2 values (max; softmax sums; loss and gradient)
__global__ void __launch_bounds__(kStnKThreads) k_stn_kps_losses(int B, int J, int S, const float* __restrict__ hm,
                                                                 const float* __restrict__ kps, int cols, float kps_weight,
                                                                 float hm_weight, float* grad_roi, float* grad_hm,
                                                                 float2* __restrict__ partial) {
    __shared__ float s_red[3][kStnKThreads / 32];
    __shared__ float s_v[3];
    const int bj = blockIdx.x, tid = threadIdx.x, w = tid >> 5, l = tid & 31, nw = kStnKThreads / 32;
    const int HW = S * S;
    const float* h = hm + (size_t)bj * HW;
    float m = -INFINITY;
    for (int p = tid; p < HW; p += kStnKThreads) m = fmaxf(m, 10.f * __ldg(h + p));
    m = warp_max(m);
    if (l == 0) s_red[0][w] = m;
    __syncthreads();
    if (tid == 0) { float x = s_red[0][0]; for (int i = 1; i < nw; ++i) x = fmaxf(x, s_red[0][i]); s_v[0] = x; }
    __syncthreads();
    m = s_v[0];
    float se = 0.f, sx = 0.f, sy = 0.f;
    for (int p = tid; p < HW; p += kStnKThreads) {
        const float e = expf(10.f * __ldg(h + p) - m);
        se += e; sx = fmaf(e, (float)(p % S), sx); sy = fmaf(e, (float)(p / S), sy);
    }
    se = warp_sum(se); sx = warp_sum(sx); sy = warp_sum(sy);
    __syncthreads();
    if (l == 0) { s_red[0][w] = se; s_red[1][w] = sx; s_red[2][w] = sy; }
    __syncthreads();
    if (tid == 0) {
        float a = 0.f, bx = 0.f, by = 0.f;
        for (int i = 0; i < nw; ++i) { a += s_red[0][i]; bx += s_red[1][i]; by += s_red[2][i]; }
        s_v[0] = a; s_v[1] = bx / a; s_v[2] = by / a;
    }
    __syncthreads();
    se = s_v[0];
    const float cx = s_v[1], cy = s_v[2];                         // soft-argmax in pixel units
    const float* kp = kps + (size_t)bj * cols;
    float gcx, gcy;
    const float lroi = stn_roi(cx / (0.5f * (float)S) - 1.f, cy / (0.5f * (float)S) - 1.f, kp, cols, kps_weight, B, &gcx, &gcy);
    const bool hm_on = hm_weight != 0.f;
    const HmWin win = hm_window(kp[0], kp[1], S);
    const float ghm = hm_weight / ((float)B * (float)J * (float)HW), inv = 1.f / se;
    float lh = 0.f;
    for (int p = tid; p < HW; p += kStnKThreads) {
        const float hv = __ldg(h + p);
        const StnPix r = stn_pixel(hv, expf(10.f * hv - m) * inv, p % S, p / S, S, cx, cy, gcx, gcy, win, ghm, hm_on);
        lh += r.l;
        stn_store(grad_roi, grad_hm, (size_t)bj * HW + p, r);
    }
    lh = warp_sum(lh);
    __syncthreads();
    if (l == 0) s_red[0][w] = lh;
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
        for (int i = 0; i < nw; ++i) t += s_red[0][i];
        partial[bj] = make_float2(lroi, t);
    }
}

__global__ void __launch_bounds__(256) k_stn_finish(const float2* partial, int n, int B, int J, int HW, float kps_weight,
                                                    float hm_weight, float* losses) {
    __shared__ double sm[2][256];
    double s0 = 0.0, s1 = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) { s0 += partial[i].x; s1 += partial[i].y; }
    sm[0][threadIdx.x] = s0; sm[1][threadIdx.x] = s1;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) { sm[0][threadIdx.x] += sm[0][threadIdx.x + o]; sm[1][threadIdx.x] += sm[1][threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        losses[0] = (float)(sm[0][0] * (double)kps_weight / (double)B);
        losses[1] = (float)(sm[1][0] * (double)hm_weight / ((double)B * J * HW));
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// part_iuv_targets
// ---------------------------------------------------------------------------------------------------------------------
// utils/smpl_utlis.py:55-79 dp2smpl_mapping: the six DensePose channels of each SMPL part crop
#define DANET_DP2SMPL_MAPPING                                                                                           \
    {{7, 8, 9, 10, 1, 2}, {1, 2, 8, 10, 12, 14}, {1, 2, 7, 9, 11, 13}, {7, 8, 9, 10, 1, 2}, {1, 2, 8, 10, 12, 14},      \
     {1, 2, 7, 9, 11, 13}, {7, 8, 9, 10, 1, 2}, {8, 10, 12, 14, 5, 5}, {7, 9, 11, 13, 6, 6}, {7, 8, 9, 10, 1, 2},        \
     {8, 10, 12, 14, 5, 5}, {7, 9, 11, 13, 6, 6}, {1, 2, 23, 24, 23, 24}, {1, 2, 15, 17, 19, 21},                       \
     {1, 2, 16, 18, 20, 22}, {1, 2, 23, 24, 23, 24}, {1, 2, 15, 17, 19, 21}, {1, 2, 16, 18, 20, 22},                    \
     {1, 2, 15, 17, 19, 21}, {1, 2, 16, 18, 20, 22}, {15, 17, 19, 21, 4, 4}, {16, 18, 20, 22, 3, 3},                    \
     {15, 17, 19, 21, 4, 4}, {16, 18, 20, 22, 3, 3}}
__constant__ signed char c_dp2smpl[24][6] = DANET_DP2SMPL_MAPPING;
#ifdef DANET_LOSSES_HOST_CHECK
static const signed char h_dp2smpl[24][6] = DANET_DP2SMPL_MAPPING;
#endif

// the 21 channels (U, V, I x [background, 6 mapped]) of part `i`'s crop at output pixel (px, py) of image b:
// affine_grid + grid_sample (bilinear, zeros) of part_iuv_simp's maps.  The I background (sum of the 6 mapped I
// channels < 0.5, repeats counted twice) is evaluated at the source pixels and then interpolated, like the reference.
__host__ __device__ inline void part_target_pixel(const float* U, const float* V, const float* I, int S,
                                                  const float* th, int align, int i, int px, int py, const signed char* map,
                                                  float* out, size_t ostride) {
    const float xb = affine_base(px, S, align), yb = affine_base(py, S, align);
    const float gx = RN_ADD(RN_ADD(RN_MUL(th[0], xb), RN_MUL(th[1], yb)), th[2]);
    const float gy = RN_ADD(RN_ADD(RN_MUL(th[3], xb), RN_MUL(th[4], yb)), th[5]);
    const Foot f = make_foot(grid_unnormalize(gx, S, align), grid_unnormalize(gy, S, align), S);
    const size_t HW = (size_t)S * S;
    float acc[3][7];
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int k = 0; k < 7; ++k) acc[m][k] = 0.f;
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
        const int xx = f.x0 + (k4 & 1), yy = f.y0 + (k4 >> 1);
        if (xx < 0 || xx >= S || yy < 0 || yy >= S) continue;
        const size_t q = (size_t)yy * S + xx;
        const float w = f.w[k4];
        float isum = 0.f;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            const size_t e = (size_t)map[k] * HW + q;
            const float iv = DANET_LDG(I + e);
            isum += iv;
            acc[0][k + 1] += DANET_LDG(U + e) * w;
            acc[1][k + 1] += DANET_LDG(V + e) * w;
            acc[2][k + 1] += iv * w;
        }
        acc[2][0] += (isum < 0.5f ? 1.f : 0.f) * w;
    }
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int k = 0; k < 7; ++k) out[(m * 7 + k) * ostride] = acc[m][k];
}

// one CTA per (image, part); threads run over the crop's pixels (coalesced 21-plane writes)
__global__ void __launch_bounds__(256) k_part_iuv_targets(int S, int C, const float* __restrict__ U,
                                                          const float* __restrict__ V, const float* __restrict__ I,
                                                          const float* __restrict__ theta, int align, float* __restrict__ out) {
    const int bp = blockIdx.x, b = bp / 24, i = bp - b * 24;
    const size_t HW = (size_t)S * S, img = (size_t)b * C * HW;
    __shared__ float s_th[6];
    __shared__ signed char s_map[6];
    if (threadIdx.x < 6) { s_th[threadIdx.x] = theta[(size_t)bp * 6 + threadIdx.x]; s_map[threadIdx.x] = c_dp2smpl[i][threadIdx.x]; }
    __syncthreads();
    float* o = out + (size_t)bp * 21 * HW;
    for (int p = threadIdx.x; p < (int)HW; p += blockDim.x)
        part_target_pixel(U + img, V + img, I + img, S, s_th, align, i, p % S, p / S, s_map, o + p, HW);
}

}  // namespace danet

using namespace danet;

extern "C" int64_t danet_dp_uvia_losses_workspace_bytes(int32_t N, int32_t HW) {
    if (N < 0 || HW < 0) return -1;
    const long long blocks = (long long)N * ((HW + kDpThreads - 1) / kDpThreads);
    return (blocks > 0 ? blocks : 1) * (long long)sizeof(float4);
}

extern "C" int danet_dp_uvia_losses(int32_t N, int32_t S, int32_t Cann, int32_t P, const float* u_pred, const float* v_pred,
                                    const float* index_pred, const float* ann_pred, const float* X_points,
                                    const float* Y_points, const float* I_points, const float* U_points,
                                    const float* V_points, const float* point_weights, const float* ann_labels,
                                    const uint8_t* has_dp, int32_t align_corners, float point_weight, float part_weight,
                                    float index_weight, float* losses, float* grad_u, float* grad_v, float* grad_index,
                                    float* grad_ann, void* workspace, danet_stream_t stream) {
    DANET_CHECK(N >= 0 && S >= 1 && Cann >= 1 && P >= 1 && P <= kDpMaxPts,
                "dp_uvia_losses: bad sizes N=%d S=%d Cann=%d P=%d (1 <= P <= %d)", N, S, Cann, P, kDpMaxPts);
    DANET_CHECK(S <= 4096, "dp_uvia_losses: S=%d too large", S);
    DANET_CHECK(u_pred && v_pred && index_pred && ann_pred && X_points && Y_points && I_points && U_points && V_points &&
                point_weights && ann_labels && losses && workspace, "dp_uvia_losses: null pointer");
    const int HW = S * S, tiles = (HW + kDpThreads - 1) / kDpThreads;
    float4* partial = reinterpret_cast<float4*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    DpArgs a;
    a.N = N; a.S = S; a.Cann = Cann; a.P = P; a.align = align_corners ? 1 : 0;
    a.u = u_pred; a.v = v_pred; a.idx = index_pred; a.ann = ann_pred;
    a.X = X_points; a.Y = Y_points; a.I = I_points; a.Up = U_points; a.Vp = V_points; a.Wp = point_weights; a.A = ann_labels;
    a.has = has_dp; a.pw = point_weight; a.part_w = part_weight; a.index_w = index_weight;
    a.gu = grad_u; a.gv = grad_v; a.gidx = grad_index; a.gann = grad_ann;
    if (N > 0) {
        DANET_CHECK(N <= 65535, "dp_uvia_losses: N=%d above 65535", N);
        k_dp_uvia_losses<<<dim3(tiles, N), kDpThreads, 0, st>>>(a, partial);
        DANET_LAUNCH_CHECK();
    }
    k_dp_finish<<<1, 256, 0, st>>>(partial, N * tiles, has_dp, N, P, HW, point_weight, part_weight, index_weight, losses);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int64_t danet_stn_kps_losses_workspace_bytes(int32_t B, int32_t J) {
    if (B < 0 || J < 0) return -1;
    const long long n = (long long)B * J;
    return (n > 0 ? n : 1) * (long long)sizeof(float2);
}

extern "C" int danet_stn_kps_losses(int32_t B, int32_t J, int32_t S, const float* hm, const float* kps, int32_t kps_cols,
                                    float kps_weight, float hm_weight, float* losses, float* grad_roi, float* grad_hm,
                                    void* workspace, danet_stream_t stream) {
    DANET_CHECK(B >= 0 && J >= 1 && S >= 1 && (kps_cols == 2 || kps_cols == 3),
                "stn_kps_losses: bad sizes B=%d J=%d S=%d cols=%d", B, J, S, kps_cols);
    DANET_CHECK(hm && kps && losses && workspace, "stn_kps_losses: null pointer");
    DANET_CHECK((long long)B * J < (1LL << 31) && (long long)S * S < (1LL << 30), "stn_kps_losses: too large");
    cudaStream_t st = (cudaStream_t)stream;
    float2* partial = reinterpret_cast<float2*>(workspace);
    if (B > 0) {
        k_stn_kps_losses<<<B * J, kStnKThreads, 0, st>>>(B, J, S, hm, kps, kps_cols, kps_weight, hm_weight, grad_roi, grad_hm,
                                                       partial);
        DANET_LAUNCH_CHECK();
    }
    k_stn_finish<<<1, 256, 0, st>>>(partial, B * J, B > 0 ? B : 1, J, S * S, kps_weight, hm_weight, losses);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_part_iuv_targets(int32_t B, int32_t S, int32_t C, const float* Umap, const float* Vmap,
                                      const float* Imap, const float* theta, int32_t align_corners, float* out,
                                      danet_stream_t stream) {
    DANET_CHECK(B >= 0 && S >= 2 && C >= 25, "part_iuv_targets: bad sizes B=%d S=%d C=%d (C >= 25, S >= 2)", B, S, C);
    DANET_CHECK(Umap && Vmap && Imap && theta && out, "part_iuv_targets: null pointer");
    DANET_CHECK((long long)B * 24 < (1LL << 31) && (long long)S * S < (1LL << 30), "part_iuv_targets: too large");
    if (B == 0) return 0;
    k_part_iuv_targets<<<B * 24, 256, 0, (cudaStream_t)stream>>>(S, C, Umap, Vmap, Imap, theta, align_corners ? 1 : 0, out);
    DANET_LAUNCH_CHECK();
    return 0;
}

#ifdef DANET_LOSSES_HOST_CHECK
// Test-only (never part of libdanet_b200.so: the flag is set by the CPU tests alone): the same per-point / per-pixel
// functions walked on the host over HOST arrays, in the kernels' order of summation per point / pixel.
extern "C" int danet_test_dp_uvia_losses_host(int32_t N, int32_t S, int32_t Cann, int32_t P, const float* u, const float* v,
                                              const float* idx, const float* ann, const float* X, const float* Y,
                                              const float* I, const float* Up, const float* Vp, const float* Wp,
                                              const float* A, const uint8_t* has, int32_t align, float pw, float part_w,
                                              float index_w, float* losses, float* gu, float* gv, float* gidx, float* gann) {
    if (P < 1 || P > kDpMaxPts) return -1;
    DpArgs a;
    a.N = N; a.S = S; a.Cann = Cann; a.P = P; a.align = align ? 1 : 0;
    a.u = u; a.v = v; a.idx = idx; a.ann = ann; a.X = X; a.Y = Y; a.I = I; a.Up = Up; a.Vp = Vp; a.Wp = Wp; a.A = A;
    a.has = has; a.pw = pw; a.part_w = part_w; a.index_w = index_w; a.gu = gu; a.gv = gv; a.gidx = gidx; a.gann = gann;
    const int HW = S * S;
    int nsel = 0;
    for (int n = 0; n < N; ++n) nsel += (!has || has[n]) ? 1 : 0;
    std::vector<Foot> feet(P);
    std::vector<float> coef((size_t)P * kDpC);
    double s[4] = {0, 0, 0, 0};
    float* const gs[3] = {gu, gv, gidx};
    for (int n = 0; n < N; ++n) {
        const bool on = nsel > 0 && (!has || has[n]);
        if (!on) {
            for (int m = 0; m < 3; ++m) if (gs[m]) for (size_t e = 0; e < (size_t)kDpC * HW; ++e) gs[m][(size_t)n * kDpC * HW + e] = 0.f;
            if (gann) for (size_t e = 0; e < (size_t)Cann * HW; ++e) gann[(size_t)n * Cann * HW + e] = 0.f;
            continue;
        }
        for (int p = 0; p < P; ++p) feet[p] = dp_foot(a, n, p);
        for (int m = 0; m < 3; ++m) {
            for (int p = 0; p < P; ++p) s[m] += dp_point_map(a, n, p, m, feet[p], (float)nsel * (float)P, coef.data() + (size_t)p * kDpC);
            if (gs[m]) for (int pix = 0; pix < HW; ++pix) dp_pixel_grad(a, n, m, pix, feet.data(), coef.data(), gs[m]);
        }
        for (int pix = 0; pix < HW; ++pix) s[3] += dp_pixel_ann(a, n, pix, index_w / ((float)nsel * (float)HW), true);
    }
    const bool any = nsel > 0;
    losses[0] = any ? (float)(s[0] * pw) : 0.f;
    losses[1] = any ? (float)(s[1] * pw) : 0.f;
    losses[2] = any ? (float)(s[2] * part_w / ((double)nsel * P)) : 0.f;
    losses[3] = any ? (float)(s[3] * index_w / ((double)nsel * HW)) : 0.f;
    return 0;
}

extern "C" int danet_test_stn_kps_losses_host(int32_t B, int32_t J, int32_t S, const float* hm, const float* kps,
                                              int32_t cols, float kps_weight, float hm_weight, float* losses,
                                              float* grad_roi, float* grad_hm) {
    const int HW = S * S;
    double s0 = 0.0, s1 = 0.0;
    for (int bj = 0; bj < B * J; ++bj) {
        const float* h = hm + (size_t)bj * HW;
        float m = -INFINITY;
        for (int p = 0; p < HW; ++p) m = fmaxf(m, 10.f * h[p]);
        float se = 0.f, sx = 0.f, sy = 0.f;
        for (int p = 0; p < HW; ++p) {
            const float e = expf(10.f * h[p] - m);
            se += e; sx += e * (float)(p % S); sy += e * (float)(p / S);
        }
        const float cx = sx / se, cy = sy / se;
        const float* kp = kps + (size_t)bj * cols;
        float gcx, gcy;
        s0 += stn_roi(cx / (0.5f * (float)S) - 1.f, cy / (0.5f * (float)S) - 1.f, kp, cols, kps_weight, B, &gcx, &gcy);
        const HmWin win = hm_window(kp[0], kp[1], S);
        const float ghm = hm_weight / ((float)B * (float)J * (float)HW);
        for (int p = 0; p < HW; ++p) {
            const StnPix r = stn_pixel(h[p], expf(10.f * h[p] - m) / se, p % S, p / S, S, cx, cy, gcx, gcy, win, ghm, hm_weight != 0.f);
            s1 += r.l;
            stn_store(grad_roi, grad_hm, (size_t)bj * HW + p, r);
        }
    }
    losses[0] = (float)(s0 * kps_weight / (B > 0 ? B : 1));
    losses[1] = (float)(s1 * hm_weight / ((double)(B > 0 ? B : 1) * J * HW));
    return 0;
}

extern "C" int danet_test_part_iuv_targets_host(int32_t B, int32_t S, int32_t C, const float* U, const float* V,
                                                const float* I, const float* theta, int32_t align, float* out) {
    const size_t HW = (size_t)S * S;
    for (int bp = 0; bp < B * 24; ++bp) {
        const int b = bp / 24, i = bp % 24;
        const size_t img = (size_t)b * C * HW;
        for (size_t p = 0; p < HW; ++p)
            part_target_pixel(U + img, V + img, I + img, S, theta + (size_t)bp * 6, align ? 1 : 0, i, (int)(p % S),
                              (int)(p / S), h_dp2smpl[i], out + (size_t)bp * 21 * HW + p, HW);
    }
    return 0;
}
#endif
