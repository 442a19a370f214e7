// BatchNorm2d in training and eval mode with its backward, and the 3x3 / stride 2 / padding 1 max pool with its
// backward, on fp32 NCHW tensors: the layers of the regressor's ResNet blocks (res_module.py:27-61,393-448) that train
// around the differentiable convolution (conv.py).  No float atomics and no host synchronisation: every result repeats
// bit for bit and the calls can be captured in a CUDA graph.
//
// BatchNorm (x [N][C][HW], n = N * HW values per channel):
//   Statistics.  Training mode sums x - K and (x - K)^2 per channel in double, K = x[0][c][0] (chan_sums_partial:
//       (channel, image chunk) partials with a fixed thread assignment and tree); k_bn2d_stats_finish adds the chunks
//       in order and writes mean = K + sum (x - K) / n, var = sum (x - K)^2 / n - (mean - K)^2, invstd =
//       1 / sqrt(var + eps) and the new running statistics (momentum, unbiased variance n / (n - 1)).  K is a data
//       element, so (mean - K)^2 / var <= n - 1 whatever |mean| / std is: the subtraction loses at most log2(n) bits of
//       the double sums, where unshifted sums lose 2 log2(|mean| / std).  Eval mode uses the running statistics.  save
//       [2][C] (double) keeps mean and invstd for the backward.
//   Apply.  y = ((x - m_hi) - m_lo) * (w * invstd) + b (+ r), then ReLU (NaN stays NaN): the mean as an fp32 pair
//       (hi + lo) is subtracted before scaling, so |mean| >> std does not cancel away the deviation.
//   Backward.  dz = dy with ReLU zeroed where y <= 0 (torch's threshold_backward on the output: a NaN y passes dy).
//       One reduction gives sum dz and sum dz * (x - mean) in double; dbias = sum dz, dweight = invstd * sum dz
//       (x - mean).  One apply pass writes dx = w invstd (dz - sum dz / n - xhat * sum dz xhat / n) (training) or w invstd dz (eval), and dresidual = dz.
//   The apply passes run over the flat tensor in float4 groups; a group that straddles two (n, c) planes (planes of
//       49 or 2 elements) looks up each element's channel.
//
// Max pool: the forward stores per output the window slot (0..8, row-major) of its maximum: the first maximum wins,
// and NaN wins over numbers (torch's rule, so the slots equal its indices).  The backward is a gather: an input pixel
// adds, in row-major window order, the dy of the windows (at most four) whose slot points at it.
//
// HRNet fuse: the forward adds the nearest-upsampled terms in list order, so it is bit-identical to the reference's
// F.interpolate + add + relu chain.  The backward of a term upsampled by f is a gather: one thread per term element
// sums dy * [not y <= 0] over its f x f block in row-major order (fp32: within (f^2 - 1) 2^-24 sum |dy| of the exact
// sum).  The ReLU keeps NaN forward and passes dy at a NaN output backward, as BatchNorm's does.
//
// Branch tails (their forwards are danet_global_avgpool and danet_linear of glue.cu): the average pool's backward
// spreads dy / HW over the plane; the linear layer's backward sums dx = dy W, dW = dy^T x and db = sum dy in double, in
// index order.
#include "common.cuh"
#include <math.h>

namespace danet {
namespace bn {

constexpr int kThreads = 256;
constexpr int kCoef = 8;                         // floats of per-channel apply coefficients

// workspace: chunk partials [2][nchunk][C] (double), then coefficients [C][kCoef] (float)
static int64_t part_bytes(int N, int C, int HW) { return align_up((int64_t)2 * chan_sums_chunks(N, HW) * C * 8, 256); }
static int64_t ws_bytes(int N, int C, int HW) { return part_bytes(N, C, HW) + (int64_t)C * kCoef * 4; }

// double -> fp32 pair hi + lo
__device__ __forceinline__ void split_f(double v, float* hi, float* lo) {
    *hi = (float)v;
    *lo = (float)(v - (double)*hi);
}

// Training: chunks of sum (x - K) and sum (x - K)^2 in order, K = x[0][c][0] -> save (mean, invstd), the forward
// coefficients {m_hi, m_lo, w * invstd, b} and new_running [2][C] (mean, unbiased variance).  Eval: the running
// statistics.
__global__ void k_bn2d_stats_finish(const double* __restrict__ part, int nchunk, int C, long long n, int training,
                                    const float* __restrict__ x, int HW,
                                    const float* __restrict__ w, const float* __restrict__ b, const float* __restrict__ rm,
                                    const float* __restrict__ rv, float momentum, float eps, double* __restrict__ save,
                                    float* __restrict__ coef, float* __restrict__ new_running) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double mean, invstd;
    if (training) {
        double s1 = 0.0, s2 = 0.0;
        for (int j = 0; j < nchunk; ++j) s1 += part[(size_t)j * C + c];
        for (int j = 0; j < nchunk; ++j) s2 += part[((size_t)nchunk + j) * C + c];
        const double d = s1 / (double)n;             // mean - K
        mean = (double)x[(size_t)c * HW] + d;
        const double v0 = s2 / (double)n - d * d;
        const double var = v0 < 0.0 ? 0.0 : v0;       // rounding below 0 is clamped; NaN stays (fmax would drop it)
        invstd = 1.0 / sqrt(var + (double)eps);
        if (new_running) {
            const double m = (double)momentum;
            new_running[c] = (float)((1.0 - m) * (double)rm[c] + m * mean);
            new_running[C + c] = (float)((1.0 - m) * (double)rv[c] + m * var * ((double)n / (double)(n - 1)));
        }
    } else {
        mean = (double)rm[c];
        invstd = 1.0 / sqrt((double)rv[c] + (double)eps);
    }
    save[c] = mean;
    save[C + c] = invstd;
    float* k = coef + (size_t)c * kCoef;
    split_f(mean, &k[0], &k[1]);
    k[2] = (float)((double)w[c] * invstd);
    k[3] = b[c];
}

// Backward: chunks of sum dz and sum dz (x - mean) in order -> dbias, dweight and the dx coefficients
// {m_hi, m_lo, c1 = sum dz / n, c2 = invstd^2 sum dz (x - mean) / n, w * invstd}
__global__ void k_bn2d_grad_finish(const double* __restrict__ part, int nchunk, int C, long long n, int training,
                                   const float* __restrict__ w, const double* __restrict__ save, float* __restrict__ dweight,
                                   float* __restrict__ dbias, float* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s1 = 0.0, s2 = 0.0;
    for (int j = 0; j < nchunk; ++j) s1 += part[(size_t)j * C + c];
    for (int j = 0; j < nchunk; ++j) s2 += part[((size_t)nchunk + j) * C + c];
    const double mean = save[c], invstd = save[C + c];
    if (dbias) dbias[c] = (float)s1;
    if (dweight) dweight[c] = (float)(s2 * invstd);
    float* k = coef + (size_t)c * kCoef;
    split_f(mean, &k[0], &k[1]);
    k[2] = training ? (float)(s1 / (double)n) : 0.0f;
    k[3] = training ? (float)(s2 * invstd * invstd / (double)n) : 0.0f;
    k[4] = (float)((double)w[c] * invstd);
}

// Eval-mode backward without weight / bias gradients needs no sums: only w * invstd
__global__ void k_bn2d_eval_coef(int C, const float* __restrict__ w, const double* __restrict__ save, float* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float* k = coef + (size_t)c * kCoef;
    k[0] = k[1] = k[2] = k[3] = 0.0f;
    k[4] = (float)((double)w[c] * save[C + c]);
}

// ReLU as torch's: NaN stays NaN.  Its backward passes dy except where y <= 0, so a NaN output passes dy as torch's
// threshold_backward does (and a diverging step shows in every gradient it reaches).
__device__ __forceinline__ float relu_fwd(float v) { return (v > 0.f || v != v) ? v : 0.f; }
__device__ __forceinline__ float relu_mask(float y, float g) { return y <= 0.f ? 0.f : g; }

// channel of flat element e of [N][C][HW]
__device__ __forceinline__ int chan_of(long long e, int HW, int C) { return (int)((e / HW) % C); }

struct FwdArgs { const float* x; const float* r; const float* coef; float* y; long long total; int HW, C, relu, vec; };

__device__ __forceinline__ float bn_fwd1(const FwdArgs& a, float x, float r, int c) {
    const float4 k = __ldg(reinterpret_cast<const float4*>(a.coef + (size_t)c * kCoef));
    float v = ((x - k.x) - k.y) * k.z + k.w;
    if (a.r) v += r;
    if (a.relu) v = relu_fwd(v);
    return v;
}

__global__ void __launch_bounds__(kThreads) k_bn2d_apply(const FwdArgs a) {
    const long long e = 4 * ((long long)blockIdx.x * kThreads + threadIdx.x);
    if (e >= a.total) return;
    if (a.vec && e + 3 < a.total) {
        const float4 x = __ldg(reinterpret_cast<const float4*>(a.x + e));
        const float4 r = a.r ? __ldg(reinterpret_cast<const float4*>(a.r + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
        const long long p = e / a.HW;
        const int q = (int)(e - p * a.HW);
        float4 y;
        if (q + 3 < a.HW) {                          // one plane: one channel
            const int c = (int)(p % a.C);
            y.x = bn_fwd1(a, x.x, r.x, c); y.y = bn_fwd1(a, x.y, r.y, c);
            y.z = bn_fwd1(a, x.z, r.z, c); y.w = bn_fwd1(a, x.w, r.w, c);
        } else {
            y.x = bn_fwd1(a, x.x, r.x, chan_of(e, a.HW, a.C)); y.y = bn_fwd1(a, x.y, r.y, chan_of(e + 1, a.HW, a.C));
            y.z = bn_fwd1(a, x.z, r.z, chan_of(e + 2, a.HW, a.C)); y.w = bn_fwd1(a, x.w, r.w, chan_of(e + 3, a.HW, a.C));
        }
        *reinterpret_cast<float4*>(a.y + e) = y;
        return;
    }
    for (long long i = e; i < e + 4 && i < a.total; ++i)
        a.y[i] = bn_fwd1(a, __ldg(a.x + i), a.r ? __ldg(a.r + i) : 0.0f, chan_of(i, a.HW, a.C));
}

struct BwdArgs {
    const float* dy; const float* y; const float* x; const float* coef; float* dx; float* dres;
    long long total; int HW, C, training, vec;
};

// dz, and dx when a.dx is set
__device__ __forceinline__ float bn_bwd1(const BwdArgs& a, float dy, float y, float x, int c, float* dx) {
    const float dz = a.y ? relu_mask(y, dy) : dy;
    if (a.dx) {
        const float* k = a.coef + (size_t)c * kCoef;
        const float kk = __ldg(k + 4);
        if (a.training) {
            const float4 m = __ldg(reinterpret_cast<const float4*>(k));
            *dx = (dz - m.z - ((x - m.x) - m.y) * m.w) * kk;
        } else {
            *dx = dz * kk;
        }
    }
    return dz;
}

__global__ void __launch_bounds__(kThreads) k_bn2d_bwd_apply(const BwdArgs a) {
    const long long e = 4 * ((long long)blockIdx.x * kThreads + threadIdx.x);
    if (e >= a.total) return;
    const bool need_x = a.dx && a.training;
    if (a.vec && e + 3 < a.total) {
        const float4 dy = __ldg(reinterpret_cast<const float4*>(a.dy + e));
        const float4 y = a.y ? __ldg(reinterpret_cast<const float4*>(a.y + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 x = need_x ? __ldg(reinterpret_cast<const float4*>(a.x + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
        const long long p = e / a.HW;
        const int q = (int)(e - p * a.HW);
        int c0, c1, c2, c3;
        if (q + 3 < a.HW) {
            c0 = c1 = c2 = c3 = (int)(p % a.C);
        } else {
            c0 = chan_of(e, a.HW, a.C); c1 = chan_of(e + 1, a.HW, a.C);
            c2 = chan_of(e + 2, a.HW, a.C); c3 = chan_of(e + 3, a.HW, a.C);
        }
        float4 dz, dx;
        dz.x = bn_bwd1(a, dy.x, y.x, x.x, c0, &dx.x); dz.y = bn_bwd1(a, dy.y, y.y, x.y, c1, &dx.y);
        dz.z = bn_bwd1(a, dy.z, y.z, x.z, c2, &dx.z); dz.w = bn_bwd1(a, dy.w, y.w, x.w, c3, &dx.w);
        if (a.dx) *reinterpret_cast<float4*>(a.dx + e) = dx;
        if (a.dres) *reinterpret_cast<float4*>(a.dres + e) = dz;
        return;
    }
    for (long long i = e; i < e + 4 && i < a.total; ++i) {
        float dx = 0.0f;
        const float dz = bn_bwd1(a, __ldg(a.dy + i), a.y ? __ldg(a.y + i) : 0.0f, need_x ? __ldg(a.x + i) : 0.0f,
                                 chan_of(i, a.HW, a.C), &dx);
        if (a.dx) a.dx[i] = dx;
        if (a.dres) a.dres[i] = dz;
    }
}

// ------------------------------------------------------------------------------------------------
// max pool 3x3 / stride 2 / padding 1, NCHW
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_maxpool3x3s2_fwd(long long total, int H, int W, int Ho, int Wo, const float* __restrict__ x, float* __restrict__ y,
                   uint8_t* __restrict__ slot) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= total) return;
    const long long p = i / ((long long)Ho * Wo);
    const int r = (int)(i - p * Ho * Wo), oh = r / Wo, ow = r - oh * Wo;
    const float* xp = x + p * H * W;
    const int h0 = 2 * oh - 1, w0 = 2 * ow - 1;
    const int hs = max(h0, 0), he = min(h0 + 3, H), ws = max(w0, 0), we = min(w0 + 3, W);
    float m = -INFINITY;
    int best = (hs - h0) * 3 + (ws - w0);
    for (int h = hs; h < he; ++h)
        for (int w = ws; w < we; ++w) {
            const float v = __ldg(xp + h * W + w);
            if (v > m || isnan(v)) { m = v; best = (h - h0) * 3 + (w - w0); }
        }
    y[i] = m;
    slot[i] = (uint8_t)best;
}

__global__ void __launch_bounds__(kThreads)
k_maxpool3x3s2_bwd(long long total, int H, int W, int Ho, int Wo, const float* __restrict__ dy,
                   const uint8_t* __restrict__ slot, float* __restrict__ dx) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= total) return;
    const long long p = i / ((long long)H * W);
    const int r = (int)(i - p * H * W), h = r / W, w = r - h * W;
    const size_t base = (size_t)p * Ho * Wo;
    float acc = 0.0f;
    // windows oh with 2 oh - 1 <= h <= 2 oh + 1, in row-major order
    for (int oh = h >> 1; oh <= min((h + 1) >> 1, Ho - 1); ++oh)
        for (int ow = w >> 1; ow <= min((w + 1) >> 1, Wo - 1); ++ow) {
            const size_t o = base + (size_t)oh * Wo + ow;
            const int s = __ldg(slot + o);
            if (2 * oh - 1 + s / 3 == h && 2 * ow - 1 + s % 3 == w) acc += __ldg(dy + o);
        }
    dx[i] = acc;
}

// ------------------------------------------------------------------------------------------------
// tails of the regressor branches: global average pool and linear layer, backward
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_global_avgpool_bwd(long long total, int HW, const float* __restrict__ dy, float* __restrict__ dx) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= total) return;
    dx[i] = __ldg(dy + i / HW) / (float)HW;
}

// One thread per output element over the flat index space [dx: N * In | dW: Out * In | db: Out] (a part is empty when
// its output is NULL).  Every sum runs in double in index order: no atomics, bit-identical on every run.
__global__ void __launch_bounds__(kThreads)
k_linear_bwd(int N, int In, int Out, long long ndx, long long ndw, long long ndb, const float* __restrict__ x,
             const float* __restrict__ w, const float* __restrict__ dy, float* __restrict__ dx, float* __restrict__ dw,
             float* __restrict__ db) {
    long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i < ndx) {                                  // dx[n,i] = sum_o dy[n,o] w[o,i]
        const int n = (int)(i / In), k = (int)(i - (long long)n * In);
        double s = 0.0;
        for (int o = 0; o < Out; ++o) s += (double)__ldg(dy + (size_t)n * Out + o) * (double)__ldg(w + (size_t)o * In + k);
        dx[i] = (float)s;
        return;
    }
    i -= ndx;
    if (i < ndw) {                                  // dW[o,i] = sum_n dy[n,o] x[n,i]
        const int o = (int)(i / In), k = (int)(i - (long long)o * In);
        double s = 0.0;
        for (int n = 0; n < N; ++n) s += (double)__ldg(dy + (size_t)n * Out + o) * (double)__ldg(x + (size_t)n * In + k);
        dw[i] = (float)s;
        return;
    }
    i -= ndw;
    if (i < ndb) {                                  // db[o] = sum_n dy[n,o]
        double s = 0.0;
        for (int n = 0; n < N; ++n) s += (double)__ldg(dy + (size_t)n * Out + i);
        db[i] = (float)s;
    }
}

// ------------------------------------------------------------------------------------------------
// HRNet fuse (hr_module.py:161-179): y = relu(up(t_0) + up(t_1) + ...), nearest upsampling by 1, 2, 4 or 8
// ------------------------------------------------------------------------------------------------
struct FuseArgs { const float* t[4]; int sh[4]; int n; };     // sh = log2 of the upsample factor

// Forward: a thread writes V consecutive outputs of one row (V = 4: 16-byte stores, and 16-/8-byte loads of the
// terms at factor 1 / 2).  The terms are added in list order, each sum rounded on its own, as the reference's
// y = y + term chain.
template <int V>
__global__ void __launch_bounds__(kThreads)
k_hr_fuse_fwd(long long items, int H, int W, const FuseArgs a, int relu, float* __restrict__ y) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= items) return;
    const int WV = W / V;
    const long long row = i / WV;                    // (n * C + c) * H + h
    const int w = (int)(i - row * WV) * V;
    const long long nc = row / H;
    const int h = (int)(row - nc * H);
    float acc[V];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j >= a.n) break;
        const int sh = a.sh[j], Wj = W >> sh;
        const float* src = a.t[j] + (size_t)(nc * (H >> sh) + (h >> sh)) * Wj;
        float v[V];
        if (V == 4 && sh == 0) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(src + w));
            v[0] = t.x; v[1 % V] = t.y; v[2 % V] = t.z; v[3 % V] = t.w;
        } else if (V == 4 && sh == 1) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(src + (w >> 1)));
            v[0] = t.x; v[1 % V] = t.x; v[2 % V] = t.y; v[3 % V] = t.y;
        } else {
#pragma unroll
            for (int k = 0; k < V; ++k) v[k] = __ldg(src + ((w + k) >> sh));
        }
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = j == 0 ? v[k] : __fadd_rn(acc[k], v[k]);
    }
    if (relu) {
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = relu_fwd(acc[k]);
    }
    float* o = y + (size_t)row * W + w;
    if (V == 4) *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1 % V], acc[2 % V], acc[3 % V]);
    else o[0] = acc[0];
}

// dy masked by the ReLU on the output: no gradient where y <= 0 (an exact 0 sum included), dy where y > 0 or NaN
__device__ __forceinline__ float relu_bwd(float g, const float* y, size_t e) { return y ? relu_mask(__ldg(y + e), g) : g; }

// Backward of one term upsampled by F: a thread owns one element of dterm and sums relu_mask(y, dy) over its F x F block in
// row-major order (fp32).  VEC: the block's rows are read as 8- (F = 2) or 16-byte (F = 4, 8) vectors.
template <int F, bool VEC>
__global__ void __launch_bounds__(kThreads)
k_hr_fuse_bwd(long long items, int Hj, int Wj, const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dt) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= items) return;
    const long long row = i / Wj;                    // (n * C + c) * Hj + hj
    const int wj = (int)(i - row * Wj);
    const long long nc = row / Hj;
    const int hj = (int)(row - nc * Hj), W = Wj * F;
    float acc = 0.f;
#pragma unroll
    for (int r = 0; r < F; ++r) {
        const size_t e = (size_t)((nc * Hj + hj) * F + r) * W + (size_t)wj * F;
        if (VEC && F == 2) {
            const float2 g = __ldg(reinterpret_cast<const float2*>(dy + e));
            float2 t = make_float2(1.f, 1.f);
            if (y) t = __ldg(reinterpret_cast<const float2*>(y + e));
            acc += relu_mask(t.x, g.x);
            acc += relu_mask(t.y, g.y);
        } else if (VEC && F >= 4) {
#pragma unroll
            for (int q = 0; q < F; q += 4) {
                const float4 g = __ldg(reinterpret_cast<const float4*>(dy + e + q));
                float4 t = make_float4(1.f, 1.f, 1.f, 1.f);
                if (y) t = __ldg(reinterpret_cast<const float4*>(y + e + q));
                acc += relu_mask(t.x, g.x);
                acc += relu_mask(t.y, g.y);
                acc += relu_mask(t.z, g.z);
                acc += relu_mask(t.w, g.w);
            }
        } else {
#pragma unroll
            for (int q = 0; q < F; ++q) acc += relu_bwd(__ldg(dy + e + q), y, e + q);
        }
    }
    dt[i] = acc;
}

// Backward of a term at factor 1: dterm = relu_mask(y, dy), 16-byte vectors when aligned
__global__ void __launch_bounds__(kThreads)
k_hr_fuse_bwd1(long long total, int vec, const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dt) {
    const long long e = 4 * ((long long)blockIdx.x * kThreads + threadIdx.x);
    if (e >= total) return;
    if (vec && e + 3 < total) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(dy + e));
        float4 o = g;
        if (y) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(y + e));
            o = make_float4(relu_mask(t.x, g.x), relu_mask(t.y, g.y), relu_mask(t.z, g.z), relu_mask(t.w, g.w));
        }
        *reinterpret_cast<float4*>(dt + e) = o;
        return;
    }
    for (long long k = e; k < e + 4 && k < total; ++k) dt[k] = relu_bwd(__ldg(dy + k), y, (size_t)k);
}

static unsigned grid_of(long long work) { return (unsigned)((work + kThreads - 1) / kThreads); }

}  // namespace bn
}  // namespace danet

using namespace danet;

static bool bn_shape_ok(int32_t N, int32_t C, int32_t HW) {
    return N >= 1 && C >= 1 && HW >= 1 && (long long)N * C * HW < (1LL << 31) && chan_sums_chunks(N, HW) < 65536;
}

extern "C" int64_t danet_bn2d_workspace_bytes(int32_t N, int32_t C, int32_t HW) {
    if (!bn_shape_ok(N, C, HW)) return 0;
    return bn::ws_bytes(N, C, HW);
}

extern "C" int danet_bn2d_forward(int32_t N, int32_t C, int32_t HW, const float* x, const float* weight, const float* bias,
                                  const float* running_mean, const float* running_var, int32_t training, float momentum,
                                  float eps, const float* residual, int32_t relu, float* y, double* save, float* new_running,
                                  void* workspace, danet_stream_t stream) {
    DANET_CHECK(bn_shape_ok(N, C, HW), "danet_bn2d_forward: bad sizes N=%d C=%d HW=%d", N, C, HW);
    DANET_CHECK(x && y && weight && bias && running_mean && running_var && save,
                "danet_bn2d_forward: x, y, weight, bias, running statistics and save must be non-null");
    DANET_CHECK(workspace && aligned16(workspace), "danet_bn2d_forward: workspace must be non-null and 16-byte aligned");
    DANET_CHECK(!training || (long long)N * HW > 1, "danet_bn2d_forward: training needs more than one value per channel");
    cudaStream_t st = (cudaStream_t)stream;
    double* part = (double*)workspace;
    float* coef = (float*)((char*)workspace + bn::part_bytes(N, C, HW));
    if (training) {
        const ChanSums s = {x, nullptr, x, nullptr, x};
        if (chan_sums_partial(s, true, N, C, HW, part, st) != 0) return -3;
    }
    bn::k_bn2d_stats_finish<<<cdiv(C, 128), 128, 0, st>>>(part, chan_sums_chunks(N, HW), C, (long long)N * HW, training,
                                                          x, HW, weight, bias, running_mean, running_var, momentum, eps, save, coef,
                                                          training ? new_running : nullptr);
    bn::FwdArgs a;
    a.x = x; a.r = residual; a.coef = coef; a.y = y; a.total = (long long)N * C * HW; a.HW = HW; a.C = C; a.relu = relu != 0;
    a.vec = aligned16(x) && aligned16(y) && (!residual || aligned16(residual));
    bn::k_bn2d_apply<<<bn::grid_of((a.total + 3) / 4), bn::kThreads, 0, st>>>(a);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_bn2d_backward(int32_t N, int32_t C, int32_t HW, const float* x, const float* y, const float* dy,
                                   const float* weight, const double* save, int32_t training, int32_t relu, float* dx,
                                   float* dweight, float* dbias, float* dresidual, void* workspace, danet_stream_t stream) {
    DANET_CHECK(bn_shape_ok(N, C, HW), "danet_bn2d_backward: bad sizes N=%d C=%d HW=%d", N, C, HW);
    DANET_CHECK(x && dy && weight && save, "danet_bn2d_backward: x, dy, weight and save must be non-null");
    DANET_CHECK(!relu || y, "danet_bn2d_backward: relu needs the forward's output y");
    DANET_CHECK(workspace && aligned16(workspace), "danet_bn2d_backward: workspace must be non-null and 16-byte aligned");
    DANET_CHECK(!training || (long long)N * HW > 1, "danet_bn2d_backward: training needs more than one value per channel");
    cudaStream_t st = (cudaStream_t)stream;
    double* part = (double*)workspace;
    float* coef = (float*)((char*)workspace + bn::part_bytes(N, C, HW));
    const float* mask = relu ? y : nullptr;
    const bool sums = dweight || dbias || (dx && training);
    if (sums) {
        const ChanSums s = {dy, mask, x, save, nullptr};
        if (chan_sums_partial(s, true, N, C, HW, part, st) != 0) return -3;
        bn::k_bn2d_grad_finish<<<cdiv(C, 128), 128, 0, st>>>(part, chan_sums_chunks(N, HW), C, (long long)N * HW, training,
                                                             weight, save, dweight, dbias, coef);
    } else if (dx) {
        bn::k_bn2d_eval_coef<<<cdiv(C, 128), 128, 0, st>>>(C, weight, save, coef);
    }
    if (dx || dresidual) {
        bn::BwdArgs a;
        a.dy = dy; a.y = mask; a.x = x; a.coef = coef; a.dx = dx; a.dres = dresidual;
        a.total = (long long)N * C * HW; a.HW = HW; a.C = C; a.training = training != 0;
        a.vec = aligned16(dy) && aligned16(x) && (!mask || aligned16(mask)) && (!dx || aligned16(dx)) &&
                (!dresidual || aligned16(dresidual));
        bn::k_bn2d_bwd_apply<<<bn::grid_of((a.total + 3) / 4), bn::kThreads, 0, st>>>(a);
    }
    DANET_LAUNCH_CHECK();
    return 0;
}

static bool pool_shape_ok(int32_t N, int32_t C, int32_t H, int32_t W) {
    return N >= 1 && C >= 1 && H >= 1 && W >= 1 && (long long)N * C * H * W < (1LL << 31);
}

extern "C" int danet_maxpool3x3s2_nchw_forward(int32_t N, int32_t C, int32_t H, int32_t W, const float* x, float* y,
                                               uint8_t* slot, danet_stream_t stream) {
    DANET_CHECK(pool_shape_ok(N, C, H, W), "danet_maxpool3x3s2_nchw_forward: bad sizes N=%d C=%d H=%d W=%d", N, C, H, W);
    DANET_CHECK(x && y && slot, "danet_maxpool3x3s2_nchw_forward: x, y and slot must be non-null");
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    const long long total = (long long)N * C * Ho * Wo;
    bn::k_maxpool3x3s2_fwd<<<bn::grid_of(total), bn::kThreads, 0, (cudaStream_t)stream>>>(total, H, W, Ho, Wo, x, y, slot);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_maxpool3x3s2_nchw_backward(int32_t N, int32_t C, int32_t H, int32_t W, const float* dy,
                                                const uint8_t* slot, float* dx, danet_stream_t stream) {
    DANET_CHECK(pool_shape_ok(N, C, H, W), "danet_maxpool3x3s2_nchw_backward: bad sizes N=%d C=%d H=%d W=%d", N, C, H, W);
    DANET_CHECK(dy && slot && dx, "danet_maxpool3x3s2_nchw_backward: dy, slot and dx must be non-null");
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    const long long total = (long long)N * C * H * W;
    bn::k_maxpool3x3s2_bwd<<<bn::grid_of(total), bn::kThreads, 0, (cudaStream_t)stream>>>(total, H, W, Ho, Wo, dy, slot, dx);
    DANET_LAUNCH_CHECK();
    return 0;
}

static bool fuse_factor_ok(int32_t f, int32_t H, int32_t W) {
    return (f == 1 || f == 2 || f == 4 || f == 8) && H % f == 0 && W % f == 0;
}

static int fuse_shift(int32_t f) { return f == 8 ? 3 : f == 4 ? 2 : f == 2 ? 1 : 0; }

extern "C" int danet_hr_fuse_forward(int32_t N, int32_t C, int32_t H, int32_t W, int32_t nterms, const float* const* terms,
                                     const int32_t* factors, int32_t relu, float* y, danet_stream_t stream) {
    DANET_CHECK(pool_shape_ok(N, C, H, W), "danet_hr_fuse_forward: bad sizes N=%d C=%d H=%d W=%d", N, C, H, W);
    DANET_CHECK(nterms >= 1 && nterms <= 4, "danet_hr_fuse_forward: %d terms (1 to 4 are supported)", nterms);
    DANET_CHECK(terms && factors && y, "danet_hr_fuse_forward: terms, factors and y must be non-null");
    bn::FuseArgs a;
    a.n = nterms;
    bool vec = (W % 4) == 0 && aligned16(y);
    for (int j = 0; j < 4; ++j) {
        a.t[j] = nullptr; a.sh[j] = 0;
        if (j >= nterms) continue;
        DANET_CHECK(terms[j], "danet_hr_fuse_forward: term %d is null", j);
        DANET_CHECK(fuse_factor_ok(factors[j], H, W), "danet_hr_fuse_forward: factor %d of term %d must be 1, 2, 4 or 8 and "
                    "divide H=%d and W=%d", factors[j], j, H, W);
        a.t[j] = terms[j]; a.sh[j] = fuse_shift(factors[j]);
        vec = vec && (a.sh[j] == 0 ? aligned16(terms[j]) : a.sh[j] == 1 ? ((uintptr_t)terms[j] & 7) == 0 : true);
    }
    const long long total = (long long)N * C * H * W;
    if (vec) bn::k_hr_fuse_fwd<4><<<bn::grid_of(total / 4), bn::kThreads, 0, (cudaStream_t)stream>>>(total / 4, H, W, a, relu, y);
    else bn::k_hr_fuse_fwd<1><<<bn::grid_of(total), bn::kThreads, 0, (cudaStream_t)stream>>>(total, H, W, a, relu, y);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_hr_fuse_backward(int32_t N, int32_t C, int32_t H, int32_t W, int32_t factor, const float* dy,
                                      const float* y, float* dterm, danet_stream_t stream) {
    DANET_CHECK(pool_shape_ok(N, C, H, W), "danet_hr_fuse_backward: bad sizes N=%d C=%d H=%d W=%d", N, C, H, W);
    DANET_CHECK(fuse_factor_ok(factor, H, W), "danet_hr_fuse_backward: factor %d must be 1, 2, 4 or 8 and divide H=%d and "
                "W=%d", factor, H, W);
    DANET_CHECK(dy && dterm, "danet_hr_fuse_backward: dy and dterm must be non-null");
    cudaStream_t st = (cudaStream_t)stream;
    const int Hj = H / factor, Wj = W / factor;
    const long long items = (long long)N * C * Hj * Wj;
    const bool vec = aligned16(dy) && (!y || aligned16(y));
    switch (factor) {
        case 1: bn::k_hr_fuse_bwd1<<<bn::grid_of((items + 3) / 4), bn::kThreads, 0, st>>>(items, vec && aligned16(dterm), dy, y, dterm); break;
        case 2: if (vec) bn::k_hr_fuse_bwd<2, true><<<bn::grid_of(items), bn::kThreads, 0, st>>>(items, Hj, Wj, dy, y, dterm);
                else bn::k_hr_fuse_bwd<2, false><<<bn::grid_of(items), bn::kThreads, 0, st>>>(items, Hj, Wj, dy, y, dterm);
                break;
        case 4: if (vec) bn::k_hr_fuse_bwd<4, true><<<bn::grid_of(items), bn::kThreads, 0, st>>>(items, Hj, Wj, dy, y, dterm);
                else bn::k_hr_fuse_bwd<4, false><<<bn::grid_of(items), bn::kThreads, 0, st>>>(items, Hj, Wj, dy, y, dterm);
                break;
        default: if (vec) bn::k_hr_fuse_bwd<8, true><<<bn::grid_of(items), bn::kThreads, 0, st>>>(items, Hj, Wj, dy, y, dterm);
                 else bn::k_hr_fuse_bwd<8, false><<<bn::grid_of(items), bn::kThreads, 0, st>>>(items, Hj, Wj, dy, y, dterm);
                 break;
    }
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_global_avgpool_backward(int32_t NC, int32_t HW, const float* dy, float* dx, danet_stream_t stream) {
    DANET_CHECK(NC >= 1 && HW >= 1 && (long long)NC * HW < (1LL << 31), "danet_global_avgpool_backward: bad sizes NC=%d HW=%d",
                NC, HW);
    DANET_CHECK(dy && dx, "danet_global_avgpool_backward: dy and dx must be non-null");
    const long long total = (long long)NC * HW;
    bn::k_global_avgpool_bwd<<<bn::grid_of(total), bn::kThreads, 0, (cudaStream_t)stream>>>(total, HW, dy, dx);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_linear_backward(int32_t N, int32_t In, int32_t Out, const float* x, const float* w, const float* dy,
                                     float* dx, float* dw, float* db, danet_stream_t stream) {
    DANET_CHECK(N >= 1 && In >= 1 && Out >= 1 && (long long)N * In < (1LL << 31) && (long long)Out * In < (1LL << 31) &&
                (long long)N * Out < (1LL << 31), "danet_linear_backward: bad sizes N=%d In=%d Out=%d", N, In, Out);
    DANET_CHECK(dy, "danet_linear_backward: dy must be non-null");
    DANET_CHECK(!dx || w, "danet_linear_backward: dx needs the weight w");
    DANET_CHECK(!dw || x, "danet_linear_backward: dw needs the input x");
    const long long ndx = dx ? (long long)N * In : 0, ndw = dw ? (long long)Out * In : 0, ndb = db ? Out : 0;
    const long long total = ndx + ndw + ndb;
    if (total == 0) return 0;
    bn::k_linear_bwd<<<bn::grid_of(total), bn::kThreads, 0, (cudaStream_t)stream>>>(N, In, Out, ndx, ndw, ndb, x, w, dy, dx,
                                                                                   dw, db);
    DANET_LAUNCH_CHECK();
    return 0;
}
