// Memory-bound fp32 glue kernels of the DaNet network half (NHWC activations).
// Each replaces a chain of small ATen launches in the reference; citations per kernel.
// Their launchers (launchers.cuh) are internal, run by the network program's step decoder (net.cu); the
// activations are padded to 8 channels, so the pools, the fuse and the STN sampler only have 8-channel kernels.
// danet_global_avgpool, danet_linear and danet_iuvmap_clean_nchw are C ABI entries of their own.
#include "launchers.cuh"
#include "stn_common.cuh"
#include <cuda_fp16.h>
#include <math.h>

namespace danet {

// ------------------------------------------------------------------------------------------
// NCHW image -> NHWC padded (input boundary of the network; demo.py:106 / eval.py:147 tensors)
// ------------------------------------------------------------------------------------------
__global__ void k_nchw_to_nhwc(int N, int C, int HW, int Cp, const float* __restrict__ x, ActV y) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)N * HW) return;
    const int n = (int)(i / HW), p = (int)(i % HW);
    if ((Cp & 3) == 0) {
        // 16-byte (fp32) / 8-byte (fp16 planes) stores per 4 channels; reads are coalesced across pixels
        for (int c = 0; c < Cp; c += 4) {
            float4 v;
            v.x = c + 0 < C ? x[((size_t)n * C + c + 0) * HW + p] : 0.0f;
            v.y = c + 1 < C ? x[((size_t)n * C + c + 1) * HW + p] : 0.0f;
            v.z = c + 2 < C ? x[((size_t)n * C + c + 2) * HW + p] : 0.0f;
            v.w = c + 3 < C ? x[((size_t)n * C + c + 3) * HW + p] : 0.0f;
            act_st4(y, i * Cp + c, v);
        }
        return;
    }
    for (int c = 0; c < Cp; ++c) act_st1(y, i * Cp + c, c < C ? x[((size_t)n * C + c) * HW + p] : 0.0f);
}

// 24 per-part iuvmap_clean calls of danet.py:93-98 in one pass (one thread per pixel; rows are read and
// written as 16-byte vectors when Cx, Cy are multiples of 4 -- they are, the graph pads channels)
template <bool VEC>
__global__ void k_iuv_clean_parts(int N, int HW, int Cx, int Cy, const float* __restrict__ x,
                                  ActV y, float* raw) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)N * HW) return;
    const float* h = x + i * Cx;
    float v[24];
    if (VEC) {
#pragma unroll
        for (int c = 0; c < 6; ++c) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(h) + c);
            v[4 * c] = t.x; v[4 * c + 1] = t.y; v[4 * c + 2] = t.z; v[4 * c + 3] = t.w;
        }
    } else {
#pragma unroll
        for (int c = 0; c < 21; ++c) v[c] = h[c];
    }
    const int best = argmax_first(v + 14, 7);
    float ov[24];
#pragma unroll
    for (int c = 0; c < 7; ++c) {
        const float oh = (c == best) ? 1.0f : 0.0f;
        ov[c] = oh * v[c]; ov[7 + c] = oh * v[7 + c]; ov[14 + c] = oh;
    }
    ov[21] = ov[22] = ov[23] = 0.0f;
    if (VEC) {
#pragma unroll
        for (int c = 0; c < 6; ++c) act_st4(y, i * Cy + 4 * c, make_float4(ov[4 * c], ov[4 * c + 1], ov[4 * c + 2], ov[4 * c + 3]));
        for (int c = 24; c < Cy; ++c) act_st1(y, i * Cy + c, 0.0f);
    } else {
#pragma unroll
        for (int c = 0; c < 21; ++c) act_st1(y, i * Cy + c, ov[c]);
        for (int c = 21; c < Cy; ++c) act_st1(y, i * Cy + c, 0.0f);
    }
    if (raw) {
        const size_t n = i / HW, pix = i - n * HW;
#pragma unroll
        for (int c = 0; c < 21; ++c) raw[(n * 21 + c) * HW + pix] = v[c];
    }
}

// ------------------------------------------------------------------------------------------
// soft-argmax centres + part visibility + affine thetas
// (utils/keypoints.py:372-394, iuv_estimator.py:137-140,176-184,262-301)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float bilinear_point(const uint8_t* amax, int S, unsigned mask, float gx, float gy,
                                                int align_corners) {
    float ix, iy;
    if (align_corners) { ix = (gx + 1.0f) * 0.5f * (float)(S - 1); iy = (gy + 1.0f) * 0.5f * (float)(S - 1); }
    else { ix = ((gx + 1.0f) * (float)S - 1.0f) * 0.5f; iy = ((gy + 1.0f) * (float)S - 1.0f) * 0.5f; }
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float tx = ix - fx, ty = iy - fy;
    float acc = 0.0f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const int xx = x0 + dx, yy = y0 + dy;
            if (xx < 0 || xx >= S || yy < 0 || yy >= S) continue;
            const float val = ((mask >> amax[yy * S + xx]) & 1u) ? 1.0f : 0.0f;
            acc += val * (dx ? tx : 1.0f - tx) * (dy ? ty : 1.0f - ty);
        }
    return acc;
}

constexpr int kStnThreads = 256;

__global__ void __launch_bounds__(kStnThreads)
k_stn_params(int B, int S, int Chm, const float* __restrict__ hm, const uint8_t* __restrict__ amax,
             const float* __restrict__ ratio, const float* __restrict__ offset, float vis_thresh,
             int align_corners, float* __restrict__ centers, float* __restrict__ theta) {
    __shared__ float s_red[kStnThreads / 32][24 * 3];
    __shared__ float s_max[24];
    __shared__ float s_c[24][2];
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int HW = S * S;
    const float* h = hm + (size_t)b * HW * Chm;
    // pass 1: per-joint max of 10*hm
    float mx[24];
#pragma unroll
    for (int j = 0; j < 24; ++j) mx[j] = -INFINITY;
    for (int p = tid; p < HW; p += kStnThreads) {
        const float4* r = reinterpret_cast<const float4*>(h + (size_t)p * Chm);
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            const float4 v = r[q];
            mx[q * 4 + 0] = fmaxf(mx[q * 4 + 0], 10.0f * v.x); mx[q * 4 + 1] = fmaxf(mx[q * 4 + 1], 10.0f * v.y);
            mx[q * 4 + 2] = fmaxf(mx[q * 4 + 2], 10.0f * v.z); mx[q * 4 + 3] = fmaxf(mx[q * 4 + 3], 10.0f * v.w);
        }
    }
#pragma unroll
    for (int j = 0; j < 24; ++j) { const float m = warp_max(mx[j]); if (lane == 0) s_red[warp][j] = m; }
    __syncthreads();
    if (tid < 24) {
        float m = s_red[0][tid];
        for (int w = 1; w < kStnThreads / 32; ++w) m = fmaxf(m, s_red[w][tid]);
        s_max[tid] = m;
    }
    __syncthreads();
    // pass 2: sum exp, sum exp*x, sum exp*y
    float se[24], sx[24], sy[24];
#pragma unroll
    for (int j = 0; j < 24; ++j) { se[j] = 0.f; sx[j] = 0.f; sy[j] = 0.f; mx[j] = s_max[j]; }
    for (int p = tid; p < HW; p += kStnThreads) {
        const float px = (float)(p % S), py = (float)(p / S);
        const float* r = h + (size_t)p * Chm;
#pragma unroll
        for (int j = 0; j < 24; ++j) {
            const float e = expf(10.0f * r[j] - mx[j]);
            se[j] += e; sx[j] = fmaf(e, px, sx[j]); sy[j] = fmaf(e, py, sy[j]);
        }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 24; ++j) {
        const float a = warp_sum(se[j]), bx = warp_sum(sx[j]), by = warp_sum(sy[j]);
        if (lane == 0) { s_red[warp][j * 3] = a; s_red[warp][j * 3 + 1] = bx; s_red[warp][j * 3 + 2] = by; }
    }
    __syncthreads();
    if (tid < 24) {
        float a = 0.f, bx = 0.f, by = 0.f;
        for (int w = 0; w < kStnThreads / 32; ++w) { a += s_red[w][tid * 3]; bx += s_red[w][tid * 3 + 1]; by += s_red[w][tid * 3 + 2]; }
        // stn_centers = softargmax / (0.5*S) - 1  (iuv_estimator.py:137-140)
        const float cx = (bx / a) / (0.5f * (float)S) - 1.0f;
        const float cy = (by / a) / (0.5f * (float)S) - 1.0f;
        s_c[tid][0] = cx; s_c[tid][1] = cy;
        centers[((size_t)b * 24 + tid) * 2] = cx;
        centers[((size_t)b * 24 + tid) * 2 + 1] = cy;
    }
    __syncthreads();
    if (tid < 24) {
        const int i = tid;
        float xmin = s_c[0][0], xmax = xmin, ymin = s_c[0][1], ymax = ymin;
        for (int j = 1; j < 24; ++j) {
            xmin = fminf(xmin, s_c[j][0]); xmax = fmaxf(xmax, s_c[j][0]);
            ymin = fminf(ymin, s_c[j][1]); ymax = fmaxf(ymax, s_c[j][1]);
        }
        const float scale_box = fmaxf(xmax - xmin, ymax - ymin) / 2.0f;
        float scale;
        if (i == 0) {
            scale = scale_box;
        } else {
            const int pi = c_parents0[i], ci = c_children1[i];
            const float dcx = s_c[ci][0] - s_c[i][0], dcy = s_c[ci][1] - s_c[i][1];
            const float dpx = s_c[pi][0] - s_c[i][0], dpy = s_c[pi][1] - s_c[i][1];
            const float sc = sqrtf(dcx * dcx + dcy * dcy) / 2.0f, sp = sqrtf(dpx * dpx + dpy * dpy) / 2.0f;
            scale = 2.0f * fmaxf(sc, sp);
        }
        scale = scale * fmaxf(ratio[i], 0.0f);
        scale = scale + fmaxf(offset[i], 0.0f);
        if (i != 0 && vis_thresh > 0.0f) {
            const float score = bilinear_point(amax + (size_t)b * HW, S, c_part_mask[i], s_c[i][0], s_c[i][1], align_corners);
            if (score < vis_thresh) scale = 0.8f * scale_box;
        }
        float* t = theta + ((size_t)b * 24 + i) * 3;
        t[0] = scale; t[1] = s_c[i][0]; t[2] = s_c[i][1];
    }
}

// 24x affine_grid + grid_sample (iuv_estimator.py:193-204), C % 8 == 0
// grid = one block per (crop b*24+part, output row py); threads run over (px, V-channel group) of the row: the
// per-element 64-bit div/mod chain of the first version cost more than the 16-byte store it fed
// V = channels per work item: 8 (16-byte accesses on the fp16 planes)
template <int V>
__global__ void __launch_bounds__(256)
k_stn_sample(int B, int S, int C, ActV xd, const float* __restrict__ theta,
             int align_corners, ActV crops) {
    const int CV = C / V;
    const int bp = blockIdx.x / S, py = blockIdx.x - bp * S;
    const int b = bp / 24;
    const float* t = theta + (size_t)bp * 3;
    const float s = t[0], cx = t[1], cy = t[2];
    float yb;
    if (align_corners) yb = -1.0f + 2.0f * (float)py / (float)(S - 1);
    else yb = (float)(2 * py + 1) / (float)S - 1.0f;
    const float gy = s * yb + cy;
    float iy;
    if (align_corners) iy = (gy + 1.0f) * 0.5f * (float)(S - 1);
    else iy = ((gy + 1.0f) * (float)S - 1.0f) * 0.5f;
    const float fy = floorf(iy);
    const float ty = iy - fy;
    const bool y_ok = fy > -2.0f && fy < (float)S + 1.0f;
    const int y0 = y_ok ? (int)fy : 0;
    const size_t ibase = (size_t)b * S * S * C;
    const size_t obase = ((size_t)bp * S + py) * S * CV;            // in V-channel groups
    const int items = S * CV;
    for (int i = threadIdx.x; i < items; i += blockDim.x) {
        const int px = i / CV, cv = i - px * CV;
        float xb;
        if (align_corners) xb = -1.0f + 2.0f * (float)px / (float)(S - 1);
        else xb = (float)(2 * px + 1) / (float)S - 1.0f;
        const float gx = s * xb + cx;
        float ix;
        if (align_corners) ix = (gx + 1.0f) * 0.5f * (float)(S - 1);
        else ix = ((gx + 1.0f) * (float)S - 1.0f) * 0.5f;
        const float fx = floorf(ix);
        const float tx = ix - fx;
        float acc[V];
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = 0.f;
        // guard against huge coordinates before the int conversion
        if (y_ok && fx > -2.0f && fx < (float)S + 1.0f) {
            const int x0 = (int)fx;
#pragma unroll
            for (int dy = 0; dy < 2; ++dy)
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    const int xx = x0 + dx, yy = y0 + dy;
                    if (xx < 0 || xx >= S || yy < 0 || yy >= S) continue;
                    const float w = (dx ? tx : 1.0f - tx) * (dy ? ty : 1.0f - ty);
                    const size_t e = ibase + (size_t)(yy * S + xx) * C + cv * V;
                    if (V == 8) {
                        const float8 v = act_ld8(xd, e);
                        acc[0] = fmaf(w, v.a.x, acc[0]); acc[1] = fmaf(w, v.a.y, acc[1]); acc[2] = fmaf(w, v.a.z, acc[2]); acc[3] = fmaf(w, v.a.w, acc[3]);
                        acc[4 % V] = fmaf(w, v.b.x, acc[4 % V]); acc[5 % V] = fmaf(w, v.b.y, acc[5 % V]);
                        acc[6 % V] = fmaf(w, v.b.z, acc[6 % V]); acc[7 % V] = fmaf(w, v.b.w, acc[7 % V]);
                    } else {
                        const float4 v = act_ld4(xd, e);
                        acc[0] = fmaf(w, v.x, acc[0]); acc[1] = fmaf(w, v.y, acc[1]); acc[2] = fmaf(w, v.z, acc[2]); acc[3] = fmaf(w, v.w, acc[3]);
                    }
                }
        }
        if (V == 8) {
            float8 o;
            o.a = make_float4(acc[0], acc[1], acc[2], acc[3]); o.b = make_float4(acc[4 % V], acc[5 % V], acc[6 % V], acc[7 % V]);
            act_st8(crops, (obase + i) * 8, o);
        } else {
            act_st4(crops, (obase + i) * 4, make_float4(acc[0], acc[1], acc[2], acc[3]));
        }
    }
}

// ------------------------------------------------------------------------------------------
// HRNet fuse (hr_module.py:161-179): y = relu(sum_j nearest_up(t_j))
// ------------------------------------------------------------------------------------------
struct FuseArgs { ActV t[4]; int f[4]; int n; };      // f = log2 of the upsample factor (1,2,4,8 -> 0..3)

// grid = (n*H + h, chunks of a row): no per-element 64-bit division.  V = channels per thread (8: 16-byte plane accesses)
template <int V>
__global__ void __launch_bounds__(256)
k_fuse_sum(int N, int H, int W, int CV, unsigned long long mCV, FuseArgs a, int relu, ActV y) {
    const int row = blockIdx.x;
    const int n = row / H, h = row - n * H;
    const int i = blockIdx.y * blockDim.x + threadIdx.x;
    if (i >= W * CV) return;
    const int w = (int)(((unsigned long long)(unsigned)i * mCV) >> 40), cv = i - w * CV;     // i / CV, exact (i < 2^24)
    float acc[V];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j >= a.n) break;
        const int sh = a.f[j];
        const size_t e = (((size_t)(n * (H >> sh) + (h >> sh)) * (W >> sh) + (w >> sh)) * CV + cv) * V;
        float v[V];
        if (V == 8) { const float8 t = act_ld8(a.t[j], e); v[0] = t.a.x; v[1] = t.a.y; v[2] = t.a.z; v[3] = t.a.w; v[4 % V] = t.b.x; v[5 % V] = t.b.y; v[6 % V] = t.b.z; v[7 % V] = t.b.w; }
        else { const float4 t = act_ld4(a.t[j], e); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = (j == 0) ? v[k] : acc[k] + v[k];
    }
    if (relu) {
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = fmaxf(acc[k], 0.f);
    }
    const size_t o = ((size_t)row * W * CV + i) * V;
    if (V == 8) { float8 t; t.a = make_float4(acc[0], acc[1], acc[2], acc[3]); t.b = make_float4(acc[4 % V], acc[5 % V], acc[6 % V], acc[7 % V]); act_st8(y, o, t); }
    else act_st4(y, o, make_float4(acc[0], acc[1], acc[2], acc[3]));
}

template <int V>
__global__ void __launch_bounds__(256)
k_maxpool3x3s2(int N, int H, int W, int CV, ActV x, ActV y) {
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const int row = blockIdx.x;
    const int n = row / Ho, ho = row - n * Ho;
    const int i = blockIdx.y * blockDim.x + threadIdx.x;
    if (i >= Wo * CV) return;
    const int wo = i / CV, cv = i - wo * CV;
    float m[V];
#pragma unroll
    for (int k = 0; k < V; ++k) m[k] = -INFINITY;
    for (int dy = 0; dy < 3; ++dy) {
        const int hh = ho * 2 - 1 + dy;
        if (hh < 0 || hh >= H) continue;
        for (int dx = 0; dx < 3; ++dx) {
            const int ww = wo * 2 - 1 + dx;
            if (ww < 0 || ww >= W) continue;
            const size_t e = (((size_t)(n * H + hh) * W + ww) * CV + cv) * V;
            float v[V];
            if (V == 8) { const float8 t = act_ld8(x, e); v[0] = t.a.x; v[1] = t.a.y; v[2] = t.a.z; v[3] = t.a.w; v[4 % V] = t.b.x; v[5 % V] = t.b.y; v[6 % V] = t.b.z; v[7 % V] = t.b.w; }
            else { const float4 t = act_ld4(x, e); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
#pragma unroll
            for (int k = 0; k < V; ++k) m[k] = fmaxf(m[k], v[k]);
        }
    }
    const size_t o = ((size_t)row * Wo * CV + i) * V;
    if (V == 8) { float8 t; t.a = make_float4(m[0], m[1], m[2], m[3]); t.b = make_float4(m[4 % V], m[5 % V], m[6 % V], m[7 % V]); act_st8(y, o, t); }
    else act_st4(y, o, make_float4(m[0], m[1], m[2], m[3]));
}

__global__ void k_global_avgpool(int N, int HW, int C, ActV x, float* __restrict__ y) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * C) return;
    const int n = i / C, c = i % C;
    float s = 0.f;
    for (int p = 0; p < HW; ++p) s += act_ld1(x, ((size_t)n * HW + p) * C + c);
    y[i] = s / (float)HW;
}

__global__ void k_linear(int N, int In, int Out, const float* __restrict__ x, const float* __restrict__ w,
                         const float* __restrict__ b, const float* __restrict__ add, float* __restrict__ y) {
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;     // one warp per output: 64-bit
    const int lane = threadIdx.x & 31;
    if (gw >= (long long)N * Out) return;
    const int n = (int)(gw / Out), o = (int)(gw % Out);
    float s = 0.f;
    for (int i = lane; i < In; i += 32) s = fmaf(x[(size_t)n * In + i], w[(size_t)o * In + i], s);
    s = warp_sum(s);
    if (lane == 0) y[gw] = s + (b ? b[o] : 0.f) + (add ? add[o] : 0.f);
}

// ------------------------------------------------------------------------------------------
// GCN refinement + pose head + rot6d (smpl_regressor.py:858-895,924; GCN.py:29-92)
// One CTA (256 threads) per sample; thread o owns output column o of each GraphConv.  rot6d is common.cuh's.
// ------------------------------------------------------------------------------------------
constexpr int kGcnThreads = 256;
constexpr int kGcnMaxF = 256;
constexpr int kGcnTF = 32;                 // input features per streamed weight tile

__global__ void __launch_bounds__(kGcnThreads)
k_gcn_pose_head(int B, GcnArgs g, const float* __restrict__ rot_feats, const float* __restrict__ global_para,
                float* __restrict__ para) {
    extern __shared__ __align__(16) float s_gcn[];
    float* s_x = s_gcn;                          // [24][kGcnMaxF] layer input
    float* s_ax = s_gcn + 24 * kGcnMaxF;         // [24][kGcnMaxF] adj @ x
    float* s_res = s_gcn + 2 * 24 * kGcnMaxF;    // [24][128] residual (pos_feats_init)
    float* s_adj = s_res + 24 * 128;             // [24][24]
    float* s_p6 = s_adj + 576;                   // [144]
    float* s_W = s_p6 + 144;                     // [2][kGcnTF][<= kGcnMaxF] streamed weight tiles (16-byte aligned: all sizes above are multiples of 4 floats)
    const int b = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < 24 * 128; i += kGcnThreads) s_x[(i / 128) * kGcnMaxF + (i % 128)] = rot_feats[(size_t)b * 24 * 128 + i];
    __syncthreads();
    for (int l = 0; l < 5; ++l) {
        const int F = g.din[l], Fo = g.dout[l];
        const int a_id = (l == 0) ? 0 : (l == 4 ? 2 : 1);
        for (int i = tid; i < 576; i += kGcnThreads) s_adj[i] = g.adj[a_id * 576 + i];
        __syncthreads();
        // ax = adj @ x
        for (int i = tid; i < 24 * F; i += kGcnThreads) {
            const int n = i / F, f = i % F;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 24; ++k) s = fmaf(s_adj[n * 24 + k], s_x[k * kGcnMaxF + f], s);
            s_ax[n * kGcnMaxF + f] = s;
        }
        __syncthreads();
        // y = relu(bn(ax @ W + b)); thread tid owns column o = tid.  W streams through shared memory in tiles of kGcnTF input
        // features (cp.async, double-buffered, all 256 threads, coalesced): the per-thread column walk it replaces waited
        // one L2 round trip per 4 features (33 us per layer, latency-bound)
        const float* W = g.W[l];
        const int ntile = (F + kGcnTF - 1) / kGcnTF;
        auto fetch = [&](int t) {
            const int f0 = t * kGcnTF, nf = min(kGcnTF, F - f0);
            const float* src = W + (size_t)f0 * Fo;
            float* dst = s_W + (t & 1) * kGcnTF * kGcnMaxF;
            for (int i4 = tid; i4 < nf * Fo / 4; i4 += kGcnThreads) {
                const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst + 4 * i4);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src + 4 * i4) : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        float acc[24];
#pragma unroll
        for (int n = 0; n < 24; ++n) acc[n] = 0.f;
        fetch(0);
        for (int t = 0; t < ntile; ++t) {
            if (t + 1 < ntile) { fetch(t + 1); asm volatile("cp.async.wait_group 1;" ::: "memory"); }
            else asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads();
            if (tid < Fo) {
                const float* sw = s_W + (t & 1) * kGcnTF * kGcnMaxF;
                const int f0 = t * kGcnTF, nf = min(kGcnTF, F - f0);
                for (int ff = 0; ff < nf; ff += 4) {
                    const float w0 = sw[ff * Fo + tid], w1 = sw[(ff + 1) * Fo + tid], w2 = sw[(ff + 2) * Fo + tid], w3 = sw[(ff + 3) * Fo + tid];
#pragma unroll
                    for (int n = 0; n < 24; ++n) {
                        const float4 av = *reinterpret_cast<const float4*>(&s_ax[n * kGcnMaxF + f0 + ff]);
                        acc[n] = fmaf(av.x, w0, fmaf(av.y, w1, fmaf(av.z, w2, fmaf(av.w, w3, acc[n]))));
                    }
                }
            }
            __syncthreads();                                   // the buffer is refilled two tiles later
        }
        if (tid < Fo) {
            const float bias = g.b[l][tid];
#pragma unroll
            for (int n = 0; n < 24; ++n) {
                float v = (acc[n] + bias) * g.bn_s[l][n] + g.bn_t[l][n];
                v = fmaxf(v, 0.f);
                if (l == 3) v += s_res[n * 128 + tid];          // l_pos_feat = pos_feats_init + refine (smpl_regressor.py:873)
                s_x[n * kGcnMaxF + tid] = v;
                if (l == 0) s_res[n * 128 + tid] = v;           // pos_feats_init
            }
        }
        __syncthreads();
    }
    // pose head: grouped 1x1 conv (24 groups, 128 -> 6) + mean_pose
    if (tid < 144) {
        const int j = tid / 6, k = tid % 6;
        const float* w = g.head_w + ((size_t)j * 6 + k) * 128;
        float s = 0.f;
#pragma unroll 16
        for (int f = 0; f < 128; ++f) s = fmaf(s_x[j * kGcnMaxF + f], __ldg(w + f), s);
        s_p6[tid] = s + g.head_b[tid] + g.mean_pose[tid];
    }
    __syncthreads();
    float* out = para + (size_t)b * 229;
    if (tid < 13) out[tid] = global_para[(size_t)b * 13 + tid];
    if (tid < 24) {
        float R[9];
        rot6d(s_p6 + tid * 6, R);
#pragma unroll
        for (int e = 0; e < 9; ++e) out[13 + tid * 9 + e] = R[e];
    }
}

}  // namespace danet

using namespace danet;

static int check_act(const danet_act* a, const char* what, int C) {
    DANET_CHECK(act_any(a), "%s: activation has neither an fp32 view nor fp16 planes", what);
    DANET_CHECK(!(a->lo && !a->hi), "%s: lo plane without hi plane", what);
    DANET_CHECK(!a->hi || C % 4 == 0, "%s: fp16 planes need C %% 4 == 0 (got %d)", what, C);
    return 0;
}

int danet::nchw_to_nhwc(int N, int C, int HW, int Cp, const float* x, const danet_act* y, cudaStream_t s) {
    DANET_CHECK(N >= 0 && C > 0 && Cp >= C && HW > 0, "danet_nchw_to_nhwc: bad sizes");
    if (N == 0) return 0;
    DANET_CHECK(x, "danet_nchw_to_nhwc: null pointer");
    if (check_act(y, "danet_nchw_to_nhwc", 4) != 0) return -1;
    k_nchw_to_nhwc<<<cdiv(N * HW, 256), 256, 0, s>>>(N, C, HW, Cp, x, actv(y));
    DANET_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------
// iuvmap_clean, global heads (utils/iuvmap.py:6-38 via danet.py:79 / iuv_estimator.py:127)
// ------------------------------------------------------------------------------------------
// A CTA moves PX pixels' head rows through shared memory with coalesced 16-byte loads (a thread per pixel reading its
// 384-byte row with strided 4-byte loads moved 3.3x the DRAM bytes under ncu), computes per pixel from shared memory and
// writes the NHWC views as one contiguous run.  The products keep the reference's NaN / Inf propagation of `U * mask`.
template <int PX>
__global__ void __launch_bounds__(128)
k_iuv_clean_global_staged(int npix_total, int HW, int Chead, int off_u, int off_v, int off_i, int off_a, int Cb,
                          const float* __restrict__ heads, ActV body, uint8_t* __restrict__ amax,
                          float* un, float* vn, float* in_, float* an) {
    extern __shared__ __align__(16) float sm_clean[];
    const int pin = Chead + 1, pout = Cb + 1;                 // odd pitches: a thread per row reads conflict-free
    float* s_in = sm_clean;
    float* s_out = sm_clean + PX * pin;
    const int p0 = blockIdx.x * PX, tid = threadIdx.x;
    const int npx = min(PX, npix_total - p0);
    const float4* src = reinterpret_cast<const float4*>(heads + (size_t)p0 * Chead);     // Chead % 4 == 0 (checked by the host)
    for (int i4 = tid; i4 < npx * Chead / 4; i4 += blockDim.x) {
        const float4 v = __ldg(src + i4);
        const int e = 4 * i4, p = e / Chead, c = e - p * Chead;
        float* d = s_in + p * pin + c;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
    __syncthreads();
    if (tid < npx) {
        const int i = p0 + tid, b = i / HW, pix = i - b * HW;
        const float* h = s_in + tid * pin;
        float I[25];
#pragma unroll
        for (int c = 0; c < 25; ++c) I[c] = h[off_i + c];
        const int best = argmax_first(I, 25);
        amax[i] = (uint8_t)best;
        float* o = s_out + tid * pout;
        for (int c = 0; c < 25; ++c) {
            const float oh = (c == best) ? 1.0f : 0.0f;
            const float u = oh * h[off_u + c], v = oh * h[off_v + c];       // products keep `U * mask`'s NaN / Inf propagation
            o[c] = u; o[25 + c] = v; o[50 + c] = oh;
            if (un) un[((size_t)b * 25 + c) * HW + pix] = u;
            if (vn) vn[((size_t)b * 25 + c) * HW + pix] = v;
            if (in_) in_[((size_t)b * 25 + c) * HW + pix] = oh;
        }
        for (int c = 75; c < Cb; ++c) o[c] = 0.0f;
        if (an) {
            float A[15];
#pragma unroll
            for (int c = 0; c < 15; ++c) A[c] = h[off_a + c];
            const int ba = argmax_first(A, 15);
            for (int c = 0; c < 15; ++c) an[((size_t)b * 15 + c) * HW + pix] = (c == ba) ? 1.0f : 0.0f;
        }
    }
    __syncthreads();
    const size_t obase = (size_t)p0 * Cb;
    for (int i2 = tid; i2 < npx * Cb / 2; i2 += blockDim.x) {    // Cb is even: channel pairs never straddle pixels
        const int e = 2 * i2, p = e / Cb, c = e - p * Cb;
        const float v0 = s_out[p * pout + c], v1 = s_out[p * pout + c + 1];
        if (body.f) *reinterpret_cast<float2*>(body.f + obase + e) = make_float2(v0, v1);
        if (body.hi) {
            const uint32_t hh = pack_h2_rn(v0, v1);
            *reinterpret_cast<uint32_t*>(body.hi + obase + e) = hh;
            if (body.lo) {
                const float2 t = h2_to_f2(hh);
                *reinterpret_cast<uint32_t*>(body.lo + obase + e) = pack_h2_rn(v0 - t.x, v1 - t.y);
            }
        }
    }
}

int danet::iuv_clean_global(int B, int HW, int Chead, int off_u, int off_v, int off_i, int off_a, int Cbody,
                            const float* heads, const danet_act* body_iuv, uint8_t* index_argmax, float* u_nchw,
                            float* v_nchw, float* i_nchw, float* ann_nchw, cudaStream_t s) {
    constexpr int kPx = 64;
    const size_t smem = (size_t)kPx * (Chead + 1 + Cbody + 1) * sizeof(float);
    DANET_CHECK(B >= 0 && HW > 0 && Cbody >= 75, "danet_iuv_clean_global: bad sizes");
    DANET_CHECK(off_u + 25 <= Chead && off_v + 25 <= Chead && off_i + 25 <= Chead && off_a + 15 <= Chead,
                "danet_iuv_clean_global: head offsets exceed Chead=%d", Chead);
    DANET_CHECK(Chead % 4 == 0 && Cbody % 4 == 0 && smem <= 48 * 1024,
                "danet_iuv_clean_global: Chead=%d and Cbody=%d must be multiples of 4 and fit 64 pixels in 48 KB",
                Chead, Cbody);
    if (B == 0) return 0;
    DANET_CHECK(heads && index_argmax, "danet_iuv_clean_global: null pointer");
    DANET_CHECK(aligned16(heads), "danet_iuv_clean_global: heads must be 16-byte aligned");
    if (check_act(body_iuv, "danet_iuv_clean_global", 4) != 0) return -1;
    k_iuv_clean_global_staged<kPx><<<cdiv(B * HW, kPx), 128, smem, s>>>(
        B * HW, HW, Chead, off_u, off_v, off_i, off_a, Cbody, heads, actv(body_iuv), index_argmax, u_nchw, v_nchw, i_nchw, ann_nchw);
    DANET_LAUNCH_CHECK();
    return 0;
}

int danet::iuv_clean_parts(int N, int HW, int Cx, int Cy, const float* x, const danet_act* y, float* raw_nchw,
                           cudaStream_t s) {
    DANET_CHECK(N >= 0 && HW > 0 && Cx >= 24 && Cy >= 24 && Cx % 4 == 0 && Cy % 4 == 0,
                "danet_iuv_clean_parts: bad sizes (Cx, Cy must be >= 24 and %% 4 == 0)");
    if (N == 0) return 0;
    DANET_CHECK(x, "danet_iuv_clean_parts: null pointer");
    if (check_act(y, "danet_iuv_clean_parts", Cy) != 0) return -1;
    k_iuv_clean_parts<true><<<cdiv((int64_t)N * HW, 128), 128, 0, s>>>(N, HW, Cx, Cy, x, actv(y), raw_nchw);
    DANET_LAUNCH_CHECK();
    return 0;
}

int danet::stn_params(int B, int S, int Chm, const float* hm, const uint8_t* index_argmax, const float* learned_ratio,
                      const float* learned_offset, float vis_thresh, int align_corners, float* centers, float* theta,
                      cudaStream_t s) {
    DANET_CHECK(B >= 0 && S > 1 && Chm >= 24 && Chm % 4 == 0, "danet_stn_params: bad sizes (Chm must be >=24 and %%4==0)");
    if (B == 0) return 0;
    DANET_CHECK(hm && index_argmax && learned_ratio && learned_offset && centers && theta, "danet_stn_params: null pointer");
    k_stn_params<<<B, kStnThreads, 0, s>>>(B, S, Chm, hm, index_argmax, learned_ratio, learned_offset, vis_thresh,
                                           align_corners, centers, theta);
    DANET_LAUNCH_CHECK();
    return 0;
}

int danet::stn_sample(int B, int S, int C, const danet_act* xd, const float* theta, int align_corners,
                      const danet_act* crops, cudaStream_t s) {
    DANET_CHECK(B >= 0 && S > 1 && C > 0 && C % 8 == 0, "danet_stn_sample: bad sizes (C %% 8 must be 0)");
    if (B == 0) return 0;
    DANET_CHECK(theta, "danet_stn_sample: null pointer");
    if (check_act(xd, "danet_stn_sample(xd)", C) != 0 || check_act(crops, "danet_stn_sample(crops)", C) != 0) return -1;
    DANET_CHECK((int64_t)B * 24 * S < (1LL << 31), "danet_stn_sample: batch too large for one launch");
    const int items = S * (C / 8);
    k_stn_sample<8><<<B * 24 * S, items >= 256 ? 256 : (items + 31) / 32 * 32, 0, s>>>(B, S, C, actv(xd), theta, align_corners, actv(crops));
    DANET_LAUNCH_CHECK();
    return 0;
}

int danet::fuse_sum(int N, int H, int W, int C, int nterms, const danet_act* terms, const int32_t* factors, int relu,
                    const danet_act* y, cudaStream_t s) {
    DANET_CHECK(N >= 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "danet_fuse_sum: bad sizes (C %% 8 must be 0)");
    DANET_CHECK(nterms >= 1 && nterms <= 4 && terms && factors, "danet_fuse_sum: 1..4 terms required");
    if (N == 0) return 0;
    if (check_act(y, "danet_fuse_sum(y)", C) != 0) return -1;
    FuseArgs a;
    a.n = nterms;
    for (int j = 0; j < 4; ++j) { a.t[j] = actv(nullptr); a.f[j] = 1; }
    for (int j = 0; j < nterms; ++j) {
        const int f = factors[j];
        DANET_CHECK((f == 1 || f == 2 || f == 4 || f == 8) && H % f == 0 && W % f == 0,
                    "danet_fuse_sum: term %d has bad upsample factor %d for %dx%d", j, f, H, W);
        if (check_act(&terms[j], "danet_fuse_sum(term)", C) != 0) return -1;
        a.t[j] = actv(&terms[j]); a.f[j] = f == 1 ? 0 : (f == 2 ? 1 : (f == 4 ? 2 : 3));
    }
    DANET_CHECK((int64_t)N * H < (1LL << 31) && (int64_t)W * (C / 4) < (1 << 24) && C / 4 < (1 << 16), "danet_fuse_sum: tensor too large for one launch");
    k_fuse_sum<8><<<dim3(N * H, cdiv(W * (C / 8), 256)), 256, 0, s>>>(N, H, W, C / 8, (1ull << 40) / (unsigned long long)(C / 8) + 1ull, a, relu, actv(y));
    DANET_LAUNCH_CHECK();
    return 0;
}

int danet::maxpool3x3s2(int N, int H, int W, int C, const danet_act* x, const danet_act* y, cudaStream_t s) {
    DANET_CHECK(N >= 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "danet_maxpool3x3s2: bad sizes (C %% 8 must be 0)");
    if (N == 0) return 0;
    if (check_act(x, "danet_maxpool3x3s2(x)", C) != 0 || check_act(y, "danet_maxpool3x3s2(y)", C) != 0) return -1;
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    DANET_CHECK((int64_t)N * Ho < (1LL << 31) && (int64_t)Wo * (C / 4) <= 65535LL * 256, "danet_maxpool3x3s2: tensor too large for one launch");
    k_maxpool3x3s2<8><<<dim3(N * Ho, cdiv(Wo * (C / 8), 256)), 256, 0, s>>>(N, H, W, C / 8, actv(x), actv(y));
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_global_avgpool(int32_t N, int32_t HW, int32_t C, const danet_act* x, float* y, danet_stream_t s) {
    DANET_CHECK(N >= 0 && HW > 0 && C > 0, "danet_global_avgpool: bad sizes");
    if (N == 0) return 0;
    DANET_CHECK(y, "danet_global_avgpool: null pointer");
    if (check_act(x, "danet_global_avgpool", 4) != 0) return -1;
    k_global_avgpool<<<cdiv(N * C, 256), 256, 0, (cudaStream_t)s>>>(N, HW, C, actv(x), y);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_linear(int32_t N, int32_t In, int32_t Out, const float* x, const float* w, const float* b,
                            const float* add, float* y, danet_stream_t s) {
    DANET_CHECK(N >= 0 && In > 0 && Out > 0, "danet_linear: bad sizes");
    if (N == 0) return 0;
    DANET_CHECK(x && w && y, "danet_linear: null pointer");
    const long long blocks = ((long long)N * Out + 7) / 8;            // 8 warps (outputs) per block
    DANET_CHECK(blocks < (1LL << 31), "danet_linear: N=%d x Out=%d outputs are too many for one grid", N, Out);
    k_linear<<<(unsigned)blocks, 256, 0, (cudaStream_t)s>>>(N, In, Out, x, w, b, add, y);
    DANET_LAUNCH_CHECK();
    return 0;
}

int danet::gcn_pose_head(int B, const GcnArgs& g, const float* rot_feats, const float* global_para, float* para,
                         cudaStream_t s) {
    DANET_CHECK(B >= 0, "danet_gcn_pose_head: bad arguments");
    if (B == 0) return 0;
    DANET_CHECK(rot_feats && global_para && para && g.adj && g.head_w && g.head_b && g.mean_pose,
                "danet_gcn_pose_head: null pointer");
    for (int l = 0; l < 5; ++l) {
        DANET_CHECK(g.W[l] && g.b[l] && g.bn_s[l] && g.bn_t[l], "danet_gcn_pose_head: layer %d has null params", l);
        DANET_CHECK(g.din[l] > 0 && g.din[l] <= kGcnMaxF && g.dout[l] > 0 && g.dout[l] <= kGcnMaxF &&
                    g.din[l] % 4 == 0 && g.dout[l] % 4 == 0 && aligned16(g.W[l]),
                    "danet_gcn_pose_head: layer %d dims %d->%d must be <= %d, multiples of 4, W 16-byte aligned", l, g.din[l], g.dout[l], kGcnMaxF);
    }
    DANET_CHECK(g.din[0] == 128 && g.dout[0] == 128 && g.dout[3] == 128 && g.din[4] == 128 && g.dout[4] == 128,
                "danet_gcn_pose_head: expected 128-d r2p / refine-out / p2r features");
    const size_t smem = (size_t)(2 * 24 * kGcnMaxF + 24 * 128 + 576 + 144 + 2 * kGcnTF * kGcnMaxF) * sizeof(float);
    static unsigned long long attr_devs = 0;
    if (first_use_on_current_device(&attr_devs) != 0)
        DANET_CUDA(cudaFuncSetAttribute(k_gcn_pose_head, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_gcn_pose_head<<<B, kGcnThreads, smem, s>>>(B, g, rot_feats, global_para, para);
    DANET_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------
// iuvmap_clean with the reference's own signature / layout (utils/iuvmap.py:6-38): NCHW maps
// ------------------------------------------------------------------------------------------
namespace danet {
__global__ void k_iuv_clean_nchw(int B, int C, int Ca, int HW, const float* __restrict__ U, const float* __restrict__ V,
                                 const float* __restrict__ I, const float* __restrict__ A, float* __restrict__ oU,
                                 float* __restrict__ oV, float* __restrict__ oI, float* __restrict__ oA) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * HW) return;
    const int b = i / HW, pix = i % HW;
    int best = 0; float bv = I[((size_t)b * C) * HW + pix];
    for (int c = 1; c < C; ++c) {
        const float x = I[((size_t)b * C + c) * HW + pix];
        if ((x > bv) || (x != x && bv == bv)) { bv = x; best = c; }
    }
    for (int c = 0; c < C; ++c) {
        const size_t o = ((size_t)b * C + c) * HW + pix;
        const float oh = (c == best) ? 1.0f : 0.0f;
        oI[o] = oh; oU[o] = oh * U[o]; oV[o] = oh * V[o];
    }
    if (A && oA) {
        int ba = 0; float av = A[((size_t)b * Ca) * HW + pix];
        for (int c = 1; c < Ca; ++c) {
            const float x = A[((size_t)b * Ca + c) * HW + pix];
            if ((x > av) || (x != x && av == av)) { av = x; ba = c; }
        }
        for (int c = 0; c < Ca; ++c) oA[((size_t)b * Ca + c) * HW + pix] = (c == ba) ? 1.0f : 0.0f;
    }
}
}  // namespace danet

extern "C" int danet_iuvmap_clean_nchw(int32_t B, int32_t C, int32_t Ca, int32_t HW, const float* U, const float* V,
                                       const float* I, const float* A, float* oU, float* oV, float* oI, float* oA,
                                       danet_stream_t s) {
    DANET_CHECK(B >= 0 && C > 0 && HW > 0, "danet_iuvmap_clean_nchw: bad sizes");
    if (B == 0) return 0;
    DANET_CHECK(U && V && I && oU && oV && oI, "danet_iuvmap_clean_nchw: null pointer");
    danet::k_iuv_clean_nchw<<<danet::cdiv(B * HW, 256), 256, 0, (cudaStream_t)s>>>(B, C, Ca, HW, U, V, I, A, oU, oV, oI, oA);
    DANET_LAUNCH_CHECK();
    return 0;
}
