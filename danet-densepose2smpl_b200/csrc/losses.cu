// Dense IUV losses of the training step, forward and backward in one pass.
// Replaces models/danet/iuv_estimator.py:304-341 (IUV_Estimator.body_uv_losses) and the autograd graph torch builds
// for it: masked smooth-L1 on the U / V maps, per-pixel cross-entropy on the part-index and annotation logits.
// The 24 per-part calls of iuv_estimator.py:232-255 are ONE launch over the (batch, part)-flattened image axis
// (image stride = 3 * 7 * HW inside part_iuv_pred [B,24,3,7,S,S]).
//
// One thread per pixel, channels walked with stride HW (NCHW: coalesced across the pixels of a warp).  A thread keeps
// the running arg-max of the target map (first maximum, like torch.argmax on the one-hot maps of iuv_img2map), an
// online log-sum-exp of the logits, and the smooth-L1 sums; the second walk over the logits (L1-resident) writes the
// gradients.  Loss sums: fp32 per thread and block, block partials to the workspace, one finishing block adds them in
// double in a fixed order -- the result does not depend on the launch schedule.
#include "common.cuh"
#include "loss_common.cuh"

namespace danet {

struct LossArgs {
    int N, C, Cann, HW;
    long long pred_stride, map_stride;        // elements between consecutive images of the prediction / target tensors
    const float *u, *v, *idx, *ann, *U, *V, *I, *A;
    const uint8_t* has;
    float inv_batch_pw;                       // point weight / batch size: scale of the smooth-L1 sums and gradients
    float *gu, *gv, *gidx, *gann;
    int* nsel; float4* partial; float* losses;
};

// number of images that carry IUV ground truth (has_iuv, iuv_estimator.py:311-318)
__global__ void k_loss_count(const uint8_t* has, int N, int* nsel) {
    __shared__ int s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
    int c = 0;
    for (int i = threadIdx.x; i < N; i += blockDim.x) c += (has == nullptr || has[i]) ? 1 : 0;
    atomicAdd(&s, c);                         // integer: order-independent
    __syncthreads();
    if (threadIdx.x == 0) *nsel = s;
}

#ifdef __CUDA_ARCH__
#define DANET_LDG(p) __ldg(p)
#else
#define DANET_LDG(p) (*(p))
#endif

// cross-entropy of one pixel: loss = lse(x) - x[target]; d/dx = (softmax - onehot) * scale.  The target is
// torch.argmax of the target map: the first maximum, NaN counting as maximal, channel 0 when every entry is -inf; the
// loss and the gradient use that one channel.
// The channel loops are unrolled by 4 over restrict-qualified pointers so that a thread has 8 / 4 independent loads in
// flight (the first version, one load pair per iteration, was latency-bound: 18 long-scoreboard stalls per issue, ncu).
__host__ __device__ inline float pixel_ce(const float* __restrict__ x, const float* __restrict__ t, float* __restrict__ g,
                                          int C, int HW, float scale, bool on) {
    float tmax = -INFINITY, m = -INFINITY, s = 0.f, xt = 0.f;
    int arg = 0;
    if (on) {
#pragma unroll 4
        for (int c = 0; c < C; ++c) {
            const float tv = DANET_LDG(t + (size_t)c * HW), xv = DANET_LDG(x + (size_t)c * HW);
            if (c == 0 || tv > tmax || (tv != tv && tmax == tmax)) { tmax = tv; arg = c; xt = xv; }
            lse_step(xv, m, s);
        }
    }
    const float lse = on ? m + logf(s) : 0.f;
    if (g) {
        const float inv = on ? 1.f / s : 0.f;
#pragma unroll 4
        for (int c = 0; c < C; ++c) {
            float gv = 0.f;
            if (on) gv = (expf(DANET_LDG(x + (size_t)c * HW) - m) * inv - (c == arg ? 1.f : 0.f)) * scale;
            g[(size_t)c * HW] = gv;
        }
    }
    return on ? lse - xt : 0.f;
}

// everything one pixel (image n, position p) contributes: the four loss terms (returned un-normalised) and its
// gradient entries.  Shared by the kernel and by the host walk the CPU tests compile (DANET_LOSSES_HOST_CHECK).
__host__ __device__ inline float4 pixel_body_uv(const LossArgs& a, int n, int p, int nsel) {
    float lu = 0.f, lv = 0.f;
    const bool on = nsel > 0 && (a.has == nullptr || a.has[n] != 0);
    const size_t po = (size_t)n * a.pred_stride + p, mo = (size_t)n * a.map_stride + p;
    // smooth-L1 (beta = 1, summed) where the target part map is positive: iuv_estimator.py:325-326
    const float sc = a.inv_batch_pw;
    const float* __restrict__ pu = a.u + po; const float* __restrict__ pv = a.v + po;
    const float* __restrict__ tU = a.U + mo; const float* __restrict__ tV = a.V + mo; const float* __restrict__ tI = a.I + mo;
    float* __restrict__ gup = a.gu ? a.gu + po : nullptr; float* __restrict__ gvp = a.gv ? a.gv + po : nullptr;
    const int HW = a.HW;
#pragma unroll 4
    for (int c = 0; c < a.C; ++c) {
        const size_t e = (size_t)c * HW;
        float gu = 0.f, gv = 0.f;
        const float iv = on ? DANET_LDG(tI + e) : 0.f;
        if (iv > 0.f) {
            const float du = DANET_LDG(pu + e) - DANET_LDG(tU + e), dv = DANET_LDG(pv + e) - DANET_LDG(tV + e);
            const float au = fabsf(du), av = fabsf(dv);
            lu += au < 1.f ? 0.5f * du * du : au - 0.5f;
            lv += av < 1.f ? 0.5f * dv * dv : av - 0.5f;
            gu = sl1_grad(du) * sc;
            gv = sl1_grad(dv) * sc;
        }
        if (gup) gup[e] = gu;
        if (gvp) gvp[e] = gv;
    }
    // cross-entropy, mean over the pixels of the selected images: iuv_estimator.py:320-327,335-339
    const float cs = on ? 1.f / ((float)nsel * (float)a.HW) : 0.f;
    const float li = pixel_ce(a.idx + po, a.I + mo, a.gidx ? a.gidx + po : nullptr, a.C, a.HW, cs, on);
    float la = 0.f;
    if (a.ann) {
        const size_t ao = (size_t)n * a.Cann * a.HW + p;
        la = pixel_ce(a.ann + ao, a.A + ao, a.gann ? a.gann + ao : nullptr, a.Cann, a.HW, cs, on);
    }
    return make_float4(lu, lv, li, la);
}

__global__ void __launch_bounds__(256) k_body_uv_losses(const LossArgs a) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)a.N * a.HW;
    float lu = 0.f, lv = 0.f, li = 0.f, la = 0.f;
    if (gid < total) {
        const int n = (int)(gid / a.HW), p = (int)(gid - (long long)n * a.HW);
        const float4 t = pixel_body_uv(a, n, p, *a.nsel);
        lu = t.x; lv = t.y; li = t.z; la = t.w;
    }
    // block partial (fixed shuffle / shared-memory order)
    __shared__ float4 sm[8];
    lu = warp_sum(lu); lv = warp_sum(lv); li = warp_sum(li); la = warp_sum(la);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) sm[w] = make_float4(lu, lv, li, la);
    __syncthreads();
    if (threadIdx.x == 0) {
        float4 t = sm[0];
        for (int i = 1; i < (int)(blockDim.x >> 5); ++i) { t.x += sm[i].x; t.y += sm[i].y; t.z += sm[i].z; t.w += sm[i].w; }
        a.partial[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(256) k_loss_finish(const float4* partial, int nblocks, const int* nsel, int HW,
                                                     float inv_batch_pw, int has_ann, float* losses) {
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
        const int n = *nsel;
        const double ce = n > 0 ? 1.0 / ((double)n * (double)HW) : 0.0;
        losses[0] = (float)(sm[0][0] * (double)inv_batch_pw);
        losses[1] = (float)(sm[1][0] * (double)inv_batch_pw);
        losses[2] = (float)(sm[2][0] * ce);
        losses[3] = has_ann ? (float)(sm[3][0] * ce) : 0.f;
    }
}

}  // namespace danet

using namespace danet;

extern "C" int64_t danet_body_uv_losses_workspace_bytes(int32_t N, int32_t HW) {
    if (N < 0 || HW < 0) return -1;
    const long long blocks = ((long long)N * HW + 63) / 64;          // smallest block the launch may choose
    return 256 + (blocks > 0 ? blocks : 1) * (long long)sizeof(float4);
}

extern "C" int danet_body_uv_losses(int32_t N, int32_t C, int32_t Cann, int32_t HW, int64_t pred_stride, int64_t map_stride,
                                    const float* u_pred, const float* v_pred, const float* index_pred, const float* ann_pred,
                                    const float* Umap, const float* Vmap, const float* Imap, const float* Annmap,
                                    const uint8_t* has_iuv, float batch_size, float point_weight, float* losses,
                                    float* grad_u, float* grad_v, float* grad_index, float* grad_ann, void* workspace,
                                    danet_stream_t stream) {
    DANET_CHECK(N >= 0 && C >= 1 && HW >= 1, "body_uv_losses: bad sizes N=%d C=%d HW=%d", N, C, HW);
    DANET_CHECK(u_pred && v_pred && index_pred && Umap && Vmap && Imap && losses && workspace, "body_uv_losses: null pointer");
    DANET_CHECK((ann_pred == nullptr) == (Annmap == nullptr), "body_uv_losses: ann_pred and Annmap come together");
    DANET_CHECK(ann_pred == nullptr || Cann >= 1, "body_uv_losses: Cann=%d", Cann);
    DANET_CHECK(!grad_ann || ann_pred, "body_uv_losses: grad_ann without ann_pred");
    DANET_CHECK(batch_size > 0.f, "body_uv_losses: batch_size must be positive");
    if (pred_stride == 0) pred_stride = (int64_t)C * HW;
    if (map_stride == 0) map_stride = (int64_t)C * HW;
    DANET_CHECK(pred_stride >= (int64_t)C * HW && map_stride >= (int64_t)C * HW, "body_uv_losses: image stride below C*HW");
    cudaStream_t st = (cudaStream_t)stream;
    const long long total = (long long)N * HW;
    DANET_CHECK((total + 63) / 64 < (1LL << 31), "body_uv_losses: too many pixels");
    // few pixels (the global heads of a 16-image batch: 50 K): smaller blocks, so that every SM gets several
    const int bt = total >= 132LL * 2048 * 2 ? 256 : (total >= 132LL * 2048 / 2 ? 128 : 64);
    const int blocks = (int)((total + bt - 1) / bt);
    LossArgs a;
    a.N = N; a.C = C; a.Cann = Cann; a.HW = HW; a.pred_stride = pred_stride; a.map_stride = map_stride;
    a.u = u_pred; a.v = v_pred; a.idx = index_pred; a.ann = ann_pred; a.U = Umap; a.V = Vmap; a.I = Imap; a.A = Annmap;
    a.has = has_iuv; a.inv_batch_pw = point_weight / batch_size;
    a.gu = grad_u; a.gv = grad_v; a.gidx = grad_index; a.gann = grad_ann;
    a.nsel = reinterpret_cast<int*>(workspace);
    a.partial = reinterpret_cast<float4*>(reinterpret_cast<uint8_t*>(workspace) + 256);
    a.losses = losses;
    k_loss_count<<<1, 256, 0, st>>>(has_iuv, N, a.nsel);
    DANET_LAUNCH_CHECK();
    if (blocks > 0) {
        k_body_uv_losses<<<blocks, bt, 0, st>>>(a);
        DANET_LAUNCH_CHECK();
    }
    k_loss_finish<<<1, 256, 0, st>>>(a.partial, blocks, a.nsel, HW, a.inv_batch_pw, ann_pred ? 1 : 0, losses);
    DANET_LAUNCH_CHECK();
    return 0;
}

#ifdef DANET_LOSSES_HOST_CHECK
// Test-only (never part of libdanet_b200.so: the flag is set by tests/test_losses_cpu.py alone): the same per-pixel
// function walked on the host over HOST arrays, so that the arithmetic of the kernel is pinned against the
// reference-generated golden without a GPU.
extern "C" int danet_test_body_uv_losses_host(int32_t N, int32_t C, int32_t Cann, int32_t HW, int64_t pred_stride,
                                              int64_t map_stride, const float* u, const float* v, const float* idx,
                                              const float* ann, const float* U, const float* V, const float* I, const float* A,
                                              const uint8_t* has, float batch_size, float point_weight, float* losses,
                                              float* gu, float* gv, float* gidx, float* gann) {
    LossArgs a;
    a.N = N; a.C = C; a.Cann = Cann; a.HW = HW;
    a.pred_stride = pred_stride ? pred_stride : (int64_t)C * HW; a.map_stride = map_stride ? map_stride : (int64_t)C * HW;
    a.u = u; a.v = v; a.idx = idx; a.ann = ann; a.U = U; a.V = V; a.I = I; a.A = A; a.has = has;
    a.inv_batch_pw = point_weight / batch_size;
    a.gu = gu; a.gv = gv; a.gidx = gidx; a.gann = gann; a.nsel = nullptr; a.partial = nullptr; a.losses = losses;
    int nsel = 0;
    for (int n = 0; n < N; ++n) nsel += (!has || has[n]) ? 1 : 0;
    double s[4] = {0, 0, 0, 0};
    for (int n = 0; n < N; ++n)
        for (int p = 0; p < HW; ++p) {
            const float4 t = pixel_body_uv(a, n, p, nsel);
            s[0] += t.x; s[1] += t.y; s[2] += t.z; s[3] += t.w;
        }
    const double ce = nsel > 0 ? 1.0 / ((double)nsel * HW) : 0.0;
    losses[0] = (float)(s[0] * a.inv_batch_pw); losses[1] = (float)(s[1] * a.inv_batch_pw);
    losses[2] = (float)(s[2] * ce); losses[3] = ann ? (float)(s[3] * ce) : 0.f;
    return 0;
}
#endif
