// Part dropout and iuvmap_clean of the IUV estimator's outputs for training (models/danet/danet.py:193-205, 247-283
// with utils/iuvmap.py:6-38), forward and backward.  One thread per (image, pixel) of the global maps and per (image,
// part crop, pixel) of the part maps, in one launch each way.
//
// The one-hot of the reference is built from thresholds of the float argmax: 1 at the argmax, -0.0 on the channels
// below it and +0.0 above it, and the cleaned U / V are products with it.  Dropping multiplies by 0.0f, so NaN and
// +-inf become NaN.  The backward is what torch autograd gives for those expressions: d(oh * x) = g * oh; a dropped
// entry gets (g * oh) * 0; and every entry of a tensor the reference passes through index_put_ (the dropped global
// maps) or assembles from per-crop slices (the part maps) is a sum with +0.0, which turns -0.0 into +0.0.
#include "common.cuh"
#include "stn_common.cuh"

namespace danet {

constexpr int kPdC = 25;          // U / V / Index channels of the global maps
constexpr int kPdCrop = 7;        // channels of one part crop: background + 6 mapped DensePose parts
constexpr int kPdParts = 24;
constexpr int kPdThreads = 256;

struct PdTable { unsigned char part[kPdParts][kPdCrop]; };   // DensePose part of (crop, channel); 0 = background

struct PdArgs {
    int B, HW, S, Ca;
    const float *u, *v, *idx, *ann;                     // [B,25,HW] x3, [B,Ca,HW]
    const float* parts;                                 // [B,24,3,7,S,S] through strides
    long long ps[6];                                    // element strides of parts
    const uint8_t* drop;                                // [B,24] or NULL (no dropout)
    PdTable tab;
};

__device__ __forceinline__ float onehot_ref(int c, int best) { return c == best ? 1.f : (c < best ? -0.f : 0.f); }

__device__ __forceinline__ bool dropped(const uint8_t* drop, int b, int part) {
    return drop && part > 0 && drop[b * kPdParts + part - 1];
}

__global__ void __launch_bounds__(kPdThreads) k_part_drop_clean_fwd(PdArgs a, float* __restrict__ oU,
        float* __restrict__ oV, float* __restrict__ oI, float* __restrict__ oA, float* __restrict__ oP,
        uint8_t* __restrict__ am_g, uint8_t* __restrict__ am_p) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long ng = (long long)a.B * a.HW;
    if (t < ng) {
        const int b = (int)(t / a.HW), pix = (int)(t % a.HW);
        const size_t base = (size_t)b * kPdC * a.HW + pix;
        float x[kPdC];
#pragma unroll
        for (int c = 0; c < kPdC; ++c) {
            x[c] = a.idx[base + (size_t)c * a.HW];
            if (dropped(a.drop, b, c)) x[c] = x[c] * 0.f;
        }
        const int best = argmax_first(x, kPdC);
        am_g[t] = (uint8_t)best;
#pragma unroll
        for (int c = 0; c < kPdC; ++c) {
            const size_t o = base + (size_t)c * a.HW;
            const bool d = dropped(a.drop, b, c);
            const float oh = onehot_ref(c, best);
            const float uu = d ? a.u[o] * 0.f : a.u[o], vv = d ? a.v[o] * 0.f : a.v[o];
            oI[o] = oh; oU[o] = oh * uu; oV[o] = oh * vv;
        }
        const size_t abase = (size_t)b * a.Ca * a.HW + pix;
        const int ba = argmax_first(a.ann + abase, a.Ca, (size_t)a.HW);
        for (int c = 0; c < a.Ca; ++c) oA[abase + (size_t)c * a.HW] = onehot_ref(c, ba);
        return;
    }
    if (t >= ng * (kPdParts + 1)) return;
    const long long q = t - ng;                         // (b, crop, pix)
    const int pix = (int)(q % a.HW), bc = (int)(q / a.HW), b = bc / kPdParts, k = bc % kPdParts;
    const long long in0 = b * a.ps[0] + k * a.ps[1] + (long long)(pix / a.S) * a.ps[4] + (long long)(pix % a.S) * a.ps[5];
    float x[kPdCrop];
    bool d[kPdCrop];
#pragma unroll
    for (int c = 0; c < kPdCrop; ++c) {
        d[c] = dropped(a.drop, b, a.tab.part[k][c]);
        x[c] = a.parts[in0 + 2 * a.ps[2] + c * a.ps[3]];
        if (d[c]) x[c] = x[c] * 0.f;
    }
    const int best = argmax_first(x, kPdCrop);
    am_p[q] = (uint8_t)best;
    const size_t o0 = (size_t)bc * 3 * kPdCrop * a.HW + pix;
#pragma unroll
    for (int c = 0; c < kPdCrop; ++c) {
        const float oh = onehot_ref(c, best);
        float uu = a.parts[in0 + c * a.ps[3]], vv = a.parts[in0 + a.ps[2] + c * a.ps[3]];
        if (d[c]) { uu = uu * 0.f; vv = vv * 0.f; }
        oP[o0 + (size_t)c * a.HW] = oh * uu;
        oP[o0 + (size_t)(kPdCrop + c) * a.HW] = oh * vv;
        oP[o0 + (size_t)(2 * kPdCrop + c) * a.HW] = oh;
    }
}

// gradient of one entry: g * oh, times 0 when dropped, plus +0.0 when the entry's tensor is summed with zeros
__device__ __forceinline__ float pd_grad(float g, float oh, bool d, bool canon) {
    float r = g * oh;
    if (d) r = r * 0.f;
    return canon ? __fadd_rn(r, 0.f) : r;
}

__global__ void __launch_bounds__(kPdThreads) k_part_drop_clean_bwd(int B, int HW, const uint8_t* __restrict__ drop,
        PdTable tab, const uint8_t* __restrict__ am_g, const uint8_t* __restrict__ am_p, const float* __restrict__ gU,
        const float* __restrict__ gV, const float* __restrict__ gP, float* __restrict__ dU, float* __restrict__ dV,
        float* __restrict__ dP) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long ng = (long long)B * HW;
    if (t < ng) {
        const int b = (int)(t / HW), pix = (int)(t % HW);
        const size_t base = (size_t)b * kPdC * HW + pix;
        const int best = am_g[t];
        const bool canon = drop != nullptr;             // the dropped maps went through index_put_
#pragma unroll
        for (int c = 0; c < kPdC; ++c) {
            const size_t o = base + (size_t)c * HW;
            const float oh = onehot_ref(c, best);
            const bool d = dropped(drop, b, c);
            dU[o] = pd_grad(gU[o], oh, d, canon);
            dV[o] = pd_grad(gV[o], oh, d, canon);
        }
        return;
    }
    if (t >= ng * (kPdParts + 1)) return;
    const long long q = t - ng;
    const int pix = (int)(q % HW), bc = (int)(q / HW), b = bc / kPdParts, k = bc % kPdParts;
    const int best = am_p[q];
    const size_t o0 = (size_t)bc * 3 * kPdCrop * HW + pix;
#pragma unroll
    for (int c = 0; c < kPdCrop; ++c) {
        const float oh = onehot_ref(c, best);
        const bool d = dropped(drop, b, tab.part[k][c]);
        const size_t ou = o0 + (size_t)c * HW, ov = o0 + (size_t)(kPdCrop + c) * HW;
        dP[ou] = pd_grad(gP[ou], oh, d, true);
        dP[ov] = pd_grad(gP[ov], oh, d, true);
        dP[o0 + (size_t)(2 * kPdCrop + c) * HW] = 0.f;
    }
}

static int pd_table(const char* where, const int8_t* dp2smpl, PdTable* tab) {
    DANET_CHECK(dp2smpl, "%s: null dp2smpl table", where);
    for (int k = 0; k < kPdParts; ++k) {
        tab->part[k][0] = 0;
        for (int m = 0; m < kPdCrop - 1; ++m) {
            const int p = dp2smpl[k * (kPdCrop - 1) + m];
            DANET_CHECK(p >= 1 && p <= kPdParts, "%s: dp2smpl[%d][%d] = %d is not a DensePose part 1..24", where, k, m, p);
            tab->part[k][m + 1] = (unsigned char)p;
        }
    }
    return 0;
}

}  // namespace danet

extern "C" int danet_part_drop_clean_forward(int32_t B, int32_t S, int32_t Ca, const float* u, const float* v,
                                             const float* index, const float* ann, const float* parts,
                                             const int64_t* part_strides, const uint8_t* drop, const int8_t* dp2smpl,
                                             float* u_out, float* v_out, float* index_out, float* ann_out,
                                             float* parts_out, uint8_t* argmax_global, uint8_t* argmax_parts,
                                             danet_stream_t stream) {
    const char* where = "danet_part_drop_clean_forward";
    DANET_CHECK(B >= 0 && S > 0 && Ca > 0, "%s: bad sizes B=%d S=%d Ca=%d", where, B, S, Ca);
    DANET_CHECK((long long)B * 25 * 3 * 7 * S * S < (1LL << 31), "%s: B=%d S=%d is too large", where, B, S);
    if (B == 0) return 0;
    DANET_CHECK(u && v && index && ann && parts && part_strides && u_out && v_out && index_out && ann_out &&
                parts_out && argmax_global && argmax_parts, "%s: null pointer", where);
    danet::PdArgs a;
    a.B = B; a.S = S; a.HW = S * S; a.Ca = Ca;
    a.u = u; a.v = v; a.idx = index; a.ann = ann; a.parts = parts; a.drop = drop;
    for (int i = 0; i < 6; ++i) a.ps[i] = part_strides[i];
    if (danet::pd_table(where, dp2smpl, &a.tab)) return -1;
    const long long n = (long long)B * a.HW * (danet::kPdParts + 1);
    danet::k_part_drop_clean_fwd<<<(unsigned)((n + danet::kPdThreads - 1) / danet::kPdThreads), danet::kPdThreads, 0,
                                   (cudaStream_t)stream>>>(a, u_out, v_out, index_out, ann_out, parts_out,
                                                           argmax_global, argmax_parts);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_part_drop_clean_backward(int32_t B, int32_t S, const uint8_t* drop, const int8_t* dp2smpl,
                                              const uint8_t* argmax_global, const uint8_t* argmax_parts,
                                              const float* grad_u_out, const float* grad_v_out,
                                              const float* grad_parts_out, float* grad_u, float* grad_v,
                                              float* grad_parts, danet_stream_t stream) {
    const char* where = "danet_part_drop_clean_backward";
    DANET_CHECK(B >= 0 && S > 0, "%s: bad sizes B=%d S=%d", where, B, S);
    DANET_CHECK((long long)B * 25 * 3 * 7 * S * S < (1LL << 31), "%s: B=%d S=%d is too large", where, B, S);
    if (B == 0) return 0;
    DANET_CHECK(argmax_global && argmax_parts && grad_u_out && grad_v_out && grad_parts_out && grad_u && grad_v &&
                grad_parts, "%s: null pointer", where);
    danet::PdTable tab;
    if (danet::pd_table(where, dp2smpl, &tab)) return -1;
    const long long n = (long long)B * S * S * (danet::kPdParts + 1);
    danet::k_part_drop_clean_bwd<<<(unsigned)((n + danet::kPdThreads - 1) / danet::kPdThreads), danet::kPdThreads, 0,
                                   (cudaStream_t)stream>>>(B, S * S, drop, tab, argmax_global, argmax_parts, grad_u_out,
                                                           grad_v_out, grad_parts_out, grad_u, grad_v, grad_parts);
    DANET_LAUNCH_CHECK();
    return 0;
}
