// One-pass multi-tensor Adam: torch.optim.Adam's CUDA default (_multi_tensor_adam, capturable=False, amsgrad=False,
// maximize=False, weight_decay=0) bit for bit, in one read of p, g, exp_avg, exp_avg_sq and one write of p, exp_avg,
// exp_avg_sq per element (28 B per parameter; torch's seven foreach passes move about 72 B).
//
// Per element, each step rounded to fp32 as torch's kernels round it:
//   m = lerp(m, g, w1)                 ATen/native/Lerp.h, its FMA contraction as nvcc compiles torch
//   v = v * beta2                      _foreach_mul_
//   v = fma(c2, g * g, v)              _foreach_addcmul_, DeviceAddCmulCdiv.cuh: fma(alpha, op(t1, t2), input)
//   d = sqrt(v) / bc2 + eps            _foreach_sqrt, _foreach_div_ (scalar list), _foreach_add_
//   p = fma(s, m / d, p)               _foreach_addcdiv_ (scalar list), the same fma form
// The scalars are fp32 roundings of the doubles torch's Python computes from the step count (optim.py); every tensor of
// one call shares them.  The intrinsics pin each rounding so that nvcc cannot contract differently.
//
// The tensor table travels in the kernel's parameter block (__grid_constant__, up to 32764 bytes since CUDA 12.1), so a
// step needs no copy, no staging buffer and no host synchronisation.  A block takes one 4096-element chunk of one tensor;
// blocks find their tensor by a binary search over the table's chunk offsets.  16-byte loads and stores where all four
// pointers of a tensor are 16-byte aligned, scalar accesses otherwise and for the tail: both compute the same function.
#include "common.cuh"

namespace danet {

constexpr int kAdamTensors = 720;              // 40 B of pointers and count + 4 B of chunk offset per tensor
constexpr int kAdamThreads = 256;
constexpr int kAdamChunk = kAdamThreads * 4 * 4; // four float4 per thread

struct AdamTable {
    float* p[kAdamTensors];
    const float* g[kAdamTensors];
    float* m[kAdamTensors];
    float* v[kAdamTensors];
    long long n[kAdamTensors];
    int chunk0[kAdamTensors + 1];              // first chunk (block) of each tensor; chunk0[count] = grid size
    int count;
    float w1, beta2, c2, bc2, eps, s;
};
static_assert(sizeof(AdamTable) <= 32764, "the Adam table must fit in one kernel parameter block");

__device__ __forceinline__ void adam_elem(const AdamTable& t, float& p, float g, float& m, float& v) {
    // Lerp.h: |w| < 0.5 ? self + w * (end - self) : end - (end - self) * (1 - w), each a contracted multiply-add
    const float diff = __fsub_rn(g, m);
    m = fabsf(t.w1) < 0.5f ? __fmaf_rn(t.w1, diff, m) : __fmaf_rn(-diff, __fsub_rn(1.0f, t.w1), g);
    v = __fmul_rn(v, t.beta2);
    v = __fmaf_rn(t.c2, __fmul_rn(g, g), v);
    const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), t.bc2), t.eps);
    p = __fmaf_rn(t.s, __fdiv_rn(m, d), p);
}

__global__ void __launch_bounds__(kAdamThreads) k_adam(const __grid_constant__ AdamTable t) {
    const int b = blockIdx.x;
    int lo = 0, hi = t.count - 1;              // the last tensor whose first chunk is <= b
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (t.chunk0[mid] <= b) lo = mid; else hi = mid - 1;
    }
    const long long begin = (long long)(b - t.chunk0[lo]) * kAdamChunk;
    const long long end = min(t.n[lo], begin + kAdamChunk);
    float* __restrict__ P = t.p[lo];
    const float* __restrict__ G = t.g[lo];
    float* __restrict__ M = t.m[lo];
    float* __restrict__ V = t.v[lo];
    long long i = begin;
    if ((((uintptr_t)P | (uintptr_t)G | (uintptr_t)M | (uintptr_t)V) & 15) == 0) {
        const long long vend = begin + ((end - begin) & ~3LL);
        for (long long j = begin + 4LL * threadIdx.x; j < vend; j += 4LL * kAdamThreads) {
            float4 p = *reinterpret_cast<const float4*>(P + j);
            const float4 g = __ldcs(reinterpret_cast<const float4*>(G + j));
            float4 m = *reinterpret_cast<const float4*>(M + j);
            float4 v = *reinterpret_cast<const float4*>(V + j);
            adam_elem(t, p.x, g.x, m.x, v.x);
            adam_elem(t, p.y, g.y, m.y, v.y);
            adam_elem(t, p.z, g.z, m.z, v.z);
            adam_elem(t, p.w, g.w, m.w, v.w);
            *reinterpret_cast<float4*>(P + j) = p;
            *reinterpret_cast<float4*>(M + j) = m;
            *reinterpret_cast<float4*>(V + j) = v;
        }
        i = vend;
    }
    for (long long j = i + threadIdx.x; j < end; j += kAdamThreads) {
        float p = P[j], m = M[j], v = V[j];
        adam_elem(t, p, G[j], m, v);
        P[j] = p;
        M[j] = m;
        V[j] = v;
    }
}

}  // namespace danet

extern "C" int danet_adam_step(int32_t count, float* const* params, const float* const* grads, float* const* exp_avgs,
                               float* const* exp_avg_sqs, const int64_t* numels, double lerp_weight, double beta2,
                               double one_minus_beta2, double bias_correction2_sqrt, double eps, double step_size,
                               danet_stream_t stream) {
    const char* where = "danet_adam_step";
    DANET_CHECK(count >= 0, "%s: count must be >= 0 (got %d)", where, count);
    if (count == 0) return 0;
    DANET_CHECK(params && grads && exp_avgs && exp_avg_sqs && numels, "%s: null table", where);
    danet::AdamTable t;
    t.w1 = (float)lerp_weight;
    t.beta2 = (float)beta2;
    t.c2 = (float)one_minus_beta2;
    t.bc2 = (float)bias_correction2_sqrt;
    t.eps = (float)eps;
    t.s = (float)step_size;
    for (int k = 0; k < count; ++k) {
        DANET_CHECK(numels[k] >= 0, "%s: numels[%d] = %lld is negative", where, k, (long long)numels[k]);
        DANET_CHECK(numels[k] == 0 || (params[k] && grads[k] && exp_avgs[k] && exp_avg_sqs[k]),
                    "%s: null pointer in tensor %d", where, k);
        DANET_CHECK((numels[k] + danet::kAdamChunk - 1) / danet::kAdamChunk < (1LL << 31) - 1,
                    "%s: tensor %d has too many elements (%lld)", where, k, (long long)numels[k]);
    }
    // fill the table tensor by tensor; launch when it is full or the next tensor would overflow the grid
    int k = 0;
    while (k < count) {
        int n = 0;
        long long chunks = 0;
        for (; k < count && n < danet::kAdamTensors; ++k) {
            const long long c = (numels[k] + danet::kAdamChunk - 1) / danet::kAdamChunk;
            if (c == 0) continue;                  // empty tensors take no block
            if (chunks + c > (1LL << 31) - 1) break;
            t.p[n] = params[k];
            t.g[n] = grads[k];
            t.m[n] = exp_avgs[k];
            t.v[n] = exp_avg_sqs[k];
            t.n[n] = numels[k];
            t.chunk0[n] = (int)chunks;
            chunks += c;
            ++n;
        }
        if (n == 0) continue;
        t.chunk0[n] = (int)chunks;
        t.count = n;
        danet::k_adam<<<(unsigned)chunks, danet::kAdamThreads, 0, (cudaStream_t)stream>>>(t);
        DANET_LAUNCH_CHECK();
    }
    return 0;
}
