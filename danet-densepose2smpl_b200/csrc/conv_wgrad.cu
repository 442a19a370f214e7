// Convolution backward for sm_90a: the weight gradient on a wgmma kernel of its own, and the small kernels that let the
// forward engine (conv_tc.cu, unchanged) compute the input gradient.  Exact (split-fp16, fp32-grade) arithmetic only.
//
// Weight gradient (k_wgrad).  dW[s][co][tap][ci] = sum over the images n of weight set s (n % wsets == s) and their
// output pixels p of dy[n,p,co] * x_tap[n,p,ci]: per tap an implicit GEMM with M = Cout, N = Cin, K = pixels.
//   Loads: a stage is four TMA boxes of 64 channels x (8 x 8) pixels, 128-byte swizzled: dy hi / lo at an 8 x 8 patch
//       of output pixels, x hi / lo at the input pixels that tap (r, s) reads for them (elementStrides = stride).  The
//       convolution's padding and the patch's overhang are the out-of-bounds zero fill, so they contribute nothing.
//       Both operands come from NHWC planes, so both are MN-major in shared memory (a K row is a pixel's 64 channels)
//       and wgmma reads both transposed.
//   MMA: one consumer warpgroup per CTA issues m64n64k16 with three products per K step, as the forward's exact mode:
//       hi*hi into the main chain, hi*lo and lo*hi into the small terms.  Every kSegStages stages (8 main-chain MMAs)
//       the chain drains and both accumulators are added, main first, to a running fp32 sum in round-to-nearest: the
//       tensor core's own accumulation truncates.
//   Split K: a work unit is (pixel chunk, weight set, Cout block, Cin block, tap).  Each writes its fp32 partial;
//       k_wgrad_finish adds the chunks in chunk order in double.  There are no float atomics, so the results repeat bit
//       for bit.  db (channel sums of the fp32 dy) uses the same scheme: k_db_partial / k_db_finish.
//
// Operand scales.  Gradients can be orders of magnitude below 1, where the lo half of an fp16 split is subnormal or zero,
// and activations can lie far from 1 either way (past 65504 the split saturates).  So dy, and the forward's x, are each
// scaled by a power of two 2^s, found on the device from the tensor's max |v| (no host synchronisation), before the split
// (k_split_scaled), and the scales are removed exactly in k_wgrad_finish (both) and k_scatter_nchw (one per output).
//
// Input gradient.  For stride 1, dx = conv(dy, W') with W' the filter rotated by 180 degrees and Cin / Cout swapped,
// padding k/2: a forward problem of the engine.  For stride 2, output-parity class (a, b) of dx is a stride-1
// correlation of dy with the taps of W of that parity.  Per dimension, the taps at dy offsets -1..1 form one centred 1-
// or 3-wide kernel; a tap at offset 2 (the fourth tap of a 7x7/s2 parity) becomes a 3-wide kernel whose one tap sits
// at +1, read back shifted by one output pixel.  Each piece is a 1x1 or 3x3 stride-1 problem of the engine; the pieces
// run as multi-problem launches (up to 6 per launch) and k_scatter_nchw sums them per dx element in a fixed order,
// removes the dy scale and writes the NCHW dx.  Executed taps: 3x3/s2 1 + 9 + 9 + 9 = 28 for 9; 7x7/s2 9 + 2*18 + 36 = 81
// for 49 (nine 3x3 problems); 1x1/s2 one 1x1 piece, the other three classes are zero.
#include "common.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <string.h>

namespace danet {
namespace wg {
using namespace tc;

constexpr int kBox = 8;                          // a K block is an 8 x 8 patch of output pixels
constexpr int kKBlk = kBox * kBox;               // 64 pixels: four k16 steps
constexpr int kCh = 64;                          // channels per M (Cout) and N (Cin) block: one 128-byte swizzle row
constexpr int kPlane = kKBlk * kCh * 2;          // one operand plane of a stage: 8 KB
constexpr int kStageBytes = 4 * kPlane;          // dy hi, dy lo, x hi, x lo
constexpr int kStages = 3;
constexpr int kSegStages = 2;                    // 2 stages x 4 k16 steps = 8 main-chain MMAs per K segment
constexpr int kThreads = 160;                    // one consumer warpgroup + one producer warp
constexpr int kSmem = kStages * kStageBytes + 1024 + 64;   // + 1024-byte alignment slack + barriers
constexpr int kTargetUnits = 8 * 132;            // split K until there are about 8 waves of work units
constexpr int kMinStages = 4;                    // ... but keep at least 4 stages (2 segments) per unit

struct alignas(64) Args {
    CUtensorMap tm[4];                           // dy hi, dy lo, x hi, x lo
    float* part;                                 // [nchunk][wsets][taps][Cout][Cin]
    int Cin, Cout, ks, stride, pad, wsets, taps, ncib, ncob;
    int tiles_w, tiles_img, tiles_set, tpc;
};

// host: geometry of a weight-gradient problem (d describes the forward convolution)
struct Geo {
    int Ho, Wo, taps, ncib, ncob, tiles_w, tiles_h, tiles_img, tiles_set, units0, nchunk, tpc;
    long long part_elems;
};
static bool make_geo(const danet_conv_desc* d, Geo* g) {
    if (!(d->stride == 1 || d->stride == 2) || !(d->ksize == 1 || d->ksize == 3 || d->ksize == 7) || d->pad != d->ksize / 2) return false;
    if (d->Cin % 8 != 0 || d->Cout % 8 != 0 || d->H < 1 || d->W < 1 || d->N < 1 || d->wsets < 1 || d->N % d->wsets != 0) return false;
    g->Ho = (d->H + 2 * d->pad - d->ksize) / d->stride + 1;
    g->Wo = (d->W + 2 * d->pad - d->ksize) / d->stride + 1;
    g->taps = d->ksize * d->ksize;
    g->ncib = cdiv(d->Cin, kCh); g->ncob = cdiv(d->Cout, kCh);
    g->tiles_w = cdiv(g->Wo, kBox); g->tiles_h = cdiv(g->Ho, kBox);
    g->tiles_img = g->tiles_w * g->tiles_h;
    const long long ts = (long long)(d->N / d->wsets) * g->tiles_img;
    if (ts >= (1LL << 30)) return false;
    g->tiles_set = (int)ts;
    const long long u0 = (long long)d->wsets * g->taps * g->ncib * g->ncob;
    if (u0 >= (1LL << 24)) return false;
    g->units0 = (int)u0;
    int nchunk = (int)((kTargetUnits + u0 - 1) / u0);
    const int cap = g->tiles_set / kMinStages > 1 ? g->tiles_set / kMinStages : 1;
    if (nchunk > cap) nchunk = cap;
    g->tpc = cdiv(g->tiles_set, nchunk);
    g->nchunk = cdiv(g->tiles_set, g->tpc);
    g->part_elems = (long long)g->nchunk * d->wsets * g->taps * d->Cout * d->Cin;
    if ((long long)d->N * d->H * d->W * d->Cin >= (1LL << 31) || (long long)d->N * g->Ho * g->Wo * d->Cout >= (1LL << 31)) return false;
    return true;
}
static int64_t part_bytes(const Geo& g) { return align_up(g.part_elems * 4, 256); }

// MN-major, 128-byte-swizzled wgmma operand (the TMA image of a 64-channel box): 8-row K groups 1024 bytes apart (SBO);
// each operand is a single 64-element MN block, so the LBO is not used
__device__ __forceinline__ uint64_t desc_mn(uint32_t saddr) {
    const uint32_t lo = ((saddr >> 4) & 0x3FFFu) | (1u << 16);
    const uint32_t hi = (1024u >> 4) | (1u << 30);
    return ((uint64_t)hi << 32) | lo;
}
// wgmma m64n64k16, fp16 x fp16 -> fp32, A and B MN-major (transposed); acc = 0 overwrites the accumulator
__device__ __forceinline__ void mma64t(float* d, uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, "
                 "%13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, "
                 "1, 1, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
                   "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
                   "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
                   "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(acc));
}

__global__ void __launch_bounds__(kThreads, 2)
k_wgrad(const __grid_constant__ Args a) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = (smem_u32(smem) + 1023u) & ~1023u;          // swizzle atoms need 1024-byte alignment
    const uint32_t bar_full = sbase + kStages * kStageBytes, bar_empty = bar_full + 8 * kStages;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    // work unit: tap fastest, so the units that read the same dy patches run side by side
    int u = blockIdx.x;
    const int tap = u % a.taps; u /= a.taps;
    const int cib = u % a.ncib; u /= a.ncib;
    const int cob = u % a.ncob; u /= a.ncob;
    const int set = u % a.wsets;
    const int chunk = u / a.wsets;
    const int t0 = chunk * a.tpc;
    const int nst = min(a.tpc, a.tiles_set - t0);
    if (threadIdx.x == 0) {
        for (int i = 0; i < kStages; ++i) { mbar_init(bar_full + 8 * i, 1); mbar_init(bar_empty + 8 * i, 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (warp == 4 && lane < 4) tma_prefetch_desc(&a.tm[lane]);
    __syncthreads();

    if (warp == 4) {
        // ================= producer: one thread issues the four TMA boxes of every stage =================
        if (lane == 0) {
            const int r = tap / a.ks, s = tap - r * a.ks;
            pdl_wait();
            for (int it = 0; it < nst; ++it) {
                const int slot = it % kStages;
                mbar_wait(bar_empty + 8 * slot, ((it / kStages) & 1) ^ 1);
                const int tile = t0 + it;
                const int img = tile / a.tiles_img, rem = tile - img * a.tiles_img;
                const int th = rem / a.tiles_w, tw = rem - th * a.tiles_w;
                const int n = img * a.wsets + set;
                const int oh0 = th * kBox, ow0 = tw * kBox;
                const int ih0 = oh0 * a.stride - a.pad + r, iw0 = ow0 * a.stride - a.pad + s;
                const uint32_t dst = sbase + slot * kStageBytes, bar = bar_full + 8 * slot;
                mbar_expect_tx(bar, (uint32_t)kStageBytes);
                tma_load_4d(dst, &a.tm[0], cob * kCh, ow0, oh0, n, bar);
                tma_load_4d(dst + kPlane, &a.tm[1], cob * kCh, ow0, oh0, n, bar);
                tma_load_4d(dst + 2 * kPlane, &a.tm[2], cib * kCh, iw0, ih0, n, bar);
                tma_load_4d(dst + 3 * kPlane, &a.tm[3], cib * kCh, iw0, ih0, n, bar);
            }
        }
        return;
    }

    // ================= consumer warpgroup =================
    const bool leader = threadIdx.x == 0;                  // releases ring slots
    float m[32], sm[32], sum[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) { m[j] = 0.f; sm[j] = 0.f; sum[j] = 0.f; }
    pdl_wait();                                            // the partials may still be read by the previous launch
    int seg = 0, pend = -1;
    for (int it = 0; it < nst; ++it) {
        const int slot = it % kStages;
        mbar_wait_inl(bar_full + 8 * slot, (uint32_t)(it / kStages) & 1u);
        const uint32_t st = sbase + slot * kStageBytes;
        const uint64_t dh = desc_mn(st), dl = desc_mn(st + kPlane), xh = desc_mn(st + 2 * kPlane), xl = desc_mn(st + 3 * kPlane);
        const uint32_t a0 = seg == 0 ? 0u : 1u;            // the first stage of a K segment overwrites the accumulators
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) mma64t(m, dh + 128 * kk, xh + 128 * kk, kk == 0 ? a0 : 1u);   // 16 rows = 2048 bytes
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) mma64t(sm, dh + 128 * kk, xl + 128 * kk, kk == 0 ? a0 : 1u);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) mma64t(sm, dl + 128 * kk, xh + 128 * kk, 1u);
        wg_commit();
        if (++seg == kSegStages || it == nst - 1) {
            // close the K segment: the whole chain must have landed
            wg_wait_all();
            reg_fence<32>(m); reg_fence<32>(sm);
#pragma unroll
            for (int j = 0; j < 32; ++j) { sum[j] += m[j]; sum[j] += sm[j]; }
            seg = 0;
            mbar_arrive_if(bar_empty + 8 * pend, leader && pend >= 0);
            mbar_arrive_if(bar_empty + 8 * slot, leader);
            pend = -1;
        } else {
            // the stage before this one is done: free its slot, keep this one's until the next wait
            wg_wait_1();
            mbar_arrive_if(bar_empty + 8 * pend, leader && pend >= 0);
            pend = slot;
        }
    }
    wg_wait_all();
    reg_fence<32>(sum);
    // accumulator fragment of m64n64: rows (Cout) 16 w + 8 r + lane / 4, columns (Cin) 8 j + 2 (lane % 4) + {0, 1}
    float* out = a.part + (((size_t)chunk * a.wsets + set) * a.taps + tap) * (size_t)a.Cout * a.Cin;
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int co = cob * kCh + 16 * warp + 8 * r + (lane >> 2);
        if (co >= a.Cout) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int ci = cib * kCh + 8 * j + cq;
            if (ci < a.Cin) *reinterpret_cast<float2*>(out + (size_t)co * a.Cin + ci) = make_float2(sum[4 * j + 2 * r], sum[4 * j + 2 * r + 1]);
        }
    }
}

// dW in the layout of nn.Conv2d.weight with groups = wsets: [wsets * cout_r][cin_r][k][k]; chunks added in order, in
// double, then the dy and x scales removed one after the other (powers of two: exact in double, where their product
// could underflow in fp32) before the one rounding to fp32
__global__ void k_wgrad_finish(const float* __restrict__ part, int nchunk, int wsets, int taps, int Cout, int Cin, int cout_r,
                               int cin_r, const float* __restrict__ dy_scale, const float* __restrict__ x_scale,
                               float* __restrict__ dW) {
    const long long total = (long long)wsets * cout_r * cin_r * taps;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int t = (int)(i % taps);
    const int ci = (int)((i / taps) % cin_r);
    const int o = (int)(i / ((long long)taps * cin_r));
    const int s = o / cout_r, co = o - s * cout_r;
    const size_t step = (size_t)wsets * taps * Cout * Cin;
    const float* p = part + (((size_t)s * taps + t) * Cout + co) * Cin + ci;
    double acc = 0.0;
    for (int c = 0; c < nchunk; ++c) acc += (double)p[(size_t)c * step];
    if (dy_scale) acc *= (double)__ldg(dy_scale + 1);
    if (x_scale) acc *= (double)__ldg(x_scale + 1);
    dW[i] = (float)acc;
}

// Per-channel sums of an fp32 NCHW tensor [N][C][HW] (db here, BatchNorm's statistics and gradient sums in
// bn_train.cu): block (channel c, image chunk j) sums its images' planes with a fixed thread assignment and a fixed
// tree, in double; the finishing kernels add the chunks in order.  u = a (0 where mask <= 0 when a mask is given) - K;
// sum 0 = sum u, and with kTwo sum 1 = sum u * (b - shift), shift = b_shift[c] or K (common.cuh, ChanSums).  Without
// k_src, K = 0 and each term is the double of the fp32 value, so db's bits do not depend on the shift.  Sum k of
// chunk j lands at part[(k * nchunk + j) * C + c].
constexpr int kDbThreads = 256;
constexpr int kDbElems = 16384;                  // elements of one channel per db partial (at least one image)
static int db_images_per_chunk(int HW) { return HW >= kDbElems ? 1 : kDbElems / HW; }
template <bool kTwo>
__global__ void __launch_bounds__(kDbThreads)
k_db_partial(ChanSums s, int N, int C, int HW, int ipc, double* __restrict__ part) {
    __shared__ double red[kTwo ? 2 : 1][kDbThreads];
    const int c = blockIdx.x, j = blockIdx.y;
    const int n0 = j * ipc, n1 = min(N, n0 + ipc);
    const double k = s.k_src ? (double)__ldg(s.k_src + (size_t)c * HW) : 0.0;
    const double shift = kTwo && s.b_shift ? s.b_shift[c] : k;
    double acc = 0.0, acc2 = 0.0;
    for (int n = n0; n < n1; ++n) {
        const size_t off = ((size_t)n * C + c) * HW;
        for (int q = threadIdx.x; q < HW; q += kDbThreads) {
            float v = __ldg(s.a + off + q);
            if (s.mask && __ldg(s.mask + off + q) <= 0.0f) v = 0.0f;
            const double u = (double)v - k;
            acc += u;
            if (kTwo) acc2 += u * ((double)__ldg(s.b + off + q) - shift);
        }
    }
    red[0][threadIdx.x] = acc;
    if (kTwo) red[kTwo ? 1 : 0][threadIdx.x] = acc2;
    __syncthreads();
    for (int o = kDbThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            red[0][threadIdx.x] += red[0][threadIdx.x + o];
            if (kTwo) red[kTwo ? 1 : 0][threadIdx.x] += red[kTwo ? 1 : 0][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        part[(size_t)j * C + c] = red[0][0];
        if (kTwo) part[((size_t)gridDim.y + j) * C + c] = red[kTwo ? 1 : 0][0];
    }
}
__global__ void k_db_finish(const double* __restrict__ part, int nchunk, int C, float* __restrict__ db) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double acc = 0.0;
    for (int j = 0; j < nchunk; ++j) acc += part[(size_t)j * C + c];
    db[c] = (float)acc;
}

// ---------------------------------------------------------------------------------------------
// dy (and the forward's x) as scaled split-fp16 planes
// ---------------------------------------------------------------------------------------------
// v is scaled by the power of two 2^s that brings max |v| into [2^13, 2^14) before the split (pow2_scale), as the
// packed weights are: without it the lo half of a small value is a subnormal (or zero) fp16 number and the split loses
// its 22 bits, and a value past 65504 saturates.  scale[0] = 2^s, scale[1] = 2^-s, scale[2] = scratch for the absolute
// maximum (float bits).  Every finite scaled value is below 2^14, so the conversion does not saturate: NaN and +-inf
// stay non-finite (a diverging step shows in every output it reaches, as it does in torch).
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__global__ void k_split_scaled(int N, int C, int HW, int Cp, const float* __restrict__ x, const float* __restrict__ scale,
                               __half* __restrict__ hi, __half* __restrict__ lo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)N * HW) return;
    const int n = (int)(i / HW), p = (int)(i % HW);
    const float sc = __ldg(scale);
    for (int c = 0; c < Cp; c += 4) {                 // Cp % 8 == 0; reads coalesced across pixels
        float4 v;
        v.x = c + 0 < C ? x[((size_t)n * C + c + 0) * HW + p] * sc : 0.0f;
        v.y = c + 1 < C ? x[((size_t)n * C + c + 1) * HW + p] * sc : 0.0f;
        v.z = c + 2 < C ? x[((size_t)n * C + c + 2) * HW + p] * sc : 0.0f;
        v.w = c + 3 < C ? x[((size_t)n * C + c + 3) * HW + p] * sc : 0.0f;
        const uint32_t h0 = pack_h2(v.x, v.y), h1 = pack_h2(v.z, v.w);
        const float2 a = h2_to_f2(h0), b = h2_to_f2(h1);
        *reinterpret_cast<uint2*>(hi + i * Cp + c) = make_uint2(h0, h1);
        *reinterpret_cast<uint2*>(lo + i * Cp + c) = make_uint2(pack_h2(v.x - a.x, v.y - a.y), pack_h2(v.z - b.x, v.w - b.y));
    }
}

// ---------------------------------------------------------------------------------------------
// input gradient helpers
// ---------------------------------------------------------------------------------------------
// taps of one dimension for output parity a: r = r0 + stride * j (j < T) feeds dx[stride * u + a] from dy[u + c - j]
struct Par { int r0, T, c; };
__host__ __device__ __forceinline__ Par parity_taps(int k, int stride, int a) {
    const int pad = k / 2;
    Par p;
    p.r0 = (a + pad) % stride;
    p.T = p.r0 <= k - 1 ? (k - 1 - p.r0) / stride + 1 : 0;
    p.c = (a + pad - p.r0) / stride;
    return p;
}
// Pieces of one dimension.  The taps whose dy offset c - j lies in [-1, 1] form one centred window (K = 1 for a single
// centred tap, else 3).  Every other tap (the offset-2 tap of a 4-tap 7x7/s2 parity) is a piece of its own: a K = 3
// kernel whose only tap sits at the window's edge, read back shifted by t = offset - 1 (or offset + 1) output pixels.
struct P1 { int K, t, j0, j1; };
static int pieces_1d(int k, int stride, int a, P1* out) {
    const Par p = parity_taps(k, stride, a);
    if (p.T == 0) return 0;
    int n = 0;
    const int jlo = p.c - 1 > 0 ? p.c - 1 : 0, jhi = p.c + 1 < p.T - 1 ? p.c + 1 : p.T - 1;
    if (jlo <= jhi) out[n++] = {(jlo == jhi && jlo == p.c) ? 1 : 3, 0, jlo, jhi};
    for (int j = 0; j < p.T; ++j) {
        if (j >= jlo && j <= jhi) continue;
        const int o = p.c - j;
        out[n++] = {3, o > 0 ? o - 1 : o + 1, j, j};
    }
    return n;
}

// forward SIMT layout [wsets][k*k*Cin][Cout] of nn.Conv2d.weight [wsets*cout_r][cin_r][k][k] (padded channels zero)
__global__ void k_weights_simt(int wsets, int cout_r, int cin_r, int k, int Cin, int Cout, const float* __restrict__ w,
                               float* __restrict__ out) {
    const int kk = k * k;
    const long long total = (long long)wsets * kk * Cin * Cout;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int co = (int)(i % Cout);
    const int ci = (int)((i / Cout) % Cin);
    const int t = (int)((i / ((long long)Cout * Cin)) % kk);
    const int s = (int)(i / ((long long)Cout * Cin * kk));
    out[i] = (co < cout_r && ci < cin_r) ? w[(((size_t)s * cout_r + co) * cin_r + ci) * kk + t] : 0.0f;
}
// The kernel of one dgrad piece in the SIMT layout of its problem: [wsets][K*K*Cout][Cin] (the problem's input channels
// are the forward's outputs).  The piece's output at u + t is dx[stride u + a], so tap (qr, qs) holds W[.][.][r0 + stride
// j][...] with j = K/2 + c - qr - t, for j in the piece's range (the same in the other dimension), zero elsewhere.
// Stride 1: the 180-degree rotation, W'[q] = W[k-1-q].
__global__ void k_dgrad_weights(int wsets, int cout_r, int cin_r, int k, int stride, danet_dgrad_piece pc, int Cout, int Cin,
                                const float* __restrict__ w, float* __restrict__ out) {
    const int K = pc.K, KK = K * K;
    const long long total = (long long)wsets * KK * Cout * Cin;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ci = (int)(i % Cin);
    const int co = (int)((i / Cin) % Cout);
    const int q = (int)((i / ((long long)Cin * Cout)) % KK);
    const int s = (int)(i / ((long long)Cin * Cout * KK));
    const int qr = q / K, qs = q - qr * K;
    const Par pr = parity_taps(k, stride, pc.a), ps = parity_taps(k, stride, pc.b);
    const int jr = K / 2 + pr.c - qr - pc.tr, js = K / 2 + ps.c - qs - pc.tc;
    float v = 0.0f;
    if (jr >= pc.jr0 && jr <= pc.jr1 && js >= pc.jc0 && js <= pc.jc1 && co < cout_r && ci < cin_r) {
        const int r = pr.r0 + stride * jr, c = ps.r0 + stride * js;
        v = w[(((size_t)s * cout_r + co) * cin_r + ci) * k * k + r * k + c];
    }
    out[i] = v;
}

// y[n][c][h][w] (NCHW, C real channels) = sum, in piece order, over the pieces of class (h % S, w % S) of the piece's map
// at [n][h / S + tr][w / S + tc][c] (NHWC, Cp channels; 0 outside the map), times scale[1] when a scale is given, plus
// bias[(n % G) * C + c] when a bias is given (after the scale: a bias never enters a scaled sum).  A block moves a
// 32-channel x 32-column tile of one output row through shared memory, so both the reads (channels) and the writes
// (columns) are coalesced.
constexpr int kMaxPieces = 9;
struct Pieces { const float* p[kMaxPieces]; int cls[kMaxPieces], tr[kMaxPieces], tc[kMaxPieces]; int n; };
__global__ void k_scatter_nchw(int N, int C, int H, int W, int Cp, int S, int Hc, int Wc, const __grid_constant__ Pieces pc,
                               const float* __restrict__ scale, const float* __restrict__ bias, int G, float* __restrict__ y) {
    __shared__ float tile[32][33];
    const int nh = blockIdx.x, n = nh / H, h = nh - n * H;
    const int w0 = blockIdx.y * 32, c0 = blockIdx.z * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int a = h % S, u = h / S;
    const float inv = scale ? __ldg(scale + 1) : 1.0f;
    const float* bn = bias ? bias + (size_t)(n % G) * C : nullptr;
    for (int wl = ty; wl < 32; wl += 8) {
        const int w = w0 + wl, c = c0 + tx;
        float v = 0.0f;
        if (w < W && c < C) {
            const int cl = a * S + w % S, vv = w / S;
            for (int i = 0; i < pc.n; ++i) {
                const int uu = u + pc.tr[i], vi = vv + pc.tc[i];
                if (pc.cls[i] == cl && uu >= 0 && uu < Hc && vi >= 0 && vi < Wc)
                    v += __ldg(pc.p[i] + (((size_t)n * Hc + uu) * Wc + vi) * Cp + c);
            }
        }
        v *= inv;
        if (bn && c < C) v += __ldg(bn + c);
        tile[wl][tx] = v;
    }
    __syncthreads();
    for (int cl = ty; cl < 32; cl += 8) {
        const int c = c0 + cl, w = w0 + tx;
        if (c < C && w < W) y[(((size_t)n * C + c) * H + h) * W + w] = tile[tx][cl];
    }
}

}  // namespace wg

static unsigned long long g_wgrad_devs = 0;

int chan_sums_chunks(int N, int HW) {
    const int ipc = wg::db_images_per_chunk(HW);
    return (N + ipc - 1) / ipc;
}

int chan_sums_partial(const ChanSums& s, bool two, int N, int C, int HW, double* part, cudaStream_t st) {
    const int ipc = wg::db_images_per_chunk(HW), nchunk = chan_sums_chunks(N, HW);
    DANET_CHECK(nchunk < 65536, "per-channel sums: too many images");
    if (two) wg::k_db_partial<true><<<dim3(C, nchunk), wg::kDbThreads, 0, st>>>(s, N, C, HW, ipc, part);
    else wg::k_db_partial<false><<<dim3(C, nchunk), wg::kDbThreads, 0, st>>>(s, N, C, HW, ipc, part);
    DANET_LAUNCH_CHECK();
    return 0;
}

}  // namespace danet

using namespace danet;

extern "C" int64_t danet_conv_wgrad_workspace_bytes(const danet_conv_desc* d) {
    wg::Geo g;
    if (!d || !wg::make_geo(d, &g)) return 0;
    return wg::part_bytes(g);
}

extern "C" int danet_conv_wgrad(const danet_conv_desc* d, int32_t cout_r, int32_t cin_r, const danet_act* x,
                                const danet_act* dy, const float* dy_scale, const float* x_scale, float* dW, void* workspace,
                                danet_stream_t stream) {
    wg::Geo g;
    DANET_CHECK(d && wg::make_geo(d, &g), "danet_conv_wgrad: shape not supported (k in {1,3,7}, pad k/2, stride 1|2, "
                                          "channels %% 8, N %% wsets == 0)");
    DANET_CHECK(cout_r >= 1 && cout_r <= d->Cout && cin_r >= 1 && cin_r <= d->Cin, "danet_conv_wgrad: bad real channel counts");
    DANET_CHECK(workspace && aligned16(workspace), "danet_conv_wgrad: workspace must be non-null and 16-byte aligned");
    DANET_CHECK(dW && x && dy && x->hi && x->lo && dy->hi && dy->lo, "danet_conv_wgrad: needs dW and the hi and lo planes of x and dy");
    cudaStream_t st = (cudaStream_t)stream;
    int dev = 0;
    DANET_CUDA(cudaGetDevice(&dev));
    if (first_use_on_current_device(&g_wgrad_devs) != 0)
        DANET_CUDA(cudaFuncSetAttribute(wg::k_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, wg::kSmem));
    wg::Args* a = new wg::Args();
    memset(a, 0, sizeof(*a));
    int rc = 0;
    // boxes of 64 channels x 8 x 8 pixels, 128-byte swizzled: dy hi, dy lo, then x hi, x lo at the convolution's stride
    const void* planes[4] = {dy->hi, dy->lo, x->hi, x->lo};
    for (int i = 0; i < 4; ++i)
        rc |= tc::encode_nhwc_f16(&a->tm[i], planes[i], d->N, i < 2 ? g.Ho : d->H, i < 2 ? g.Wo : d->W, i < 2 ? d->Cout : d->Cin,
                                  wg::kCh, wg::kBox, wg::kBox, CU_TENSOR_MAP_SWIZZLE_128B, i < 2 ? 1 : d->stride);
    if (rc != 0) { delete a; return -1; }
    a->part = (float*)workspace;
    a->Cin = d->Cin; a->Cout = d->Cout; a->ks = d->ksize; a->stride = d->stride; a->pad = d->pad; a->wsets = d->wsets;
    a->taps = g.taps; a->ncib = g.ncib; a->ncob = g.ncob;
    a->tiles_w = g.tiles_w; a->tiles_img = g.tiles_img; a->tiles_set = g.tiles_set; a->tpc = g.tpc;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)((long long)g.units0 * g.nchunk)); cfg.blockDim = dim3(wg::kThreads);
    cfg.dynamicSmemBytes = wg::kSmem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, wg::k_wgrad, *a);
    delete a;
    DANET_CUDA(e);
    const long long total = (long long)d->wsets * cout_r * cin_r * g.taps;
    wg::k_wgrad_finish<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const float*)workspace, g.nchunk, d->wsets, g.taps, d->Cout,
                                                                      d->Cin, cout_r, cin_r, dy_scale, x_scale, dW);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int64_t danet_conv_bias_grad_workspace_bytes(int32_t N, int32_t C, int32_t HW) {
    if (N < 1 || C < 1 || HW < 1) return 0;
    return (int64_t)chan_sums_chunks(N, HW) * C * 8;
}

extern "C" int danet_conv_bias_grad(int32_t N, int32_t C, int32_t HW, const float* dy, float* db, void* workspace,
                                    danet_stream_t stream) {
    DANET_CHECK(N >= 1 && C >= 1 && HW >= 1 && dy && db && workspace && ((uintptr_t)workspace & 7) == 0,
                "danet_conv_bias_grad: bad arguments");
    const int nchunk = chan_sums_chunks(N, HW);
    DANET_CHECK(nchunk < 65536, "danet_conv_bias_grad: too many images");
    cudaStream_t st = (cudaStream_t)stream;
    const ChanSums s = {dy, nullptr, nullptr, nullptr, nullptr};
    if (chan_sums_partial(s, false, N, C, HW, (double*)workspace, st) != 0) return -3;
    wg::k_db_finish<<<cdiv(C, 128), 128, 0, st>>>((const double*)workspace, nchunk, C, db);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_conv_grad_split(int32_t N, int32_t C, int32_t HW, int32_t Cp, const float* dy, void* hi, void* lo,
                                     float* scale, danet_stream_t stream) {
    DANET_CHECK(N >= 1 && C >= 1 && HW >= 1 && Cp >= C && Cp % 8 == 0 && dy && hi && lo && scale,
                "danet_conv_grad_split: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = pow2_scale(dy, (long long)N * C * HW, scale, 2, st);
    if (rc != 0) return rc;
    wg::k_split_scaled<<<(unsigned)(((long long)N * HW + 255) / 256), 256, 0, st>>>(N, C, HW, Cp, dy, scale, (__half*)hi, (__half*)lo);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_conv_weights_simt(int32_t wsets, int32_t cout_r, int32_t cin_r, int32_t ksize, int32_t Cout, int32_t Cin,
                                       const float* w, float* w_simt, danet_stream_t stream) {
    DANET_CHECK(w && w_simt && wsets >= 1 && ksize >= 1 && cout_r >= 1 && cin_r >= 1 && Cout >= cout_r && Cin >= cin_r,
                "danet_conv_weights_simt: bad arguments");
    const long long total = (long long)wsets * ksize * ksize * Cin * Cout;
    wg::k_weights_simt<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(wsets, cout_r, cin_r, ksize, Cin, Cout, w,
                                                                                         w_simt);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int32_t danet_conv_dgrad_pieces(int32_t ksize, int32_t stride, danet_dgrad_piece* pieces) {
    if (!pieces || !(ksize == 1 || ksize == 3 || ksize == 7) || !(stride == 1 || stride == 2)) return -1;
    if (ksize == 7 && stride == 1) return -1;         // not a forward shape of the engine either
    int n = 0;
    for (int a = 0; a < stride; ++a)
        for (int b = 0; b < stride; ++b) {
            wg::P1 pr[8], pc[8];
            const int nr = wg::pieces_1d(ksize, stride, a, pr), nc = wg::pieces_1d(ksize, stride, b, pc);
            for (int i = 0; i < nr; ++i)
                for (int j = 0; j < nc; ++j) {
                    if (n == wg::kMaxPieces) return -1;
                    danet_dgrad_piece& p = pieces[n++];
                    p.a = a; p.b = b; p.K = pr[i].K > pc[j].K ? pr[i].K : pc[j].K;
                    p.tr = pr[i].t; p.tc = pc[j].t;
                    p.jr0 = pr[i].j0; p.jr1 = pr[i].j1; p.jc0 = pc[j].j0; p.jc1 = pc[j].j1;
                }
        }
    return n;
}

extern "C" int danet_conv_dgrad_weights(int32_t wsets, int32_t cout_r, int32_t cin_r, int32_t ksize, int32_t stride,
                                        const danet_dgrad_piece* piece, int32_t Cout, int32_t Cin, const float* w, float* w_out,
                                        danet_stream_t stream) {
    DANET_CHECK(piece && (piece->K == 1 || piece->K == 3), "danet_conv_dgrad_weights: bad piece");
    DANET_CHECK(w && w_out && wsets >= 1 && cout_r >= 1 && cin_r >= 1 && Cout >= cout_r && Cin >= cin_r && (stride == 1 || stride == 2),
                "danet_conv_dgrad_weights: bad arguments");
    const long long total = (long long)wsets * piece->K * piece->K * Cout * Cin;
    wg::k_dgrad_weights<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(wsets, cout_r, cin_r, ksize, stride, *piece,
                                                                                          Cout, Cin, w, w_out);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_conv_dgrad_scatter(int32_t N, int32_t C, int32_t H, int32_t W, int32_t Cp, int32_t stride, int32_t Hc,
                                        int32_t Wc, int32_t npieces, const danet_dgrad_piece* pieces, const float* const* maps,
                                        const float* scale, const float* bias, int32_t groups, float* y, danet_stream_t stream) {
    DANET_CHECK(pieces && maps && y && N >= 1 && C >= 1 && Cp >= C && H >= 1 && W >= 1 && (stride == 1 || stride == 2) &&
                npieces >= 0 && npieces <= wg::kMaxPieces && groups >= 1, "danet_conv_dgrad_scatter: bad arguments");
    DANET_CHECK(Hc >= (H + stride - 1) / stride && Wc >= (W + stride - 1) / stride, "danet_conv_dgrad_scatter: maps too small");
    DANET_CHECK((long long)N * H < (1LL << 31), "danet_conv_dgrad_scatter: too many rows");
    wg::Pieces p = {};
    p.n = npieces;
    for (int i = 0; i < npieces; ++i) {
        DANET_CHECK(maps[i] && pieces[i].a >= 0 && pieces[i].a < stride && pieces[i].b >= 0 && pieces[i].b < stride,
                    "danet_conv_dgrad_scatter: bad piece %d", i);
        p.p[i] = maps[i]; p.cls[i] = pieces[i].a * stride + pieces[i].b; p.tr[i] = pieces[i].tr; p.tc[i] = pieces[i].tc;
    }
    const dim3 grid((unsigned)(N * H), (unsigned)cdiv(W, 32), (unsigned)cdiv(C, 32));
    wg::k_scatter_nchw<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(N, C, H, W, Cp, stride, Hc, Wc, p, scale, bias, groups,
                                                                       y);
    DANET_LAUNCH_CHECK();
    return 0;
}
