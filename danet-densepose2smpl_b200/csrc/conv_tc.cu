// wgmma implicit-GEMM convolution engine for sm_90a (Hopper).
// The tensor-core path of models/module/hr_module.py:161-179,334-378 + res_module.py:27-97,281-390,393-535
// convolutions (conv + folded BN + residual + ReLU): 1x1 / 3x3 / 7x7, stride 1 or 2, weight sets (the
// reference's grouped convolutions over the (batch, part)-flattened image axis).
//
// Numerics.  Activations and weights are SPLIT-FP16: v = hi + lo with hi = rn_f16(v), lo = rn_f16(v - hi)
// (22 significant bits, fp16 exponent range; plain fp32 numbers below 6e-5 keep an absolute error <= 3e-8).
// "exact" mode issues three products per K step, hi*hi + hi*lo + lo*hi, in fp32 accumulators (the dropped lo*lo
// term is 2^-22 relative): fp32-grade results from the fp16 tensor pipe, which is what lets the default path meet
// the reference's fp32 outputs to 1e-4.  "fast" mode issues hi*hi only.
//
// Structure (one persistent CTA per SM, up to kMaxProb independent convolutions -- e.g. the parallel branches of one
// HRNet stage -- in ONE launch over a concatenated space of work units: tiles in fast mode, tile pairs in exact mode):
//   A (activations): fp16 NHWC planes in HBM.  One TMA tensor-map load (cp.async.bulk.tensor.4d, SWIZZLE_128B/64B/32B,
//       out-of-bounds zero fill = the convolution's padding, elementStrides = 2 for the parity planes of a
//       stride-2 convolution) brings the input HALO of a tile -- (16+k-1) x (8+k-1) pixels x <= 64 channels --
//       into shared memory, one 128/64/32-byte row per pixel.  Eight consecutive MMA rows are eight consecutive
//       pixels of one halo row, the next 8-row group is the next image row (SBO = halo pitch), so every filter
//       tap is just a different descriptor start address: an input element crosses L2->SM ~1.3x, not 9x.
//   B (weights): pre-packed once (danet_conv_tc_pack) into the swizzled shared-memory image of every
//       (N tile, channel chunk, parity plane, tap group[, hi/lo]) block; streamed with 1-D cp.async.bulk.
//   MMA: two consumer warpgroups per tile, each owning 64 of the tile's 128 output pixels (8 image rows x 8 columns), issue
//       wgmma.mma_async m64nNk16 (N = the tile's output channels) with fp32 accumulators in registers.
//       exact mode: the lo and hi weight rows are concatenated along N, so hi*[lo|hi] is ONE MMA of width 2N whose
//       first half lands in a separate small-term accumulator; lo*hi joins the small terms.  Per weight block all
//       hi*[lo|hi] MMAs are issued first, then all lo*hi MMAs (two same-shape chains).
//       Every MMA has a compile-time width (one tile body per N tile width); a warpgroup commits one group per
//       weight block and waits only for the block before it, so the MMAs of consecutive blocks stay in flight.
//   K segments (exact mode): the tensor core's fp32 accumulation truncates, which biases long chains; after every
//       kSegMmas main-chain MMAs the accumulators are added in fp32 round-to-nearest to a running sum that starts at
//       bias + residual.
//   Epilogue: each consumer thread holds 2 pixels x 2 consecutive channels per 8-channel group; ReLU, output as
//       split-fp16 planes and/or fp32.
//   Kernels: one per precision mode, each with its own tile body; they share the prologue, the scheduler, the output
//       mapping and the epilogue.  One thread runs the scheduler and issues every TMA / bulk copy in consumption order.
//       k_conv_tc_fast (288 threads, fast_tile): a producer warp after the two consumer warpgroups.  k_conv_tc_exact
//       (512 threads, exact_tile): four consumer warpgroups, two per tile of a pair (same weight set and N tile,
//       pair_coord), so one weight stream feeds 256 pixels.  A 17th warp would cut every thread to 96 registers, so
//       warp 0 issues the copies (one elected lane) where its warpgroup frees ring slots (produce).
//   Launch: programmatic dependent launch; every mbarrier wait is bounded (traps instead of hanging).
#include "common.cuh"
#include "wgmma_f16.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <mutex>
#include <utility>
#include <string.h>
#include <math.h>

namespace danet {
namespace tc {

constexpr int kTileH = 16, kTileW = 8;
// Fast mode: two consumer warpgroups (64 pixels = 8 tile rows each) and a producer warp.  Exact mode: four consumer
// warpgroups, two per tile of a tile pair, and no producer warp (warp 0 issues the copies): 16 warps x 32 lanes x 128
// registers fill the register file, which a 17th warp would cut to 96 registers per thread.
constexpr int kConsFast = 2, kThreadsFast = (4 * kConsFast + 1) * 32;
constexpr int kWarpProd = 4 * kConsFast;               // fast mode: the producer warp follows the consumer warpgroups
constexpr int kConsExact = 4, kThreadsExact = 4 * kConsExact * 32;
constexpr int kNtMaxExact = 64, kNtMaxFast = 256;      // output channels per N tile: bounded by the register accumulators
constexpr int kMaxAStages = 8, kMaxBStages = 8;
constexpr int kSmemMax = 227 * 1024;                   // opt-in dynamic shared memory per CTA on sm_90
constexpr int kSmemFixed = 2048;                       // barriers + 1024-byte alignment slack
constexpr int kSchedDepth = 4, kSchedAhead = 2, kSchedStatic = 3;
constexpr int kPackHeader = 1024;                      // packed weights start with a header: float[0] = 2^s applied to the weights, float[1] = 2^-s
constexpr int kSegMmas = 8;                            // exact mode: close a K segment after a weight block once it holds >= 8 main-chain MMAs
// The close rule, asked after every weight block: the tile's last block always closes; seg_mmas counts the main-chain
// MMAs since the last close, this block included.  exact_tile and danet_conv_tc_dispatch both ask here.
__host__ __device__ constexpr bool seg_close(bool last_block, int seg_mmas) { return last_block || seg_mmas >= kSegMmas; }

struct alignas(64) Prob {
    CUtensorMap tm[2];                   // input planes: hi, lo
    const uint8_t* wpk; const float* bias;
    const float* res_f; const __half* res_hi; const __half* res_lo;
    float* y_f; __half* y_hi; __half* y_lo;
    int N, H, W, Cin, Cout, Ho, Wo, ks, stride, pad, relu, wsets, exact;
    int npa;                             // active parity planes (1 for stride 1, up to 4 for stride 2)
    int SWB, KCH, nchunks;               // swizzle bytes per pixel row, channels per chunk, chunks
    int TG;                              // filter taps per weight block
    int NT, ntn;                         // output channels per N tile, N tiles
    int nstack, hs, box_h;               // small maps: nstack images share one tile; image n's rows start at group n*hs
                                         // (hs = H + pad: the zero rows between images are the TMA out-of-bounds fill)
    int bpc;                             // weight blocks per channel chunk
    int par_py[4], par_px[4], ntap[4], ngrp[4], stage_bytes, sbo_a;   // a plane's halo box (the largest): bytes, row pitch
    int tapoff16[4][16];                 // smem offset (16-byte units) of each tap's shifted view inside the plane
    int tapidx[4][16];                   // original filter tap index r*ks+s (weight packing)
    int tiles_w, tiles_h, tile_count;
    int rows_blk;                        // rows of one weight block per tap
    int tap_bytes, b_block_bytes, nblk;  // nblk: weight blocks per (weight set, N tile)
    long long blocks_per_set;
    unsigned long long m_ntn, m_tw, m_th, m_ws;
};

constexpr int kMaxProb = 6;
struct ArgsN {
    int nprob, total_units, na_stages, a_slot_bytes, nb_stages, b_slot_bytes;
    unsigned* sched;                     // [2]: dynamic unit counter, finished-CTA counter (self-resetting); NULL = static round-robin
    Prob p[kMaxProb];
    // the scheduled work units, tiles in fast mode and tile pairs (pair_coord) in exact mode: problem i owns units
    // unit_base[i] .. + unit_count[i]
    int unit_base[kMaxProb], unit_count[kMaxProb];
};

static unsigned long long magic40(int d) { return (1ull << 40) / (unsigned long long)d + 1ull; }

// ---------------------------------------------------------------------------------------------
// host: geometry of one problem (everything but the shared-memory ring sizes, which belong to the launch)
// ---------------------------------------------------------------------------------------------
static bool make_prob(const danet_conv_desc* d, Prob* g) {
    if (!(d->stride == 1 || d->stride == 2) || !(d->ksize == 1 || d->ksize == 3 || d->ksize == 7) || d->pad != d->ksize / 2) return false;
    if (d->Cin % 8 != 0 || d->Cout % 8 != 0 || d->H < 1 || d->W < 1 || d->N < 1 || d->wsets < 1) return false;
    g->N = d->N; g->H = d->H; g->W = d->W; g->Cin = d->Cin; g->Cout = d->Cout; g->ks = d->ksize;
    g->pad = d->pad; g->stride = d->stride; g->relu = d->relu; g->wsets = d->wsets;
    g->exact = (d->flags & DANET_CONV_EXACT) ? 1 : 0;
    g->Ho = (d->H + 2 * d->pad - d->ksize) / d->stride + 1;
    g->Wo = (d->W + 2 * d->pad - d->ksize) / d->stride + 1;
    if (g->Ho < 1 || g->Wo < 1) return false;
    // N tiling: equal tiles of a multiple of 16 channels, at most kNtMax* (exact mode keeps three register
    // accumulators per output -- main, small terms, running sum -- so its tiles are narrower)
    const int np = (d->Cout + 15) / 16 * 16;
    const int ntmax = g->exact ? kNtMaxExact : kNtMaxFast;
    g->ntn = (np + ntmax - 1) / ntmax;
    g->NT = ((np + g->ntn - 1) / g->ntn + 15) / 16 * 16;
    // parity decomposition: a stride-2 convolution is the sum over the input parities (py,px) of dense
    // stride-1 sub-convolutions; each parity plane is one TMA box with elementStrides = 2
    g->npa = 0;
    int max_ntap = 0, tr_max = 0, tc_max = 0;
    int tc_[4];
    for (int py = 0; py < d->stride; ++py)
        for (int px = 0; px < d->stride; ++px) {
            const int tr = py < d->ksize ? (d->ksize - 1 - py) / d->stride + 1 : 0;     // taps r = py + stride*i
            const int tcn = px < d->ksize ? (d->ksize - 1 - px) / d->stride + 1 : 0;
            if (tr * tcn == 0) continue;
            if (tr * tcn > 16) return false;
            const int a = g->npa++;
            g->par_py[a] = py; g->par_px[a] = px; g->ntap[a] = tr * tcn; tc_[a] = tcn;
            max_ntap = tr * tcn > max_ntap ? tr * tcn : max_ntap;
            tr_max = tr > tr_max ? tr : tr_max; tc_max = tcn > tc_max ? tcn : tc_max;
        }
    // every parity plane is loaded with the box of the largest one (one tensor map per input plane)
    const int Hb = kTileH + tr_max - 1, Wb = kTileW + tc_max - 1;
    // Small maps: several images share the 16 row groups of a tile, each loaded by its own TMA box at row offset n * hs.
    //   stride 1 (H + pad <= 8): box = H + 2 pad rows, hs = H + pad -- the bottom halo of one image and the top halo of
    //     the next are the same shared-memory rows, both filled with out-of-bounds zeros;
    //   stride 2 (Ho + tr - 1 <= 8): one box of Ho + tr - 1 rows per image and parity plane, hs = the box height.
    // Row groups that fall outside an image's Ho output rows produce garbage outputs the epilogue never stores.  With
    // several weight sets a tile stacks images n, n + wsets, n + 2 wsets, ...: all of them use one weight set.
    g->nstack = 1; g->hs = kTileH; g->box_h = Hb;
    if (d->stride == 1 && d->H + d->pad <= kTileH / 2) {
        g->hs = d->H + d->pad;
        g->box_h = d->H + 2 * d->pad;
    } else if (d->stride == 2 && g->Ho + tr_max - 1 <= kTileH / 2) {
        g->hs = g->box_h = g->Ho + tr_max - 1;
    }
    // swizzle width: the widest row unless the channel count is tiny
    int swb = 128;
    const int c16 = (d->Cin + 15) / 16 * 16;
    while (swb > 32 && swb / 2 >= 2 * c16) swb /= 2;
    // Stacked image n's box lands at shared-memory offset n * hs * Wb * SWB, and a TMA destination must be 128-byte
    // aligned.  With 32- and 64-byte rows some heights give an odd offset (2x2 maps of <= 16 channels under a 3x3
    // filter: 3 rows x 10 pixels x 32 bytes); those maps get a tile per image.
    if (g->hs < kTileH && (g->hs * Wb * swb) % 128 != 0) { g->hs = kTileH; g->box_h = Hb; }
    if (g->hs < kTileH) g->nstack = kTileH / g->hs;
    g->SWB = swb; g->KCH = swb / 2;
    g->nchunks = (d->Cin + g->KCH - 1) / g->KCH;
    g->rows_blk = g->NT * (g->exact ? 2 : 1);
    g->tap_bytes = g->rows_blk * swb;
    int tg = max_ntap;
    // weight block size: larger blocks mean fewer barrier round trips; exact mode keeps more ring slots instead
    while (tg > 1 && tg * g->tap_bytes > (g->exact ? 24 : 48) * 1024) --tg;
    g->TG = tg;
    g->b_block_bytes = (tg * g->tap_bytes + 1023) / 1024 * 1024;
    g->stage_bytes = Hb * Wb * swb; g->sbo_a = Wb * swb;
    g->bpc = 0;
    for (int a = 0; a < 4; ++a) {
        if (a >= g->npa) { g->par_py[a] = g->par_px[a] = g->ntap[a] = g->ngrp[a] = 0;
                           for (int k = 0; k < 16; ++k) g->tapoff16[a][k] = g->tapidx[a][k] = 0; continue; }
        g->ngrp[a] = (g->ntap[a] + tg - 1) / tg;
        g->bpc += g->ngrp[a];
        for (int k = 0; k < 16; ++k) { g->tapoff16[a][k] = 0; g->tapidx[a][k] = 0; }
        for (int k = 0; k < g->ntap[a]; ++k) {
            const int ti = k / tc_[a], tj = k % tc_[a];
            g->tapoff16[a][k] = ((ti * Wb + tj) * swb) >> 4;
            g->tapidx[a][k] = (g->par_py[a] + d->stride * ti) * d->ksize + (g->par_px[a] + d->stride * tj);
        }
    }
    g->nblk = g->nchunks * g->bpc;
    g->blocks_per_set = (long long)g->ntn * g->nblk;
    g->tiles_w = (g->Wo + kTileW - 1) / kTileW; g->tiles_h = (g->Ho + kTileH - 1) / kTileH;
    // image groups: one image each, or (stacked) wsets x ceil(images per set / nstack)
    const long long groups = g->nstack == 1 ? d->N
                           : (long long)d->wsets * (((d->N + d->wsets - 1) / d->wsets + g->nstack - 1) / g->nstack);
    const long long tiles = groups * g->tiles_h * g->tiles_w * g->ntn;
    if (tiles >= (1 << 24) || g->wsets >= (1 << 16)) return false;
    if ((long long)d->N * g->Ho * g->Wo * d->Cout >= (1LL << 31) || (long long)d->N * d->H * d->W * d->Cin >= (1LL << 31)) return false;   // 32-bit element offsets
    g->tile_count = (int)tiles;
    g->m_ntn = magic40(g->ntn); g->m_tw = magic40(g->tiles_w); g->m_th = magic40(g->tiles_h); g->m_ws = magic40(g->wsets);
    return true;
}

// Exact mode's tile pairs (pair_coord).  The two tiles of a pair have the same weight set and N tile, so one weight
// stream feeds both:
//   - maps of two or more tile rows: tile rows 2q and 2q + 1 of one image group, same tile column;
//   - maps of one tile row (small and stacked maps, the 1x1-tile maps): image groups 2q wsets + ws and (2q + 1) wsets + ws
//     of one weight set ws, same tile column.
// A pair without a partner (an odd number of tile rows, or of image groups per weight set) gets a second tile past the
// map: its rows are >= Ho or its images >= N, so TMA fills its halo with zeros and it stores nothing.
static int pair_count(const Prob& g) {
    const int U = g.tiles_h * g.tiles_w * g.ntn;
    const int groups = g.tile_count / U;
    if (g.tiles_h > 1) return groups * ((g.tiles_h + 1) / 2) * g.tiles_w * g.ntn;
    const int per_set = (groups + g.wsets - 1) / g.wsets;
    return (per_set + 1) / 2 * g.wsets * U;
}

// ring sizes of a launch over n problems; false if they cannot fit
static bool plan_rings(ArgsN* a) {
    int amax = 0, bmax = 0, need_a = 2, max_a = kMaxAStages;
    bool exact = false;
    for (int i = 0; i < a->nprob; ++i) {
        amax = a->p[i].stage_bytes > amax ? a->p[i].stage_bytes : amax;
        bmax = a->p[i].b_block_bytes > bmax ? a->p[i].b_block_bytes : bmax;
        if (a->p[i].exact) exact = true;
    }
    a->a_slot_bytes = (amax + 1023) / 1024 * 1024;
    a->b_slot_bytes = (bmax + 1023) / 1024 * 1024;
    if (exact) {
        // an A slot holds the halos of both tiles of a pair.  Three slots: the current parity plane's hi and lo and one
        // prefetch; the rest goes to weight blocks
        a->a_slot_bytes *= 2;
        need_a = max_a = 3;
    }
    int nb = 3;
    int na = (kSmemMax - kSmemFixed - nb * a->b_slot_bytes) / a->a_slot_bytes;
    if (na < need_a) { nb = 2; na = (kSmemMax - kSmemFixed - nb * a->b_slot_bytes) / a->a_slot_bytes; }
    if (na < need_a) return false;
    if (na > max_a) na = max_a;
    // spend what is left on deeper weight prefetch
    while (nb < kMaxBStages && kSmemFixed + na * a->a_slot_bytes + (nb + 1) * a->b_slot_bytes <= kSmemMax) ++nb;
    a->na_stages = na; a->nb_stages = nb;
    return true;
}

// ---------------------------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------------------------
// K-major swizzled shared-memory matrix descriptor of wgmma: start address and SBO (the stride between 8-row groups)
// in 16-byte units, LBO unused for swizzled K-major layouts, swizzle mode in bits 62-63 (128B = 1, 64B = 2, 32B = 3).
// The swizzle phase follows the absolute shared-memory address (the TMA writes the same pattern), so a start
// address that is only row-aligned (a filter tap shifted by a few pixels) needs no base offset.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t sbo_bytes, uint32_t swb) {
    const uint32_t mode = swb == 128 ? 1u : (swb == 64 ? 2u : 3u);
    const uint32_t lo = ((saddr >> 4) & 0x3FFFu) | (1u << 16);
    const uint32_t hi = ((sbo_bytes >> 4) & 0x3FFFu) | (mode << 30);
    return ((uint64_t)hi << 32) | lo;
}
// physical offset of logical byte offset `off` inside a 1024-byte-aligned swizzled region
__host__ __device__ __forceinline__ uint32_t swz(uint32_t off, uint32_t mask) { return off ^ (((off >> 7) & mask) << 4); }
__host__ __device__ __forceinline__ int mdiv(int x, unsigned long long m) { return (int)(((unsigned long long)(unsigned)x * m) >> 40); }

// img0: the tile's first image; stacked image n is img0 + n * wsets.  ws: the tile's weight set.
struct TileCoord { int nt, tw, th, img0, ws; };
// image group grp: weight set grp % wsets; with stacking, the group holds images img0, img0 + wsets, ...
__host__ __device__ __forceinline__ void group_coord(const Prob& g, int grp, TileCoord& c) {
    const int bg = mdiv(grp, g.m_ws);
    c.ws = grp - bg * g.wsets;
    c.img0 = c.ws + g.wsets * bg * g.nstack;          // = grp without stacking
}
__device__ __forceinline__ TileCoord decode_tile(const Prob& g, int t) {
    TileCoord c;
    int r = mdiv(t, g.m_ntn); c.nt = t - r * g.ntn;
    int r2 = mdiv(r, g.m_tw); c.tw = r - r2 * g.tiles_w;
    const int grp = mdiv(r2, g.m_th); c.th = r2 - grp * g.tiles_h;
    group_coord(g, grp, c);
    return c;
}

// exact mode: tile h (0, 1) of pair pp (problem-relative); pair_count describes the pairing.  Pair index =
// (outer * tiles_w + tw) * ntn + nt, outer = group * ceil(tiles_h / 2) + q (tile rows 2q, 2q + 1) or, with one tile
// row, q * wsets + ws (image groups 2q wsets + ws, (2q + 1) wsets + ws).
__host__ __device__ __forceinline__ TileCoord pair_coord(const Prob& g, int pp, int h) {
    TileCoord c;
    const int r = mdiv(pp, g.m_ntn); c.nt = pp - r * g.ntn;
    const int outer = mdiv(r, g.m_tw); c.tw = r - outer * g.tiles_w;
    int grp;
    if (g.tiles_h > 1) {
        const int th2 = (g.tiles_h + 1) >> 1;
        grp = outer / th2;
        c.th = 2 * (outer - grp * th2) + h;
    } else {
        const int q = mdiv(outer, g.m_ws);
        grp = (2 * q + h) * g.wsets + (outer - q * g.wsets);
        c.th = 0;
    }
    group_coord(g, grp, c);
    return c;
}

// ring positions of one consumer warpgroup (every consumer walks the A and B rings in the producer's order)
struct Ring { int as, bs; uint32_t aph, bph; };

// shared-memory addresses of the rings and their barriers
struct Smem { uint32_t sA, sB, bar_a_full, bar_a_empty, bar_b_full, bar_b_empty; };

// barrier region (at bar_a_full): A / B ring barriers, then the tile scheduler's ring and, in exact mode, the copy cursor
constexpr uint32_t kOffSchedFull = 512, kOffSchedEmpty = kOffSchedFull + 8 * kSchedDepth;
constexpr uint32_t kOffSchedRing = kOffSchedFull + 16 * kSchedDepth, kOffCursor = 640, kOffPark = 768;

// Exact mode's copy cursor.  Warp 0 walks the copy sequence of its CTA's tile pairs (each pair: per channel chunk and
// parity plane, the hi and lo halos of both tiles, then the plane's weight blocks) and runs it ahead of consumption by
// the ring depths.  Its state is a row of ints in shared memory between runs, so that it costs no registers while the
// tile body runs with every accumulator live; produce() holds the row in registers only while warp 0's own loop state
// is parked (exact_tile).  Every lane of warp 0 reads and writes the same values.
enum CursorField {
    kCurSeq, kCurPub, kCurPubEnd,        // pair being loaded, next scheduler ring entry to publish, the last one is out
    kCurPi,                              // problem of the pair being loaded (-1: take the next pair)
    kCurC, kCurSlot, kCurStep,           // channel chunk, parity plane, step (0, 1: halo planes hi, lo; 2..: weight blocks)
    kCurH0, kCurH1, kCurW0,              // halo origin: rows of the pair's two tiles, columns (shared)
    kCurImg0, kCurImg1, kCurBlk,         // first image of each tile; the pair's next weight block
    kCurFa, kCurFb,                      // A / B ring fills issued
    kCurRa, kCurRb,                      // A / B ring uses warpgroup 0 has released
    kCurAs, kCurBs, kCurAph, kCurBph,    // next A / B slot and the empty-barrier phases
    kCurFields
};
constexpr int kCurWords = (kCurFields + 3) / 4 * 4;   // the row padded to whole 16-byte vectors (cur_load)
static_assert(kOffCursor % 16 == 0 && kOffCursor + 4 * kCurWords <= kOffPark && kOffPark + 4 * 32 <= 1024, "barrier region layout");

// consumer side of the scheduler ring: one lane waits for entry `seq`, reads the work unit and frees the entry
__device__ __forceinline__ int sched_next(const Smem& S, int seq) {
    const int slot = seq & (kSchedDepth - 1);
    mbar_wait(S.bar_a_full + kOffSchedFull + 8 * slot, (seq / kSchedDepth) & 1);
    int unit;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(unit) : "r"(S.bar_a_full + kOffSchedRing + 4 * slot) : "memory");
    mbar_arrive(S.bar_a_full + kOffSchedEmpty + 8 * slot);
    return unit;
}

// the problem that owns work unit u (u < total_units)
__device__ __forceinline__ int unit_prob(const ArgsN& a, int u) {
    for (int pi = 0;; ++pi) if (u < a.unit_base[pi] + a.unit_count[pi]) return pi;
}

// The work unit that scheduler entry pub of this CTA names, total_units once they are all taken.  A CTA's first
// kSchedStatic entries are its round-robin share (no atomic latency at start-up); later ones come from the global
// counter, which take() increments (heaviest problems first): greedy list scheduling over heterogeneous units.
template <class Take>
__device__ __forceinline__ int sched_unit(const ArgsN& a, int pub, Take take) {
    const int t = pub < kSchedStatic || !a.sched ? (int)blockIdx.x + pub * (int)gridDim.x : take() + kSchedStatic * (int)gridDim.x;
    return t < a.total_units ? t : a.total_units;
}
__device__ __forceinline__ int cur_get(uint32_t cur, int f) {
    int v;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(cur + 4 * f) : "memory");
    return v;
}
__device__ __forceinline__ void cur_set(uint32_t cur, int f, int v) {
    asm volatile("st.shared.s32 [%0], %1;" ::"r"(cur + 4 * f), "r"(v) : "memory");
}

// The cursor's row as 16-byte vectors: produce() reads it once into registers and writes it back once, so its steps do
// not wait on a shared-memory load each.
__device__ __forceinline__ void cur_load(uint32_t cur, int* f) {
#pragma unroll
    for (int k = 0; k < kCurWords; k += 4)
        asm volatile("ld.shared.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(f[k]), "=r"(f[k + 1]), "=r"(f[k + 2]), "=r"(f[k + 3])
                     : "r"(cur + 4 * k) : "memory");
}
__device__ __forceinline__ void cur_store(uint32_t cur, const int* f) {
#pragma unroll
    for (int k = 0; k < kCurWords; k += 4)
        asm volatile("st.shared.v4.s32 [%0], {%1, %2, %3, %4};" ::"r"(cur + 4 * k), "r"(f[k]), "r"(f[k + 1]), "r"(f[k + 2]),
                     "r"(f[k + 3]) : "memory");
}

// Exact mode, warp 0 only, every lane (uniform control flow; the elected lane issues): the copy cursor's steps on its row f
// (cur_load).  Issue the copies whose slots warpgroup 0 no longer holds (ring fills below the releases f[kCurRa],
// f[kCurRb] plus the ring depths), in consumption order, waiting for the other warpgroups to free each slot.  Those never
// wait on a copy at or after the one waited for: a warpgroup frees a weight block once the next block's MMAs are issued,
// and a halo slot at the end of its parity plane (drained), so only earlier copies are needed.  Stops at the first copy
// whose slot warpgroup 0 still holds.
__device__ __forceinline__ void cursor_steps(const ArgsN& a, const Smem& S, int* f) {
#pragma unroll 1
    for (;;) {
        if (f[kCurPi] < 0) {
            // publish scheduler entries up to kSchedAhead pairs past the one loaded next, then take that one
#pragma unroll 1
            while (f[kCurPub] <= f[kCurSeq] + kSchedAhead && !f[kCurPubEnd]) {
                const int pub = f[kCurPub], rs = pub & (kSchedDepth - 1);
                mbar_wait_inl(S.bar_a_full + kOffSchedEmpty + 8 * rs, ((pub / kSchedDepth) & 1) ^ 1);
                const int t = sched_unit(a, pub, [&] { return __shfl_sync(0xffffffffu, atom_inc_elect(a.sched), 0); });
                if (t == a.total_units) f[kCurPubEnd] = 1;
                st_arrive_elect(S.bar_a_full + kOffSchedRing + 4 * rs, t, S.bar_a_full + kOffSchedFull + 8 * rs);
                f[kCurPub] = pub + 1;
            }
            int pair;
            asm volatile("ld.shared.s32 %0, [%1];" : "=r"(pair)
                         : "r"(S.bar_a_full + kOffSchedRing + 4 * (f[kCurSeq] & (kSchedDepth - 1))) : "memory");
            pair = __shfl_sync(0xffffffffu, pair, 0);            // the elected lane 0 wrote it
            if (pair >= a.total_units) return;
            const int pi = unit_prob(a, pair);
            const Prob& P = a.p[pi];
            const int pp = pair - a.unit_base[pi];
            {
                const TileCoord tc = pair_coord(P, pp, 0);
                f[kCurH0] = tc.th * kTileH * P.stride - P.pad;
                f[kCurW0] = tc.tw * kTileW * P.stride - P.pad;
                f[kCurImg0] = tc.img0;
                f[kCurBlk] = tc.ws * (int)P.blocks_per_set + tc.nt * P.nblk;
            }
            {
                const TileCoord tc = pair_coord(P, pp, 1);
                f[kCurH1] = tc.th * kTileH * P.stride - P.pad;
                f[kCurImg1] = tc.img0;
            }
            f[kCurC] = 0; f[kCurSlot] = 0; f[kCurStep] = 0;
            f[kCurPi] = pi;
        }
        const Prob& P = a.p[f[kCurPi]];
        const int step = f[kCurStep], slot = f[kCurSlot];
        if (step < 2) {
            // the hi (step 0) or lo (step 1) halo plane of both tiles, into one A slot
            if (f[kCurFa] >= f[kCurRa] + a.na_stages) return;
            const int as = f[kCurAs];
            mbar_wait_inl(S.bar_a_empty + 8 * as, ((f[kCurAph] >> as) & 1) ^ 1);
            mbar_expect_tx_elect(S.bar_a_full + 8 * as, 2u * P.nstack * P.box_h * P.sbo_a);
            // box k: the first tile's nstack images, then the second tile's (rows or images beyond the map are out of
            // bounds: zero fill)
#pragma unroll 1
            for (int k = 0; k < 2 * P.nstack; ++k) {
                const int h = k >= P.nstack ? 1 : 0, n = k - h * P.nstack;
                tma_load_4d_elect(S.sA + as * a.a_slot_bytes + h * (a.a_slot_bytes >> 1) + n * P.hs * P.sbo_a,
                                  &P.tm[step], f[kCurC] * P.KCH, f[kCurW0] + P.par_px[slot],
                                  (h ? f[kCurH1] : f[kCurH0]) + P.par_py[slot], (h ? f[kCurImg1] : f[kCurImg0]) + n * P.wsets,
                                  S.bar_a_full + 8 * as);
            }
            f[kCurAph] ^= 1 << as;
            f[kCurAs] = as + 1 == a.na_stages ? 0 : as + 1;
            f[kCurFa] += 1;
            f[kCurStep] = step + 1;
        } else {
            if (f[kCurFb] >= f[kCurRb] + a.nb_stages) return;
            const int bs = f[kCurBs];
            mbar_wait_inl(S.bar_b_empty + 8 * bs, ((f[kCurBph] >> bs) & 1) ^ 1);
            const uint32_t bar = S.bar_b_full + 8 * bs;
            mbar_expect_tx_elect(bar, (uint32_t)P.b_block_bytes);
            bulk_g2s_elect(S.sB + bs * a.b_slot_bytes, P.wpk + kPackHeader + (long long)f[kCurBlk] * P.b_block_bytes,
                           (uint32_t)P.b_block_bytes, bar);
            f[kCurBph] ^= 1 << bs;
            f[kCurBs] = bs + 1 == a.nb_stages ? 0 : bs + 1;
            f[kCurFb] += 1;
            f[kCurBlk] += 1;
            if (step - 1 < P.ngrp[slot]) f[kCurStep] = step + 1;
            else {                                            // the parity plane is complete
                f[kCurStep] = 0;
                if (slot + 1 < P.npa) f[kCurSlot] = slot + 1;
                else {
                    f[kCurSlot] = 0;
                    if (f[kCurC] + 1 < P.nchunks) f[kCurC] += 1;
                    else { f[kCurPi] = -1; f[kCurSeq] += 1; }
                }
            }
        }
    }
}

// Exact mode, warp 0 only: warpgroup 0 has just released dA A and dB B ring uses; run the copy cursor.
__device__ __forceinline__ void produce(const ArgsN& a, const Smem& S, int dA, int dB) {
    const uint32_t cur = S.bar_a_full + kOffCursor;
    int f[kCurWords];
    cur_load(cur, f);
    f[kCurRa] += dA; f[kCurRb] += dB;
    cursor_steps(a, S, f);
    cur_store(cur, f);
}

// ---------------------------------------------------------------------------------------------
// the tile bodies: one consumer warpgroup's share of one tile, at a compile-time N tile width
// ---------------------------------------------------------------------------------------------
// NT: the problem's N tile width (P.NT).  Every wgmma has a fixed width and a fixed accumulator set, so ptxas keeps
// them in flight: one commit group per weight block, and the warpgroup waits only for the block before it (wait_group
// 1) -- that block's B slot is freed once the next block's MMAs are issued.

// the next slot of a ring: wait until it is full, flip its phase bit, advance
__device__ __forceinline__ int ring_take(uint32_t bar_full, int& idx, uint32_t& ph, int n) {
    const int s = idx;
    mbar_wait_inl(bar_full + 8 * s, (ph >> s) & 1u);
    ph ^= 1u << s; if (++idx == n) idx = 0;
    return s;
}

// This thread's outputs in warpgroup wg's 64 pixels of a tile.  The accumulator fragment of m64nNk16 holds tile rows
// prow0, prow0 + 1 at column pcol and channels 8 j + cq, 8 j + cq + 1 of every 8-channel group j: registers 4 j + 2 r
// + {0, 1} for row prow0 + r.  Row prow is tile row prow of image tc.img0, or (stacked small maps) row prow % hs of image
// tc.img0 + (prow / hs) * wsets -- rows Ho.. of a stacked image's hs rows produce no output.  eoff[r]: offset of the
// pixel's channel tc.nt * NT + cq in the output; cw: channels of the N tile that exist (multiple of 8); boff: bias offset.
struct TileOut { uint32_t eoff[2]; bool ok[2]; int cw, boff; };
template <int NT>
__device__ __forceinline__ TileOut tile_out(const Prob& P, const TileCoord& tc, int wg, int w4, int lane) {
    TileOut o;
    const int prow0 = 8 * wg + 2 * w4, pcol = lane >> 2, cq = 2 * (lane & 3);
    const int Cout = P.Cout, Wo = P.Wo, Ho = P.Ho;
    const int ow = tc.tw * kTileW + pcol;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int prow = prow0 + r;
        int oh = tc.th * kTileH + prow, img = tc.img0;
        bool row_ok = oh < Ho;
        if (P.nstack > 1) {
            const int n = prow / P.hs;
            oh = prow - n * P.hs; img = tc.img0 + n * P.wsets;
            row_ok = oh < Ho && n < P.nstack && img < P.N;
        }
        o.ok[r] = row_ok && ow < Wo;
        o.eoff[r] = ((uint32_t)(img * Ho + oh) * Wo + ow) * Cout + tc.nt * NT + cq;
    }
    o.cw = Cout - tc.nt * NT;
    o.boff = tc.ws * Cout + tc.nt * NT + cq;
    return o;
}

// The MMAs of taps k0 .. k0 + ntk - 1 of a weight block, kv K steps each (K steps wholly beyond Cin are not issued), of
// width W into (d0, d1).  The first one overwrites the accumulators when acc is 0; returns the next acc (1).  Off: the
// type of the caller's per-tap B stride tap16 (exact mode keeps it in an int that warp 0 can park).
template <int W, class Off>
__device__ __forceinline__ uint32_t mma_taps(float* d0, float* d1, uint64_t ad, uint64_t bd, const Prob& P, int slot, int k0,
                                             int ntk, int kv, Off tap16, uint32_t acc) {
#pragma unroll 1
    for (int tt = 0; tt < ntk; ++tt) {
        const uint32_t toff = (uint32_t)P.tapoff16[slot][k0 + tt];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if (kk >= kv) break;
            Wgmma<W>::mma(d0, d1, ad + toff + 2 * kk, bd + tt * tap16 + 2 * kk, acc);
            acc = 1;
        }
    }
    return acc;
}

// x 2^-s, ReLU, split, store.  value(j, r): the float2 of channel group j, row r, in the packed weights' 2^s scale.
template <int NT, class Value>
__device__ __forceinline__ void store_out(const Prob& P, const TileOut& o, float inv_scale, Value value) {
    const int relu = P.relu;
    float* __restrict__ y_f = P.y_f; __half* __restrict__ y_hi = P.y_hi; __half* __restrict__ y_lo = P.y_lo;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
        if (8 * j >= o.cw) continue;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!o.ok[r]) continue;
            const float2 v = value(j, r);
            float x0 = v.x * inv_scale, x1 = v.y * inv_scale;
            if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
            const uint32_t e = o.eoff[r] + 8 * j;
            if (y_f) *reinterpret_cast<float2*>(y_f + e) = make_float2(x0, x1);
            if (y_hi) {
                const uint32_t hv = pack_h2_rn(x0, x1);
                *reinterpret_cast<uint32_t*>(y_hi + e) = hv;
                if (y_lo) {
                    const float2 t = h2_to_f2(hv);
                    *reinterpret_cast<uint32_t*>(y_lo + e) = pack_h2_rn(x0 - t.x, x1 - t.y);
                }
            }
        }
    }
}

// Fast mode: warpgroup wg's 64 pixels (tile rows 8 wg ..) of a tile, hi * hi into the accumulator m.  Bias and residual
// are added to the finished accumulator in the epilogue.  A parity plane's A slot is held, like a B slot, until the
// wait after the next block.
template <int NT>
__device__ __forceinline__ void fast_tile(const ArgsN& a, const Prob& P, const TileCoord tc, const Smem S, Ring& R, int wg, int w4,
                                          int lane, bool leader, float* m) {
    constexpr int NV = NT / 2;            // fp32 accumulator registers per thread (64 x NT warpgroup tile)
    const TileOut o = tile_out<NT>(P, tc, wg, w4, lane);
    // the packed weights carry a power-of-two scale 2^s (so that their lo halves are normal fp16 numbers): bias and
    // residual enter the sum times 2^s and the result leaves it times 2^-s -- exact in fp32
    const float2 wsc = __ldg(reinterpret_cast<const float2*>(P.wpk));
    // bias + residual of this thread's outputs (channel group j, row r)
    auto init_term = [&](int j, int r) {
        float2 t = make_float2(0.f, 0.f);
        if (8 * j < o.cw) {
            if (P.bias) t = __ldg(reinterpret_cast<const float2*>(P.bias + o.boff + 8 * j));
            if (o.ok[r]) {
                if (P.res_f) {
                    const float2 q = __ldg(reinterpret_cast<const float2*>(P.res_f + o.eoff[r] + 8 * j));
                    t.x += q.x; t.y += q.y;
                } else if (P.res_hi) {
                    const float2 q = h2_to_f2(__ldg(reinterpret_cast<const unsigned*>(P.res_hi + o.eoff[r] + 8 * j)));
                    t.x += q.x; t.y += q.y;
                    if (P.res_lo) {
                        const float2 q2 = h2_to_f2(__ldg(reinterpret_cast<const unsigned*>(P.res_lo + o.eoff[r] + 8 * j)));
                        t.x += q2.x; t.y += q2.y;
                    }
                }
            }
        }
        return t;
    };
    const int nchunks = P.nchunks, npa = P.npa, TG = P.TG, SWB = P.SWB, kmma = P.KCH / 16;   // K = 16 halves per MMA
    const uint32_t tap16 = P.tap_bytes >> 4;
    const uint64_t bd0 = make_desc(0, 8 * SWB, SWB);
    uint32_t acc = 0;
    // ring slots whose MMAs may still be in flight: freed once a later wait covers them (-1: none)
    int pend_b = -1, pend_a = -1;
    auto release_pending = [&]() {
        mbar_arrive_if(S.bar_b_empty + 8 * pend_b, leader && pend_b >= 0);
        mbar_arrive_if(S.bar_a_empty + 8 * pend_a, leader && pend_a >= 0);
        pend_b = pend_a = -1;
    };
    for (int c = 0; c < nchunks; ++c) {
        const int kreal = (P.Cin - c * P.KCH + 15) >> 4;
        const int kv = kreal < kmma ? kreal : kmma;
        for (int slot = 0; slot < npa; ++slot) {
            const int as = ring_take(S.bar_a_full, R.as, R.aph, a.na_stages);
            // this warpgroup's 8 tile rows start 8 halo rows further down for the second warpgroup
            const uint64_t ad0 = make_desc(0, (uint32_t)P.sbo_a, SWB) + ((uint32_t)(wg * 8 * P.sbo_a) >> 4);
            const uint64_t ad = ad0 + ((S.sA + as * a.a_slot_bytes) >> 4);
            const int ngrp = P.ngrp[slot], ntap = P.ntap[slot];
            for (int tg = 0; tg < ngrp; ++tg) {
                const int k0 = tg * TG;
                const int ntk = min(TG, ntap - k0);
                const int bs = ring_take(S.bar_b_full, R.bs, R.bph, a.nb_stages);
                const uint64_t bd = bd0 + ((S.sB + bs * a.b_slot_bytes) >> 4);
                wg_fence();
                acc = mma_taps<NT>(m, m + NT / 4, ad, bd, P, slot, k0, ntk, kv, tap16, acc);
                wg_commit();
                // the block before this one is done: free its slots, keep this one's until the next wait
                wg_wait_1();
                release_pending();
                pend_b = bs;
                if (tg == ngrp - 1) pend_a = as;
            }
        }
    }
    wg_wait_all();
    reg_fence<NV>(m);
    release_pending();
    store_out<NT>(P, o, wsc.y, [&](int j, int r) {
        const float2 t = init_term(j, r);
        return make_float2(m[4 * j + 2 * r] + t.x * wsc.x, m[4 * j + 2 * r + 1] + t.y * wsc.x);
    });
}

// Exact mode: warpgroup wg's 64 pixels of tile `half` of a pair (the second tile's halo is the second half of each A
// slot); warp 0 (prod) also runs the copy cursor.  Per weight block, hi * [lo | hi] and then lo * hi: the main chain in
// m, the small terms in s.  At every K segment close both are added to the running sum, which starts at bias + residual.
// A parity plane's end drains too and frees its two A slots.
template <int NT>
__device__ __forceinline__ void exact_tile(const ArgsN& a, const Prob& P, const TileCoord tc, const Smem S, Ring& R, int wg, int w4,
                                           int lane, bool leader, int half, bool prod, float* accs, float* sum) {
    constexpr int NV = NT / 2, nj = NT / 8;   // accumulator registers per thread and set; 8-channel groups
    float* s = accs;                      // small terms hi*lo + lo*hi
    float* m = accs + NV;                 // main chain
    TileOut o = tile_out<NT>(P, tc, wg, w4, lane);
    if (tc.img0 >= P.N) o.ok[0] = o.ok[1] = false;       // the second tile of a pair without a partner stores nothing
    // the packed weights' scale 2^s: bias and residual enter the sum times 2^s, the result leaves it times 2^-s
    const float2 wsc = __ldg(reinterpret_cast<const float2*>(P.wpk));
    {
        // The running sum starts at bias + residual, before the tile's first MMA.  The loads of two channel groups are
        // issued together and the adds follow, so that the loads' latencies overlap instead of adding up.  q holds the
        // residual of output (j, r): an fp32 pair, or the hi and lo half2 words.  Two groups at a time: the accumulators
        // are live here, and a larger q spills.
        const float* const bias = P.bias, * const rf = P.res_f;
        const __half* const rh = P.res_hi, * const rl = P.res_lo;
        constexpr int kJ = 2;                         // nj = NT / 8 is even
#pragma unroll
        for (int j0 = 0; j0 < nj; j0 += kJ) {
            uint32_t q[4 * kJ];
#pragma unroll
            for (int j = j0; j < j0 + kJ; ++j)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int i = 4 * j + 2 * r, k = i - 4 * j0;
                    const bool in = 8 * j < o.cw && o.ok[r];
                    float2 b = make_float2(0.f, 0.f);
                    if (8 * j < o.cw && bias) b = __ldg(reinterpret_cast<const float2*>(bias + o.boff + 8 * j));
                    sum[i] = b.x; sum[i + 1] = b.y;
                    q[k] = q[k + 1] = 0u;
                    if (in && rf) {
                        const float2 v = __ldg(reinterpret_cast<const float2*>(rf + o.eoff[r] + 8 * j));
                        q[k] = __float_as_uint(v.x); q[k + 1] = __float_as_uint(v.y);
                    } else if (in && rh) {
                        q[k] = __ldg(reinterpret_cast<const unsigned*>(rh + o.eoff[r] + 8 * j));
                        if (rl) q[k + 1] = __ldg(reinterpret_cast<const unsigned*>(rl + o.eoff[r] + 8 * j));
                    }
                }
#pragma unroll
            for (int j = j0; j < j0 + kJ; ++j)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int i = 4 * j + 2 * r, k = i - 4 * j0;
                    float tx = sum[i], ty = sum[i + 1];
                    if (8 * j < o.cw && o.ok[r]) {
                        if (rf) { tx += __uint_as_float(q[k]); ty += __uint_as_float(q[k + 1]); }
                        else if (rh) {
                            const float2 h = h2_to_f2(q[k]);
                            tx += h.x; ty += h.y;
                            if (rl) { const float2 l = h2_to_f2(q[k + 1]); tx += l.x; ty += l.y; }
                        }
                    }
                    sum[i] = tx * wsc.x; sum[i + 1] = ty * wsc.x;
                }
        }
    }
    // ints, not consts: warp 0 parks these while it runs the copy cursor (below)
    int nchunks = P.nchunks, npa = P.npa, TG = P.TG, SWB = P.SWB, kmma = P.KCH / 16;   // K = 16 halves per MMA
    int tap16 = P.tap_bytes >> 4, hi16 = (NT * SWB) >> 4;                            // the hi weight rows follow the NT lo rows
    uint32_t acc = 0;
    int seg_cnt = 0;
    int pend_b = -1;                                      // the previous block's B slot until a later wait covers it
    for (int c = 0; c < nchunks; ++c) {
        const int kreal = (P.Cin - c * P.KCH + 15) >> 4;
        int kv = kreal < kmma ? kreal : kmma;
        for (int slot = 0; slot < npa; ++slot) {
            int as_hi = ring_take(S.bar_a_full, R.as, R.aph, a.na_stages);
            int as_lo = ring_take(S.bar_a_full, R.as, R.aph, a.na_stages);
            int ngrp = P.ngrp[slot], ntap = P.ntap[slot];
            for (int tg = 0; tg < ngrp; ++tg) {
                const int k0 = tg * TG;
                const int ntk = min(TG, ntap - k0);
                const int bs = ring_take(S.bar_b_full, R.bs, R.bph, a.nb_stages);
                const uint64_t bd = make_desc(0, 8 * SWB, SWB) + ((S.sB + bs * a.b_slot_bytes) >> 4);
                wg_fence();
                // the A operands: the pair's second tile is the slot's second half.  Computed here, per block, because
                // warp 0 parks as_hi / as_lo while it runs the copy cursor (below).
                const uint32_t tile_a = S.sA + half * (a.a_slot_bytes >> 1) + wg * 8 * P.sbo_a;
                const uint64_t ad1 = make_desc(0, (uint32_t)P.sbo_a, SWB);
                const uint64_t ad_hi = ad1 + ((tile_a + as_hi * a.a_slot_bytes) >> 4);
                const uint64_t ad_lo = ad1 + ((tile_a + as_lo * a.a_slot_bytes) >> 4);
                // hi * [lo | hi]: small terms in s, main chain in m; then lo * hi into s.  The instruction's accumulator
                // is (s, m) in that order: ptxas keeps the wgmmas in flight only if the lo * hi accumulator s is the
                // start of the wide one, not its second half.
                acc = mma_taps<2 * NT>(s, m, ad_hi, bd, P, slot, k0, ntk, kv, tap16, acc);
                mma_taps<NT>(s, s + NT / 4, ad_lo, bd + hi16, P, slot, k0, ntk, kv, tap16, 1u);
                wg_commit();
                const bool plane_end = tg == ngrp - 1;
                seg_cnt += ntk * kv;
                const bool close = seg_close(c == nchunks - 1 && slot == npa - 1 && plane_end, seg_cnt);
                // A parity plane's end drains too, so that its two A slots are free before the next plane's halos are
                // loaded: with three A slots, that is what lets the next plane's lo halo in.  The chain goes on (acc
                // stays 1) unless the K segment closes, so the MMA sequence is unchanged.
                const int db = pend_b >= 0 ? 1 : 0;
                int dA = 0, dB = db;
                if (close || plane_end) {
                    wg_wait_all();
                    reg_fence<NV>(m);
                    reg_fence<NV>(s);
                    if (close) {
#pragma unroll
                        for (int j = 0; j < NV; ++j) {
                            sum[j] += m[j];
                            sum[j] += s[j];
                        }
                        acc = 0; seg_cnt = 0;
                    }
                    mbar_arrive_if(S.bar_b_empty + 8 * pend_b, leader && pend_b >= 0);
                    pend_b = -1;
                    mbar_arrive_if(S.bar_b_empty + 8 * bs, leader);
                    mbar_arrive_if(S.bar_a_empty + 8 * as_hi, leader && plane_end);
                    mbar_arrive_if(S.bar_a_empty + 8 * as_lo, leader && plane_end);
                    dA = plane_end ? 2 : 0; dB = db + 1;
                } else {
                    wg_wait_1();
                    mbar_arrive_if(S.bar_b_empty + 8 * pend_b, leader && pend_b >= 0);
                    pend_b = bs;
                }
                if (prod && (dA | dB)) {
                    // Warp 0 runs the copy cursor, unless the block released no slot: then the cursor would stop at
                    // the copy it stopped at last time.  Its loop state waits in shared memory meanwhile: with every
                    // accumulator live, the cursor has no registers to spare otherwise.  The reloads go through a
                    // shuffle so that ptxas still sees warp-uniform values (a loop bound it cannot prove uniform
                    // would serialise the wgmmas).
                    const uint32_t pk = S.bar_a_full + kOffPark;
                    int* const v[] = {&c, &slot, &tg, &kv, &ngrp, &ntap, &as_hi, &as_lo, &seg_cnt, &pend_b, &R.as, &R.bs,
                                      &nchunks, &npa, &TG, &SWB, &kmma, &tap16, &hi16};
                    constexpr int nv = sizeof(v) / sizeof(v[0]);
#pragma unroll
                    for (int i = 0; i < nv; ++i) cur_set(pk, i, *v[i]);
                    cur_set(pk, nv, (int)acc); cur_set(pk, nv + 1, (int)R.aph); cur_set(pk, nv + 2, (int)R.bph);
                    produce(a, S, dA, dB);
#pragma unroll
                    for (int i = 0; i < nv; ++i) *v[i] = __shfl_sync(0xffffffffu, cur_get(pk, i), 0);
                    acc = (uint32_t)__shfl_sync(0xffffffffu, cur_get(pk, nv), 0);
                    R.aph = (uint32_t)__shfl_sync(0xffffffffu, cur_get(pk, nv + 1), 0);
                    R.bph = (uint32_t)__shfl_sync(0xffffffffu, cur_get(pk, nv + 2), 0);
                }
            }
        }
    }
    // the last segment closed (drained) already; the wait tells ptxas that no MMA is in flight past here
    wg_wait_all();
    reg_fence<NV>(m);
    reg_fence<NV>(s);
    store_out<NT>(P, o, wsc.y, [&](int j, int r) { return make_float2(sum[4 * j + 2 * r], sum[4 * j + 2 * r + 1]); });
}

// ---------------------------------------------------------------------------------------------
// the kernels, one per precision mode
// ---------------------------------------------------------------------------------------------
// shared memory: the A ring, the B ring, then the barrier region (1024-byte aligned: the swizzle atoms need it)
__device__ __forceinline__ Smem carve_smem(const ArgsN& a) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sA = (smem_u32(smem) + 1023u) & ~1023u, sB = sA + a.na_stages * a.a_slot_bytes;
    const uint32_t sBar = sB + a.nb_stages * a.b_slot_bytes;       // barriers: A full, A empty, B full, B empty, ...
    return {sA, sB, sBar, sBar + 8 * kMaxAStages, sBar + 16 * kMaxAStages, sBar + 16 * kMaxAStages + 8 * kMaxBStages};
}

// the warp index through a shuffle: ptxas then knows it is warp-uniform, and so is every branch on the warp role (a
// role branch it cannot prove uniform makes it serialise the wgmmas behind it)
__device__ __forceinline__ int warp_index() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }

// Barrier set-up of both kernels.  A ring slot is freed by one arrival of each of the cons consumer warpgroups, a
// scheduler entry by lane 0 of every consumer warp.  copy_warp, which issues the copies, prefetches the first `maps`
// tensor maps of every problem.
__device__ __forceinline__ void start_cta(const ArgsN& a, const Smem& S, int cons, int copy_warp, int maps, int warp, int lane) {
    if (threadIdx.x == 0) {
        for (int i = 0; i < a.na_stages; ++i) { mbar_init(S.bar_a_full + 8 * i, 1); mbar_init(S.bar_a_empty + 8 * i, cons); }
        for (int i = 0; i < a.nb_stages; ++i) { mbar_init(S.bar_b_full + 8 * i, 1); mbar_init(S.bar_b_empty + 8 * i, cons); }
        for (int i = 0; i < kSchedDepth; ++i) { mbar_init(S.bar_a_full + kOffSchedFull + 8 * i, 1); mbar_init(S.bar_a_full + kOffSchedEmpty + 8 * i, 4 * cons); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (warp == copy_warp && lane < a.nprob)
#pragma unroll
        for (int i = 0; i < maps; ++i) tma_prefetch_desc(&a.p[lane].tm[i]);
    __syncthreads();
    pdl_launch_dependents();            // the next launch may fill SMs as our CTAs retire
}

// the last CTA to finish re-arms the scheduler for the next launch (or graph replay) that uses this slot
__device__ __forceinline__ void sched_rearm(const ArgsN& a) {
    __syncthreads();
    if (threadIdx.x == 0 && a.sched) {
        __threadfence();
        if (atomicAdd(a.sched + 1, 1u) == gridDim.x - 1) { a.sched[0] = 0u; a.sched[1] = 0u; __threadfence(); }
    }
}

// Exact mode: four consumer warpgroups over tile pairs; warp 0 also issues every copy (produce).
__global__ void __launch_bounds__(kThreadsExact, 1)
k_conv_tc_exact(const __grid_constant__ ArgsN a) {
    const Smem S = carve_smem(a);
    const int warp = warp_index(), lane = threadIdx.x & 31;
    if (threadIdx.x == 0)                                   // the copy cursor: no pair taken yet
        for (int f = 0; f < kCurWords; ++f) cur_set(S.bar_a_full + kOffCursor, f, f == kCurPi ? -1 : 0);
    start_cta(a, S, kConsExact, 0, 2, warp, lane);
    const int wg = warp >> 2, w4 = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;          // releases ring slots for its warpgroup
    const bool prod = warp == 0;
    Ring R = {0, 0, 0u, 0u};
    constexpr int NVMAX = kNtMaxExact / 2;
    float accs[2 * NVMAX];                 // small terms then main chain
    float sum[NVMAX];                      // bias + residual + every closed K segment, fp32 round-to-nearest
    pdl_wait();                            // activations come from the previous kernel; residual reads / output writes
    if (prod) produce(a, S, 0, 0);         // the first copies and scheduler entries
    for (int seq = 0;; ++seq) {
        int pair = 0;
        if (lane == 0) pair = sched_next(S, seq);
        pair = __shfl_sync(0xffffffffu, pair, 0);
        if (pair >= a.total_units) break;
        const int pi = unit_prob(a, pair);
        const Prob& P = a.p[pi];
        // warpgroups 0, 1 take the pair's first tile, 2, 3 the second (the same tile of the next image group)
        const int half = wg >> 1;
        const TileCoord tc = pair_coord(P, pair - a.unit_base[pi], half);
#define DANET_NT_CASE(N) case N: exact_tile<N>(a, P, tc, S, R, wg & 1, w4, lane, leader, half, prod, accs, sum); break;
        switch (P.NT) {
            DANET_NT_CASE(16) DANET_NT_CASE(32) DANET_NT_CASE(48) DANET_NT_CASE(64)
            default: __trap();
        }
#undef DANET_NT_CASE
    }
    sched_rearm(a);
}

// Fast mode: two consumer warpgroups over tiles and a producer warp that runs the tile scheduler and issues every copy.
__global__ void __launch_bounds__(kThreadsFast, 1)
k_conv_tc_fast(const __grid_constant__ ArgsN a) {
    const Smem S = carve_smem(a);
    const int warp = warp_index(), lane = threadIdx.x & 31;
    start_cta(a, S, kConsFast, kWarpProd, 1, warp, lane);
    if (warp == kWarpProd) {
        // ================= producer: tile scheduler + every TMA / bulk copy, in consumption order =================
        if (lane == 0) {
            int as = 0, bs = 0; uint32_t aph = 0, bph = 0;
            // tile scheduler: this thread publishes tile indices kSchedAhead tiles ahead of its own loads
            int pub = 0; bool ended = false;
            for (int seq = 0;; ++seq) {
                while (pub <= seq + kSchedAhead && !ended) {
                    const int slot = pub & (kSchedDepth - 1);
                    mbar_wait(S.bar_a_full + kOffSchedEmpty + 8 * slot, ((pub / kSchedDepth) & 1) ^ 1);
                    const int t = sched_unit(a, pub, [&] { return (int)atomicAdd(a.sched, 1u); });
                    ended = t == a.total_units;
                    asm volatile("st.shared.s32 [%0], %1;" ::"r"(S.bar_a_full + kOffSchedRing + 4 * slot), "r"(t) : "memory");
                    mbar_arrive(S.bar_a_full + kOffSchedFull + 8 * slot);
                    ++pub;
                }
                int tile;
                asm volatile("ld.shared.s32 %0, [%1];" : "=r"(tile) : "r"(S.bar_a_full + kOffSchedRing + 4 * (seq & (kSchedDepth - 1))) : "memory");
                if (tile >= a.total_units) break;
                if (seq == 0) pdl_wait();                            // activations come from the previous kernel
                const int pi = unit_prob(a, tile);
                const Prob& P = a.p[pi];
                const TileCoord tc = decode_tile(P, tile - a.unit_base[pi]);
                const int h0 = tc.th * kTileH * P.stride - P.pad, w0 = tc.tw * kTileW * P.stride - P.pad;
                const uint8_t* src = P.wpk + kPackHeader + ((long long)tc.ws * P.blocks_per_set + (long long)tc.nt * P.nblk) * P.b_block_bytes;
                int b = 0;
                for (int c = 0; c < P.nchunks; ++c)
                    for (int slot = 0; slot < P.npa; ++slot) {
                        mbar_wait(S.bar_a_empty + 8 * as, ((aph >> as) & 1u) ^ 1u);
                        if (P.nstack > 1) {
                            const uint32_t box_bytes = (uint32_t)(P.box_h * P.sbo_a);
                            mbar_expect_tx(S.bar_a_full + 8 * as, box_bytes * P.nstack);
                            for (int n = 0; n < P.nstack; ++n)       // images beyond N are out of bounds: zero rows
                                tma_load_4d(S.sA + as * a.a_slot_bytes + n * P.hs * P.sbo_a, &P.tm[0], c * P.KCH,
                                            w0 + P.par_px[slot], h0 + P.par_py[slot], tc.img0 + n * P.wsets, S.bar_a_full + 8 * as);
                        } else {
                            mbar_expect_tx(S.bar_a_full + 8 * as, (uint32_t)P.stage_bytes);
                            tma_load_4d(S.sA + as * a.a_slot_bytes, &P.tm[0], c * P.KCH, w0 + P.par_px[slot], h0 + P.par_py[slot],
                                        tc.img0, S.bar_a_full + 8 * as);
                        }
                        aph ^= 1u << as;
                        if (++as == a.na_stages) as = 0;
                        for (int t = 0; t < P.ngrp[slot]; ++t, ++b) {
                            mbar_wait(S.bar_b_empty + 8 * bs, ((bph >> bs) & 1u) ^ 1u);
                            mbar_expect_tx(S.bar_b_full + 8 * bs, (uint32_t)P.b_block_bytes);
                            bulk_g2s(S.sB + bs * a.b_slot_bytes, src + (long long)b * P.b_block_bytes, (uint32_t)P.b_block_bytes,
                                     S.bar_b_full + 8 * bs);
                            bph ^= 1u << bs;
                            if (++bs == a.nb_stages) bs = 0;
                        }
                    }
            }
        }
    } else {
        // ================= consumer warpgroups: wgmma main loop + epilogue =================
        const int wg = warp >> 2, w4 = warp & 3;
        const bool leader = (threadIdx.x & 127) == 0;          // releases ring slots for its warpgroup
        Ring R = {0, 0, 0u, 0u};
        float accs[kNtMaxFast / 2];                              // the main chain (the only accumulator set)
        pdl_wait();                                              // residual reads / output writes
        for (int seq = 0;; ++seq) {
            int tile = 0;
            if (lane == 0) tile = sched_next(S, seq);
            tile = __shfl_sync(0xffffffffu, tile, 0);
            if (tile >= a.total_units) break;
            const int pi = unit_prob(a, tile);
            const Prob& P = a.p[pi];
            const TileCoord tc = decode_tile(P, tile - a.unit_base[pi]);
            // one tile body per N tile width make_prob can produce; every body uses a prefix of the same accumulator
            // array, so the widths share their registers
#define DANET_NT_CASE(N) case N: fast_tile<N>(a, P, tc, S, R, wg, w4, lane, leader, accs); break;
            switch (P.NT) {
                DANET_NT_CASE(16) DANET_NT_CASE(32) DANET_NT_CASE(48) DANET_NT_CASE(64) DANET_NT_CASE(80) DANET_NT_CASE(96)
                DANET_NT_CASE(112) DANET_NT_CASE(128) DANET_NT_CASE(144) DANET_NT_CASE(160) DANET_NT_CASE(176) DANET_NT_CASE(192)
                DANET_NT_CASE(208) DANET_NT_CASE(224) DANET_NT_CASE(240) DANET_NT_CASE(256)
                default: __trap();
            }
#undef DANET_NT_CASE
        }
    }
    sched_rearm(a);
}

// pow2_scale (common.cuh): k_absmax leaves the largest finite |x| in word 2 of the header, k_pow2_scale turns it into
// the power-of-two scale 2^s that brings it into [2^13, 2^14) -- the lo halves (2^-11 of the value) of all but the
// tiniest values are then normal fp16 numbers and the split keeps its 22 bits -- and writes the header words.  s is
// clamped to [-126, 126] so that 2^s and 2^-s are both finite, normal fp32 numbers: a maximum below 2^-112 gets the
// largest scale there is instead of an infinite one (and a zero inverse).
__global__ void k_absmax(long long n, const float* __restrict__ x, unsigned* __restrict__ out) {
    unsigned m = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned b = __float_as_uint(fabsf(x[i]));
        if (b < 0x7f800000u && b > m) m = b;           // finite values only; non-negative floats order like their bit patterns
    }
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);   // a maximum: the same result in any order
}
__global__ void k_pow2_scale(float* __restrict__ hdr, int words) {
    __shared__ float sc;
    if (threadIdx.x == 0) {
        const float amax = __uint_as_float(reinterpret_cast<const unsigned*>(hdr)[2]);
        float scale = 1.0f;
        if (amax > 0.0f) { int e = 0; frexpf(amax, &e); scale = ldexpf(1.0f, min(max(14 - e, -126), 126)); }
        sc = scale;
    }
    __syncthreads();
    if ((int)threadIdx.x < words) hdr[threadIdx.x] = threadIdx.x == 0 ? sc : (threadIdx.x == 1 ? 1.0f / sc : 0.0f);
}

// weight packing: SIMT layout [wsets][ks*ks*Cin][Cout] fp32 -> swizzled smem-image blocks of split fp16.
// block (ws, nt, chunk, parity plane, tap group[, plane]) = [TG taps][rows][SWB bytes]; rows = output channels
// (exact mode: NT lo rows then NT hi rows).  The header's scale 2^s (pow2_scale) multiplies every weight.
__device__ __forceinline__ void pack_one(const Prob& g, const float* __restrict__ w, __half* __restrict__ out, float scale) {
    const int blk_halves = g.b_block_bytes / 2;
    const long long total = (long long)g.wsets * g.blocks_per_set * blk_halves;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int taps = g.ks * g.ks;
    long long blk = i / blk_halves;
    const uint32_t poff = (uint32_t)(i % blk_halves) * 2;             // physical byte offset inside the block
    const uint32_t smask = g.SWB == 128 ? 7u : (g.SWB == 64 ? 3u : 1u);
    const uint32_t loff = swz(poff, smask);                            // the XOR swizzle is an involution
    const int tt = loff / g.tap_bytes;
    float v = 0.f;
    int want_lo = 0;
    if (tt < g.TG) {
        const uint32_t r = loff - tt * g.tap_bytes;
        int n = r / g.SWB; const int kk = (r % g.SWB) / 2;
        if (g.exact) { if (n < g.NT) want_lo = 1; else n -= g.NT; }
        int bi = (int)(blk % g.bpc); blk /= g.bpc;
        int slot = 0, base = 0;
        for (;;) { const int nb = g.ngrp[slot]; if (bi < base + nb || slot + 1 >= g.npa) break; base += nb; ++slot; }
        const int tgi = bi - base;
        const int c = (int)(blk % g.nchunks); blk /= g.nchunks;
        const int nt = (int)(blk % g.ntn);
        const int ws = (int)(blk / g.ntn);
        const int k = tgi * g.TG + tt;
        if (k < g.ntap[slot]) {
            const int t = g.tapidx[slot][k];
            const int cin = c * g.KCH + kk;
            const int co = nt * g.NT + n;
            if (co < g.Cout && cin < g.Cin) v = w[((size_t)ws * taps * g.Cin + (size_t)t * g.Cin + cin) * g.Cout + co] * scale;
        }
    }
    // every finite v is below 2^14 after the scale, so no clamp: NaN and +-inf stay NaN and +-inf (their lo half is NaN),
    // and a diverging weight makes the convolution's output non-finite as torch's would be
    const __half h = __float2half_rn(v);
    out[i] = want_lo ? __float2half_rn(v - __half2float(h)) : h;
}
__global__ void k_pack(const Prob g, const float* __restrict__ w, __half* __restrict__ out, const float* __restrict__ hdr) {
    pack_one(g, w, out, __ldg(hdr));
}

// fp32 NHWC -> split-fp16 planes (test / boundary helper) and back
__global__ void k_act_split(long long n, const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = fminf(fmaxf(x[i], -65504.f), 65504.f);
    const __half h = __float2half_rn(v);
    hi[i] = h;
    if (lo) lo[i] = __float2half_rn(v - __half2float(h));
}
__global__ void k_act_merge(long long n, const __half* __restrict__ hi, const __half* __restrict__ lo, float* __restrict__ y) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    y[i] = __half2float(hi[i]) + (lo ? __half2float(lo[i]) : 0.f);
}

// ---------------------------------------------------------------------------------------------
// host: tensor maps + launch
// ---------------------------------------------------------------------------------------------
}  // namespace tc

int pow2_scale(const float* x, long long n, float* hdr, int words, cudaStream_t st) {
    DANET_CUDA(cudaMemsetAsync(hdr + 2, 0, 4, st));
    tc::k_absmax<<<264, 256, 0, st>>>(n, x, reinterpret_cast<unsigned*>(hdr + 2));
    tc::k_pow2_scale<<<1, 256, 0, st>>>(hdr, words);
    DANET_LAUNCH_CHECK();
    return 0;
}

static int g_sm_count[64];
static unsigned* g_sched[64];              // per device: kSchedSlots x {tile counter, done counter}, zero-initialised, self-resetting
static unsigned g_sched_seq[64];
constexpr int kSchedSlots = 1024;
static std::mutex g_tc_mu;
static unsigned long long g_tc_devs = 0;

// geometry of every problem + the shared-memory rings of the launch (1 <= n <= kMaxProb: the callers check n)
static int configure_group(int n, const danet_conv_desc* const* descs, tc::ArgsN* a) {
    using namespace tc;
    memset(a, 0, sizeof(*a));
    a->nprob = n;
    for (int i = 0; i < n; ++i)
        if (!make_prob(descs[i], &a->p[i])) { set_error("danet_conv_tc_group: problem %d has an unsupported shape", i); return -1; }
    for (int i = 1; i < n; ++i)
        DANET_CHECK(a->p[i].exact == a->p[0].exact, "danet_conv_tc_group: exact and fast problems cannot share a launch");
    DANET_CHECK(plan_rings(a), "danet_conv_tc_group: shared-memory plan does not fit");
    return 0;
}

int conv_tc_group_launch(int n, const danet_conv_problem* probs, cudaStream_t stream) {
    using namespace tc;
    ArgsN a;
    {
        const danet_conv_desc* dp[kMaxProb];
        DANET_CHECK(n >= 1 && n <= kMaxProb, "danet_conv_tc_group: 1..%d problems per launch (got %d)", kMaxProb, n);
        for (int i = 0; i < n; ++i) dp[i] = &probs[i].d;
        if (configure_group(n, dp, &a) != 0) return -1;
    }
    // tiles are dealt round-robin over the persistent CTAs in problem order: the problems with the most expensive
    // tiles go first, so that the long tiles start early and the cheap ones fill the tail
    // (a stable insertion sort of a.p in place; order[i] is the caller's index of a.p[i])
    int order[kMaxProb];
    double tcost[kMaxProb];
    for (int i = 0; i < n; ++i) {
        const Prob& P = a.p[i];
        int taps = 0;
        for (int s2 = 0; s2 < P.npa; ++s2) taps += P.ntap[s2];
        tcost[i] = (double)taps * ((P.Cin + 15) / 16) * (P.exact ? 2.0 : 1.0) * (128 + P.NT * (P.exact ? 1.5 : 1.0));
        order[i] = i;
    }
    for (int i = 1; i < n; ++i)
        for (int j = i; j > 0 && tcost[j] > tcost[j - 1]; --j) {
            std::swap(a.p[j], a.p[j - 1]); std::swap(tcost[j], tcost[j - 1]); std::swap(order[j], order[j - 1]);
        }
    int tiles = 0;
    for (int i = 0; i < n; ++i) {
        Prob& P = a.p[i];
        const danet_conv_problem& q = probs[order[i]];
        DANET_CHECK(q.x.hi && q.w_packed && (q.y.hi || q.y.f32), "danet_conv_tc_group: problem %d: null x.hi / weights / output", order[i]);
        DANET_CHECK(!P.exact || q.x.lo, "danet_conv_tc_group: problem %d: exact mode needs the x.lo plane", order[i]);
        P.wpk = (const uint8_t*)q.w_packed; P.bias = q.bias;
        P.res_f = q.res.f32; P.res_hi = (const __half*)q.res.hi; P.res_lo = (const __half*)q.res.lo;
        if (P.res_f) { P.res_hi = nullptr; P.res_lo = nullptr; }
        P.y_f = q.y.f32; P.y_hi = (__half*)q.y.hi; P.y_lo = (__half*)q.y.lo;
        // the input planes as tensor maps whose box is a parity plane's halo: KCH channels x (sbo_a / SWB) x box_h
        // pixels.  One map serves every parity plane: make_prob sizes them all with the largest box.
        const CUtensorMapSwizzle sw = P.SWB == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (P.SWB == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
        for (int h = 0; h < (P.exact ? 2 : 1); ++h)
            if (encode_nhwc_f16(&P.tm[h], h ? q.x.lo : q.x.hi, P.N, P.H, P.W, P.Cin, P.KCH, P.sbo_a / P.SWB, P.box_h, sw, P.stride) != 0) return -1;
        if (!P.exact) P.tm[1] = P.tm[0];
        tiles += P.tile_count;
        DANET_CHECK(tiles < (1 << 24), "danet_conv_tc_group: too many tiles");
        a.unit_base[i] = a.total_units;
        a.unit_count[i] = P.exact ? pair_count(P) : P.tile_count;
        a.total_units += a.unit_count[i];
    }
    int dev = 0;
    DANET_CUDA(cudaGetDevice(&dev));
    DANET_CHECK(dev >= 0 && dev < 64, "conv_tc: device ordinal %d out of range", dev);
    {
        std::lock_guard<std::mutex> lk(g_tc_mu);
        if (first_use_on_current_device(&g_tc_devs) != 0) {          // function attributes are per device
            DANET_CUDA(cudaDeviceGetAttribute(&g_sm_count[dev], cudaDevAttrMultiProcessorCount, dev));
            DANET_CUDA(cudaFuncSetAttribute(k_conv_tc_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
            DANET_CUDA(cudaFuncSetAttribute(k_conv_tc_exact, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
            DANET_CUDA(cudaMalloc((void**)&g_sched[dev], kSchedSlots * 2 * sizeof(unsigned)));
            DANET_CUDA(cudaMemset(g_sched[dev], 0, kSchedSlots * 2 * sizeof(unsigned)));
        }
        // every launch takes the next counter pair (a CUDA graph keeps the one it captured: the kernel re-arms it)
        a.sched = g_sched[dev] + 2 * (g_sched_seq[dev]++ % kSchedSlots);
    }
    const int smem_bytes = kSmemFixed + a.na_stages * a.a_slot_bytes + a.nb_stages * a.b_slot_bytes;
    const int cap = g_sm_count[dev];
    const int grid = a.total_units < cap ? a.total_units : cap;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(a.p[0].exact ? kThreadsExact : kThreadsFast);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    if (a.p[0].exact) { DANET_CUDA(cudaLaunchKernelEx(&cfg, k_conv_tc_exact, a)); }
    else { DANET_CUDA(cudaLaunchKernelEx(&cfg, k_conv_tc_fast, a)); }
    DANET_LAUNCH_CHECK();
    return 0;
}

}  // namespace danet

using namespace danet;

extern "C" int danet_conv_tc_supported(const danet_conv_desc* d) {
    tc::Prob g;
    if (!d || !tc::make_prob(d, &g)) return 0;
    tc::ArgsN* a = new tc::ArgsN();
    a->nprob = 1; a->p[0] = g;
    const bool ok = tc::plan_rings(a);
    delete a;
    return ok ? 1 : 0;
}

extern "C" int64_t danet_conv_tc_packed_bytes(const danet_conv_desc* d) {
    tc::Prob g;
    if (!d || !tc::make_prob(d, &g)) return 0;
    return tc::kPackHeader + (int64_t)d->wsets * g.blocks_per_set * g.b_block_bytes;
}

extern "C" int danet_conv_tc_geometry(const danet_conv_desc* d, int64_t* out) {
    tc::Prob g;
    if (!d || !out || !tc::make_prob(d, &g)) return -1;
    int64_t ksteps = 0, taps = 0, a_bytes = 0;
    for (int c = 0; c < g.nchunks; ++c) {
        const int kreal = (g.Cin - c * g.KCH + 15) / 16;
        ksteps += kreal < g.KCH / 16 ? kreal : g.KCH / 16;
    }
    for (int s = 0; s < g.npa; ++s) {
        taps += g.ntap[s];
        a_bytes += g.nstack > 1 ? (int64_t)g.nstack * g.box_h * g.sbo_a : g.stage_bytes;
    }
    out[0] = tc::kTileH; out[1] = tc::kTileW; out[2] = g.tile_count; out[3] = g.nstack;
    out[4] = g.exact ? 3 : 1;                                              // products per MAC (exact: hi*hi + hi*lo + lo*hi)
    out[5] = (int64_t)tc::kTileH * tc::kTileW * g.NT * 16 * ksteps * taps;  // issued MACs of one product
    out[6] = a_bytes * g.nchunks * (g.exact ? 2 : 1);                      // activation halo bytes (TMA)
    out[7] = (int64_t)g.nblk * g.b_block_bytes;                            // weight bytes (bulk copies)
    return 0;
}

extern "C" int danet_conv_tc_cta_geometry(const danet_conv_desc* d, int64_t* out) {
    int64_t t[8];
    if (danet_conv_tc_geometry(d, t) != 0) return -1;
    tc::Prob g;
    tc::make_prob(d, &g);
    const int tiles = g.exact ? 2 : 1;                  // exact mode: a tile pair shares one weight stream
    out[0] = tiles;
    out[1] = g.exact ? tc::pair_count(g) : g.tile_count;
    out[2] = t[7];
    out[3] = t[6] * tiles;
    return 0;
}

extern "C" int danet_conv_tc_dispatch(const danet_conv_desc* d, int64_t* out) {
    tc::Prob g;
    if (!d || !out || !tc::make_prob(d, &g)) return -1;
    const int kmma = g.KCH / 16;
    int kv_last = 0, max_ntap = 0, max_ngrp = 0;
    // the K segments of one tile: consume_tile's (chunk, parity plane, tap group) loop and its close rule
    int64_t closes = 0, longest = 0, at_plane_end = 0, mid_plane = 0;
    int seg = 0;
    for (int c = 0; c < g.nchunks; ++c) {
        const int kreal = (g.Cin - c * g.KCH + 15) >> 4;
        const int kv = kreal < kmma ? kreal : kmma;
        kv_last = kv;
        for (int slot = 0; slot < g.npa; ++slot) {
            max_ntap = g.ntap[slot] > max_ntap ? g.ntap[slot] : max_ntap;
            max_ngrp = g.ngrp[slot] > max_ngrp ? g.ngrp[slot] : max_ngrp;
            for (int tg = 0; tg < g.ngrp[slot]; ++tg) {
                const int ntk = g.TG < g.ntap[slot] - tg * g.TG ? g.TG : g.ntap[slot] - tg * g.TG;
                const bool plane_end = tg == g.ngrp[slot] - 1;
                const bool last = c == g.nchunks - 1 && slot == g.npa - 1 && plane_end;
                seg += ntk * kv;
                if (!g.exact || !tc::seg_close(last, seg)) continue;
                ++closes;
                longest = seg > longest ? seg : longest;
                if (!last) ++(plane_end ? at_plane_end : mid_plane);
                seg = 0;
            }
        }
    }
    // the tile pairs of one (tile column, N tile): pair_coord says where each second tile lies
    int64_t pairs = 0, past = 0;
    if (g.exact) {
        pairs = tc::pair_count(g);
        const int inner = g.tiles_w * g.ntn;
        for (int64_t o = 0; o < pairs / inner; ++o) {
            const tc::TileCoord t = tc::pair_coord(g, (int)(o * inner), 1);
            if (g.tiles_h > 1 ? t.th >= g.tiles_h : t.img0 >= g.N) past += inner;
        }
    }
    const int64_t r[DANET_CONV_DISPATCH_FIELDS] = {
        g.NT, g.ntn, g.Cout - (g.ntn - 1) * g.NT, g.SWB, g.KCH, g.nchunks, kv_last, g.npa, max_ntap, g.TG, max_ngrp,
        g.nstack, g.hs, g.tiles_h, g.tiles_w, g.nblk, closes, longest, at_plane_end, mid_plane,
        g.exact ? (g.tiles_h > 1 ? 1 : 2) : 0, pairs, past};
    for (int i = 0; i < DANET_CONV_DISPATCH_FIELDS; ++i) out[i] = r[i];
    return 0;
}

extern "C" int danet_conv_tc_pack(const danet_conv_desc* d, const float* w_simt, void* w_packed, danet_stream_t stream) {
    tc::Prob g;
    DANET_CHECK(d && tc::make_prob(d, &g), "danet_conv_tc_pack: shape not supported by the tensor-core path");
    DANET_CHECK(w_simt && w_packed, "danet_conv_tc_pack: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const long long nw = (long long)d->wsets * d->ksize * d->ksize * d->Cin * d->Cout;
    const int rc = pow2_scale(w_simt, nw, (float*)w_packed, tc::kPackHeader / 4, st);
    if (rc != 0) return rc;
    const long long total = (long long)g.wsets * g.blocks_per_set * (g.b_block_bytes / 2);
    tc::k_pack<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(g, w_simt, (__half*)((uint8_t*)w_packed + tc::kPackHeader),
                                                                 (const float*)w_packed);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_conv_tc_config(int32_t n, const danet_conv_desc* descs, int32_t* stages) {
    DANET_CHECK(descs && stages, "danet_conv_tc_config: null pointer");
    const danet_conv_desc* dp[tc::kMaxProb];
    DANET_CHECK(n >= 1 && n <= tc::kMaxProb, "danet_conv_tc_config: 1..%d problems (got %d)", tc::kMaxProb, n);
    for (int i = 0; i < n; ++i) dp[i] = &descs[i];
    tc::ArgsN* a = new tc::ArgsN();
    const int rc = configure_group(n, dp, a);
    if (rc == 0) { stages[0] = a->na_stages; stages[1] = a->nb_stages; }
    delete a;
    return rc;
}

extern "C" int danet_conv_tc_group(int32_t n, const danet_conv_problem* probs, danet_stream_t stream) {
    DANET_CHECK(probs, "danet_conv_tc_group: null problem list");
    for (int i = 0; i < n; ++i) if (probs[i].d.N == 0) { DANET_CHECK(n == 1, "danet_conv_tc_group: empty problem in a group"); return 0; }
    return conv_tc_group_launch(n, probs, (cudaStream_t)stream);
}

extern "C" int danet_act_split(int64_t n, const float* x, void* hi, void* lo, danet_stream_t stream) {
    DANET_CHECK(n >= 0 && (n == 0 || (x && hi)), "danet_act_split: bad arguments");
    if (n == 0) return 0;
    tc::k_act_split<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n, x, (__half*)hi, (__half*)lo);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_act_merge(int64_t n, const void* hi, const void* lo, float* y, danet_stream_t stream) {
    DANET_CHECK(n >= 0 && (n == 0 || (hi && y)), "danet_act_merge: bad arguments");
    if (n == 0) return 0;
    tc::k_act_merge<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n, (const __half*)hi, (const __half*)lo, y);
    DANET_LAUNCH_CHECK();
    return 0;
}
