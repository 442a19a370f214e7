// LSP mask and part-segmentation scoring for sm_90a: the rendered 224 x 224 maps put back into each original image
// (utils/imutils.py:89-113 `uncrop`) and counted against the ground truth (eval.py:219-266), for a whole batch of images
// of different sizes in two launches.  Replaces a D2H copy of the renders, a per-image numpy uncrop and scipy resize,
// and the per-class numpy comparisons.
//   k_seg_tables  one thread per (image, axis): the nearest-neighbour source index of every crop row / column
//   k_seg_count   a (blocks, image) grid over the original pixels: one joint (mask, part) histogram per block in shared
//                 memory, added into the image's int64 tables
//
// The resize is scipy.misc.imresize(..., interp='nearest'), i.e. Pillow's Image.resize(NEAREST), whose source index for
// output pixel i of n is built by a sequential double recurrence: s = R / n, v = s / 2, idx[i] = (int)v, v += s.  The
// closed form floor((i + 0.5) * R / n) differs from it for most n, and so would any reassociated (parallel) sum, so
// each table is built by one thread, one add after another.
// The counts are integers: shared-memory and per-image atomics in any order give the same sums, so the tables are exact
// and repeatable.  Nothing here synchronises with the host.
#include "common.cuh"

namespace danet {

constexpr int kSegThreads = 256;
constexpr int kSegPartRows = 9;          // ground-truth part rows: 0..6, 255, any other value
constexpr int kSegPartCols = 7;          // predicted part columns: 0..6
constexpr int kSegPartBins = 64;         // 63 (row, col) pairs, then bin 63: a predicted value past 6 (not counted)
constexpr int kSegBins = 2 * 2 * kSegPartBins;   // joint histogram: (gt mask, pred mask) x part bin

struct SegGeom {
    int64_t ul_x, ul_y, crop_h, crop_w, orig_h, orig_w, gt_offset, table_offset;
};

__host__ __device__ __forceinline__ double seg_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

// Pillow's NEAREST source index along one axis: n output pixels from R input pixels (Geometry.c, ImagingScaleAffine:
// xo = a[2] + a[0] * 0.5 with a[0] = R / n and a[2] = 0, then one `xo += a[0]` per pixel; every v is >= 0).
__host__ __device__ __forceinline__ void seg_nearest_table(int n, int R, int32_t* out) {
    const double s = (double)R / (double)n;
    double v = s * 0.5;
    for (int i = 0; i < n; ++i) {
        out[i] = (int32_t)v;
        v = seg_add(v, s);
    }
}

// The rendered-map pixel that uncrop puts at original pixel (y, x): uncrop pastes the resized crop's window
// [max(0, ul), min(orig, br)) at the same place, so (y, x) of the image takes the resized crop's pixel (y - ul_y,
// x - ul_x) when that lies inside the crop, and 0 otherwise.  Returns the offset r * R + c, or -1 for "0".
__host__ __device__ __forceinline__ int seg_source(const SegGeom& g, const int32_t* rows, const int32_t* cols, int R,
                                                   int64_t y, int64_t x) {
    const int64_t cy = y - g.ul_y, cx = x - g.ul_x;
    if (cy < 0 || cy >= g.crop_h || cx < 0 || cx >= g.crop_w) return -1;
    return rows[cy] * R + cols[cx];
}

// The ground-truth row of a part label: 0..6 as they are, 255 (UP-3D's "ignore") row 7, any other value row 8.
__host__ __device__ __forceinline__ int seg_part_row(int g) { return g <= 6 ? g : (g == 255 ? 7 : 8); }

__global__ void k_seg_tables(int B, int R, const SegGeom* __restrict__ geom, int32_t* __restrict__ tables) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * B) return;
    const SegGeom g = geom[t >> 1];
    const bool cols = t & 1;
    seg_nearest_table((int)(cols ? g.crop_w : g.crop_h), R,
                      tables + g.table_offset + (cols ? g.crop_h : 0));
}

__global__ void __launch_bounds__(kSegThreads)
k_seg_count(int R, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ parts, const SegGeom* __restrict__ geom,
            const uint8_t* __restrict__ mask_gt, const uint8_t* __restrict__ parts_gt,
            const int32_t* __restrict__ tables, unsigned long long* __restrict__ mask_conf,
            unsigned long long* __restrict__ part_conf) {
    __shared__ unsigned int hist[kSegBins];
    const int b = blockIdx.y;
    const SegGeom g = geom[b];
    for (int i = threadIdx.x; i < kSegBins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const int32_t* rows = tables + g.table_offset;
    const int32_t* cols = rows + g.crop_h;
    const uint8_t* m = mask + (size_t)b * R * R;
    const uint8_t* p = parts + (size_t)b * R * R;
    const uint8_t* gm = mask_gt + g.gt_offset;
    const uint8_t* gp = parts_gt + g.gt_offset;
    const int64_t npix = g.orig_h * g.orig_w;
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31));
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = warp0; base < npix; base += stride) {          // warp-uniform trip count
        const int64_t q = base + lane;
        int key = -1;
        if (q < npix) {
            const unsigned y = (unsigned)q / (unsigned)g.orig_w, x = (unsigned)q - y * (unsigned)g.orig_w;
            const int src = seg_source(g, rows, cols, R, y, x);
            const int pm = src >= 0 && m[src] != 0;
            const int pp = src >= 0 ? p[src] : 0;
            const int pbin = pp < kSegPartCols ? seg_part_row(gp[q]) * kSegPartCols + pp : kSegPartBins - 1;
            key = ((gm[q] != 0) * 2 + pm) * kSegPartBins + pbin;
        }
        // one shared atomic per distinct bin in the warp (most pixels of a warp share a bin)
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        if (key >= 0 && lane == __ffs(peers) - 1) atomicAdd(&hist[key], (unsigned)__popc(peers));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kSegBins; i += blockDim.x) {
        const unsigned c = hist[i];
        if (c == 0) continue;
        const int mb = i / kSegPartBins, pb = i % kSegPartBins;
        atomicAdd(&mask_conf[(size_t)b * 4 + mb], (unsigned long long)c);
        if (pb < kSegPartRows * kSegPartCols) atomicAdd(&part_conf[(size_t)b * kSegPartRows * kSegPartCols + pb],
                                                        (unsigned long long)c);
    }
}

}  // namespace danet

using namespace danet;

extern "C" int danet_seg_confusion(int32_t B, int32_t R, const uint8_t* mask, const uint8_t* parts, const int64_t* geom,
                                   const uint8_t* mask_gt, const uint8_t* parts_gt, int64_t max_pixels, int32_t* tables,
                                   int64_t* mask_conf, int64_t* part_conf, danet_stream_t stream) {
    DANET_CHECK(B >= 0 && R > 0 && max_pixels >= 0 && max_pixels <= INT32_MAX,
                "danet_seg_confusion: bad sizes (B=%d, R=%d, max_pixels=%lld)", B, R, (long long)max_pixels);
    if (B == 0) return 0;
    DANET_CHECK(B <= 65535, "danet_seg_confusion: at most 65535 images per call (B=%d)", B);
    DANET_CHECK(mask && parts && geom && mask_gt && parts_gt && tables && mask_conf && part_conf,
                "danet_seg_confusion: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    DANET_CUDA(cudaMemsetAsync(mask_conf, 0, sizeof(int64_t) * 4 * B, st));
    DANET_CUDA(cudaMemsetAsync(part_conf, 0, sizeof(int64_t) * kSegPartRows * kSegPartCols * B, st));
    const SegGeom* g = reinterpret_cast<const SegGeom*>(geom);
    k_seg_tables<<<cdiv(2 * B, 128), 128, 0, st>>>(B, R, g, tables);
    DANET_LAUNCH_CHECK();
    if (max_pixels == 0) return 0;
    // ~8 pixels per thread for the largest image, at most 128 blocks per image
    const int64_t want = (max_pixels + kSegThreads * 8 - 1) / (kSegThreads * 8);
    const dim3 grid((unsigned)(want < 128 ? want : 128), (unsigned)B);
    k_seg_count<<<grid, kSegThreads, 0, st>>>(R, mask, parts, g, mask_gt, parts_gt, tables,
                                              reinterpret_cast<unsigned long long*>(mask_conf),
                                              reinterpret_cast<unsigned long long*>(part_conf));
    DANET_LAUNCH_CHECK();
    return 0;
}

#ifdef DANET_SEG_HOST_CHECK
// The device's per-axis table and per-pixel mapping walked on the host.  geom: the 8 int64 of one image (see
// include/danet_b200.h); map [R,R] -> out [orig_h, orig_w], 0 where uncrop leaves 0.
extern "C" int danet_test_seg_table_host(int32_t n, int32_t R, int32_t* out) {
    seg_nearest_table(n, R, out);
    return 0;
}

extern "C" int danet_test_seg_uncrop_host(int32_t R, const uint8_t* map, const int64_t* geom, uint8_t* out) {
    const SegGeom g = *reinterpret_cast<const SegGeom*>(geom);
    std::vector<int32_t> tab((size_t)(g.crop_h + g.crop_w));
    seg_nearest_table((int)g.crop_h, R, tab.data());
    seg_nearest_table((int)g.crop_w, R, tab.data() + g.crop_h);
    for (int64_t y = 0; y < g.orig_h; ++y)
        for (int64_t x = 0; x < g.orig_w; ++x) {
            const int src = seg_source(g, tab.data(), tab.data() + g.crop_h, R, y, x);
            out[y * g.orig_w + x] = src >= 0 ? map[src] : 0;
        }
    return 0;
}
#endif
