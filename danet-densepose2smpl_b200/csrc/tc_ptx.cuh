// PTX helpers shared by the wgmma kernels (conv_tc.cu, conv_wgrad.cu): mbarriers, TMA / bulk copies, programmatic
// dependent launch, wgmma fences and groups, and the driver's tensor-map encoder.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <mutex>
#include <stdint.h>
#include "common.cuh"

namespace danet {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive only where pred holds, as one predicated instruction: an `if (leader)` branch between wgmmas looks divergent
// to ptxas, which then serialises them
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(bar), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// one out-of-line copy: the bounded polling loop is ~40 SASS instructions and there are many wait sites
static __device__ __noinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
#pragma unroll 1
    for (uint32_t it = 0; it < (1u << 22); ++it) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (done) return;
    }
    __trap();                                        // bounded wait: never hang the device
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, int c3, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}
// Elected forms: the whole (converged) warp executes them and one lane, the lowest, issues the operation.  The exact-mode
// conv engine issues its copies from inside a consumer warp, where an `if (lane == 0)` branch would serialise its wgmmas.
__device__ __forceinline__ void mbar_expect_tx_elect(uint32_t bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\t@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}"
                 ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s_elect(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\t"
                 "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n\t}"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_4d_elect(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, int c3, uint32_t bar) {
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\t"
                 "@p cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];\n\t}"
                 ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}
// st.shared of v at addr, then mbarrier.arrive on bar, both by the elected lane (the arrive releases the store)
__device__ __forceinline__ void st_arrive_elect(uint32_t addr, int v, uint32_t bar) {
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\t@p st.shared.s32 [%0], %1;\n\t"
                 "@p mbarrier.arrive.shared::cta.b64 _, [%2];\n\t}" ::"r"(addr), "r"(v), "r"(bar) : "memory");
}
// atomicAdd(ctr, 1) by the elected lane (lane 0 of a converged warp); the other lanes get 0
__device__ __forceinline__ int atom_inc_elect(unsigned* ctr) {
    int v = 0;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\t@p atom.global.add.u32 %0, [%1], 1;\n\t}"
                 : "+r"(v) : "l"(ctr) : "memory");
    return v;
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}
// programmatic dependent launch: this grid may start while the previous kernel of the stream drains; nothing the
// previous kernel wrote (activations, residual) or still reads (our output may be its input) is touched before pdl_wait()
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads across wgmma.wait_group
template <int NV> __device__ __forceinline__ void reg_fence(float* d) {
#pragma unroll
    for (int i = 0; i < NV; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Consumer-side wait: inlined, so that no call sits between wgmmas in flight (a call makes ptxas serialise them).
// Still bounded: traps instead of hanging.
__device__ __forceinline__ void mbar_wait_inl(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
#pragma unroll 1
    for (uint32_t it = 0; it < (1u << 22); ++it) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (done) return;
    }
    __trap();
}
__device__ __forceinline__ void wg_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
    });
    return fn;
}

// An fp16 NHWC tensor [N][H][W][C] as a 4-D tensor map.  A box reads box_c channels of box_w x box_h pixels, taking
// every stride-th column and row (elementStrides = stride); elements outside the tensor are zero filled.
static int encode_nhwc_f16(CUtensorMap* tm, const void* base, int N, int H, int W, int C, int box_c, int box_w, int box_h,
                           CUtensorMapSwizzle sw, int stride) {
    PFN_encodeTiled fn = encode_fn();
    DANET_CHECK(fn, "cuTensorMapEncodeTiled is not available from this driver");
    DANET_CHECK(base && aligned16(base), "tensor map: activation planes must be non-null and 16-byte aligned");
    cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t gstr[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)(stride * (box_w - 1) + 1), (cuuint32_t)(stride * (box_h - 1) + 1), 1u};
    cuuint32_t estr[4] = {1u, (cuuint32_t)stride, (cuuint32_t)stride, 1u};
    const CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), gdim, gstr, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    DANET_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) for [%d,%d,%d,%d] box [%u,%u,%u]", (int)r, N, H, W, C,
                box[0], box[1], box[2]);
    return 0;
}

}  // namespace tc
}  // namespace danet
