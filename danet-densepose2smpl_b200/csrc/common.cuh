// Shared helpers for libdanet_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/danet_b200.h"

namespace danet {

void set_error(const char* fmt, ...);

#define DANET_CHECK(cond, ...)                                   \
    do { if (!(cond)) { danet::set_error(__VA_ARGS__); return -1; } } while (0)

#define DANET_CUDA(expr)                                                              \
    do { cudaError_t _e = (expr);                                                     \
         if (_e != cudaSuccess) {                                                     \
             danet::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                              __FILE__, __LINE__);                                    \
             return -2; } } while (0)

#define DANET_LAUNCH_CHECK()                                                          \
    do { cudaError_t _e = cudaGetLastError();                                         \
         if (_e != cudaSuccess) {                                                     \
             danet::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), \
                              __FILE__, __LINE__);                                    \
             return -3; } } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int64_t align_up(int64_t a, int64_t b) { return (a + b - 1) / b * b; }
static inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// Hands out the regions of a caller's workspace in order, each 256-byte aligned.  On a null base it only counts, so one
// layout serves an entry's *_workspace_bytes query and the entry itself, and the two cannot disagree.
struct WsCarve {
    char* base;
    int64_t bytes = 0;
    template <typename T> T* take(int64_t count) {
        T* p = base ? (T*)(base + bytes) : nullptr;
        bytes = align_up(bytes + count * (int64_t)sizeof(T), 256);
        return p;
    }
};

template <typename T>
int upload(T** dptr, const T* host, size_t count) {
    DANET_CUDA(cudaMalloc((void**)dptr, count * sizeof(T) + 16));
    DANET_CUDA(cudaMemcpy(*dptr, host, count * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross3(V3 a, V3 b) { return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }

// rot6d_to_rotmat (utils/geometry.py:47-61): x viewed [3,2], a1 = x[:,0], a2 = x[:,1]; b1 = a1 / max(|a1|, 1e-12),
// u = a2 - (b1 . a2) b1, b2 = u / max(|u|, 1e-12), b3 = b1 x b2; R has the columns (b1, b2, b3).  The SMPL front-end,
// the inference pose head and the training head all run this one definition, so they agree to the last bit.  The state
// keeps what the training head's backward needs: the raw norms n1r, n2r, the clamped n1, n2 and dd = b1 . a2.
struct Rot6dState { V3 a1, a2, b1, u, b2; float n1r, n1, dd, n2r, n2; };
__device__ __forceinline__ Rot6dState rot6d_state(const float* x) {
    Rot6dState s;
    s.a1 = v3(x[0], x[2], x[4]); s.a2 = v3(x[1], x[3], x[5]);
    s.n1r = sqrtf(dot3(s.a1, s.a1)); s.n1 = fmaxf(s.n1r, 1e-12f);
    s.b1 = v3(s.a1.x / s.n1, s.a1.y / s.n1, s.a1.z / s.n1);
    s.dd = dot3(s.b1, s.a2);
    s.u = v3(s.a2.x - s.dd * s.b1.x, s.a2.y - s.dd * s.b1.y, s.a2.z - s.dd * s.b1.z);
    s.n2r = sqrtf(dot3(s.u, s.u)); s.n2 = fmaxf(s.n2r, 1e-12f);
    s.b2 = v3(s.u.x / s.n2, s.u.y / s.n2, s.u.z / s.n2);
    return s;
}
__device__ __forceinline__ void rot6d(const float* x, float* R) {
    const Rot6dState s = rot6d_state(x);
    const V3 b3 = cross3(s.b1, s.b2);
    R[0] = s.b1.x; R[1] = s.b2.x; R[2] = b3.x;
    R[3] = s.b1.y; R[4] = s.b2.y; R[5] = b3.y;
    R[6] = s.b1.z; R[7] = s.b2.z; R[8] = b3.z;
}

// batch_rodrigues (utils/geometry.py:9-45, the quaternion route): axis-angle v -> row-major R.  danet_batch_rodrigues and
// the training targets' 229-wide `target` (csrc/targets.cu) run this one definition.
__device__ __forceinline__ void rodrigues_quat(const float* v, float* R) {
    const float ax = v[0] + 1e-8f, ay = v[1] + 1e-8f, az = v[2] + 1e-8f;
    const float l = sqrtf(ax * ax + ay * ay + az * az);
    const float nx = v[0] / l, ny = v[1] / l, nz = v[2] / l;
    const float h = l * 0.5f;
    const float sn = sinf(h);
    float w = cosf(h), x = sn * nx, y = sn * ny, z = sn * nz;
    const float qn = sqrtf(w * w + x * x + y * y + z * z);
    w /= qn; x /= qn; y /= qn; z /= qn;
    const float w2 = w * w, x2 = x * x, y2 = y * y, z2 = z * z;
    const float wx = w * x, wy = w * y, wz = w * z, xy = x * y, xz = x * z, yz = y * z;
    R[0] = w2 + x2 - y2 - z2; R[1] = 2 * xy - 2 * wz;   R[2] = 2 * wy + 2 * xz;
    R[3] = 2 * wz + 2 * xy;   R[4] = w2 - x2 + y2 - z2; R[5] = 2 * yz - 2 * wx;
    R[6] = 2 * xz - 2 * wy;   R[7] = 2 * wx + 2 * yz;   R[8] = w2 - x2 - y2 + z2;
}

// perspective_projection (utils/geometry.py:63-91) of one point p: rotation R (row-major), translation t, focal f,
// centre c -> out[2].  danet_perspective_projection and the training targets' key points run this one definition.
__device__ __forceinline__ void persp_point(const float* R, const float* t, float f, const float* c, float px, float py,
                                            float pz, float* out) {
    const float x = R[0] * px + R[1] * py + R[2] * pz + t[0];
    const float y = R[3] * px + R[4] * py + R[5] * pz + t[1];
    const float z = R[6] * px + R[7] * py + R[8] * pz + t[2];
    const float xn = x / z, yn = y / z, zn = z / z;
    out[0] = f * xn + c[0] * zn;
    out[1] = f * yn + c[1] * zn;
}

// cudaFuncSetAttribute is per device: true the first time the calling thread's current device is seen by this
// call site (`mask` is the site's static bit set, one bit per device ordinal; -1 on error)
inline std::mutex& first_use_mutex() { static std::mutex m; return m; }
inline int first_use_on_current_device(unsigned long long* mask) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return -1;
    std::lock_guard<std::mutex> lk(first_use_mutex());       // host threads may make their first launch concurrently
    const bool first = !((*mask >> dev) & 1ull);
    *mask |= 1ull << dev;
    return first ? 1 : 0;
}

// two fp32 -> packed fp16x2 (lo in the lower half), round-to-nearest-even, saturating: the conversion the
// tensor-core convolution applies to its activations (conv_tc.cu), shared by the kernels that may write
// fp16 activation buffers for it
__device__ __forceinline__ uint32_t pack_h2_rn(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// Device view of a danet_act (include/danet_b200.h): fp32 tensor and/or split-fp16 planes of one NHWC activation.
// Readers prefer the fp32 view when present; writers fill every view that is present.  The split is the one the
// tensor-core convolution's epilogue applies: hi = rn_f16(v) (saturating), lo = rn_f16(v - hi).
struct ActV { float* f; __half* hi; __half* lo; };
static inline ActV actv(const danet_act* a) {
    ActV v; v.f = a ? a->f32 : nullptr; v.hi = a ? (__half*)a->hi : nullptr; v.lo = a ? (__half*)a->lo : nullptr;
    return v;
}
__device__ __forceinline__ float2 h2_to_f2(uint32_t u) {
    float2 r;
    asm("{\n\t.reg .f16 a, b;\n\tmov.b32 {a, b}, %2;\n\tcvt.f32.f16 %0, a;\n\tcvt.f32.f16 %1, b;\n\t}" : "=f"(r.x), "=f"(r.y) : "r"(u));
    return r;
}
// four consecutive channels starting at element e (e % 4 == 0; planes are 8-byte aligned there)
__device__ __forceinline__ float4 act_ld4(const ActV& a, size_t e) {
    if (a.f) return __ldg(reinterpret_cast<const float4*>(a.f + e));
    const uint2 h = __ldg(reinterpret_cast<const uint2*>(a.hi + e));
    float2 p = h2_to_f2(h.x), q = h2_to_f2(h.y);
    if (a.lo) {
        const uint2 l = __ldg(reinterpret_cast<const uint2*>(a.lo + e));
        const float2 pl = h2_to_f2(l.x), ql = h2_to_f2(l.y);
        p.x += pl.x; p.y += pl.y; q.x += ql.x; q.y += ql.y;
    }
    return make_float4(p.x, p.y, q.x, q.y);
}
__device__ __forceinline__ void act_st4(const ActV& a, size_t e, float4 v) {
    if (a.f) *reinterpret_cast<float4*>(a.f + e) = v;
    if (a.hi) {
        const uint32_t h0 = pack_h2_rn(v.x, v.y), h1 = pack_h2_rn(v.z, v.w);
        *reinterpret_cast<uint2*>(a.hi + e) = make_uint2(h0, h1);
        if (a.lo) {
            const float2 p = h2_to_f2(h0), q = h2_to_f2(h1);
            *reinterpret_cast<uint2*>(a.lo + e) = make_uint2(pack_h2_rn(v.x - p.x, v.y - p.y), pack_h2_rn(v.z - q.x, v.w - q.y));
        }
    }
}
// eight consecutive channels starting at element e (e % 8 == 0): 16-byte accesses on the fp16 planes
struct float8 { float4 a, b; };
__device__ __forceinline__ float8 act_ld8(const ActV& a, size_t e) {
    float8 r;
    if (a.f) { r.a = __ldg(reinterpret_cast<const float4*>(a.f + e)); r.b = __ldg(reinterpret_cast<const float4*>(a.f + e + 4)); return r; }
    const uint4 h = __ldg(reinterpret_cast<const uint4*>(a.hi + e));
    float2 p0 = h2_to_f2(h.x), p1 = h2_to_f2(h.y), p2 = h2_to_f2(h.z), p3 = h2_to_f2(h.w);
    if (a.lo) {
        const uint4 l = __ldg(reinterpret_cast<const uint4*>(a.lo + e));
        const float2 q0 = h2_to_f2(l.x), q1 = h2_to_f2(l.y), q2 = h2_to_f2(l.z), q3 = h2_to_f2(l.w);
        p0.x += q0.x; p0.y += q0.y; p1.x += q1.x; p1.y += q1.y; p2.x += q2.x; p2.y += q2.y; p3.x += q3.x; p3.y += q3.y;
    }
    r.a = make_float4(p0.x, p0.y, p1.x, p1.y); r.b = make_float4(p2.x, p2.y, p3.x, p3.y);
    return r;
}
__device__ __forceinline__ void act_st8(const ActV& a, size_t e, const float8& v) {
    if (a.f) { *reinterpret_cast<float4*>(a.f + e) = v.a; *reinterpret_cast<float4*>(a.f + e + 4) = v.b; }
    if (a.hi) {
        uint4 h;
        h.x = pack_h2_rn(v.a.x, v.a.y); h.y = pack_h2_rn(v.a.z, v.a.w); h.z = pack_h2_rn(v.b.x, v.b.y); h.w = pack_h2_rn(v.b.z, v.b.w);
        *reinterpret_cast<uint4*>(a.hi + e) = h;
        if (a.lo) {
            const float2 p0 = h2_to_f2(h.x), p1 = h2_to_f2(h.y), p2 = h2_to_f2(h.z), p3 = h2_to_f2(h.w);
            uint4 l;
            l.x = pack_h2_rn(v.a.x - p0.x, v.a.y - p0.y); l.y = pack_h2_rn(v.a.z - p1.x, v.a.w - p1.y);
            l.z = pack_h2_rn(v.b.x - p2.x, v.b.y - p2.y); l.w = pack_h2_rn(v.b.z - p3.x, v.b.w - p3.y);
            *reinterpret_cast<uint4*>(a.lo + e) = l;
        }
    }
}
__device__ __forceinline__ float act_ld1(const ActV& a, size_t e) {
    if (a.f) return __ldg(a.f + e);
    float v = __half2float(a.hi[e]);
    if (a.lo) v += __half2float(a.lo[e]);
    return v;
}
__device__ __forceinline__ void act_st1(const ActV& a, size_t e, float v) {
    if (a.f) a.f[e] = v;
    if (a.hi) {
        const __half h = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
        a.hi[e] = h;
        if (a.lo) a.lo[e] = __float2half_rn(v - __half2float(h));
    }
}
static inline bool act_any(const danet_act* a) { return a && (a->f32 || a->hi); }

// Power-of-two scale of n floats x (conv_tc.cu), on the device: hdr[0] = 2^s and hdr[1] = 2^-s, where 2^s brings the
// largest finite |x| into [2^13, 2^14) (1 when there is none).  hdr[2] is scratch for that maximum; hdr[2 .. words) are
// zeroed afterwards (words <= 256).  The packed conv weights' header and the dy scale of conv_wgrad.cu use it.
int pow2_scale(const float* x, long long n, float* hdr, int words, cudaStream_t st);

// Fixed-order per-channel sums of an fp32 NCHW tensor [N][C][HW] in double (conv_wgrad.cu, k_db_partial): with u = a
// (0 where mask <= 0 when mask is given; a NaN mask keeps a) minus K, sum 0 = sum of u; with `two`, sum 1 = sum of
// u * (b - b_shift[c]).  K = k_src[c * HW] (element 0 of channel c, the first image's) when k_src is given, else 0;
// with k_src and no b_shift, b is shifted by K too, so sum 1 = sum (a - K)^2 for b = a: the shift keeps the variance
// sum from cancelling when |mean| >> std.  b_shift and k_src may be NULL.  part receives
// [two ? 2 : 1][chan_sums_chunks(N, HW)][C] chunk partials, to be added in chunk order.
struct ChanSums { const float* a; const float* mask; const float* b; const double* b_shift; const float* k_src; };
int chan_sums_chunks(int N, int HW);
int chan_sums_partial(const ChanSums& s, bool two, int N, int C, int HW, double* part, cudaStream_t st);

}  // namespace danet
