// Fused SMPL layer for sm_90a: pose front-ends (rot-mat / axis-angle / rot6d), 24-joint
// kinematic chain, blend shapes + pose correctives + linear blend skinning for 6890 vertices,
// and the vertex-regressed joints (extra 9, H36M 17, 21 picked vertices) -> 49-joint output.
//
// Replaces models/smpl.py:15-46 + smplx.lbs (third-party, see oracle/lbs.py) and
// utils/geometry.py:9-91; rot6d is common.cuh's, the one both pose heads use.  Two routes:
//  * small batches (B < kGemmMinB): everything fp32 SIMT in one fused kernel (below);
//  * large batches: the blend-shape + pose-corrective contraction  v_posed[B, 20670] = template +
//    [pose_feature | betas][B, 224] x [posedirs ; shapedirs][224, 20670]  is a genuine GEMM (4.5 MMAC per body,
//    88 % of the layer's arithmetic) and runs on the wgmma engine of conv_tc.cu as a 1x1 "convolution" whose
//    pixels are the bodies (exact mode: split-fp16 operands, 3 MMAs, fp32 accumulation -> fp32-grade), in chunks
//    of kGemmChunk bodies so that the fp32 v_posed chunk (42 MB) stays in the 50 MB L2 until the skinning
//    kernel (the same k_smpl_verts, phase 1 replaced by a coalesced load) has consumed it.
// Fused SIMT route, three launches per forward:
//   k_smpl_pose    one warp per body, lane = joint: rotations, rest joints (linear in beta, precomputed
//                  J_template + J_shapedirs*beta), chain level by level -> A[B,24,3x4], pose_feature[B,208]
//   k_smpl_verts   grid (54 vertex tiles, B/NB body chunks), 128 threads:
//                    phase 1 (coordinate-parallel, coalesced 4-byte lanes): v_posed for NB bodies,
//                            posedirs/shapedirs rows reused from registers across the NB bodies
//                    phase 2 (vertex-parallel): skinning from smem-resident A, result staged in smem
//                    phase 3: coalesced store + per-tile partial sums of the sparse joint regressors
//   k_smpl_joints  one CTA per body: reduce partials in fixed tile order (deterministic), pick
//                  vertices, apply joint_map.
#include "common.cuh"
#include <string.h>

namespace danet {

constexpr int kJ = 24;
constexpr int kTileV = 128;             // vertices per CTA tile
constexpr int kTileC = kTileV * 3;      // coordinates per CTA tile
constexpr int kPF = 208;                // padded pose-feature length (207 -> 208)
constexpr int kMaxBetas = 16;
constexpr int kGF = 224;                // GEMM route: feature row = 207 pose features | 0 | betas (<= 16) at 208..
constexpr int kGemmMinB = 512;          // batches at least this large take the tensor-core GEMM route
constexpr int kGemmChunk = 512;         // bodies per GEMM + skinning round (fp32 v_posed chunk = 42 MB, L2-resident)

struct SmplView {
    int nv, ntiles, nvpad, npad, nbetas;
    const float* vt;          // [npad]
    const float* sd;          // [nbetas][npad]
    const float* pd;          // [kPF][npad]
    const float* Jt;          // [72]
    const float* Jsd;         // [72][nbetas]
    int parents[kJ];
    int skin_packed;          // 1: <=4 influences per vertex
    const uint32_t* skin_idx; // [nvpad] 4 x u8
    const float4* skin_w;     // [nvpad]
    const float* skin_dense;  // [24][nvpad]
    const float* reg_rows;    // [nrows][nvpad]
    int nrows, npairs;
    const int* tile_pair_off; // [ntiles+1]
    const int* tile_pair_row; // [npairs]
    const int* row_pair_off;  // [nrows+1]
    const int* row_pair_slot; // [npairs]
    int nsel; const int* sel; // picked vertices
    int nextra, nh36m;
    int nout; const int* joint_map;
};

int conv_tc_group_launch(int n, const danet_conv_problem* probs, cudaStream_t stream);   // conv_tc.cu

}  // namespace danet

struct danet_smpl {
    danet::SmplView v;
    std::vector<void*> allocs;
    // GEMM route: packed [posedirs ; shapedirs] weights, template as bias
    void* gemm_w = nullptr;
    float* gemm_bias = nullptr;
    int gemm_cout = 0;
};

namespace danet {

// ---------------------------------------------------------------------------------------------
// rotation front-ends
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void rodrigues_smplx(const float* v, float* R) {
    // smplx.lbs.batch_rodrigues: angle = |v + 1e-8|, d = v / angle, R = I + sin K + (1-cos) K K
    const float ax = v[0] + 1e-8f, ay = v[1] + 1e-8f, az = v[2] + 1e-8f;
    const float angle = sqrtf(ax * ax + ay * ay + az * az);
    const float x = v[0] / angle, y = v[1] / angle, z = v[2] / angle;
    const float s = sinf(angle), c1 = 1.0f - cosf(angle);
    R[0] = 1.0f + c1 * (-(z * z) - y * y); R[1] = s * (-z) + c1 * (x * y);      R[2] = s * y + c1 * (x * z);
    R[3] = s * z + c1 * (x * y);           R[4] = 1.0f + c1 * (-(z * z) - x * x); R[5] = s * (-x) + c1 * (y * z);
    R[6] = s * (-y) + c1 * (x * z);        R[7] = s * x + c1 * (y * z);          R[8] = 1.0f + c1 * (-(y * y) - x * x);
}

// rodrigues_quat (utils/geometry.py:9-45) is common.cuh's, shared with the training targets (csrc/targets.cu)

__global__ void k_rot6d(int n, const float* __restrict__ x, float* __restrict__ R) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float in[6], out[9];
#pragma unroll
    for (int k = 0; k < 6; ++k) in[k] = x[(size_t)i * 6 + k];
    rot6d(in, out);
#pragma unroll
    for (int k = 0; k < 9; ++k) R[(size_t)i * 9 + k] = out[k];
}

__global__ void k_rodrigues(int n, const float* __restrict__ aa, float* __restrict__ R, int flavor) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float in[3] = {aa[(size_t)i * 3], aa[(size_t)i * 3 + 1], aa[(size_t)i * 3 + 2]}, out[9];
    if (flavor == 1) rodrigues_smplx(in, out); else rodrigues_quat(in, out);
#pragma unroll
    for (int k = 0; k < 9; ++k) R[(size_t)i * 9 + k] = out[k];
}

__global__ void k_persp(int B, int N, const float* __restrict__ pts, const float* __restrict__ rot,
                        const float* __restrict__ tr, const float* __restrict__ focal,
                        const float* __restrict__ center, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * N) return;
    const int b = i / N;
    persp_point(rot + (size_t)b * 9, tr + b * 3, focal[b], center + b * 2, pts[(size_t)i * 3], pts[(size_t)i * 3 + 1],
                pts[(size_t)i * 3 + 2], out + (size_t)i * 2);
}

__global__ void k_mpjpe(int B, const float* __restrict__ j17, const float* __restrict__ gt14,
                        float* __restrict__ out) {
    // eval.py:202-212 with constants.H36M_TO_J14 (constants.py:95-96)
    const int sel[14] = {6, 5, 4, 1, 2, 3, 16, 15, 14, 11, 12, 13, 8, 10};
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float* p = j17 + (size_t)b * 51;
    float acc = 0.0f;
    for (int j = 0; j < 14; ++j) {
        float s = 0.0f;
        for (int c = 0; c < 3; ++c) {
            const float d = (p[sel[j] * 3 + c] - p[c]) - gt14[((size_t)b * 14 + j) * 3 + c];
            s += d * d;
        }
        acc += sqrtf(s);
    }
    out[b] = acc / 14.0f;
}

// ---------------------------------------------------------------------------------------------
// k_smpl_pose
// ---------------------------------------------------------------------------------------------
constexpr int kPoseWarps = 4;                       // bodies per CTA of k_smpl_pose (one warp each)
__global__ void __launch_bounds__(kPoseWarps * 32)
k_smpl_pose(int B, int pose_kind, const float* __restrict__ betas,
            const float* __restrict__ pose, SmplView m, float* __restrict__ rot_out,
            float* __restrict__ G, float* __restrict__ A, float* __restrict__ pf,
            float* __restrict__ posed, __half* __restrict__ feat_hi, __half* __restrict__ feat_lo) {
    // One warp per body, lane i < 24 = joint i.  The kinematic chain runs level by level: a lane fetches its
    // parent's world transform with shuffles (tree depth 8 for SMPL), so the per-body serial work is 8 small
    // matrix products instead of 24, every global access is a contiguous run of one body's data, and the
    // expressions (and their order) are those of the one-thread-per-body form this replaces.
    __shared__ float s_pf[kPoseWarps][kGF];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * kPoseWarps + warp;
    if (b >= B) return;                                  // whole warps leave together
    const int i = lane < kJ ? lane : 0;                  // lanes 24..31 shadow joint 0 (they write nothing)
    const bool act = lane < kJ;
    float beta[kMaxBetas];
    for (int l = 0; l < m.nbetas; ++l) beta[l] = betas[(size_t)b * m.nbetas + l];
    float Ji[3];
    for (int r = 0; r < 3; ++r) {
        const int e = i * 3 + r;
        float v = m.Jt[e];
        for (int l = 0; l < m.nbetas; ++l) v = fmaf(beta[l], m.Jsd[e * m.nbetas + l], v);
        Ji[r] = v;
    }
    float R[9];
    if (pose_kind == DANET_POSE_ROTMAT) {
        for (int e = 0; e < 9; ++e) R[e] = pose[((size_t)b * kJ + i) * 9 + e];
    } else if (pose_kind == DANET_POSE_AXIS_ANGLE) {
        const float v[3] = {pose[((size_t)b * kJ + i) * 3], pose[((size_t)b * kJ + i) * 3 + 1],
                            pose[((size_t)b * kJ + i) * 3 + 2]};
        rodrigues_smplx(v, R);
    } else {
        float v[6];
        for (int e = 0; e < 6; ++e) v[e] = pose[((size_t)b * kJ + i) * 6 + e];
        rot6d(v, R);
    }
    if (rot_out && act) for (int e = 0; e < 9; ++e) rot_out[((size_t)b * kJ + i) * 9 + e] = R[e];
    if (act && i > 0) for (int e = 0; e < 9; ++e) s_pf[warp][(i - 1) * 9 + e] = R[e] - ((e % 4 == 0) ? 1.0f : 0.0f);
    // depth of this joint in the tree, and the deepest level
    const int p = i > 0 ? m.parents[i] : 0;
    int depth = 0;
    for (int q = i; q > 0; q = m.parents[q]) ++depth;
    int maxd = act ? depth : 0;
    for (int o = 16; o > 0; o >>= 1) maxd = max(maxd, __shfl_xor_sync(0xffffffffu, maxd, o));
    float rel[3];
    for (int r = 0; r < 3; ++r) rel[r] = Ji[r] - __shfl_sync(0xffffffffu, Ji[r], p);
    float g[12];
    for (int r = 0; r < 3; ++r) {                        // the root's transform; every other lane overwrites it at its level
        g[r * 4 + 0] = R[r * 3 + 0]; g[r * 4 + 1] = R[r * 3 + 1]; g[r * 4 + 2] = R[r * 3 + 2];
        g[r * 4 + 3] = Ji[r];
    }
    for (int d = 1; d <= maxd; ++d) {
        float gp[12];
#pragma unroll
        for (int e = 0; e < 12; ++e) gp[e] = __shfl_sync(0xffffffffu, g[e], p);
        if (depth == d) {
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const float a0 = gp[r * 4], a1 = gp[r * 4 + 1], a2 = gp[r * 4 + 2], a3 = gp[r * 4 + 3];
                g[r * 4 + 0] = a0 * R[0] + a1 * R[3] + a2 * R[6];
                g[r * 4 + 1] = a0 * R[1] + a1 * R[4] + a2 * R[7];
                g[r * 4 + 2] = a0 * R[2] + a1 * R[5] + a2 * R[8];
                g[r * 4 + 3] = a0 * rel[0] + a1 * rel[1] + a2 * rel[2] + a3;
            }
        }
    }
    if (act) {
        if (G) {                                         // world transforms (backward pass)
            float4* Gv = reinterpret_cast<float4*>(G + ((size_t)b * kJ + i) * 12);
            Gv[0] = make_float4(g[0], g[1], g[2], g[3]); Gv[1] = make_float4(g[4], g[5], g[6], g[7]); Gv[2] = make_float4(g[8], g[9], g[10], g[11]);
        }
        float a[12];
        for (int r = 0; r < 3; ++r) {
            posed[((size_t)b * kJ + i) * 3 + r] = g[r * 4 + 3];
            a[r * 4 + 0] = g[r * 4 + 0]; a[r * 4 + 1] = g[r * 4 + 1]; a[r * 4 + 2] = g[r * 4 + 2];
            a[r * 4 + 3] = g[r * 4 + 3] - (g[r * 4 + 0] * Ji[0] + g[r * 4 + 1] * Ji[1] + g[r * 4 + 2] * Ji[2]);
        }
        float4* Av = reinterpret_cast<float4*>(A + ((size_t)b * kJ + i) * 12);
        Av[0] = make_float4(a[0], a[1], a[2], a[3]); Av[1] = make_float4(a[4], a[5], a[6], a[7]); Av[2] = make_float4(a[8], a[9], a[10], a[11]);
    }
    __syncwarp();
    // pose feature [207 | 0] (fp32) and, on the GEMM route, [pose feature | 0 | betas | 0 ...] as split-fp16 planes
    // (hi = rn(v), lo = rn(v - hi)): lanes sweep the row, coalesced
    for (int k = lane; k < kGF; k += 32) {
        float v = 0.0f;
        if (k < 207) v = s_pf[warp][k];
        if (k < kPF) pf[(size_t)b * kPF + k] = v;
        if (feat_hi) {
            if (k >= 208 && k - 208 < m.nbetas) v = beta[k - 208];
            const __half h = __float2half_rn(v);
            feat_hi[(size_t)b * kGF + k] = h;
            feat_lo[(size_t)b * kGF + k] = __float2half_rn(v - __half2float(h));
        }
    }
}

// ---------------------------------------------------------------------------------------------
// k_smpl_verts
// ---------------------------------------------------------------------------------------------
// k_smpl_skin: the skinning + store + regressor-partial phases of k_smpl_verts for the tensor-core route, where
// v_posed is already in memory (L2-resident GEMM output).  One CTA walks TL consecutive vertex tiles of its NB bodies:
// the bone transforms are loaded once (they were 38 % of the old kernel's read traffic: 54 tiles x 1152 B per body) and
// tile k+1's v_posed rows stream into the second shared-memory buffer (cp.async, 16-byte chunks) while tile k is skinned.
__device__ __forceinline__ void cp_async16_zfill(float* smem_dst, const float* gsrc, int src_bytes) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
template <int NB, int TL>
__global__ void __launch_bounds__(kTileV)
k_smpl_skin(int B, const float* __restrict__ A, SmplView m, float* __restrict__ verts, float* __restrict__ partials,
            const float* __restrict__ vposed, int vp_stride) {
    extern __shared__ __align__(16) float smem_lbs[];
    float (*s_A)[kJ * 12] = reinterpret_cast<float (*)[kJ * 12]>(smem_lbs);
    float* s_vbuf = smem_lbs + NB * kJ * 12;                       // [2][NB][kTileC]
    const int b0 = blockIdx.y * NB, tid = threadIdx.x, t0 = blockIdx.x * TL;
    constexpr int kChunks = kTileC / 4;                              // 16-byte chunks per body row of a tile

    auto issue = [&](int tile, int buf) {
        for (int i = tid; i < NB * kChunks; i += kTileV) {
            const int b = i / kChunks, c = i - b * kChunks, bb = min(b0 + b, B - 1);
            const int n = tile * kTileC + 4 * c;
            const bool ok = n + 4 <= vp_stride;                      // the last tile runs past the row: zero fill
            cp_async16_zfill(s_vbuf + ((size_t)(buf * NB + b) * kTileC + 4 * c), vposed + (size_t)bb * vp_stride + (ok ? n : 0), ok ? 16 : 0);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    issue(t0, 0);
    for (int i = tid; i < NB * kJ * 12; i += kTileV) {
        const int b = i / (kJ * 12), k = i % (kJ * 12), bb = min(b0 + b, B - 1);
        s_A[b][k] = A[(size_t)bb * kJ * 12 + k];
    }
    const int ncoord = m.nv * 3;
    const int warp = tid >> 5, lane = tid & 31;
#pragma unroll 1
    for (int kt = 0; kt < TL; ++kt) {
        const int tile = t0 + kt;
        // everything this tile needs from global memory that does not depend on v_posed is requested before the wait:
        // the vertex's bones and weights, the tile's regressor rows (first pair of this warp)
        const int v = tile * kTileV + tid;
        const uint32_t idx = __ldg(m.skin_idx + v);
        const float4 w = __ldg(m.skin_w + v);
        const int off = m.tile_pair_off[tile], npair = m.tile_pair_off[tile + 1] - off;
        float r4n[kTileV / 32];
        auto load_pair = [&](int pr, float* r4) {
            if (pr < npair) {
                const float* rr = m.reg_rows + (size_t)m.tile_pair_row[off + pr] * m.nvpad + (size_t)tile * kTileV;
#pragma unroll
                for (int i = 0; i < kTileV / 32; ++i) r4[i] = __ldg(rr + lane + i * 32);
            }
        };
        load_pair(warp, r4n);
        if (kt + 1 < TL) {
            issue(tile + 1, (kt + 1) & 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        float (*s_v)[kTileC] = reinterpret_cast<float (*)[kTileC]>(s_vbuf + (size_t)(kt & 1) * NB * kTileC);
        // ---- skinning, thread = vertex (<= 4 bones per vertex) ----
        {
            const int j0 = idx & 255, j1 = (idx >> 8) & 255, j2 = (idx >> 16) & 255, j3 = idx >> 24;
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                const float x = s_v[b][3 * tid], y = s_v[b][3 * tid + 1], z = s_v[b][3 * tid + 2];
                const float4* A0 = reinterpret_cast<const float4*>(&s_A[b][j0 * 12]);
                const float4* A1 = reinterpret_cast<const float4*>(&s_A[b][j1 * 12]);
                const float4* A2 = reinterpret_cast<const float4*>(&s_A[b][j2 * 12]);
                const float4* A3 = reinterpret_cast<const float4*>(&s_A[b][j3 * 12]);
                float o[3];
#pragma unroll
                for (int r = 0; r < 3; ++r) {                    // one 16-byte row of each bone's 3x4 transform
                    const float4 a0 = A0[r], a1 = A1[r], a2 = A2[r], a3 = A3[r];
                    const float t0 = w.x * a0.x + w.y * a1.x + w.z * a2.x + w.w * a3.x;
                    const float t1 = w.x * a0.y + w.y * a1.y + w.z * a2.y + w.w * a3.y;
                    const float t2 = w.x * a0.z + w.y * a1.z + w.z * a2.z + w.w * a3.z;
                    const float t3 = w.x * a0.w + w.y * a1.w + w.z * a2.w + w.w * a3.w;
                    o[r] = t0 * x + t1 * y + t2 * z + t3;
                }
                s_v[b][3 * tid] = o[0]; s_v[b][3 * tid + 1] = o[1]; s_v[b][3 * tid + 2] = o[2];
            }
        }
        __syncthreads();
        // ---- coalesced store + joint-regressor partial sums ----
        if (verts) {
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                if (b0 + b < B) {
#pragma unroll
                    for (int j = 0; j < 3; ++j) {
                        const int gn = tile * kTileC + tid + j * kTileV;
                        if (gn < ncoord) verts[(size_t)(b0 + b) * ncoord + gn] = s_v[b][tid + j * kTileV];
                    }
                }
            }
        }
        // one warp per (tile, regressor row) pair, all NB bodies at once: 3 NB partial sums per lane, reduced across the
        // warp by halving the value set at every shuffle step (27 shuffles instead of 15 per body)
        static_assert(NB == 8, "the transposed reduction below is written for 8 bodies (24 values over 32 lanes)");
        for (int pr = warp; pr < npair; pr += kTileV / 32) {
            float r4[kTileV / 32];
#pragma unroll
            for (int i = 0; i < kTileV / 32; ++i) r4[i] = r4n[i];
            load_pair(pr + kTileV / 32, r4n);                        // next pair's row while this one is reduced
            float acc[NB * 3];
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
                for (int i = 0; i < kTileV / 32; ++i) {
                    const int vv = lane + i * 32;
                    s0 = fmaf(r4[i], s_v[b][3 * vv], s0);
                    s1 = fmaf(r4[i], s_v[b][3 * vv + 1], s1);
                    s2 = fmaf(r4[i], s_v[b][3 * vv + 2], s2);
                }
                acc[3 * b] = s0; acc[3 * b + 1] = s1; acc[3 * b + 2] = s2;
            }
            const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
            float w12[12], w6[6], w3[3];
#pragma unroll
            for (int k = 0; k < 12; ++k) {
                const float keep = h16 ? acc[k + 12] : acc[k], send = h16 ? acc[k] : acc[k + 12];
                w12[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                const float keep = h8 ? w12[k + 6] : w12[k], send = h8 ? w12[k] : w12[k + 6];
                w6[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float keep = h4 ? w6[k + 3] : w6[k], send = h4 ? w6[k] : w6[k + 3];
                float v = keep + __shfl_xor_sync(0xffffffffu, send, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                w3[k] = v;
            }
            const int body = lane >> 2;                            // lanes 4g hold body g = bit4*4 + bit3*2 + bit2
            if ((lane & 3) == 0 && b0 + body < B) {
                float* dst = partials + ((size_t)(b0 + body) * m.npairs + off + pr) * 3;
                dst[0] = w3[0]; dst[1] = w3[1]; dst[2] = w3[2];
            }
        }
        __syncthreads();                                             // the buffer is refilled two tiles later
    }
}

template <int NB>
__global__ void __launch_bounds__(kTileV)
k_smpl_verts(int B, const float* __restrict__ betas, const float* __restrict__ pf,
             const float* __restrict__ A, SmplView m, float* __restrict__ verts,
             float* __restrict__ partials, const float* __restrict__ vposed, int vp_stride) {
    extern __shared__ __align__(16) float smem_lbs[];
    float (*s_pf)[kPF] = reinterpret_cast<float (*)[kPF]>(smem_lbs);
    float (*s_A)[kJ * 12] = reinterpret_cast<float (*)[kJ * 12]>(smem_lbs + NB * kPF);
    float (*s_v)[kTileC] = reinterpret_cast<float (*)[kTileC]>(smem_lbs + NB * (kPF + kJ * 12));
    float (*s_beta)[kMaxBetas] = reinterpret_cast<float (*)[kMaxBetas]>(smem_lbs + NB * (kPF + kJ * 12 + kTileC));

    const int tile = blockIdx.x, b0 = blockIdx.y * NB, tid = threadIdx.x;
    if (!vposed)
    for (int i = tid; i < NB * kPF; i += kTileV) {
        const int b = i / kPF, k = i % kPF, bb = min(b0 + b, B - 1);
        s_pf[b][k] = pf[(size_t)bb * kPF + k];
    }
    for (int i = tid; i < NB * kJ * 12; i += kTileV) {
        const int b = i / (kJ * 12), k = i % (kJ * 12), bb = min(b0 + b, B - 1);
        s_A[b][k] = A[(size_t)bb * kJ * 12 + k];
    }
    for (int i = tid; i < NB * kMaxBetas; i += kTileV) {
        const int b = i / kMaxBetas, l = i % kMaxBetas, bb = min(b0 + b, B - 1);
        s_beta[b][l] = l < m.nbetas ? betas[(size_t)bb * m.nbetas + l] : 0.0f;
    }
    __syncthreads();

    // ---- phase 1: v_posed[n] for n = tile*384 + tid + {0,128,256}, NB bodies ----
    const size_t n0 = (size_t)tile * kTileC + tid;
    if (vposed) {
        // GEMM route: v_posed comes from the tensor-core contraction (row b of vposed, vp_stride floats apart)
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const int bb = min(b0 + b, B - 1);
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const int n = (int)n0 + j * kTileV;
                s_v[b][tid + j * kTileV] = n < vp_stride ? __ldg(vposed + (size_t)bb * vp_stride + n) : 0.0f;
            }
        }
    } else {
    float acc[3][NB];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float t = __ldg(m.vt + n0 + j * kTileV);
#pragma unroll
        for (int b = 0; b < NB; ++b) acc[j][b] = t;
    }
    for (int l = 0; l < m.nbetas; ++l) {
        float s[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) s[j] = __ldg(m.sd + (size_t)l * m.npad + n0 + j * kTileV);
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const float bl = s_beta[b][l];
#pragma unroll
            for (int j = 0; j < 3; ++j) acc[j][b] = fmaf(bl, s[j], acc[j][b]);
        }
    }
#pragma unroll 2
    for (int k = 0; k < kPF; k += 4) {
        float p[4][3];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int j = 0; j < 3; ++j) p[kk][j] = __ldg(m.pd + (size_t)(k + kk) * m.npad + n0 + j * kTileV);
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const float4 f = *reinterpret_cast<const float4*>(&s_pf[b][k]);
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                float a = acc[j][b];
                a = fmaf(f.x, p[0][j], a);
                a = fmaf(f.y, p[1][j], a);
                a = fmaf(f.z, p[2][j], a);
                a = fmaf(f.w, p[3][j], a);
                acc[j][b] = a;
            }
        }
    }
#pragma unroll
    for (int b = 0; b < NB; ++b)
#pragma unroll
        for (int j = 0; j < 3; ++j) s_v[b][tid + j * kTileV] = acc[j][b];
    }
    __syncthreads();

    // ---- phase 2: skinning, thread = vertex ----
    const int v = tile * kTileV + tid;
    if (m.skin_packed) {
        const uint32_t idx = __ldg(m.skin_idx + v);
        const float4 w = __ldg(m.skin_w + v);
        const int j0 = idx & 255, j1 = (idx >> 8) & 255, j2 = (idx >> 16) & 255, j3 = idx >> 24;
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const float x = s_v[b][3 * tid], y = s_v[b][3 * tid + 1], z = s_v[b][3 * tid + 2];
            float o[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                float t[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int e = r * 4 + c;
                    t[c] = w.x * s_A[b][j0 * 12 + e] + w.y * s_A[b][j1 * 12 + e] +
                           w.z * s_A[b][j2 * 12 + e] + w.w * s_A[b][j3 * 12 + e];
                }
                o[r] = t[0] * x + t[1] * y + t[2] * z + t[3];
            }
            s_v[b][3 * tid] = o[0]; s_v[b][3 * tid + 1] = o[1]; s_v[b][3 * tid + 2] = o[2];
        }
    } else {
        float w[kJ];
#pragma unroll
        for (int j = 0; j < kJ; ++j) w[j] = __ldg(m.skin_dense + (size_t)j * m.nvpad + v);
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const float x = s_v[b][3 * tid], y = s_v[b][3 * tid + 1], z = s_v[b][3 * tid + 2];
            float o[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int j = 0; j < kJ; ++j)
#pragma unroll
                    for (int c = 0; c < 4; ++c) t[c] = fmaf(w[j], s_A[b][j * 12 + r * 4 + c], t[c]);
                o[r] = t[0] * x + t[1] * y + t[2] * z + t[3];
            }
            s_v[b][3 * tid] = o[0]; s_v[b][3 * tid + 1] = o[1]; s_v[b][3 * tid + 2] = o[2];
        }
    }
    __syncthreads();

    // ---- phase 3: coalesced store + joint-regressor partial sums ----
    const int ncoord = m.nv * 3;
    if (verts) {
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            if (b0 + b < B) {
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    const int gn = tile * kTileC + tid + j * kTileV;
                    if (gn < ncoord) verts[(size_t)(b0 + b) * ncoord + gn] = s_v[b][tid + j * kTileV];
                }
            }
        }
    }
    const int warp = tid >> 5, lane = tid & 31;
    const int off = m.tile_pair_off[tile], npair = m.tile_pair_off[tile + 1] - off;
    for (int q = warp; q < npair * NB; q += kTileV / 32) {
        const int pr = q / NB, b = q % NB;
        const int row = m.tile_pair_row[off + pr];
        const float* rr = m.reg_rows + (size_t)row * m.nvpad + (size_t)tile * kTileV;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < kTileV / 32; ++i) {
            const int vv = lane + i * 32;
            const float r = __ldg(rr + vv);
            s0 = fmaf(r, s_v[b][3 * vv], s0);
            s1 = fmaf(r, s_v[b][3 * vv + 1], s1);
            s2 = fmaf(r, s_v[b][3 * vv + 2], s2);
        }
        s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
        if (lane == 0 && b0 + b < B) {
            float* dst = partials + ((size_t)(b0 + b) * m.npairs + off + pr) * 3;
            dst[0] = s0; dst[1] = s1; dst[2] = s2;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// k_smpl_joints
// ---------------------------------------------------------------------------------------------
__global__ void k_smpl_joints(int B, SmplView m, const float* __restrict__ posed,
                              const float* __restrict__ verts, const float* __restrict__ partials,
                              float* __restrict__ joints, float* __restrict__ smpl_joints,
                              float* __restrict__ joints_h36m) {
    extern __shared__ float s_j[];          // [(24 + nsel + nrows) * 3]
    const int b = blockIdx.x;
    const int ncat = kJ + m.nsel + m.nrows;
    for (int t = threadIdx.x; t < ncat * 3; t += blockDim.x) {
        const int i = t / 3, c = t % 3;
        float val;
        if (i < kJ) {
            val = posed[((size_t)b * kJ + i) * 3 + c];
        } else if (i < kJ + m.nsel) {
            val = verts[((size_t)b * m.nv + m.sel[i - kJ]) * 3 + c];
        } else {
            const int row = i - kJ - m.nsel;
            val = 0.0f;
            for (int q = m.row_pair_off[row]; q < m.row_pair_off[row + 1]; ++q)
                val += partials[((size_t)b * m.npairs + m.row_pair_slot[q]) * 3 + c];
        }
        s_j[t] = val;
    }
    __syncthreads();
    if (joints)
        for (int t = threadIdx.x; t < m.nout * 3; t += blockDim.x)
            joints[(size_t)b * m.nout * 3 + t] = s_j[m.joint_map[t / 3] * 3 + t % 3];
    if (smpl_joints)
        for (int t = threadIdx.x; t < kJ * 3; t += blockDim.x) smpl_joints[(size_t)b * kJ * 3 + t] = s_j[t];
    if (joints_h36m && m.nh36m > 0)
        for (int t = threadIdx.x; t < m.nh36m * 3; t += blockDim.x)
            joints_h36m[(size_t)b * m.nh36m * 3 + t] = s_j[(kJ + m.nsel + m.nextra) * 3 + t];
}

// ---------------------------------------------------------------------------------------------
// backward of the SMPL layer (the piece of the training step, train/trainer.py:148-215 + smpl_regressor.py:131-221,
// that has a hard oracle): given dL/dverts and dL/d(smpl joints), dL/dbetas and dL/dR (R = the 24 rotation matrices
// the layer consumed, pose2rot=False).  fp32 SIMT; everything is recomputed from (betas, R), nothing is kept from
// the forward pass.  No float atomics: every sum has a fixed order, so the result is bit-for-bit repeatable and a
// body's gradient does not depend on the rest of the batch.
//   k_smpl_pose          (forward kernel) -> G (world transforms), A (skinning transforms), pose feature
//   k_lbs_bwd_verts      grid (vertex tile, body): recompute v_posed, dv_posed = T_v^T g, and the tile's partial
//                        dA = sum_v w (g x [v_posed;1]), each of the 24 x 12 entries summed in vertex order
//   k_lbs_bwd_dA         dA = the tile partials summed in tile order
//   k_lbs_bwd_blend      dpf = P dv_posed (207 rows), dbeta_shape = S dv_posed: one warp per (body, row)
//   k_lbs_bwd_chain      one thread per body: reverse kinematic chain -> dR, dJ -> dbeta
// ---------------------------------------------------------------------------------------------
constexpr int kTileS = kTileV + 1;      // row stride of the staged [joint][vertex] and [entry][vertex] planes (no bank conflicts)
__global__ void __launch_bounds__(kTileV)
k_lbs_bwd_verts(int B, const float* __restrict__ betas, const float* __restrict__ pf, const float* __restrict__ A,
                SmplView m, const float* __restrict__ gverts, float* __restrict__ dvp, float* __restrict__ dA_tiles) {
    __shared__ float s_pf[kPF];
    __shared__ float s_A[kJ * 12];
    __shared__ float s_v[kTileC];
    __shared__ float s_beta[kMaxBetas];
    __shared__ float s_w[kJ * kTileS];      // skinning weight of (joint, vertex), 0 past nv
    __shared__ float s_gv[12 * kTileS];     // g[r] * [v_posed; 1][c] of (entry r * 4 + c, vertex)
    const int tile = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    for (int i = tid; i < kPF; i += kTileV) s_pf[i] = pf[(size_t)b * kPF + i];
    for (int i = tid; i < kJ * 12; i += kTileV) s_A[i] = A[(size_t)b * kJ * 12 + i];
    if (tid < kMaxBetas) s_beta[tid] = tid < m.nbetas ? betas[(size_t)b * m.nbetas + tid] : 0.f;
    __syncthreads();
    // v_posed of the tile (coordinate-parallel, like the forward pass)
    const size_t n0 = (size_t)tile * kTileC + tid;
    for (int j = 0; j < 3; ++j) {
        const size_t n = n0 + j * kTileV;
        float acc = __ldg(m.vt + n);
        for (int l = 0; l < m.nbetas; ++l) acc = fmaf(s_beta[l], __ldg(m.sd + (size_t)l * m.npad + n), acc);
        for (int k = 0; k < 207; ++k) acc = fmaf(s_pf[k], __ldg(m.pd + (size_t)k * m.npad + n), acc);
        s_v[tid + j * kTileV] = acc;
    }
    __syncthreads();
    const int v = tile * kTileV + tid;
    float gx = 0.f, gy = 0.f, gz = 0.f;
    if (v < m.nv) {
        gx = gverts[((size_t)b * m.nv + v) * 3]; gy = gverts[((size_t)b * m.nv + v) * 3 + 1]; gz = gverts[((size_t)b * m.nv + v) * 3 + 2];
    }
    const float x = s_v[3 * tid], y = s_v[3 * tid + 1], z = s_v[3 * tid + 2];
    float T[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float g[3] = {gx, gy, gz};
    const float vh[4] = {x, y, z, 1.0f};
    for (int j = 0; j < kJ; ++j) {
        float w = 0.f;
        if (m.skin_packed) {
            const uint32_t idx = __ldg(m.skin_idx + v);
            const float4 ww = __ldg(m.skin_w + v);
            if ((int)(idx & 255) == j) w += ww.x;
            if ((int)((idx >> 8) & 255) == j) w += ww.y;
            if ((int)((idx >> 16) & 255) == j) w += ww.z;
            if ((int)(idx >> 24) == j) w += ww.w;
        } else {
            w = __ldg(m.skin_dense + (size_t)j * m.nvpad + v);
        }
        if (v >= m.nv) w = 0.f;
        s_w[j * kTileS + tid] = w;
        if (w == 0.f) continue;
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) T[r * 3 + c] = fmaf(w, s_A[j * 12 + r * 4 + c], T[r * 3 + c]);
    }
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) s_gv[(r * 4 + c) * kTileS + tid] = g[r] * vh[c];
    // dv_posed = T^T g
    if (v < m.nv)
        for (int c = 0; c < 3; ++c)
            dvp[(size_t)b * m.npad + 3 * v + c] = T[c] * g[0] + T[3 + c] * g[1] + T[6 + c] * g[2];
    else if (3 * v + 2 < m.npad)
        for (int c = 0; c < 3; ++c) dvp[(size_t)b * m.npad + 3 * v + c] = 0.f;
    __syncthreads();
    // the tile's partial dA: thread = (joint, entry) output, summed over the tile's vertices in order
    float* out = dA_tiles + ((size_t)b * m.ntiles + tile) * (kJ * 12);
    for (int o = tid; o < kJ * 12; o += kTileV) {
        const float* wj = s_w + (o / 12) * kTileS;
        const float* ge = s_gv + (o % 12) * kTileS;
        float s = 0.f;
        for (int u = 0; u < kTileV; ++u) s = fmaf(wj[u], ge[u], s);
        out[o] = s;
    }
}

// dA[b] = sum over the vertex tiles, in tile order, of the partials of k_lbs_bwd_verts
__global__ void k_lbs_bwd_dA(int B, int ntiles, const float* __restrict__ dA_tiles, float* __restrict__ dA) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * kJ * 12) return;
    const int b = i / (kJ * 12), o = i - b * (kJ * 12);
    const float* p = dA_tiles + (size_t)b * ntiles * (kJ * 12) + o;
    float s = 0.f;
    for (int t = 0; t < ntiles; ++t) s += p[(size_t)t * (kJ * 12)];
    dA[i] = s;
}

// rows 0..206: dL/dpose_feature; rows 207..207+nbetas-1: dL/dbeta through the shape blend shapes
__global__ void k_lbs_bwd_blend(int B, SmplView m, const float* __restrict__ dvp, float* __restrict__ dpf, float* __restrict__ dbeta) {
    const int nrow = 207 + m.nbetas;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (gw >= B * nrow) return;
    const int b = gw / nrow, r = gw % nrow;
    const float* row = r < 207 ? m.pd + (size_t)r * m.npad : m.sd + (size_t)(r - 207) * m.npad;
    const float* d = dvp + (size_t)b * m.npad;
    float s = 0.f;
    for (int n = lane; n < m.nv * 3; n += 32) s = fmaf(__ldg(row + n), d[n], s);
    s = warp_sum(s);
    if (lane == 0) { if (r < 207) dpf[(size_t)b * kPF + r] = s; else dbeta[(size_t)b * m.nbetas + (r - 207)] = s; }
}

__global__ void k_lbs_bwd_chain(int B, SmplView m, const float* __restrict__ betas, const float* __restrict__ R,
                                const float* __restrict__ G, const float* __restrict__ dA, const float* __restrict__ dpf,
                                const float* __restrict__ gjoints, float* __restrict__ dbeta, float* __restrict__ dR) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float J[kJ * 3];
    for (int e = 0; e < kJ * 3; ++e) {
        float v = m.Jt[e];
        for (int l = 0; l < m.nbetas; ++l) v = fmaf(betas[(size_t)b * m.nbetas + l], m.Jsd[e * m.nbetas + l], v);
        J[e] = v;
    }
    float dRg[kJ][9], dtg[kJ][3], dJ[kJ * 3];
    const float* Gb = G + (size_t)b * kJ * 12;
    for (int i = 0; i < kJ; ++i) {
        const float* a = dA + ((size_t)b * kJ + i) * 12;
        // A_i = [Rg_i | tg_i - Rg_i J_i]
        for (int r = 0; r < 3; ++r) {
            const float at = a[r * 4 + 3];
            for (int c = 0; c < 3; ++c) dRg[i][r * 3 + c] = a[r * 4 + c] - at * J[i * 3 + c];
            dtg[i][r] = at + (gjoints ? gjoints[((size_t)b * kJ + i) * 3 + r] : 0.f);
        }
        for (int c = 0; c < 3; ++c)
            dJ[i * 3 + c] = -(Gb[i * 12 + 0 * 4 + c] * a[3] + Gb[i * 12 + 1 * 4 + c] * a[7] + Gb[i * 12 + 2 * 4 + c] * a[11]);
    }
    for (int i = kJ - 1; i >= 0; --i) {
        const float* Ri = R + ((size_t)b * kJ + i) * 9;
        float* out = dR + ((size_t)b * kJ + i) * 9;
        if (i == 0) {
            // G_0 = [R_0 | J_0]
            for (int e = 0; e < 9; ++e) out[e] = dRg[0][e];
            for (int c = 0; c < 3; ++c) dJ[c] += dtg[0][c];
            break;
        }
        const int p = m.parents[i];
        const float* Gp = Gb + p * 12;
        const float rel[3] = {J[i * 3] - J[p * 3], J[i * 3 + 1] - J[p * 3 + 1], J[i * 3 + 2] - J[p * 3 + 2]};
        // Rg_i = Rg_p R_i ; tg_i = Rg_p rel + tg_p
        float dRi[9], drel[3];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c)
                dRi[r * 3 + c] = Gp[0 * 4 + r] * dRg[i][0 * 3 + c] + Gp[1 * 4 + r] * dRg[i][1 * 3 + c] + Gp[2 * 4 + r] * dRg[i][2 * 3 + c];
        for (int r = 0; r < 3; ++r)
            drel[r] = Gp[0 * 4 + r] * dtg[i][0] + Gp[1 * 4 + r] * dtg[i][1] + Gp[2 * 4 + r] * dtg[i][2];
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c)
                dRg[p][r * 3 + c] += dRg[i][r * 3 + 0] * Ri[c * 3 + 0] + dRg[i][r * 3 + 1] * Ri[c * 3 + 1] + dRg[i][r * 3 + 2] * Ri[c * 3 + 2]
                                     + dtg[i][r] * rel[c];
            dtg[p][r] += dtg[i][r];
        }
        for (int c = 0; c < 3; ++c) { dJ[i * 3 + c] += drel[c]; dJ[p * 3 + c] -= drel[c]; }
        // pose feature = vec(R_i - I), i >= 1
        for (int e = 0; e < 9; ++e) out[e] = dRi[e] + dpf[(size_t)b * kPF + (i - 1) * 9 + e];
    }
    for (int l = 0; l < m.nbetas; ++l) {
        float s = dbeta[(size_t)b * m.nbetas + l];
        for (int e = 0; e < kJ * 3; ++e) s = fmaf(dJ[e], m.Jsd[e * m.nbetas + l], s);
        dbeta[(size_t)b * m.nbetas + l] = s;
    }
}

template <typename T>
static int up(danet_smpl* h, const T** dst, const std::vector<T>& src) {
    T* d = nullptr;
    if (upload(&d, src.data(), src.size()) != 0) return -1;
    h->allocs.push_back(d);
    *dst = d;
    return 0;
}

// The forward's route and workspace (a null base only sizes it): skinning transforms, pose feature, posed joints,
// regressor partials and, on the GEMM route, the split-fp16 feature planes and the fp32 v_posed of one chunk.
struct SmplFwdWs {
    bool gemm;
    float *A, *pf, *posed, *partials, *vposed = nullptr;
    __half *feat_hi = nullptr, *feat_lo = nullptr;
    int64_t bytes;
    SmplFwdWs(const danet_smpl* h, int B, int bodies_per_cta, void* base)
        : gemm(B >= kGemmMinB && h->gemm_cout > 0 && bodies_per_cta >= 0) {
        WsCarve c{(char*)base};
        A = c.take<float>((int64_t)B * kJ * 12);
        pf = c.take<float>((int64_t)B * kPF);
        posed = c.take<float>((int64_t)B * kJ * 3);
        partials = c.take<float>((int64_t)B * (h->v.npairs > 0 ? h->v.npairs : 1) * 3);
        if (gemm) {
            const int64_t Bp = align_up(B, 8);
            feat_hi = c.take<__half>(Bp * kGF);
            feat_lo = c.take<__half>(Bp * kGF);
            vposed = c.take<float>((B < kGemmChunk ? Bp : kGemmChunk) * h->gemm_cout);
        }
        bytes = c.bytes;
    }
};

// The backward's workspace (a null base only sizes it): world and skinning transforms, pose feature, posed joints,
// dL/dv_posed, dL/dA, dL/dpose_feature and the per-tile partials of dL/dA.
struct SmplBwdWs {
    float *G, *A, *pf, *posed, *dvp, *dA, *dpf, *dA_tiles;
    int64_t bytes;
    SmplBwdWs(const danet_smpl* h, int B, void* base) {
        WsCarve c{(char*)base};
        G = c.take<float>((int64_t)B * kJ * 12);
        A = c.take<float>((int64_t)B * kJ * 12);
        pf = c.take<float>((int64_t)B * kPF);
        posed = c.take<float>((int64_t)B * kJ * 3);
        dvp = c.take<float>((int64_t)B * h->v.npad);
        dA = c.take<float>((int64_t)B * kJ * 12);
        dpf = c.take<float>((int64_t)B * kPF);
        dA_tiles = c.take<float>((int64_t)B * h->v.ntiles * kJ * 12);
        bytes = c.bytes;
    }
};

}  // namespace danet

using namespace danet;

extern "C" int danet_smpl_create(const danet_smpl_desc* d, danet_smpl_t* out) {
    DANET_CHECK(d && out, "danet_smpl_create: null argument");
    DANET_CHECK(d->num_joints == kJ, "danet_smpl_create: num_joints must be 24 (got %d)", d->num_joints);
    DANET_CHECK(d->num_betas >= 1 && d->num_betas <= kMaxBetas, "danet_smpl_create: num_betas %d not in 1..16", d->num_betas);
    DANET_CHECK(d->num_verts > 0 && d->v_template && d->shapedirs && d->posedirs && d->J_regressor &&
                d->lbs_weights && d->parents, "danet_smpl_create: missing model array");
    DANET_CHECK(d->parents[0] < 0, "danet_smpl_create: parents[0] must be -1");
    for (int i = 1; i < kJ; ++i)
        DANET_CHECK(d->parents[i] >= 0 && d->parents[i] < i, "danet_smpl_create: parents must precede children");
    const int nv = d->num_verts, nb = d->num_betas;
    auto* h = new danet_smpl();
    SmplView& m = h->v;
    m.nv = nv; m.ntiles = cdiv(nv, kTileV); m.nvpad = m.ntiles * kTileV; m.npad = m.nvpad * 3; m.nbetas = nb;
    for (int i = 0; i < kJ; ++i) m.parents[i] = d->parents[i];

    std::vector<float> vt(m.npad, 0.f), sd((size_t)nb * m.npad, 0.f), pd((size_t)kPF * m.npad, 0.f);
    for (int i = 0; i < nv * 3; ++i) vt[i] = d->v_template[i];
    for (int i = 0; i < nv * 3; ++i)
        for (int l = 0; l < nb; ++l) sd[(size_t)l * m.npad + i] = d->shapedirs[(size_t)i * nb + l];
    for (int k = 0; k < 207; ++k)
        for (int i = 0; i < nv * 3; ++i) pd[(size_t)k * m.npad + i] = d->posedirs[(size_t)k * nv * 3 + i];
    // rest joints are linear in beta: J = J_regressor (v_template + S beta)
    std::vector<float> Jt(kJ * 3), Jsd((size_t)kJ * 3 * nb);
    for (int j = 0; j < kJ; ++j)
        for (int c = 0; c < 3; ++c) {
            double a = 0.0;
            std::vector<double> s(nb, 0.0);
            for (int v = 0; v < nv; ++v) {
                const double r = d->J_regressor[(size_t)j * nv + v];
                if (r == 0.0) continue;
                a += r * d->v_template[v * 3 + c];
                for (int l = 0; l < nb; ++l) s[l] += r * d->shapedirs[((size_t)v * 3 + c) * nb + l];
            }
            Jt[j * 3 + c] = (float)a;
            for (int l = 0; l < nb; ++l) Jsd[(size_t)(j * 3 + c) * nb + l] = (float)s[l];
        }
    // skinning weights: packed (<= 4 influences) or dense
    int maxnnz = 0;
    for (int v = 0; v < nv; ++v) {
        int nnz = 0;
        for (int j = 0; j < kJ; ++j) nnz += d->lbs_weights[(size_t)v * kJ + j] != 0.0f;
        maxnnz = nnz > maxnnz ? nnz : maxnnz;
    }
    m.skin_packed = maxnnz <= 4;
    m.skin_idx = nullptr; m.skin_w = nullptr; m.skin_dense = nullptr;
    int rc = 0;
    if (m.skin_packed) {
        std::vector<uint32_t> idx(m.nvpad, 0u);
        std::vector<float4> w(m.nvpad, make_float4(0.f, 0.f, 0.f, 0.f));
        for (int v = 0; v < nv; ++v) {
            int k = 0; uint32_t pk = 0; float ww[4] = {0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < kJ; ++j) {
                const float x = d->lbs_weights[(size_t)v * kJ + j];
                if (x != 0.0f) { pk |= (uint32_t)j << (8 * k); ww[k] = x; ++k; }
            }
            idx[v] = pk; w[v] = make_float4(ww[0], ww[1], ww[2], ww[3]);
        }
        rc |= up(h, &m.skin_idx, idx); rc |= up(h, &m.skin_w, w);
    } else {
        std::vector<float> wd((size_t)kJ * m.nvpad, 0.f);
        for (int v = 0; v < nv; ++v)
            for (int j = 0; j < kJ; ++j) wd[(size_t)j * m.nvpad + v] = d->lbs_weights[(size_t)v * kJ + j];
        rc |= up(h, &m.skin_dense, wd);
    }
    // vertex-regressed joints: stacked rows (extra ; h36m), tile-sparse pair lists
    m.nextra = d->num_extra; m.nh36m = d->J_regressor_h36m ? d->num_h36m : 0;
    m.nrows = m.nextra + m.nh36m;
    std::vector<float> rows((size_t)(m.nrows > 0 ? m.nrows : 1) * m.nvpad, 0.f);
    for (int r = 0; r < m.nextra; ++r)
        for (int v = 0; v < nv; ++v) rows[(size_t)r * m.nvpad + v] = d->J_regressor_extra[(size_t)r * nv + v];
    for (int r = 0; r < m.nh36m; ++r)
        for (int v = 0; v < nv; ++v) rows[(size_t)(m.nextra + r) * m.nvpad + v] = d->J_regressor_h36m[(size_t)r * nv + v];
    std::vector<int> tpo(m.ntiles + 1, 0), tpr;
    std::vector<std::vector<int>> row_slots(m.nrows > 0 ? m.nrows : 1);
    for (int t = 0; t < m.ntiles; ++t) {
        tpo[t] = (int)tpr.size();
        for (int r = 0; r < m.nrows; ++r) {
            bool nz = false;
            for (int v = t * kTileV; v < (t + 1) * kTileV && !nz; ++v) nz = rows[(size_t)r * m.nvpad + v] != 0.0f;
            if (nz) { row_slots[r].push_back((int)tpr.size()); tpr.push_back(r); }
        }
    }
    tpo[m.ntiles] = (int)tpr.size();
    m.npairs = (int)tpr.size();
    std::vector<int> rpo(m.nrows + 1, 0), rps;
    for (int r = 0; r < m.nrows; ++r) { rpo[r] = (int)rps.size(); for (int s : row_slots[r]) rps.push_back(s); }
    rpo[m.nrows] = (int)rps.size();
    if (tpr.empty()) tpr.push_back(0);
    if (rps.empty()) rps.push_back(0);
    m.nsel = d->num_selected;
    std::vector<int> sel(d->selected_verts, d->selected_verts + d->num_selected);
    if (sel.empty()) sel.push_back(0);
    for (int i = 0; i < d->num_selected; ++i)
        if (sel[i] < 0 || sel[i] >= nv) { set_error("danet_smpl_create: selected vertex %d out of range", sel[i]); delete h; return -1; }
    m.nout = d->num_out_joints;
    std::vector<int> jm(d->joint_map, d->joint_map + d->num_out_joints);
    const int ncat = kJ + m.nsel + m.nextra;
    for (int i = 0; i < m.nout; ++i)
        if (jm[i] < 0 || jm[i] >= ncat) { set_error("danet_smpl_create: joint_map[%d]=%d out of range 0..%d", i, jm[i], ncat - 1); delete h; return -1; }
    if (jm.empty()) jm.push_back(0);

    rc |= up(h, &m.vt, vt); rc |= up(h, &m.sd, sd); rc |= up(h, &m.pd, pd);
    rc |= up(h, &m.Jt, Jt); rc |= up(h, &m.Jsd, Jsd);
    rc |= up(h, &m.reg_rows, rows);
    rc |= up(h, &m.tile_pair_off, tpo); rc |= up(h, &m.tile_pair_row, tpr);
    rc |= up(h, &m.row_pair_off, rpo); rc |= up(h, &m.row_pair_slot, rps);
    rc |= up(h, &m.sel, sel); rc |= up(h, &m.joint_map, jm);
    if (rc != 0) { danet_smpl_destroy(h); return -2; }
    // GEMM route operands: W [224][Cout] = [posedirs (207 rows) ; 0 ; shapedirs^T (nbetas rows) ; 0...], bias = template,
    // packed into the tensor-core engine's split-fp16 weight blocks (exact mode)
    {
        const int cout = (nv * 3 + 7) / 8 * 8;
        std::vector<float> W((size_t)kGF * cout, 0.f), bias(cout, 0.f);
        for (int k = 0; k < 207; ++k)
            for (int i = 0; i < nv * 3; ++i) W[(size_t)k * cout + i] = d->posedirs[(size_t)k * nv * 3 + i];
        for (int l = 0; l < nb; ++l)
            for (int i = 0; i < nv * 3; ++i) W[(size_t)(208 + l) * cout + i] = d->shapedirs[(size_t)i * nb + l];
        for (int i = 0; i < nv * 3; ++i) bias[i] = d->v_template[i];
        danet_conv_desc cd = {1, 128, 8, kGF, cout, 1, 1, 0, 1, 0, DANET_CONV_EXACT};
        const int64_t pbytes = danet_conv_tc_packed_bytes(&cd);
        h->gemm_cout = 0;
        if (pbytes > 0) {
            float* dW = nullptr;
            const float* dB = nullptr;
            if (upload(&dW, W.data(), W.size()) != 0 || up(h, &dB, bias) != 0) { danet_smpl_destroy(h); return -2; }
            void* pk = nullptr;
            if (cudaMalloc(&pk, (size_t)pbytes) != cudaSuccess) { cudaFree(dW); danet_smpl_destroy(h); set_error("danet_smpl_create: out of memory"); return -2; }
            h->allocs.push_back(pk);
            const int prc = danet_conv_tc_pack(&cd, dW, pk, nullptr);
            cudaDeviceSynchronize();
            cudaFree(dW);
            if (prc != 0) { danet_smpl_destroy(h); return -2; }
            h->gemm_w = pk; h->gemm_bias = const_cast<float*>(dB); h->gemm_cout = cout;
        }
    }
    *out = h;
    return 0;
}

extern "C" int danet_smpl_destroy(danet_smpl_t h) {
    if (!h) return 0;
    for (void* p : h->allocs) cudaFree(p);
    delete h;
    return 0;
}

extern "C" int64_t danet_smpl_workspace_bytes(danet_smpl_t h, int32_t B) {
    if (!h || B <= 0) return 0;
    return SmplFwdWs(h, B, 0, nullptr).bytes;
}

extern "C" int danet_smpl_forward(danet_smpl_t h, int32_t B, const float* betas, const float* pose,
                                  int32_t pose_kind, float* verts, float* joints, float* smpl_joints,
                                  float* joints_h36m, float* rotmats, void* workspace,
                                  int32_t bodies_per_cta, danet_stream_t stream_) {
    DANET_CHECK(h, "danet_smpl_forward: null handle");
    DANET_CHECK(B > 0, "danet_smpl_forward: empty batch (B=%d)", B);
    DANET_CHECK(betas && pose && workspace, "danet_smpl_forward: null input/workspace pointer");
    DANET_CHECK(pose_kind >= 0 && pose_kind <= 2, "danet_smpl_forward: bad pose_kind %d", pose_kind);
    DANET_CHECK(verts || !(joints || smpl_joints || joints_h36m),
                "danet_smpl_forward: joint outputs need the verts buffer (picked vertices are read from it)");
    DANET_CHECK(bodies_per_cta == -1 || bodies_per_cta == 0 || bodies_per_cta == 1 || bodies_per_cta == 2 ||
                bodies_per_cta == 4 || bodies_per_cta == 8 || bodies_per_cta == 16,
                "danet_smpl_forward: bodies_per_cta must be -1, 0, 1, 2, 4, 8 or 16 (got %d)", bodies_per_cta);
    cudaStream_t stream = (cudaStream_t)stream_;
    const SmplView& m = h->v;
    const SmplFwdWs ws(h, B, bodies_per_cta, workspace);
    k_smpl_pose<<<cdiv(B, kPoseWarps), kPoseWarps * 32, 0, stream>>>(B, pose_kind, betas, pose, m, rotmats, nullptr, ws.A, ws.pf, ws.posed, ws.feat_hi, ws.feat_lo);
    DANET_LAUNCH_CHECK();
    int nb = bodies_per_cta;
    if (nb <= 0) nb = B >= 32 ? 8 : (B >= 4 ? 4 : (B >= 2 ? 2 : 1));      // tools/lbs_sweep.py sweeps it
    // shared memory is sized from the blocking a launch instantiates: the GEMM route's fallback always runs 8 bodies
    // per CTA, whatever the caller's bodies_per_cta
#define DANET_LBS_LAUNCH(NBV, Bc, off, VP)                                                          \
    do {                                                                                            \
        const size_t smem = (size_t)NBV * (kPF + kJ * 12 + kTileC + kMaxBetas) * sizeof(float);     \
        static unsigned long long attr_devs = 0;                                                    \
        if (first_use_on_current_device(&attr_devs) != 0) {                                         \
            DANET_CUDA(cudaFuncSetAttribute(k_smpl_verts<NBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        }                                                                                           \
        dim3 grid(m.ntiles, cdiv(Bc, NBV));                                                         \
        k_smpl_verts<NBV><<<grid, kTileV, smem, stream>>>(Bc, betas + (size_t)(off) * m.nbetas, ws.pf + (size_t)(off) * kPF, \
            ws.A + (size_t)(off) * kJ * 12, m, verts ? verts + (size_t)(off) * m.nv * 3 : nullptr, \
            ws.partials + (size_t)(off) * (m.npairs > 0 ? m.npairs : 1) * 3, VP, h->gemm_cout);       \
    } while (0)
    if (ws.gemm) {
        // tensor-core route: per chunk, one 1x1 "convolution" over the bodies (exact mode) + the skinning phases
        for (int off = 0; off < B; off += kGemmChunk) {
            const int Bc = B - off < kGemmChunk ? B - off : kGemmChunk;
            danet_conv_problem pr;
            memset(&pr, 0, sizeof(pr));
            pr.d.N = 1; pr.d.H = cdiv(Bc, 8); pr.d.W = 8; pr.d.Cin = kGF; pr.d.Cout = h->gemm_cout; pr.d.ksize = 1; pr.d.stride = 1;
            pr.d.pad = 0; pr.d.wsets = 1; pr.d.relu = 0; pr.d.flags = DANET_CONV_EXACT;
            pr.x.hi = ws.feat_hi + (size_t)off * kGF; pr.x.lo = ws.feat_lo + (size_t)off * kGF;
            pr.y.f32 = ws.vposed; pr.w_packed = h->gemm_w; pr.bias = h->gemm_bias;
            if (conv_tc_group_launch(1, &pr, stream) != 0) return -1;
            constexpr int kSkinTL = 3;                                  // vertex tiles per CTA of the skinning pass
            if (m.skin_packed && m.ntiles % kSkinTL == 0) {
                dim3 grid(m.ntiles / kSkinTL, cdiv(Bc, 8));
                const size_t sm = (size_t)8 * (kJ * 12 + 2 * kTileC) * sizeof(float);
                k_smpl_skin<8, kSkinTL><<<grid, kTileV, sm, stream>>>(Bc, ws.A + (size_t)off * kJ * 12, m,
                    verts ? verts + (size_t)off * m.nv * 3 : nullptr, ws.partials + (size_t)off * (m.npairs > 0 ? m.npairs : 1) * 3,
                    ws.vposed, h->gemm_cout);
            } else {
                DANET_LBS_LAUNCH(8, Bc, off, ws.vposed);
            }
            DANET_LAUNCH_CHECK();
        }
    } else {
        switch (nb) {
            case 1:  DANET_LBS_LAUNCH(1, B, 0, nullptr); break;
            case 2:  DANET_LBS_LAUNCH(2, B, 0, nullptr); break;
            case 4:  DANET_LBS_LAUNCH(4, B, 0, nullptr); break;
            case 8:  DANET_LBS_LAUNCH(8, B, 0, nullptr); break;
            case 16: DANET_LBS_LAUNCH(16, B, 0, nullptr); break;        // no other value passes the check on entry
        }
        DANET_LAUNCH_CHECK();
    }
#undef DANET_LBS_LAUNCH
    if (joints || smpl_joints || joints_h36m) {
        const int ncat = kJ + m.nsel + m.nrows;
        k_smpl_joints<<<B, 192, ncat * 3 * sizeof(float), stream>>>(B, m, ws.posed, verts, ws.partials, joints,
                                                                    smpl_joints, joints_h36m);
        DANET_LAUNCH_CHECK();
    }
    return 0;
}

extern "C" int64_t danet_smpl_backward_workspace_bytes(danet_smpl_t h, int32_t B) {
    if (!h || B <= 0) return 0;
    return SmplBwdWs(h, B, nullptr).bytes;
}

extern "C" int danet_smpl_backward(danet_smpl_t h, int32_t B, const float* betas, const float* rotmats,
                                   const float* grad_verts, const float* grad_smpl_joints, float* grad_betas,
                                   float* grad_rotmats, void* workspace, danet_stream_t stream_) {
    DANET_CHECK(h, "danet_smpl_backward: null handle");
    DANET_CHECK(B > 0, "danet_smpl_backward: empty batch (B=%d)", B);
    DANET_CHECK(betas && rotmats && grad_verts && grad_betas && grad_rotmats && workspace, "danet_smpl_backward: null pointer");
    cudaStream_t stream = (cudaStream_t)stream_;
    const SmplView& m = h->v;
    const SmplBwdWs ws(h, B, workspace);
    k_smpl_pose<<<cdiv(B, kPoseWarps), kPoseWarps * 32, 0, stream>>>(B, DANET_POSE_ROTMAT, betas, rotmats, m, nullptr, ws.G, ws.A, ws.pf, ws.posed, nullptr, nullptr);
    DANET_LAUNCH_CHECK();
    k_lbs_bwd_verts<<<dim3(m.ntiles, B), kTileV, 0, stream>>>(B, betas, ws.pf, ws.A, m, grad_verts, ws.dvp, ws.dA_tiles);
    DANET_LAUNCH_CHECK();
    k_lbs_bwd_dA<<<cdiv(B * kJ * 12, 256), 256, 0, stream>>>(B, m.ntiles, ws.dA_tiles, ws.dA);
    DANET_LAUNCH_CHECK();
    const int nrow = 207 + m.nbetas;
    k_lbs_bwd_blend<<<cdiv((int64_t)B * nrow * 32, 256), 256, 0, stream>>>(B, m, ws.dvp, ws.dpf, grad_betas);
    DANET_LAUNCH_CHECK();
    k_lbs_bwd_chain<<<cdiv(B, 32), 32, 0, stream>>>(B, m, betas, rotmats, ws.G, ws.dA, ws.dpf, grad_smpl_joints, grad_betas, grad_rotmats);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_rot6d_to_rotmat(int32_t n, const float* x, float* R, danet_stream_t s) {
    DANET_CHECK(n >= 0 && (n == 0 || (x && R)), "danet_rot6d_to_rotmat: bad arguments");
    if (n == 0) return 0;
    k_rot6d<<<cdiv(n, 128), 128, 0, (cudaStream_t)s>>>(n, x, R);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_batch_rodrigues(int32_t n, const float* aa, float* R, int32_t flavor, danet_stream_t s) {
    DANET_CHECK(n >= 0 && (n == 0 || (aa && R)), "danet_batch_rodrigues: bad arguments");
    DANET_CHECK(flavor == 0 || flavor == 1, "danet_batch_rodrigues: flavor must be 0 (quaternion) or 1 (smplx)");
    if (n == 0) return 0;
    k_rodrigues<<<cdiv(n, 128), 128, 0, (cudaStream_t)s>>>(n, aa, R, flavor);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_perspective_projection(int32_t B, int32_t N, const float* points, const float* rotation,
                                            const float* translation, const float* focal, const float* center,
                                            float* out, danet_stream_t s) {
    DANET_CHECK(B >= 0 && N >= 0, "danet_perspective_projection: negative size");
    if (B * N == 0) return 0;
    DANET_CHECK(points && rotation && translation && focal && center && out, "danet_perspective_projection: null pointer");
    k_persp<<<cdiv(B * N, 256), 256, 0, (cudaStream_t)s>>>(B, N, points, rotation, translation, focal, center, out);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_mpjpe_h36m(int32_t B, const float* pred_j17, const float* gt_j14, float* mpjpe, danet_stream_t s) {
    DANET_CHECK(B >= 0, "danet_mpjpe_h36m: negative batch");
    if (B == 0) return 0;
    DANET_CHECK(pred_j17 && gt_j14 && mpjpe, "danet_mpjpe_h36m: null pointer");
    k_mpjpe<<<cdiv(B, 64), 64, 0, (cudaStream_t)s>>>(B, pred_j17, gt_j14, mpjpe);
    DANET_LAUNCH_CHECK();
    return 0;
}
