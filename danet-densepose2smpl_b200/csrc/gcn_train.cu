// Regressor head, training path: r2p_gcn -> refine_gcn (+ residual) -> p2r_gcn -> pose head + rot6d, with BatchNorm1d(24)
// on batch statistics, the intermediate heads of training mode and the backward of all of it
// (smpl_regressor.py:844-895, GCN.py:29-92, graph.py:232-261, geometry.py rot6d_to_rotmat).  rot6d and the state its
// backward reads (Rot6dState) are common.cuh's, shared with the inference pose head and the SMPL front-end.
//
// One launch per stage over the whole batch: a GraphConv layer is A.X (k_adj_mul), (A.X).W + b (k_gemm), the per-node
// batch statistics (k_bn_stats, one CTA per node: BatchNorm1d(24) normalises each node over B x F_out values, so no
// image's layer output can be normalised before every image's Y exists) and BN + ReLU (+ residual) (k_bn_act).  The
// backward mirrors it.  Every sum runs in a fixed order inside one thread or one CTA (no float atomics): results repeat
// bit for bit and nothing synchronises with the host.
#include "common.cuh"

namespace danet {
namespace {

constexpr int kDI[5] = {128, 128, 256, 256, 128};
constexpr int kDO[5] = {128, 256, 256, 128, 128};
constexpr float kBnEps = 1e-5f, kBnMomentum = 0.1f;
constexpr int kT = 256;

#define GT_TRY(x) do { int _r = (x); if (_r) return _r; } while (0)

// sum over a 256-thread CTA; every thread gets the same total (fixed shuffle tree, then the 8 warp sums in order)
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kT / 32; ++w) s += red[w];
    __syncthreads();
    return s;
}

__device__ __forceinline__ float bn_z(float y, float mean, float invstd, float g, float b) {
    return (y - mean) * invstd * g + b;
}

// The ReLU keeps NaN (fmaxf would return 0 for it), and its backward passes dy except where the input is <= 0, so a NaN
// passes dy: torch's relu and threshold_backward, and bn_train.cu's policy.
__device__ __forceinline__ float relu_keep_nan(float v) { return v <= 0.f ? 0.f : v; }
__device__ __forceinline__ bool relu_passes(float v) { return !(v <= 0.f); }

// ---- normalize_undigraph(I_n + A_mask * relu(E)) (graph.py:232-261): one CTA of 576 threads -----------------------
__global__ void k_adj_fwd(const float* __restrict__ I_n, const float* __restrict__ A_mask, const float* __restrict__ E,
                          float* __restrict__ Mout, float* __restrict__ Ahat, float* __restrict__ dout) {
    __shared__ float sM[576], sd[24];
    const int t = threadIdx.x;
    sM[t] = I_n[t] + A_mask[t] * relu_keep_nan(E[t]);
    __syncthreads();
    if (t < 24) {
        float s = 0.f;
        for (int i = 0; i < 24; ++i) s += sM[i * 24 + t];           // column sums: Dl = sum(A, 0)
        sd[t] = s > 0.f ? 1.f / sqrtf(s) : 0.f;
        dout[t] = sd[t];
    }
    __syncthreads();
    Mout[t] = sM[t];
    Ahat[t] = sd[t / 24] * sM[t] * sd[t % 24];
}

// d A_hat (summed over the three refinement layers in order) -> d edge_importance
__global__ void k_adj_bwd(const float* __restrict__ dApart, const float* __restrict__ M, const float* __restrict__ d,
                          const float* __restrict__ A_mask, const float* __restrict__ E, float* __restrict__ gE) {
    __shared__ float sG[576], sgs[24];
    const int t = threadIdx.x;
    sG[t] = (dApart[t] + dApart[576 + t]) + dApart[2 * 576 + t];
    __syncthreads();
    if (t < 24) {
        float gd = 0.f;
        for (int q = 0; q < 24; ++q) gd += sG[t * 24 + q] * M[t * 24 + q] * d[q];
        for (int p = 0; p < 24; ++p) gd += sG[p * 24 + t] * M[p * 24 + t] * d[p];
        sgs[t] = d[t] > 0.f ? -0.5f * d[t] * d[t] * d[t] * gd : 0.f;
    }
    __syncthreads();
    const int i = t / 24, j = t % 24;
    const float dM = sG[t] * d[i] * d[j] + sgs[j];
    gE[t] = relu_passes(E[t]) ? dM * A_mask[t] : 0.f;
}

// Y[b,n,f] = (add[b,n,f] +) sum_k A'[n,k] X[b,k,f], A' = A or A^T; add may be Y itself
__global__ void k_adj_mul(int B, int F, const float* __restrict__ A, int transpose, const float* __restrict__ X,
                          const float* add, float* Y) {
    __shared__ float sA[576];
    for (int i = threadIdx.x; i < 576; i += blockDim.x) sA[i] = transpose ? A[(i % 24) * 24 + i / 24] : A[i];
    __syncthreads();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 24 * F) return;
    const int f = idx % F, n = (idx / F) % 24, b = idx / (24 * F);
    const float* x = X + (size_t)b * 24 * F + f;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 24; ++k) s = fmaf(sA[n * 24 + k], x[k * F], s);
    Y[idx] = add ? add[idx] + s : s;
}

// C[M,N] = sum_k A(m,k) B(k,n) (+ bias[n]); A(m,k) = A[m*sam + k*sak], B(k,n) = B[k*sbk + n*sbn].  64 x 64 tiles,
// 4 x 4 outputs per thread, k in ascending order for every output.
constexpr int kGT = 64, kGK = 16;
__global__ void __launch_bounds__(kT) k_gemm(int M, int N, int K, const float* __restrict__ A, int sam, int sak,
                                             const float* __restrict__ Bm, int sbk, int sbn, const float* __restrict__ bias,
                                             float* __restrict__ C) {
    __shared__ float As[kGK][kGT + 4], Bs[kGK][kGT + 4];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int m0 = blockIdx.y * kGT, n0 = blockIdx.x * kGT;
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
    for (int k0 = 0; k0 < K; k0 += kGK) {
        for (int i = tid; i < kGK * kGT; i += kT) {
            int kk, mm;
            if (sam == 1) { kk = i / kGT; mm = i % kGT; } else { kk = i % kGK; mm = i / kGK; }
            const int m = m0 + mm, k = k0 + kk;
            As[kk][mm] = (m < M && k < K) ? A[(size_t)m * sam + (size_t)k * sak] : 0.f;
            int nn;
            if (sbn == 1) { kk = i / kGT; nn = i % kGT; } else { kk = i % kGK; nn = i / kGK; }
            const int n = n0 + nn, k2 = k0 + kk;
            Bs[kk][nn] = (n < N && k2 < K) ? Bm[(size_t)k2 * sbk + (size_t)n * sbn] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kGK; ++kk) {
            float a[4], b[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) a[r] = As[kk][ty + 16 * r];
#pragma unroll
            for (int c = 0; c < 4; ++c) b[c] = Bs[kk][tx + 16 * c];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(a[r], b[c], acc[r][c]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int m = m0 + ty + 16 * r;
        if (m >= M) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int n = n0 + tx + 16 * c;
            if (n < N) C[(size_t)m * N + n] = acc[r][c] + (bias ? bias[n] : 0.f);
        }
    }
}

// per-node statistics of Y [B,24,F] (one CTA per node): training -> batch mean / biased variance and the updated running
// statistics; eval -> the running statistics.  Both passes sum y - K with K = Y[0,n,0], a data element (as bn_train.cu
// does): the shifted mean dm = sum (y - K) / N is then off by a few units of the spread, not of |mean|, and the
// variance sum ((y - K) - dm)^2 / N keeps its digits when |mean| >> std.  An infinite first element would make every
// y - K NaN, so K is 0 then: the mean is infinite, as torch's is, and the running mean shows it.
__global__ void __launch_bounds__(kT) k_bn_stats(int B, int F, const float* __restrict__ Y, int training,
                                                 const float* __restrict__ rm, const float* __restrict__ rv,
                                                 float* __restrict__ mean_out, float* __restrict__ invstd_out,
                                                 float* __restrict__ new_rm, float* __restrict__ new_rv) {
    __shared__ float red[kT / 32];
    const int n = blockIdx.x, N = B * F;
    if (!training) {
        if (threadIdx.x == 0) { mean_out[n] = rm[n]; invstd_out[n] = 1.f / sqrtf(rv[n] + kBnEps); }
        return;
    }
    const float y0 = Y[(size_t)n * F];
    const float K = isfinite(y0) ? y0 : 0.f;
    float s = 0.f;
    for (int i = threadIdx.x; i < N; i += kT) s += Y[((size_t)(i / F) * 24 + n) * F + i % F] - K;
    const float dm = block_sum(s, red) / (float)N;
    const float mean = K + dm;
    float q = 0.f;
    for (int i = threadIdx.x; i < N; i += kT) {
        const float d = (Y[((size_t)(i / F) * 24 + n) * F + i % F] - K) - dm;
        q = fmaf(d, d, q);
    }
    const float var = block_sum(q, red) / (float)N;
    if (threadIdx.x == 0) {
        mean_out[n] = mean;
        invstd_out[n] = 1.f / sqrtf(var + kBnEps);
        if (new_rm) {
            new_rm[n] = (1.f - kBnMomentum) * rm[n] + kBnMomentum * mean;
            new_rv[n] = (1.f - kBnMomentum) * rv[n] + kBnMomentum * (var * (float)N / (float)(N - 1));
        }
    }
}

__global__ void k_bn_act(int B, int F, const float* __restrict__ Y, const float* __restrict__ mean,
                         const float* __restrict__ invstd, const float* __restrict__ g, const float* __restrict__ beta,
                         const float* __restrict__ res, float* __restrict__ H) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 24 * F) return;
    const int n = (idx / F) % 24;
    float v = relu_keep_nan(bn_z(Y[idx], mean[n], invstd[n], g[n], beta[n]));
    if (res) v += res[idx];                                    // l_pos_feat = pos_feats_init + refine (smpl_regressor.py:873)
    H[idx] = v;
}

// BN + ReLU backward, reduction half (one CTA per node): d gamma = sum dZ * xhat, d beta = sum dZ; sums[n] =
// (sum gamma dZ, sum gamma dZ xhat) for the input gradient
__global__ void __launch_bounds__(kT) k_bn_bwd_reduce(int B, int F, const float* __restrict__ Y, const float* __restrict__ mean,
                                                      const float* __restrict__ invstd, const float* __restrict__ g,
                                                      const float* __restrict__ beta, const float* __restrict__ dH,
                                                      float* __restrict__ g_gamma, float* __restrict__ g_beta,
                                                      float* __restrict__ sums) {
    __shared__ float red[kT / 32];
    const int n = blockIdx.x, N = B * F;
    const float mu = mean[n], is = invstd[n], ga = g[n], be = beta[n];
    float s1 = 0.f, s2 = 0.f;
    for (int i = threadIdx.x; i < N; i += kT) {
        const size_t e = ((size_t)(i / F) * 24 + n) * F + i % F;
        const float y = Y[e];
        const float dz = relu_passes(bn_z(y, mu, is, ga, be)) ? dH[e] : 0.f;
        s1 += dz;
        s2 = fmaf(dz, (y - mu) * is, s2);
    }
    s1 = block_sum(s1, red);
    s2 = block_sum(s2, red);
    if (threadIdx.x == 0) {
        g_gamma[n] = s2; g_beta[n] = s1;
        sums[2 * n] = ga * s1; sums[2 * n + 1] = ga * s2;
    }
}

__global__ void k_bn_bwd_dy(int B, int F, int training, const float* __restrict__ Y, const float* __restrict__ mean,
                            const float* __restrict__ invstd, const float* __restrict__ g, const float* __restrict__ beta,
                            const float* __restrict__ dH, const float* __restrict__ sums, float* __restrict__ dY) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 24 * F) return;
    const int n = (idx / F) % 24;
    const float y = Y[idx], mu = mean[n], is = invstd[n];
    const float dxh = relu_passes(bn_z(y, mu, is, g[n], beta[n])) ? dH[idx] * g[n] : 0.f;
    if (training) {
        const float Nf = (float)(B * F);
        dY[idx] = is / Nf * (Nf * dxh - sums[2 * n] - (y - mu) * is * sums[2 * n + 1]);
    } else {
        dY[idx] = dxh * is;
    }
}

// out[c] = sum_m X[m, c] (bias gradient over the 24 B rows)
__global__ void k_colsum(int M, int N, const float* __restrict__ X, float* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= N) return;
    float s = 0.f;
    for (int m = 0; m < M; ++m) s += X[(size_t)m * N + c];
    out[c] = s;
}

// dA[n,k] = sum_{b,f} dAX[b,n,f] X[b,k,f] (one CTA per (n,k))
__global__ void __launch_bounds__(kT) k_dadj(int B, int F, const float* __restrict__ dAX, const float* __restrict__ X,
                                             float* __restrict__ dA) {
    __shared__ float red[kT / 32];
    const int n = blockIdx.x / 24, k = blockIdx.x % 24, N = B * F;
    float s = 0.f;
    for (int i = threadIdx.x; i < N; i += kT) {
        const int b = i / F, f = i % F;
        s = fmaf(dAX[((size_t)b * 24 + n) * F + f], X[((size_t)b * 24 + k) * F + f], s);
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) dA[blockIdx.x] = s;
}

// grouped 1x1 conv, 24 groups of 128 -> K: out[b, j*K+k] = sum_f W[j*K+k, f] X[b,j,f] + bias (+ add)
__global__ void k_group_head(int B, int K, const float* __restrict__ X, const float* __restrict__ W,
                             const float* __restrict__ bias, const float* __restrict__ add, float* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 24 * K) return;
    const int jk = idx % (24 * K), b = idx / (24 * K), j = jk / K;
    const float* x = X + ((size_t)b * 24 + j) * 128;
    const float* w = W + (size_t)jk * 128;
    float s = 0.f;
    for (int f = 0; f < 128; ++f) s = fmaf(w[f], x[f], s);
    out[idx] = s + bias[jk] + (add ? add[jk] : 0.f);
}

// head backward, input half: dX[b,j,f] = (add[b,j,f] +) sum_k W[j*K+k, f] dp[b, j*K+k]; add may be dX itself
__global__ void k_head_bwd_x(int B, int K, const float* __restrict__ W, const float* __restrict__ dp,
                             const float* add, float* dX) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 24 * 128) return;
    const int f = idx % 128, j = (idx / 128) % 24, b = idx / (24 * 128);
    float s = 0.f;
    for (int k = 0; k < K; ++k) s = fmaf(W[(size_t)(j * K + k) * 128 + f], dp[(size_t)b * 24 * K + j * K + k], s);
    dX[idx] = add ? add[idx] + s : s;
}

// head backward, parameter half: dW[jk, f] = sum_b dp[b,jk] X[b,j,f]; db[jk] = sum_b dp[b,jk]
__global__ void k_head_bwd_w(int B, int K, const float* __restrict__ X, const float* __restrict__ dp,
                             float* __restrict__ dW, float* __restrict__ db) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 24 * K * 128) return;
    const int f = idx % 128, jk = idx / 128, j = jk / K;
    float s = 0.f, sb = 0.f;
    for (int b = 0; b < B; ++b) {
        const float g = dp[(size_t)b * 24 * K + jk];
        s = fmaf(g, X[((size_t)b * 24 + j) * 128 + f], s);
        sb += g;
    }
    dW[idx] = s;
    if (f == 0) db[jk] = sb;
}

__device__ __forceinline__ V3 axpy3(float s, V3 a, V3 b) { return v3(fmaf(s, a.x, b.x), fmaf(s, a.y, b.y), fmaf(s, a.z, b.z)); }
__device__ __forceinline__ V3 scale3(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }

// F.normalize backward: v / max(|v|, 1e-12); the clamp's side passes g / eps
__device__ __forceinline__ V3 normalize_bwd(float nraw, float n, V3 b, V3 g) {
    if (nraw > 1e-12f) return scale3(axpy3(-dot3(b, g), b, g), 1.f / n);
    return scale3(g, 1.f / n);
}

// rot6d_to_rotmat of the pose head: p6 [B,144] -> out[b*stride + off + j*9 + e]; para also gets global_para [B,13]
__global__ void k_rot6d_fwd(int B, const float* __restrict__ p6, float* __restrict__ out, int stride, int off,
                            const float* __restrict__ gpara) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 24) return;
    const int b = idx / 24, j = idx % 24;
    float R[9];
    rot6d(p6 + (size_t)idx * 6, R);
    float* o = out + (size_t)b * stride + off + j * 9;
#pragma unroll
    for (int e = 0; e < 9; ++e) o[e] = R[e];
    if (gpara && j < 13) out[(size_t)b * stride + j] = gpara[b * 13 + j];
}

// its backward: gR[b*stride + off + j*9 + e] -> dp6 [B,144]; g_gpara [B,13] = gR[b*stride + 0..12] when given
__global__ void k_rot6d_bwd(int B, const float* __restrict__ p6, const float* __restrict__ gR, int stride, int off,
                            float* __restrict__ dp6, float* __restrict__ g_gpara) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 24) return;
    const int b = idx / 24, j = idx % 24;
    const Rot6dState s = rot6d_state(p6 + (size_t)idx * 6);
    const float* g = gR + (size_t)b * stride + off + j * 9;
    const V3 g1 = v3(g[0], g[3], g[6]), g2 = v3(g[1], g[4], g[7]), g3 = v3(g[2], g[5], g[8]);
    const V3 c1 = cross3(s.b2, g3), c2 = cross3(g3, s.b1);
    V3 gb1 = v3(g1.x + c1.x, g1.y + c1.y, g1.z + c1.z);
    const V3 gb2 = v3(g2.x + c2.x, g2.y + c2.y, g2.z + c2.z);
    const V3 gu = normalize_bwd(s.n2r, s.n2, s.b2, gb2);
    const float gub1 = dot3(gu, s.b1);
    const V3 ga2 = axpy3(-gub1, s.b1, gu);
    gb1 = v3(gb1.x - s.a2.x * gub1 - s.dd * gu.x, gb1.y - s.a2.y * gub1 - s.dd * gu.y, gb1.z - s.a2.z * gub1 - s.dd * gu.z);
    const V3 ga1 = normalize_bwd(s.n1r, s.n1, s.b1, gb1);
    float* d = dp6 + (size_t)idx * 6;
    d[0] = ga1.x; d[1] = ga2.x; d[2] = ga1.y; d[3] = ga2.y; d[4] = ga1.z; d[5] = ga2.z;
    if (g_gpara && j < 13) g_gpara[b * 13 + j] = gR[(size_t)b * stride + j];
}

// the three head losses and their gradients, one CTA (sums in a fixed order); has[b] = 1 selects image b
__global__ void __launch_bounds__(kT) k_head_losses(int B, const float* __restrict__ pose0, const float* __restrict__ coord0,
                                                    const float* __restrict__ coord1, const float* __restrict__ target,
                                                    const float* __restrict__ gt, const uint8_t* __restrict__ has,
                                                    float rot_w, float pos_w, float* __restrict__ losses,
                                                    float* __restrict__ g_pose0, float* __restrict__ g_coord0,
                                                    float* __restrict__ g_coord1) {
    __shared__ float red[kT / 32];
    float c = 0.f;
    for (int b = threadIdx.x; b < B; b += kT) c += has[b] == 1 ? 1.f : 0.f;
    const float n = block_sum(c, red);
    const float inv = n > 0.f ? 1.f / n : 0.f;
    float s = 0.f;
    for (int i = threadIdx.x; i < B * 216; i += kT) {
        const int b = i / 216, e = i % 216;
        const float d = has[b] == 1 ? pose0[i] - target[(size_t)b * 229 + 13 + e] : 0.f;
        s = fmaf(d, d, s);
        if (g_pose0) g_pose0[i] = rot_w * 2.f * d * inv / 216.f;
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) losses[0] = rot_w * s * inv / 216.f;
    for (int k = 0; k < 2; ++k) {
        const float* cp = k ? coord1 : coord0;
        float* gc = k ? g_coord1 : g_coord0;
        float a = 0.f;
        for (int i = threadIdx.x; i < B * 72; i += kT) {
            const float d = has[i / 72] == 1 ? cp[i] - gt[i] : 0.f;
            a += fabsf(d);
            if (gc) gc[i] = pos_w * (float)((d > 0.f) - (d < 0.f)) * inv;
        }
        a = block_sum(a, red);
        if (threadIdx.x == 0) losses[1 + k] = pos_w * a * inv;
    }
}

// ---- workspace layout (floats, every region 256-byte aligned) -----------------------------------------------------
// The forward's saved activations, then one region per backward intermediate: gH[l] the full gradient of H[l] (the
// residual's and the coord heads' shares included), dY[l] the gradient of the GraphConv output, dAX[l] that of A X.
// tests/gcn_head_sweep_common.py mirrors this layout and reads every region.
struct Layout {
    size_t M, Ahat, d, AX[5], Y[5], H[5], mean[5], invstd[5], p6[2], dp6[2], gH[5], dY[5], dAX[5], dA, sums, total;
};
Layout layout(int B) {
    Layout L;
    size_t o = 0;
    auto take = [&](size_t n) { const size_t r = o; o += (n + 63) / 64 * 64; return r; };
    const size_t R = (size_t)24 * B;
    L.M = take(576); L.Ahat = take(576); L.d = take(24);
    for (int l = 0; l < 5; ++l) {
        L.AX[l] = take(R * kDI[l]); L.Y[l] = take(R * kDO[l]); L.H[l] = take(R * kDO[l]);
        L.mean[l] = take(24); L.invstd[l] = take(24);
    }
    for (int k = 0; k < 2; ++k) { L.p6[k] = take((size_t)B * 144); L.dp6[k] = take((size_t)B * 144); }
    for (int l = 0; l < 5; ++l) { L.gH[l] = take(R * kDO[l]); L.dY[l] = take(R * kDO[l]); L.dAX[l] = take(R * kDI[l]); }
    L.dA = take(3 * 576); L.sums = take(48);
    L.total = o;
    return L;
}

int gemm(cudaStream_t st, int M, int N, int K, const float* A, int sam, int sak, const float* Bm, int sbk, int sbn,
         const float* bias, float* C) {
    k_gemm<<<dim3(cdiv(N, kGT), cdiv(M, kGT)), kT, 0, st>>>(M, N, K, A, sam, sak, Bm, sbk, sbn, bias, C);
    DANET_LAUNCH_CHECK();
    return 0;
}

int adj_mul(cudaStream_t st, int B, int F, const float* A, int transpose, const float* X, const float* add, float* Y) {
    k_adj_mul<<<cdiv(B * 24 * F, kT), kT, 0, st>>>(B, F, A, transpose, X, add, Y);
    DANET_LAUNCH_CHECK();
    return 0;
}

int head_fwd(cudaStream_t st, int B, int K, const float* X, const float* W, const float* b, const float* add, float* out) {
    k_group_head<<<cdiv(B * 24 * K, kT), kT, 0, st>>>(B, K, X, W, b, add, out);
    DANET_LAUNCH_CHECK();
    return 0;
}

int head_bwd(cudaStream_t st, int B, int K, const float* X, const float* W, const float* dp, float* dW, float* db,
             const float* add, float* dX) {
    k_head_bwd_w<<<cdiv(24 * K * 128, kT), kT, 0, st>>>(B, K, X, dp, dW, db);
    DANET_LAUNCH_CHECK();
    k_head_bwd_x<<<cdiv(B * 24 * 128, kT), kT, 0, st>>>(B, K, W, dp, add, dX);
    DANET_LAUNCH_CHECK();
    return 0;
}

// The largest batch: the R-row gemms' grid.y, cdiv(24 B, 64), must stay within 65535, and every B * 24 * F element
// count (F <= 256) within int.  Both entries refuse a larger B before any launch.
constexpr int kMaxBatch = 65535 * kGT / 24;
static_assert((int64_t)kMaxBatch * 24 * 256 < ((int64_t)1 << 31), "element counts must fit in int");

int check_params(const danet_gcn_train_params* p, int training, bool grads) {
    DANET_CHECK(p, "gcn_head_train: null parameter struct");
    for (int l = 0; l < 5; ++l) {
        DANET_CHECK(p->W[l] && p->b[l] && p->bn_weight[l] && p->bn_bias[l] && p->running_mean[l] && p->running_var[l],
                    "gcn_head_train: layer %d has null parameters", l);
        DANET_CHECK(!grads || (p->gW[l] && p->gb[l] && p->g_bn_weight[l] && p->g_bn_bias[l]),
                    "gcn_head_train: layer %d has null gradient pointers", l);
    }
    DANET_CHECK(p->r2p_A && p->p2r_A && p->I_n && p->A_mask && p->edge_importance && p->mean_pose && p->pose_w[1] &&
                p->pose_b[1], "gcn_head_train: null graph buffer or pose head");
    DANET_CHECK(!training || (p->pose_w[0] && p->pose_b[0] && p->coord_w[0] && p->coord_b[0] && p->coord_w[1] && p->coord_b[1]),
                "gcn_head_train: training mode needs the intermediate heads");
    DANET_CHECK(!grads || (p->g_edge_importance && p->g_pose_w[1] && p->g_pose_b[1]), "gcn_head_train: null gradient pointers");
    DANET_CHECK(!grads || !training || (p->g_pose_w[0] && p->g_pose_b[0] && p->g_coord_w[0] && p->g_coord_b[0] &&
                                        p->g_coord_w[1] && p->g_coord_b[1]),
                "gcn_head_train: training mode needs the intermediate heads' gradient pointers");
    return 0;
}

}  // namespace
}  // namespace danet

using namespace danet;

extern "C" int64_t danet_gcn_head_train_workspace_bytes(int32_t B) {
    if (B < 1 || B > kMaxBatch) return 0;
    return (int64_t)layout(B).total * (int64_t)sizeof(float);
}

extern "C" int danet_gcn_head_train_forward(int32_t B, const danet_gcn_train_params* p, int32_t training,
                                            const float* rot_feats, const float* global_para, float* para, float* pose0,
                                            float* coord0, float* coord1, float* new_stats, void* workspace,
                                            danet_stream_t stream) {
    DANET_CHECK(B >= 1 && B <= kMaxBatch, "danet_gcn_head_train_forward: batch size %d outside 1..%d", B, kMaxBatch);
    GT_TRY(check_params(p, training, false));
    DANET_CHECK(rot_feats && global_para && para && workspace, "danet_gcn_head_train_forward: null pointer");
    DANET_CHECK(!training || (pose0 && coord0 && coord1), "danet_gcn_head_train_forward: training mode needs pose0 / coord0 / coord1");
    DANET_CHECK(aligned16(workspace), "danet_gcn_head_train_forward: workspace must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const Layout L = layout(B);
    float* w = (float*)workspace;
    k_adj_fwd<<<1, 576, 0, st>>>(p->I_n, p->A_mask, p->edge_importance, w + L.M, w + L.Ahat, w + L.d);
    DANET_LAUNCH_CHECK();
    const float* adj[5] = {p->r2p_A, w + L.Ahat, w + L.Ahat, w + L.Ahat, p->p2r_A};
    if (training) {                                             // pose_regressors[0] on rot_feats (smpl_regressor.py:849-856)
        GT_TRY(head_fwd(st, B, 6, rot_feats, p->pose_w[0], p->pose_b[0], p->mean_pose, w + L.p6[0]));
        k_rot6d_fwd<<<cdiv(B * 24, kT), kT, 0, st>>>(B, w + L.p6[0], pose0, 216, 0, nullptr);
        DANET_LAUNCH_CHECK();
    }
    const float* X = rot_feats;
    const int R = 24 * B;
    for (int l = 0; l < 5; ++l) {
        const int Fi = kDI[l], Fo = kDO[l];
        GT_TRY(adj_mul(st, B, Fi, adj[l], 0, X, nullptr, w + L.AX[l]));
        GT_TRY(gemm(st, R, Fo, Fi, w + L.AX[l], Fi, 1, p->W[l], Fo, 1, p->b[l], w + L.Y[l]));
        const bool upd = training && new_stats;
        k_bn_stats<<<24, kT, 0, st>>>(B, Fo, w + L.Y[l], training, p->running_mean[l], p->running_var[l], w + L.mean[l],
                                      w + L.invstd[l], upd ? new_stats + l * 24 : nullptr, upd ? new_stats + 120 + l * 24 : nullptr);
        DANET_LAUNCH_CHECK();
        k_bn_act<<<cdiv(R * Fo, kT), kT, 0, st>>>(B, Fo, w + L.Y[l], w + L.mean[l], w + L.invstd[l], p->bn_weight[l],
                                                  p->bn_bias[l], l == 3 ? w + L.H[0] : nullptr, w + L.H[l]);
        DANET_LAUNCH_CHECK();
        if (training && (l == 0 || l == 3)) {                  // coord_regressors[0/1] (smpl_regressor.py:863-882)
            const int k = l == 0 ? 0 : 1;
            GT_TRY(head_fwd(st, B, 3, w + L.H[l], p->coord_w[k], p->coord_b[k], nullptr, k ? coord1 : coord0));
        }
        X = w + L.H[l];
    }
    GT_TRY(head_fwd(st, B, 6, X, p->pose_w[1], p->pose_b[1], p->mean_pose, w + L.p6[1]));
    k_rot6d_fwd<<<cdiv(B * 24, kT), kT, 0, st>>>(B, w + L.p6[1], para, 229, 13, global_para);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_gcn_head_train_backward(int32_t B, const danet_gcn_train_params* p, int32_t training,
                                             const float* rot_feats, const float* g_para, const float* g_pose0,
                                             const float* g_coord0, const float* g_coord1, float* g_rot_feats,
                                             float* g_global_para, void* workspace, danet_stream_t stream) {
    DANET_CHECK(B >= 1 && B <= kMaxBatch, "danet_gcn_head_train_backward: batch size %d outside 1..%d", B, kMaxBatch);
    GT_TRY(check_params(p, training, true));
    DANET_CHECK(rot_feats && g_para && g_rot_feats && g_global_para && workspace, "danet_gcn_head_train_backward: null pointer");
    DANET_CHECK(!training || (g_pose0 && g_coord0 && g_coord1),
                "danet_gcn_head_train_backward: training mode needs g_pose0 / g_coord0 / g_coord1");
    DANET_CHECK(aligned16(workspace), "danet_gcn_head_train_backward: workspace must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const Layout L = layout(B);
    float* w = (float*)workspace;
    const int R = 24 * B;
    const float* adj[5] = {p->r2p_A, w + L.Ahat, w + L.Ahat, w + L.Ahat, p->p2r_A};
    // one GraphConv + BN + ReLU layer: dH -> gradients of its parameters, dY[l], dAX[l] and dX = (add +) A^T dAX[l]
    auto layer = [&](int l, const float* dH, const float* add, float* dX) -> int {
        const int Fi = kDI[l], Fo = kDO[l];
        const float* Xin = l == 0 ? rot_feats : w + L.H[l - 1];
        float* dY = w + L.dY[l]; float* dAX = w + L.dAX[l];
        k_bn_bwd_reduce<<<24, kT, 0, st>>>(B, Fo, w + L.Y[l], w + L.mean[l], w + L.invstd[l], p->bn_weight[l], p->bn_bias[l],
                                           dH, p->g_bn_weight[l], p->g_bn_bias[l], w + L.sums);
        DANET_LAUNCH_CHECK();
        k_bn_bwd_dy<<<cdiv(R * Fo, kT), kT, 0, st>>>(B, Fo, training, w + L.Y[l], w + L.mean[l], w + L.invstd[l],
                                                     p->bn_weight[l], p->bn_bias[l], dH, w + L.sums, dY);
        DANET_LAUNCH_CHECK();
        k_colsum<<<cdiv(Fo, 128), 128, 0, st>>>(R, Fo, dY, p->gb[l]);
        DANET_LAUNCH_CHECK();
        GT_TRY(gemm(st, Fi, Fo, R, w + L.AX[l], 1, Fi, dY, Fo, 1, nullptr, p->gW[l]));        // dW = (A X)^T dY
        GT_TRY(gemm(st, R, Fi, Fo, dY, Fo, 1, p->W[l], 1, Fo, nullptr, dAX));                // d(A X) = dY W^T
        if (l >= 1 && l <= 3) {
            k_dadj<<<576, kT, 0, st>>>(B, Fi, dAX, Xin, w + L.dA + (l - 1) * 576);
            DANET_LAUNCH_CHECK();
        }
        return adj_mul(st, B, Fi, adj[l], 1, dAX, add, dX);
    };
    float* gH[5];
    for (int l = 0; l < 5; ++l) gH[l] = w + L.gH[l];
    // pose_regressors[1] + rot6d; global_para's gradient is para's first 13 columns
    k_rot6d_bwd<<<cdiv(B * 24, kT), kT, 0, st>>>(B, w + L.p6[1], g_para, 229, 13, w + L.dp6[1], g_global_para);
    DANET_LAUNCH_CHECK();
    GT_TRY(head_bwd(st, B, 6, w + L.H[4], p->pose_w[1], w + L.dp6[1], p->g_pose_w[1], p->g_pose_b[1], nullptr, gH[4]));
    GT_TRY(layer(4, gH[4], nullptr, gH[3]));                           // gH[3] = d l_pos_feat
    if (training) GT_TRY(head_bwd(st, B, 3, w + L.H[3], p->coord_w[1], g_coord1, p->g_coord_w[1], p->g_coord_b[1], gH[3], gH[3]));
    GT_TRY(layer(3, gH[3], nullptr, gH[2]));
    GT_TRY(layer(2, gH[2], nullptr, gH[1]));
    GT_TRY(layer(1, gH[1], gH[3], gH[0]));                             // + the residual's share, gH[3]
    if (training) GT_TRY(head_bwd(st, B, 3, w + L.H[0], p->coord_w[0], g_coord0, p->g_coord_w[0], p->g_coord_b[0], gH[0], gH[0]));
    GT_TRY(layer(0, gH[0], nullptr, g_rot_feats));
    if (training) {
        k_rot6d_bwd<<<cdiv(B * 24, kT), kT, 0, st>>>(B, w + L.p6[0], g_pose0, 216, 0, w + L.dp6[0], nullptr);
        DANET_LAUNCH_CHECK();
        GT_TRY(head_bwd(st, B, 6, rot_feats, p->pose_w[0], w + L.dp6[0], p->g_pose_w[0], p->g_pose_b[0], g_rot_feats,
                        g_rot_feats));
    }
    k_adj_bwd<<<1, 576, 0, st>>>(w + L.dA, w + L.M, w + L.d, p->A_mask, p->edge_importance, p->g_edge_importance);
    DANET_LAUNCH_CHECK();
    return 0;
}

extern "C" int danet_gcn_head_losses(int32_t B, const float* pose0, const float* coord0, const float* coord1,
                                     const float* target, const float* gt_joints, const uint8_t* has, float rot_w,
                                     float pos_w, float* losses, float* g_pose0, float* g_coord0, float* g_coord1,
                                     danet_stream_t stream) {
    DANET_CHECK(B >= 1, "danet_gcn_head_losses: bad batch size %d", B);
    DANET_CHECK(pose0 && coord0 && coord1 && target && gt_joints && has && losses, "danet_gcn_head_losses: null pointer");
    k_head_losses<<<1, kT, 0, (cudaStream_t)stream>>>(B, pose0, coord0, coord1, target, gt_joints, has, rot_w, pos_w, losses,
                                                      g_pose0, g_coord0, g_coord1);
    DANET_LAUNCH_CHECK();
    return 0;
}
