// fp32 implicit-GEMM convolution on the FMA pipe (NHWC) -- the independent fp32 check path of the network half
// (conv_algo='simt'); its launcher (launchers.cuh) runs the network program's conv2d steps.
// Replaces nn.Conv2d (+ folded BatchNorm2d + ReLU + residual add) of models/module/hr_module.py,
// models/module/res_module.py; grouped convolutions (res_module.py:335-342,500-535) are expressed
// as `wsets` weight sets over the (batch,part)-flattened image axis (see include/danet_b200.h).
//
// CTA tile: 64 (image, output pixel) rows of one weight set x 64 output channels, 256 threads, 4x4 outputs per
// thread (32 x 32, 2x2 per thread, when the 64 x 64 grid would have fewer than 120 CTAs), K streamed in
// (tap, 16-channel) chunks through shared memory with register prefetch.
#include "launchers.cuh"

namespace danet {

constexpr int kKC = 16;      // input channels per K chunk

struct ConvArgs {
    int N, H, W, Cin, Cout, ks, stride, pad, Ho, Wo, wsets, relu;
    const float* x; const float* w; const float* bias; const float* res; float* y;
};

// TM x TN output tile per CTA (64x64: 4x4 outputs per thread; 32x32: 2x2, for problems whose 64x64
// grid would leave most SMs idle, e.g. the 2x2-pixel 512-channel layers of the ResNet tail)
template <int TM, int TN>
__global__ void __launch_bounds__(256)
k_conv_simt(ConvArgs a) {
    constexpr int MT = TM / 16, NTH = TN / 16;       // outputs per thread
    constexpr int APITCH = TM + 4;
    __shared__ __align__(16) float As[kKC][APITCH];
    __shared__ __align__(16) float Bs[kKC][TN];
    // rows of the implicit GEMM = (image of this weight set, output pixel), flattened: image
    // n = g + wsets * (row / HoWo).  Tiny maps (4x4, 2x2) then still fill the row tile.
    const int tid = threadIdx.x;
    const int g = blockIdx.z;
    const int q0 = blockIdx.x * TM;
    const int co0 = blockIdx.y * TN;
    const int HoWo = a.Ho * a.Wo;
    const int rows = ((a.N - g + a.wsets - 1) / a.wsets) * HoWo;
    const int K = a.ks * a.ks * a.Cin;
    const float* wg = a.w + (size_t)g * K * a.Cout;

    // A-load role (threads < TM*4): row lp = tid/4, channel vec lv = tid%4
    const bool a_role = tid < TM * 4;
    const int lp = tid >> 2, lv = tid & 3;
    const int lq = q0 + lp;
    const bool lvalid = a_role && lq < rows;
    const int lk = lvalid ? lq / HoWo : 0, lpix = lvalid ? lq - lk * HoWo : 0;
    const int loh = lpix / a.Wo, low = lpix - loh * a.Wo;
    const float* xn = a.x + (size_t)(g + a.wsets * lk) * a.H * a.W * a.Cin;
    // B-load role (threads < 16*TN/4): row bk, col vec bv
    const bool b_role = tid < kKC * (TN / 4);
    const int bk = tid / (TN / 4), bv = tid % (TN / 4);
    // compute role
    const int ty = tid >> 4, tx = tid & 15;

    float acc[MT][NTH];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NTH; ++j) acc[i][j] = 0.f;

    const int cchunks = (a.Cin + kKC - 1) / kKC;
    const int nchunks = a.ks * a.ks * cchunks;

    auto load = [&](int chunk, float4& ra, float4& rb) {
        const int tap = chunk / cchunks, c0 = (chunk % cchunks) * kKC;
        const int r = tap / a.ks, s = tap % a.ks;
        ra = make_float4(0.f, 0.f, 0.f, 0.f);
        const int ih = loh * a.stride - a.pad + r, iw = low * a.stride - a.pad + s;
        const int c = c0 + lv * 4;
        if (lvalid && ih >= 0 && ih < a.H && iw >= 0 && iw < a.W && c < a.Cin)
            ra = __ldg(reinterpret_cast<const float4*>(xn + ((size_t)ih * a.W + iw) * a.Cin + c));
        rb = make_float4(0.f, 0.f, 0.f, 0.f);
        const int kc = c0 + bk, co = co0 + bv * 4;
        if (b_role && kc < a.Cin && co < a.Cout)
            rb = __ldg(reinterpret_cast<const float4*>(wg + ((size_t)tap * a.Cin + kc) * a.Cout + co));
    };

    // kPF chunks of operands are in flight per thread: with one, every 16-channel chunk cost a full L2
    // round trip (288 chunks x ~0.8 us for the 2x2-pixel 512-channel layers)
    constexpr int kPF = 4;
    float4 ra[kPF], rb[kPF];
#pragma unroll
    for (int d = 0; d < kPF; ++d)
        if (d < nchunks) load(d, ra[d], rb[d]);
    for (int chunk0 = 0; chunk0 < nchunks; chunk0 += kPF) {
#pragma unroll
        for (int d = 0; d < kPF; ++d) {
            const int chunk = chunk0 + d;
            if (chunk >= nchunks) break;
            if (a_role) { As[lv * 4 + 0][lp] = ra[d].x; As[lv * 4 + 1][lp] = ra[d].y; As[lv * 4 + 2][lp] = ra[d].z; As[lv * 4 + 3][lp] = ra[d].w; }
            if (b_role) *reinterpret_cast<float4*>(&Bs[bk][bv * 4]) = rb[d];
            __syncthreads();
            if (chunk + kPF < nchunks) load(chunk + kPF, ra[d], rb[d]);
#pragma unroll
            for (int k = 0; k < kKC; ++k) {
                float am[MT], bm[NTH];
                if (MT == 4) {
                    const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
                    am[0] = av.x; am[1] = av.y; am[MT - 2] = av.z; am[MT - 1] = av.w;
                } else {
                    const float2 av = *reinterpret_cast<const float2*>(&As[k][ty * 2]);
                    am[0] = av.x; am[1] = av.y;
                }
                if (NTH == 4) {
                    const float4 bv4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
                    bm[0] = bv4.x; bm[1] = bv4.y; bm[NTH - 2] = bv4.z; bm[NTH - 1] = bv4.w;
                } else {
                    const float2 bv2 = *reinterpret_cast<const float2*>(&Bs[k][tx * 2]);
                    bm[0] = bv2.x; bm[1] = bv2.y;
                }
#pragma unroll
                for (int i = 0; i < MT; ++i)
#pragma unroll
                    for (int j = 0; j < NTH; ++j) acc[i][j] = fmaf(am[i], bm[j], acc[i][j]);
            }
            __syncthreads();
        }
    }

    const int co = co0 + tx * NTH;
    if (co >= a.Cout) return;
    float bias[NTH];
#pragma unroll
    for (int j = 0; j < NTH; ++j) bias[j] = a.bias ? __ldg(a.bias + (size_t)g * a.Cout + co + j) : 0.f;
#pragma unroll
    for (int i = 0; i < MT; ++i) {
        const int q = q0 + ty * MT + i;
        if (q >= rows) continue;
        const int qk = q / HoWo, qp = q - qk * HoWo;
        const size_t o = ((size_t)(g + a.wsets * qk) * HoWo + qp) * a.Cout + co;
        float v[NTH];
#pragma unroll
        for (int j = 0; j < NTH; ++j) {
            v[j] = acc[i][j] + bias[j];
            if (a.res) v[j] += __ldg(a.res + o + j);
            if (a.relu) v[j] = fmaxf(v[j], 0.f);
        }
        if (NTH == 4) *reinterpret_cast<float4*>(a.y + o) = make_float4(v[0], v[1], v[NTH - 2], v[NTH - 1]);
        else *reinterpret_cast<float2*>(a.y + o) = make_float2(v[0], v[1]);
    }
}

int conv2d(const danet_conv_desc& d, const float* x, const float* w, const float* bias, const float* residual, float* y,
           cudaStream_t stream) {
    DANET_CHECK(d.N >= 0 && d.H > 0 && d.W > 0 && d.Cin > 0 && d.Cout > 0, "danet_conv2d: bad sizes");
    DANET_CHECK(d.Cin % 4 == 0 && d.Cout % 4 == 0, "danet_conv2d: Cin (%d) and Cout (%d) must be multiples of 4 (pad channels)", d.Cin, d.Cout);
    DANET_CHECK(d.ksize >= 1 && d.ksize <= 7 && d.stride >= 1 && d.stride <= 2 && d.pad >= 0, "danet_conv2d: bad ksize/stride/pad");
    DANET_CHECK(d.wsets >= 1, "danet_conv2d: wsets must be >= 1");
    DANET_CHECK(d.H + 2 * d.pad >= d.ksize && d.W + 2 * d.pad >= d.ksize, "danet_conv2d: kernel larger than padded input");
    DANET_CHECK(d.wsets <= 65535, "danet_conv2d: wsets=%d exceeds 65535", d.wsets);
    if (d.N == 0) return 0;
    DANET_CHECK(x && w && y, "danet_conv2d: null pointer");
    DANET_CHECK(d.flags == 0, "danet_conv2d: flags are only taken by the tensor-core path");
    ConvArgs a;
    a.N = d.N; a.H = d.H; a.W = d.W; a.Cin = d.Cin; a.Cout = d.Cout; a.ks = d.ksize;
    a.stride = d.stride; a.pad = d.pad; a.wsets = d.wsets; a.relu = d.relu;
    a.Ho = (d.H + 2 * d.pad - d.ksize) / d.stride + 1;
    a.Wo = (d.W + 2 * d.pad - d.ksize) / d.stride + 1;
    a.x = x; a.w = w; a.bias = bias; a.res = residual; a.y = y;
    const int rows = cdiv(a.N, a.wsets) * a.Ho * a.Wo;
    const long long ctas64 = (long long)cdiv(rows, 64) * cdiv(a.Cout, 64) * a.wsets;
    if (ctas64 < 120) {
        dim3 grid(cdiv(rows, 32), cdiv(a.Cout, 32), a.wsets);
        k_conv_simt<32, 32><<<grid, 256, 0, stream>>>(a);
    } else {
        dim3 grid(cdiv(rows, 64), cdiv(a.Cout, 64), a.wsets);
        k_conv_simt<64, 64><<<grid, 256, 0, stream>>>(a);
    }
    DANET_LAUNCH_CHECK();
    return 0;
}

}  // namespace danet
