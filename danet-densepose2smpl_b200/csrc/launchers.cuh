// Launchers of the network half's inference kernels (glue.cu, conv_simt.cu).  They are internal: their one caller is
// the step decoder of net.cu, so every inference launch -- the Python plan's through danet_net_run_step and a loaded
// program's -- is a step record.  Each checks its arguments (a program file is outside input), returns 0, or -1 with
// danet_last_error() set, and launches on `s`.  Activations are NHWC danet_act views: fp32 and/or split-fp16 planes;
// a launcher reads the fp32 view when present, else hi(+lo), and writes every view that is present.
#pragma once
#include "common.cuh"

namespace danet {

// GCN refinement + pose head parameters, device pointers prepared once: adj [3][24*24] (r2p_A, normalised refine
// adjacency, p2r_A); per GCN layer l (5 layers: r2p, refine0..2, p2r) W_l [din,dout], b_l [dout], BN scale / shift
// [24]; head_w [24][6][128], head_b [24*6], mean_pose [144].  Passed to k_gcn_pose_head as it is.
struct GcnArgs {
    const float* adj;
    const float* W[5]; const float* b[5]; const float* bn_s[5]; const float* bn_t[5];
    int din[5], dout[5];
    const float* head_w; const float* head_b; const float* mean_pose;
};

// input boundary: x NCHW [N,C,HW] -> y NHWC [N,HW,Cp] with Cp >= C zero-padded channels (demo.py:106, eval.py:147)
int nchw_to_nhwc(int N, int C, int HW, int Cp, const float* x, const danet_act* y, cudaStream_t s);
// fp32 FMA implicit-GEMM convolution (the conv_algo='simt' check path): fp32 views only, weights w
// [wsets][ksize*ksize*Cin][Cout] (tap-major, then cin), bias [wsets][Cout] (BN folded), residual (or NULL) of the
// output's shape added before the ReLU (res_module.py:40-56,77-97).  d.flags must be 0.
int conv2d(const danet_conv_desc& d, const float* x, const float* w, const float* bias, const float* residual, float* y,
           cudaStream_t s);
// hr_module.py:161-179 fuse: y = relu(sum_j up_{f_j}(t_j)), t_j [N,H/f_j,W/f_j,C] nearest-upsampled by f_j in
// {1,2,4,8}, 1..4 terms summed in argument order; C % 8 == 0
int fuse_sum(int N, int H, int W, int C, int nterms, const danet_act* terms, const int32_t* factors, int relu,
             const danet_act* y, cudaStream_t s);
// nn.MaxPool2d(3,2,1) (res_module.py:409); C % 8 == 0
int maxpool3x3s2(int N, int H, int W, int C, const danet_act* x, const danet_act* y, cudaStream_t s);
// utils/iuvmap.py:6-38 iuvmap_clean on the global heads [B,HW,Chead] (U 25 | V 25 | Index 25 | Ann 15 at off_u / off_v
// / off_i / off_a) -> body_iuv [B,HW,Cbody >= 75] (cat[U,V,I] of danet.py:85, pad channels zeroed), the uint8 argmax
// map [B,HW] and optional NCHW u / v / i [B,25,HW], ann [B,15,HW] (danet.py:81).  Chead, Cbody % 4 == 0, 64 pixels of
// both rows fit in 48 KB of shared memory, heads 16-byte aligned.
int iuv_clean_global(int B, int HW, int Chead, int off_u, int off_v, int off_i, int off_a, int Cbody, const float* heads,
                     const danet_act* body_iuv, uint8_t* index_argmax, float* u_nchw, float* v_nchw, float* i_nchw,
                     float* ann_nchw, cudaStream_t s);
// danet.py:93-98, the 24 per-part iuvmap_clean calls: x [N,HW,Cx] with (U 7 | V 7 | I 7) in its first 21 channels
// (N = batch*24) -> y [N,HW,Cy] (pad channels zeroed) and an optional raw copy part_iuv_pred [N,21,HW]
// (iuv_estimator.py:208-211).  Cx, Cy >= 24 and % 4 == 0.
int iuv_clean_parts(int N, int HW, int Cx, int Cy, const float* x, const danet_act* y, float* raw_nchw, cudaStream_t s);
// iuv_estimator.py:137-140,176-184,262-301: soft-argmax centres of 10*hm [B,HW,Chm] (24 heat-map channels first), part
// visibility from index_argmax [B,HW], affine thetas -> centers [B,24,2], theta [B,24,3] = (scale, cx, cy).
// align_corners: 0 = torch >= 1.3 semantics, 1 = torch 1.1.
int stn_params(int B, int S, int Chm, const float* hm, const uint8_t* index_argmax, const float* learned_ratio,
               const float* learned_offset, float vis_thresh, int align_corners, float* centers, float* theta,
               cudaStream_t s);
// iuv_estimator.py:193-204: 24x affine_grid + grid_sample (bilinear, zeros) of xd [B,S,S,C] -> crops [B*24,S,S,C]
// (image b*24 + part); C % 8 == 0
int stn_sample(int B, int S, int C, const danet_act* xd, const float* theta, int align_corners, const danet_act* crops,
               cudaStream_t s);
// smpl_regressor.py:858-895 + GCN.py:29-92 + geometry.py:47-61: r2p_gcn -> refine_gcn(+res) -> p2r_gcn -> grouped 1x1
// pose head + mean_pose -> rot6d_to_rotmat, after global_para [B,13] (cam, shape) -> para [B,229]; rot_feats [B,24,128]
int gcn_pose_head(int B, const GcnArgs& g, const float* rot_feats, const float* global_para, float* para, cudaStream_t s);

}  // namespace danet
