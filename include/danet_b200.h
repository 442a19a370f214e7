/* libdanet_b200.so -- C ABI of the H100-native DaNet inference hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  Every entry point replaces one piece of the
 * reference's Python/ATen path (file:line of the reference cited per function).  Conventions:
 *   - all data pointers are DEVICE pointers (fp32 / int32 / uint8, contiguous, caller-owned)
 *     unless the name says `host`; no torch types cross this boundary;
 *   - every call takes a `cudaStream_t` (passed as void*) and is asynchronous on it;
 *   - return value: 0 = ok, <0 = error; `danet_last_error()` returns a thread-local message;
 *   - no allocation inside hot calls: handles own their constants, callers own activations and
 *     workspaces (sizes from the `*_workspace_bytes` helpers);
 *   - handles are not thread-safe: one handle per stream / rank.
 *
 * Activations of the network half are fp32 NHWC ("pixels x channels"); tensors that the
 * reference returns to its callers in NCHW are written in NCHW by the kernel that produces them.
 */
#ifndef DANET_B200_H
#define DANET_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef void* danet_stream_t;                 /* cudaStream_t */
typedef struct danet_smpl*   danet_smpl_t;
typedef struct danet_raster* danet_raster_t;

const char* danet_last_error(void);
int danet_version(void);                      /* ABI version, bumped on any signature change */
int danet_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------
 * SMPL layer.  Replaces models/smpl.py:15-46 (SMPL.__init__/forward) and the third-party
 * smplx.lbs it calls (lbs, batch_rodrigues, batch_rigid_transform, vertices2joints,
 * VertexJointSelector), plus utils/geometry.py:9-61 (batch_rodrigues, rot6d_to_rotmat) as
 * pose front-ends and eval.py:78,186,202 (J_regressor_h36m matmul).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int32_t num_verts;                 /* 6890 */
    int32_t num_joints;                /* 24 */
    int32_t num_betas;                 /* 10 */
    const float* v_template;           /* HOST [V,3] */
    const float* shapedirs;            /* HOST [V,3,num_betas] */
    const float* posedirs;             /* HOST [(J-1)*9, V*3]  (smplx layout) */
    const float* J_regressor;          /* HOST [J,V] */
    const float* lbs_weights;          /* HOST [V,J] */
    const int32_t* parents;            /* HOST [J], parents[0] = -1 */
    int32_t num_selected;              /* 21 vertices appended by VertexJointSelector */
    const int32_t* selected_verts;     /* HOST [num_selected] */
    int32_t num_extra;                 /* 9 rows of J_regressor_extra (models/smpl.py:21-22) */
    const float* J_regressor_extra;    /* HOST [num_extra,V] */
    int32_t num_h36m;                  /* 17 rows of J_regressor_h36m (eval.py:78) or 0 */
    const float* J_regressor_h36m;     /* HOST [num_h36m,V] or NULL */
    int32_t num_out_joints;            /* 49 */
    const int32_t* joint_map;          /* HOST [num_out_joints] into cat(J posed, selected, extra) */
} danet_smpl_desc;

enum { DANET_POSE_ROTMAT = 0,          /* pose [B,24,3,3]   (pose2rot=False)                       */
       DANET_POSE_AXIS_ANGLE = 1,      /* pose [B,24,3]     smplx Rodrigues (pose2rot=True)         */
       DANET_POSE_ROT6D = 2 };         /* pose [B,24,6]     utils/geometry.py:47-61                 */

int danet_smpl_create(const danet_smpl_desc* desc, danet_smpl_t* out);
int danet_smpl_destroy(danet_smpl_t h);
/* bytes of scratch `danet_smpl_forward` needs for a batch of B bodies */
int64_t danet_smpl_workspace_bytes(danet_smpl_t h, int32_t B);
/* outputs may be NULL to skip: verts [B,V,3]; joints [B,num_out_joints,3];
 * smpl_joints [B,J,3]; joints_h36m [B,num_h36m,3]; rotmats [B,J,3,3].
 * `bodies_per_cta` 0 = auto (tuning knob: 1,2,4,8,16). */
int danet_smpl_forward(danet_smpl_t h, int32_t B, const float* betas, const float* pose,
                       int32_t pose_kind, float* verts, float* joints, float* smpl_joints,
                       float* joints_h36m, float* rotmats, void* workspace,
                       int32_t bodies_per_cta, danet_stream_t stream);

/* Backward of the SMPL layer -- the first piece of the training step (train/trainer.py:148-215 back-propagates
 * vertex / joint losses through models/smpl.py:27-46 into the regressed betas and rotation matrices,
 * models/danet/smpl_regressor.py:131-221).  rotmats [B,24,3,3] are the matrices the forward consumed (pose2rot=False,
 * treated as free 3x3 inputs); grad_verts [B,V,3]; grad_smpl_joints [B,24,3] or NULL (gradients w.r.t. the regressed
 * joints are folded into grad_verts by the caller: J_regressor^T g); outputs grad_betas [B,num_betas],
 * grad_rotmats [B,24,3,3].  Recomputes the forward intermediates; fp32, with no float atomics: every sum runs in a
 * fixed order, so the result is bit-for-bit repeatable and a body's gradient does not depend on the rest of the batch. */
int64_t danet_smpl_backward_workspace_bytes(danet_smpl_t h, int32_t B);
int danet_smpl_backward(danet_smpl_t h, int32_t B, const float* betas, const float* rotmats,
                        const float* grad_verts, const float* grad_smpl_joints, float* grad_betas,
                        float* grad_rotmats, void* workspace, danet_stream_t stream);

/* utils/geometry.py:47-61 rot6d_to_rotmat: x [n,6] (viewed [n,3,2]) -> R [n,3,3] */
int danet_rot6d_to_rotmat(int32_t n, const float* x, float* R, danet_stream_t stream);
/* utils/geometry.py:9-45 batch_rodrigues (quaternion route): aa [n,3] -> R [n,3,3];
 * flavor 1 = smplx.lbs.batch_rodrigues (matrix exponential form) */
int danet_batch_rodrigues(int32_t n, const float* aa, float* R, int32_t flavor, danet_stream_t stream);
/* utils/geometry.py:63-91 perspective_projection: points [B,N,3], rotation [B,3,3],
 * translation [B,3], focal [B] , center [B,2] -> out [B,N,2] */
int danet_perspective_projection(int32_t B, int32_t N, const float* points, const float* rotation,
                                 const float* translation, const float* focal, const float* center,
                                 float* out, danet_stream_t stream);
/* eval.py:202-212: pred_j17 [B,17,3] (J_regressor_h36m joints), gt_j14 [B,14,3] (already
 * pelvis-centred + H36M_TO_J14-selected) -> mpjpe [B] */
int danet_mpjpe_h36m(int32_t B, const float* pred_j17, const float* gt_j14, float* mpjpe,
                     danet_stream_t stream);
/* eval.py:219-266 with utils/imutils.py:89-113 (uncrop): LSP mask and part scoring of B rendered maps at their
 * original image sizes (csrc/seg_eval.cu).  mask / parts [B,R,R] uint8 (the render: mask nonzero = covered -- the
 * caller applies toimage's bytescale, which empties an all-covered float mask; parts 0..6); geom [B,8] int64 per image
 * = { ul_x, ul_y, crop_h, crop_w, orig_h, orig_w, gt_offset, table_offset } where ul and crop = br - ul are uncrop's
 * integers and the crop overlaps or touches the image; mask_gt / parts_gt: the ground-truth images, row-major
 * [orig_h, orig_w] uint8 at gt_offset of one packed buffer each; tables: int32 workspace of sum(crop_h + crop_w)
 * entries, image b's at table_offset; max_pixels: the largest orig_h * orig_w (it sizes the grid, <= INT32_MAX) ->
 *   mask_conf [B,2,2] int64   pixel counts of (gt > 0, pred > 0)
 *   part_conf [B,9,7] int64   pixel counts of (gt row, pred part): rows 0..6 the labels, 7 the label 255, 8 any other
 *                             label; a predicted part past 6 is counted in no column
 * The crop is resized like scipy.misc.imresize(interp='nearest') = Pillow's NEAREST (a sequential double recurrence
 * per axis).  Integer counts: exact and repeatable. */
int danet_seg_confusion(int32_t B, int32_t R, const uint8_t* mask, const uint8_t* parts, const int64_t* geom,
                        const uint8_t* mask_gt, const uint8_t* parts_gt, int64_t max_pixels, int32_t* tables,
                        int64_t* mask_conf, int64_t* part_conf, danet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training targets (csrc/targets.cu).  No entry synchronises with the host, so a step's target
 * preparation can be captured in one CUDA graph.
 * ------------------------------------------------------------------------------------------ */
/* utils/geometry.py:94-157 estimate_translation (with estimate_translation_np): S [B,49,3] joints and joints_2d
 * [B,49,3] key points (x, y in pixels, confidence), of which joints 25..48 are used -> trans [B,3].  Weights are the
 * fp32 sqrt of the confidences; the normal equations are formed and solved (LU with partial pivoting) in fp64 and
 * rounded once to fp32.  Where numpy raises LinAlgError (an exactly zero pivot: every confidence 0), the row is NaN. */
int danet_estimate_translation(int32_t B, const float* S, const float* joints_2d, double focal_length, double img_size,
                               float* trans, danet_stream_t stream);
/* train/trainer.py:157-161 and :177-191: fit_pose [B,72] / fit_betas [B,10] (the SPIN fits) with a row's betas zeroed
 * when any |beta| > 3, then replaced by gt_pose / gt_betas where has_smpl -> opt_pose, opt_betas; valid_fit [B] =
 * has_smpl | fit_valid (fit_valid NULL = has_smpl alone); has_iuv [B] = iuv_annotated & valid_fit.  Flags are uint8,
 * nonzero = true; the outputs are 0 / 1. */
int danet_fit_merge(int32_t B, const float* fit_pose, const float* fit_betas, const float* gt_pose, const float* gt_betas,
                    const uint8_t* has_smpl, const uint8_t* fit_valid, const uint8_t* iuv_annotated, float* opt_pose,
                    float* opt_betas, uint8_t* valid_fit, uint8_t* has_iuv, danet_stream_t stream);
/* train/trainer.py:163-212 after the SMPL forward of the merged fits, and models/danet/danet.py:159-162.
 * opt_joints [B,49,3] and smpl_joints [B,24,3] of that forward, keypoints [B,49,3] (x, y in [-1,1], confidence),
 * opt_pose [B,72], opt_betas [B,10], has_iuv / has_dp [B] uint8, smpl_2dkps [B,24,3] ->
 *   opt_cam_t [B,3]        danet_estimate_translation of opt_joints on the de-normalised key points (:168-175)
 *   target_cam [B,3]       [2 f / img_res / t_z, t_x, t_y] (:208-212)
 *   target_smpl_kps [B,24,3]  smpl_joints projected with R = I, t = opt_cam_t, centre img_res / 2, normalised to
 *                          [-1,1], confidence (has_iuv == 1); the row is smpl_2dkps where has_dp == 1 (:194-204)
 *   target [B,229]         cat(target_cam, opt_betas, batch_rodrigues(opt_pose)), quaternion route (danet.py:159-162) */
int danet_train_targets(int32_t B, const float* opt_joints, const float* smpl_joints, const float* keypoints,
                        const float* opt_pose, const float* opt_betas, const uint8_t* has_iuv, const uint8_t* has_dp,
                        const float* smpl_2dkps, double focal_length, int32_t img_res, float* opt_cam_t, float* target_cam,
                        float* target_smpl_kps, float* target, danet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Dense IUV losses of the training step (SURVEY section 8f-2), forward and backward in one pass.
 * Replaces models/danet/iuv_estimator.py:304-341 (IUV_Estimator.body_uv_losses) and the autograd
 * graph torch records for it.  Predictions u/v/index [N,C,HW] and targets U/V/I [N,C,HW] (fp32,
 * channel stride HW, image strides `pred_stride` / `map_stride` in elements, 0 = dense C*HW), optional
 * annotation logits / targets [N,Cann,HW] (dense, both NULL to skip), optional has_iuv [N] (uint8, NULL =
 * every image).  losses[4] = { point_weight/batch_size * sum smooth_l1(u - U | I > 0), the same for v,
 * mean cross-entropy(index, argmax I), mean cross-entropy(ann, argmax Ann) } over the images with
 * has_iuv (all zero when none has).  grad_* (NULL to skip; laid out like the predictions) receive
 * d losses[k] / d prediction.  The 24 per-part calls of iuv_estimator.py:232-255 are one call over the
 * (batch, part)-flattened axis: N = 24 B, batch_size = 24 B, strides 3*7*HW, has_iuv repeated per part.
 * Deterministic (fixed summation order). */
int64_t danet_body_uv_losses_workspace_bytes(int32_t N, int32_t HW);
int danet_body_uv_losses(int32_t N, int32_t C, int32_t Cann, int32_t HW, int64_t pred_stride, int64_t map_stride,
                         const float* u_pred, const float* v_pred, const float* index_pred, const float* ann_pred,
                         const float* Umap, const float* Vmap, const float* Imap, const float* Annmap,
                         const uint8_t* has_iuv, float batch_size, float point_weight, float* losses,
                         float* grad_u, float* grad_v, float* grad_index, float* grad_ann, void* workspace,
                         danet_stream_t stream);

/* Sparse DensePose-point losses, forward and backward in one pass.  Replaces
 * models/danet/iuv_estimator.py:343-419 (IUV_Estimator.dp_uvia_losses, called from :106-121) and its autograd graph.
 * Predictions u/v/index [N,25,S,S], ann [N,Cann,S,S]; per image P point slots (196): X / Y / I points [N,P]
 * (pixel coordinates, float labels truncated toward zero), U / V points and point weights [N,25,P] (patch-major),
 * ann_labels [N,S*S] (float labels); has_dp [N] uint8 or NULL (= every image).  The points are sampled bilinearly
 * with zeros padding at grid (X - S/2) * 2/S (align_corners 0 = torch >= 1.3, 1 = torch 1.1).
 * losses[4] = { point_weight * sum w * SL1(w * (u - U)) (a sum, not divided by the batch), the same for v,
 * part_weight * mean cross-entropy of the sampled index logits over nsel*P points, index_weight * mean cross-entropy
 * of ann over nsel*S*S pixels }, all zero when no image is selected.  grad_* (NULL to skip) receive d losses[k] /
 * d prediction; the grid_sample backward is a gather in point order.  Labels outside [0, C) contribute nothing (the
 * Python layer rejects them).  Deterministic.  Workspace: danet_dp_uvia_losses_workspace_bytes(N, S*S). */
int64_t danet_dp_uvia_losses_workspace_bytes(int32_t N, int32_t HW);
int danet_dp_uvia_losses(int32_t N, int32_t S, int32_t Cann, int32_t P, const float* u_pred, const float* v_pred,
                         const float* index_pred, const float* ann_pred, const float* X_points, const float* Y_points,
                         const float* I_points, const float* U_points, const float* V_points, const float* point_weights,
                         const float* ann_labels, const uint8_t* has_dp, int32_t align_corners, float point_weight,
                         float part_weight, float index_weight, float* losses, float* grad_u, float* grad_v,
                         float* grad_index, float* grad_ann, void* workspace, danet_stream_t stream);

/* STN key-point losses, forward and backward in one pass.  Replaces iuv_estimator.py:137-171 with
 * utils/keypoints.py:268-331 (generate_heatmap) and :334-394 (softmax_integral_tensor).  hm [B,J,S,S] (NCHW),
 * kps [B,J,kps_cols] (x, y in [-1, 1], third column = weight).  Centre of joint j: soft-argmax of 10*hm / (0.5*S) - 1.
 * losses[2] = { kps_weight / B * sum_{w != 0} w * (SL1(cx - x) + SL1(cy - y))  (0 when kps_cols == 2),
 * hm_weight * mean SL1(hm - G) with G the sigma-1 7x7 Gaussian at int(k*S + 0.5), k = 0.5*gt + 0.5 }.
 * grad_roi / grad_hm [B,J,S,S] (NULL to skip) = d losses[0] / d hm and d losses[1] / d hm; the same pointer twice
 * receives their sum.  Deterministic.
 * Workspace: danet_stn_kps_losses_workspace_bytes(B, J). */
int64_t danet_stn_kps_losses_workspace_bytes(int32_t B, int32_t J);
int danet_stn_kps_losses(int32_t B, int32_t J, int32_t S, const float* hm, const float* kps, int32_t kps_cols,
                         float kps_weight, float hm_weight, float* losses, float* grad_roi, float* grad_hm,
                         void* workspace, danet_stream_t stream);

/* Part-crop IUV targets.  Replaces iuv_estimator.py:217-230 with part_iuv_simp :422-445.  Umap / Vmap / Imap
 * [B,C,S,S] (C >= 25, iuv_img2map), theta [B,24,2,3] (affine_para) -> out [B,24,3,7,S,S]: per part i and map, channel 0
 * = background (0 for U and V; for I: sum of the 6 mapped I channels < 0.5 at the source pixel), then the 6 channels
 * of dp2smpl_mapping[i], each resampled by affine_grid + grid_sample (bilinear, zeros padding). */
int danet_part_iuv_targets(int32_t B, int32_t S, int32_t C, const float* Umap, const float* Vmap, const float* Imap,
                           const float* theta, int32_t align_corners, float* out, danet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * IUV rasteriser.  Replaces utils/renderer.py:207-298 (IUV_Renderer) and the third-party
 * neural_renderer forward pass it calls; optionally fuses utils/iuvmap.py:103-151 (iuv_img2map).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int32_t num_smpl_verts;            /* 6890 */
    int32_t num_mesh_verts;            /* 7829 */
    const int32_t* vert_mapping;       /* HOST [num_mesh_verts], 0-based into SMPL vertices */
    int32_t num_faces;                 /* 13774 */
    const int32_t* faces;              /* HOST [num_faces,3] into mesh verts */
    const float* textures;             /* HOST [num_faces,3]  (I/24, mean U, mean V) */
    int32_t orig_size;                 /* 224 */
    int32_t out_size;                  /* 56 */
    float focal_length;                /* 5000 (already scaled by orig_size/224 like renderer.py:222-227) */
    float near_plane, far_plane;       /* 0.1, 100 */
    int32_t tex_mode;                  /* 0 = face texture exactly; 1 = neural_renderer texture_size==1 blend */
} danet_raster_desc;

int danet_raster_create(const danet_raster_desc* desc, danet_raster_t* out);
int danet_raster_destroy(danet_raster_t h);
int64_t danet_raster_workspace_bytes(danet_raster_t h, int32_t B);
/* verts [B,V,3], cam [B,3] (s,tx,ty) -> img [B,3,S,S].  Optional (NULL to skip):
 * face_idx [B,S,S] int32 (-1 background), maps_u/v/i [B,25,S,S], maps_ann [B,15,S,S]. */
int danet_raster_iuv(danet_raster_t h, int32_t B, const float* verts, const float* cam, float* img,
                     int32_t* face_idx, float* maps_u, float* maps_v, float* maps_i, float* maps_ann,
                     void* workspace, danet_stream_t stream);
/* danet_raster_iuv for the images b with select[b] != 0 (select [B] uint8; NULL = every image), as
 * models/danet/danet.py:163-165 renders verts2uvimg(target_verts[has_iuv], target_cam[has_iuv]) into a zero image:
 * the other images cost no rasterisation and come out as background (the zero image, face -1, its maps), whatever
 * their vertices and camera hold.  danet_raster_iuv is this entry with select = NULL. */
int danet_raster_iuv_select(danet_raster_t h, int32_t B, const float* verts, const float* cam, const uint8_t* select,
                            float* img, int32_t* face_idx, float* maps_u, float* maps_v, float* maps_i, float* maps_ann,
                            void* workspace, danet_stream_t stream);
/* utils/iuvmap.py:103-151 on an arbitrary IUV image [B,3,S,S] */
int danet_iuv_img2map(int32_t B, int32_t S, const float* img, float* maps_u, float* maps_v,
                      float* maps_i, float* maps_ann, danet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Network half (models/danet/, models/module/).  NHWC activations as danet_act views (fp32 and/or
 * split-fp16 planes): an entry reads the fp32 view when present, else hi(+lo), and writes every view that is
 * present.  The network's other layers (input conversion, fp32-FMA convolution, HRNet fuse, pools, iuvmap_clean,
 * STN, GCN head) run as steps of a network program (danet_net_*, below).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int32_t N, H, W, Cin;              /* input  [N,H,W,Cin]                                      */
    int32_t Cout, ksize, stride, pad;  /* output [N,Ho,Wo,Cout], Ho = (H+2*pad-ksize)/stride+1     */
    int32_t wsets;                     /* weight sets: image n uses set n % wsets (grouped convs of
                                          res_module.py:335-342,500-535 become wsets=24 over the
                                          (batch,part)-flattened image axis)                       */
    int32_t relu;                      /* apply ReLU last                                         */
    int32_t flags;                     /* tensor-core path: DANET_CONV_EXACT                      */
} danet_conv_desc;
/* tensor-core path, exact mode: three MMAs per K step on split-fp16 operands (hi*hi + hi*lo + lo*hi,
 * fp32 accumulation): fp32-grade results (the reference computes these layers in fp32).  Without the flag
 * only hi*hi is issued (fp16-operand precision, ~1e-3 on the network output). */
#define DANET_CONV_EXACT 4

/* An activation tensor of the network half, NHWC.  Any subset of the three views may be present:
 *   f32      fp32 [N,H,W,C]
 *   hi / lo  SPLIT-FP16 planes, each IEEE fp16 [N,H,W,C], C % 8 == 0, 16-byte aligned:
 *            value = float(hi) + float(lo), hi = rn(value), lo = rn(value - hi)  (22 significant bits);
 *            lo == NULL means "hi only" (fast mode).
 * Tensor-core convolutions read hi/lo through TMA tensor maps and write any of the views. */
typedef struct { float* f32; void* hi; void* lo; } danet_act;

/* Tensor-core path.  One launch runs up to 6 independent convolutions (e.g. the parallel branches of an
 * HRNet stage, hr_module.py:165-166) over one persistent grid.  w_packed comes from danet_conv_tc_pack with
 * the SAME descriptor (flags included).  x needs hi (+ lo in exact mode); res: f32, or hi(+lo), or all NULL;
 * y: f32 and/or hi(+lo).  Cin % 8 == 0, Cout % 8 == 0 (pad channels carry zero weights / zero data). */
typedef struct {
    danet_conv_desc d;
    danet_act x, res, y;
    const void* w_packed;
    const float* bias;                 /* [wsets][Cout] or NULL */
} danet_conv_problem;
int danet_conv_tc_group(int32_t n, const danet_conv_problem* problems, danet_stream_t stream);
/* The depth of the shared activation / weight rings (stages[0], stages[1]) a launch over a group of n problems would
 * get; the rings are sized for the largest member.  Nonzero if the group cannot share one launch. */
int danet_conv_tc_config(int32_t n, const danet_conv_desc* descs, int32_t* stages);
/* bytes / packing helper: converts weights in the SIMT layout w [wsets][ksize*ksize*Cin][Cout] (tap-major, then cin)
 * into the swizzled shared-memory image blocks of split-fp16 weights the wgmma kernel bulk-copies (device -> device,
 * stream-ordered, no host synchronisation or allocation: capturable in a CUDA graph).  Header word 2 of w_packed is its
 * scratch while it runs. */
int64_t danet_conv_tc_packed_bytes(const danet_conv_desc* d);
int danet_conv_tc_pack(const danet_conv_desc* d, const float* w_simt, void* w_packed, danet_stream_t stream);
int danet_conv_tc_supported(const danet_conv_desc* d);
/* Host-only geometry of one problem, as the engine tiles it: out[0..7] = tile rows, tile columns, tiles, images per tile
 * (small maps stack several), products per MAC (exact 3, fast 1), issued MACs of one product per tile, activation
 * bytes and weight bytes copied into shared memory per tile.  -1 if the shape is not supported. */
int danet_conv_tc_geometry(const danet_conv_desc* d, int64_t* out);
/* Host-only geometry of the engine's CTA work unit (exact mode: a pair of tiles that share one weight stream; fast mode:
 * one tile): out[0..3] = tiles per work unit, work units, weight bytes and activation bytes copied into shared memory
 * per work unit.  -1 if the shape is not supported. */
int danet_conv_tc_cta_geometry(const danet_conv_desc* d, int64_t* out);
/* Host-only report of what the kernel will do with one problem, from the engine's own make_prob, pairing and K segment
 * close rule (for tests that must know which tile body, swizzle, tap grouping, stacking and pairing form a shape runs):
 *   out[0..2]   N tile width NT (the compiled tile body), N tiles, output channels in the last N tile
 *   out[3..6]   swizzle bytes per pixel row, channels per chunk, chunks, K steps (16 channels) of the last chunk
 *   out[7..10]  parity planes, filter taps of the largest plane, taps per weight block TG, weight blocks of that plane
 *   out[11..14] images stacked per tile, tile rows per stacked image hs (16 without stacking), tile rows and tile
 *               columns of a map
 *   out[15]     weight blocks per (weight set, N tile)
 *   out[16..19] exact mode, per tile: K segment closes, main-chain MMAs of the longest segment, closes at the end of a
 *               parity plane other than the tile's last block, closes inside a parity plane (fast mode: 0)
 *   out[20..22] exact mode: pairing kind (1 = tile rows 2q, 2q + 1; 2 = image groups of one weight set; fast mode 0),
 *               tile pairs, pairs whose second tile lies past the map (it computes zeros and stores nothing)
 * -1 if the shape is not supported. */
#define DANET_CONV_DISPATCH_FIELDS 23
int danet_conv_tc_dispatch(const danet_conv_desc* d, int64_t* out);
/* fp32 -> split-fp16 planes (lo may be NULL) and back (lo may be NULL); n elements */
int danet_act_split(int64_t n, const float* x, void* hi, void* lo, danet_stream_t stream);
int danet_act_merge(int64_t n, const void* hi, const void* lo, float* y, danet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Convolution backward (csrc/conv_wgrad.cu), exact mode: the gradients of torch.nn.functional.conv2d for the shapes the
 * tensor-core path accepts (k in {1,3,7}, pad k/2, stride 1|2, groups = wsets over the (batch, group)-flattened image
 * axis).  Weights use the layout of nn.Conv2d.weight: w [wsets*cout][cin][k][k], where cout / cin are the real
 * per-group channel counts and Cout / Cin >= them the multiples of 8 of the activation planes.  No float atomics: every
 * result repeats bit for bit.  No host synchronisation: capturable in a CUDA graph.
 * ------------------------------------------------------------------------------------------ */
/* forward weights in the SIMT layout [wsets][k*k*Cin][Cout] that danet_conv_tc_pack takes */
int danet_conv_weights_simt(int32_t wsets, int32_t cout, int32_t cin, int32_t ksize, int32_t Cout, int32_t Cin,
                            const float* w, float* w_simt, danet_stream_t stream);
/* Input gradient.  Output-parity class (a, b) of dx (rows a mod stride, columns b mod stride) is a stride-1
 * correlation of dy with the taps of w of that parity.  It is computed as one or more PIECES, each a 1x1 or 3x3
 * stride-1 forward problem of the engine (input channels Cout, output channels Cin, padding K/2) whose output map at
 * [u + tr][v + tc] adds to dx[stride*u + a][stride*v + b].  Taps jr0..jr1 / jc0..jc1 (tap r = r0 + stride*j of the
 * class's parity) are the piece's.  Stride 1 has one piece: the filter rotated by 180 degrees.  7x7/s2: nine 3x3 pieces
 * (81 taps executed for 49); 3x3/s2: four (28 for 9); 1x1/s2: one. */
typedef struct { int32_t a, b, K, tr, tc, jr0, jr1, jc0, jc1; } danet_dgrad_piece;
/* fills pieces[<= 9]; returns their number, or -1 for an unsupported ksize / stride (7x7 needs stride 2) */
int32_t danet_conv_dgrad_pieces(int32_t ksize, int32_t stride, danet_dgrad_piece* pieces);
/* the piece's kernel in the SIMT layout of its problem: w_out [wsets][K*K*Cout][Cin] */
int danet_conv_dgrad_weights(int32_t wsets, int32_t cout, int32_t cin, int32_t ksize, int32_t stride,
                             const danet_dgrad_piece* piece, int32_t Cout, int32_t Cin, const float* w, float* w_out,
                             danet_stream_t stream);
/* interleave / crop / sum: y NCHW [N,C,H,W] (fp32) with y[n][c][h][w] = sum in piece order over the pieces of class
 * (h % stride, w % stride) of maps[i] at [n][h / stride + tr][w / stride + tc][c] (0 outside), times scale[1] when
 * scale (device) is not NULL, plus bias[(n % groups) * C + c] when bias (device, [groups][C]) is not NULL.  maps is a
 * HOST array of npieces device pointers, each NHWC fp32 [N,Hc,Wc,Cp].  With stride 1 and the piece {0} it is the
 * NHWC -> NCHW conversion (the forward's epilogue: the x scale removed, then the bias added). */
int danet_conv_dgrad_scatter(int32_t N, int32_t C, int32_t H, int32_t W, int32_t Cp, int32_t stride, int32_t Hc, int32_t Wc,
                             int32_t npieces, const danet_dgrad_piece* pieces, const float* const* maps,
                             const float* scale, const float* bias, int32_t groups, float* y, danet_stream_t stream);
/* v NCHW [N,C,HW] fp32 (dy, or the forward's x) -> split-fp16 NHWC planes [N,HW,Cp] (Cp % 8 == 0, pad channels 0) of
 * v * 2^s, where the power of two 2^s brings max finite |v| into [2^13, 2^14) (1 when there is none; s is clamped to
 * [-126, 126]): values far from 1 keep their 22 bits.  NaN and +-inf stay non-finite in the planes.
 * scale: device float[3]; receives scale[0] = 2^s, scale[1] = 2^-s (scale[2] is scratch).  No host synchronisation. */
int danet_conv_grad_split(int32_t N, int32_t C, int32_t HW, int32_t Cp, const float* dy, void* hi, void* lo, float* scale,
                          danet_stream_t stream);
/* Weight gradient of the forward problem d (flags ignored; N % wsets == 0): x [N,H,W,Cin] and dy [N,Ho,Wo,Cout] as hi +
 * lo split-fp16 planes; dy_scale / x_scale = the scales danet_conv_grad_split wrote for dy / x (or NULL: unscaled).  dW
 * [wsets*cout][cin][k][k] from a wgmma implicit GEMM over the pixels in split-fp16 exact arithmetic; split K over pixel
 * chunks, partials in the workspace (16-byte aligned), chunks added in a fixed order in double, both scales removed
 * exactly (one after the other, in double). */
int64_t danet_conv_wgrad_workspace_bytes(const danet_conv_desc* d);
int danet_conv_wgrad(const danet_conv_desc* d, int32_t cout, int32_t cin, const danet_act* x, const danet_act* dy,
                     const float* dy_scale, const float* x_scale, float* dW, void* workspace, danet_stream_t stream);
/* Bias gradient: db[c] = sum over n and the HW pixels of the fp32 NCHW dy [N,C,HW]; image chunks summed in double with
 * a fixed order, then added in chunk order.  Workspace 8-byte aligned. */
int64_t danet_conv_bias_grad_workspace_bytes(int32_t N, int32_t C, int32_t HW);
int danet_conv_bias_grad(int32_t N, int32_t C, int32_t HW, const float* dy, float* db, void* workspace, danet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training layers of the regressor's ResNet blocks (csrc/bn_train.cu), fp32 NCHW: BatchNorm2d with batch or running
 * statistics (res_module.py:33-36,406,433,520; smpl_regressor.py:434,496) fused with the residual add and ReLU of
 * BasicBlock.forward (res_module.py:40-56) and the stems (smpl_regressor.py:432-436,494-499, res_module.py:445-447),
 * and nn.MaxPool2d(3, 2, 1) (res_module.py:408,448), each with its backward.  No float atomics: every result repeats bit
 * for bit.  No host synchronisation: capturable in a CUDA graph.
 * ------------------------------------------------------------------------------------------ */
/* Workspace of danet_bn2d_forward / danet_bn2d_backward (16-byte aligned; 0 for unsupported sizes): the per-channel
 * partial sums [2][nchunk][C] (double, rounded up to 256 bytes) + [C][8] floats of coefficients, where nchunk =
 * ceil(N / ipc) image chunks of ipc = max(1, 16384 / HW) images. */
int64_t danet_bn2d_workspace_bytes(int32_t N, int32_t C, int32_t HW);
/* y = relu?(bn(x) + residual?) over x [N,C,HW] with F.batch_norm's semantics.  training = 1: the biased batch variance
 * normalises; new_running [2][C] (may be NULL) receives (1 - momentum) * running + momentum * (batch mean | unbiased
 * batch variance); the caller copies it into its buffers.  training = 0: running_mean / running_var normalise.
 * save [2][C] (double) receives the mean and invstd used, for the backward.  residual may be NULL.  Training needs
 * N * HW > 1. */
int danet_bn2d_forward(int32_t N, int32_t C, int32_t HW, const float* x, const float* weight, const float* bias,
                       const float* running_mean, const float* running_var, int32_t training, float momentum, float eps,
                       const float* residual, int32_t relu, float* y, double* save, float* new_running, void* workspace,
                       danet_stream_t stream);
/* Backward of the forward above (same sizes, x, save, training and relu; y = its output, needed when relu = 1):
 * dz = dy (0 where y <= 0 with relu); dresidual = dz; dbias = sum dz; dweight = invstd * sum dz (x - mean); dx = w invstd
 * (dz - sum dz / n - xhat sum dz xhat / n) in training mode, w invstd dz in eval mode.  Each output may be NULL, and
 * only the non-NULL ones are computed. */
int danet_bn2d_backward(int32_t N, int32_t C, int32_t HW, const float* x, const float* y, const float* dy,
                        const float* weight, const double* save, int32_t training, int32_t relu, float* dx, float* dweight,
                        float* dbias, float* dresidual, void* workspace, danet_stream_t stream);
/* nn.MaxPool2d(3, 2, 1) (res_module.py:408,448) NCHW x [N,C,H,W] -> y [N,C,Ho,Wo], Ho = (H - 1) / 2 + 1, and per output
 * the row-major slot (0..8) in its 3x3 window of the maximum taken: the first maximum, NaN over numbers (torch's
 * choice); padding is never taken. */
int danet_maxpool3x3s2_nchw_forward(int32_t N, int32_t C, int32_t H, int32_t W, const float* x, float* y, uint8_t* slot,
                                    danet_stream_t stream);
/* dx [N,C,H,W]: each input pixel sums, in row-major window order, dy of the windows whose slot chose it. */
int danet_maxpool3x3s2_nchw_backward(int32_t N, int32_t C, int32_t H, int32_t W, const float* dy, const uint8_t* slot,
                                     float* dx, danet_stream_t stream);
/* Backward of nn.AdaptiveAvgPool2d(1) over NC planes of HW pixels (the forward is danet_global_avgpool on the fp32 view
 * [NC, HW, 1]): dx [NC][HW] = dy [NC] / HW. */
int danet_global_avgpool_backward(int32_t NC, int32_t HW, const float* dy, float* dx, danet_stream_t stream);
/* Backward of danet_linear (y = x W^T + b + add; add is not differentiated): x [N][In], w [Out][In], dy [N][Out] ->
 * dx = dy W [N][In], dw = dy^T x [Out][In], db = sum_n dy [Out], each summed in double in index order.  Each output
 * may be NULL, and only the non-NULL ones are computed (dx needs w, dw needs x). */
int danet_linear_backward(int32_t N, int32_t In, int32_t Out, const float* x, const float* w, const float* dy, float* dx,
                          float* dw, float* db, danet_stream_t stream);

/* HRNet fuse (models/module/hr_module.py:161-179) in training: fp32 NCHW
 * y [N,C,H,W] = relu?(up(t_0) + up(t_1) + ...), term j [N,C,H/f_j,W/f_j] upsampled nearest by f_j in {1,2,4,8},
 * added in list order (bit-identical to the F.interpolate + add + relu chain).  terms / factors: host arrays of
 * nterms (1..4) entries; the ReLU keeps NaN.  The backward writes one term's gradient: dterm = the f x f block sums
 * of dy, 0 where y <= 0 (a NaN y passes dy; y NULL: no ReLU), row-major. */
int danet_hr_fuse_forward(int32_t N, int32_t C, int32_t H, int32_t W, int32_t nterms, const float* const* terms,
                          const int32_t* factors, int32_t relu, float* y, danet_stream_t stream);
int danet_hr_fuse_backward(int32_t N, int32_t C, int32_t H, int32_t W, int32_t factor, const float* dy, const float* y,
                           float* dterm, danet_stream_t stream);

/* STN part crops in training (models/danet/iuv_estimator.py:193-204): 24x F.affine_grid(theta_i, xd.size()) +
 * F.grid_sample(xd, grid) (bilinear, zeros), cat on dim 1.  xd [B,C,S,S], theta [B,24,2,3] with zero off-diagonal
 * entries (not read), crops [B,24*C,S,S], all fp32 NCHW.  The backward is the exact adjoint of the forward w.r.t. xd,
 * a gather summed in double. */
int danet_part_crops_forward(int32_t B, int32_t C, int32_t S, const float* xd, const float* theta, int32_t align_corners,
                             float* crops, danet_stream_t stream);
int danet_part_crops_backward(int32_t B, int32_t C, int32_t S, const float* dcrops, const float* theta,
                              int32_t align_corners, float* dxd, danet_stream_t stream);
/* Training-mode thetas (iuv_estimator.py:137-140,172-191,262-301): soft-argmax centres of 10 * hm [B,24,Sh,Sh], the
 * centre jitter center_jitter * (center_noise [B,24,2] - 0.5), part visibility (bilinear sample of
 * 1[argmax index_pred [B,25,Si,Si] in the part's set] < vis_score; off when vis_score <= 0) and affine_para with the
 * scale jitters scale_jitter * (scale_noise [24,2,B] - 0.5).  NULL noise: no jitter.  centers [B,24,2] (jittered),
 * theta [B,24,2,3] = [[s, 0, cx], [0, s, cy]]. */
int danet_part_thetas(int32_t B, int32_t Sh, int32_t Si, const float* hm, const float* index_pred,
                      const float* learned_ratio, const float* learned_offset, float vis_score, const float* center_noise,
                      float center_jitter, const float* scale_noise, float scale_jitter, int32_t align_corners,
                      float* centers, float* theta, danet_stream_t stream);

/* nn.AdaptiveAvgPool2d(1) NHWC [N,H,W,C] -> [N,C] */
int danet_global_avgpool(int32_t N, int32_t HW, int32_t C, const danet_act* x, float* y, danet_stream_t stream);
/* y[n,o] = sum_i x[n,i] w[o,i] + b[o] (+ add[o])  (SmplResNet.final_layer + mean_cam_shape) */
int danet_linear(int32_t N, int32_t In, int32_t Out, const float* x, const float* w, const float* b,
                 const float* add, float* y, danet_stream_t stream);

/* utils/iuvmap.py:6-38 with the reference's own signature: NCHW maps U,V,Index [B,C,HW] and
 * optional AnnIndex [B,Ca,HW] (NULL to skip) -> cleaned maps of the same shapes */
int danet_iuvmap_clean_nchw(int32_t B, int32_t C, int32_t Ca, int32_t HW, const float* U, const float* V,
                            const float* I, const float* A, float* oU, float* oV, float* oI, float* oA,
                            danet_stream_t stream);
/* ------------------------------------------------------------------------------------------
 * Regressor head, training path (csrc/gcn_train.cu): the same head as the network program's, with raw (unfolded)
 * parameters, BatchNorm1d(24) on batch statistics (training = 1) or on the running statistics (training = 0), the
 * intermediate supervision heads of training mode and the backward.  fp32 throughout; no float atomics, every
 * reduction in a fixed order (bit-repeatable), no host synchronisation (capturable in a CUDA graph).
 * Layer l = 0..4: r2p_gcn.gc.0 [128->128], refine_gcn.gc.0..2 [128->256->256->128], p2r_gcn.gc.0 [128->128];
 * W[l] [in,out] and b[l] [out] of GraphConv, bn_weight / bn_bias / running_mean / running_var [24] of act.<i>.0.
 * Graph buffers [24*24]: r2p_A, p2r_A, I_n, A_mask; edge_importance [24*24] (a parameter).
 * pose_w[k] [24*6][128], pose_b[k] [144] = pose_regressors.<k>.1; coord_w[k] [24*3][128], coord_b[k] [72] =
 * coord_regressors.<k>.1; mean_pose [144].  The g* pointers receive the gradients (written, not accumulated); the
 * pose_regressors.0 / coord_regressors gradients only in training mode (they may be NULL otherwise).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const float* W[5]; const float* b[5]; const float* bn_weight[5]; const float* bn_bias[5];
    const float* running_mean[5]; const float* running_var[5];
    const float* r2p_A; const float* p2r_A; const float* I_n; const float* A_mask; const float* edge_importance;
    const float* pose_w[2]; const float* pose_b[2]; const float* coord_w[2]; const float* coord_b[2];
    const float* mean_pose;
    float* gW[5]; float* gb[5]; float* g_bn_weight[5]; float* g_bn_bias[5];
    float* g_edge_importance;
    float* g_pose_w[2]; float* g_pose_b[2]; float* g_coord_w[2]; float* g_coord_b[2];
} danet_gcn_train_params;
/* Bytes of the workspace one forward + backward pair shares (saved activations and backward intermediates); 0 outside
 * 1 <= B <= 174760, the batch sizes the entries accept (cdiv(24 B, 64) gemm row blocks fit a grid's y dimension). */
int64_t danet_gcn_head_train_workspace_bytes(int32_t B);
/* smpl_regressor.py:849-895 + GCN.py:29-92 + graph.py:232-261 (normalize_undigraph of I_n + A_mask * relu(E), on the
 * device) + geometry.py rot6d_to_rotmat: rot_feats [B,24,128], global_para [B,13] -> para [B,229]; in training mode
 * also pose0 [B,216] (:849-856), coord0 / coord1 [B,24,3] (:863-882) and, when new_stats is not NULL, the updated
 * running statistics new_stats [2][5][24] (mean | unbiased variance, momentum 0.1) -- the caller copies them into
 * its buffers.  The workspace (16-byte aligned) keeps what the backward needs; pass the same one to it. */
int danet_gcn_head_train_forward(int32_t B, const danet_gcn_train_params* p, int32_t training, const float* rot_feats,
                                 const float* global_para, float* para, float* pose0, float* coord0, float* coord1,
                                 float* new_stats, void* workspace, danet_stream_t stream);
/* Backward of the forward above (same B, p, training, rot_feats, workspace): g_para [B,229] and, in training mode,
 * g_pose0 [B,216], g_coord0 / g_coord1 [B,24,3] -> g_rot_feats [B,24,128], g_global_para [B,13] and every g* of p. */
int danet_gcn_head_train_backward(int32_t B, const danet_gcn_train_params* p, int32_t training, const float* rot_feats,
                                  const float* g_para, const float* g_pose0, const float* g_coord0, const float* g_coord1,
                                  float* g_rot_feats, float* g_global_para, void* workspace, danet_stream_t stream);
/* smpl_regressor.py:147-166,233-238: losses [3] = joint_rotation0 = rot_w * MSE(pose0, target[:,13:]) over the
 * selected images, joint_position0/1 = pos_w * sum |coord - gt_joints| / #selected; has [B] (1 = selected).  With no
 * image selected the losses and gradients are 0.  g_pose0 / g_coord0 / g_coord1 receive d(loss k)/d(input k). */
int danet_gcn_head_losses(int32_t B, const float* pose0, const float* coord0, const float* coord1, const float* target,
                          const float* gt_joints, const uint8_t* has, float rot_w, float pos_w, float* losses,
                          float* g_pose0, float* g_coord0, float* g_coord1, danet_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Whole-network entry (csrc/net.cu).  Replaces the network half of DaNet.infer_net
 * (models/danet/danet.py:78-98: img2iuv -> iuvmap_clean -> iuv2smpl, up to `para`) for hosts without Python.
 * A "network program" is what danet_b200.plan.Plan.export() writes for ONE batch size: the launch steps (each one
 * kernel launch, with its arguments), the activation buffer table and the BN-folded, packed weights.  Loading
 * allocates everything on the CURRENT device; infer replays the steps (optionally as one CUDA graph, captured on the
 * first call).  danet_net_run_step runs one step record directly; the Python plan launches every kernel through it, so
 * it and a loaded program decode the same records with the same code.  A danet_net_t owns its buffers: one infer at a
 * time per handle (load one handle per host thread / stream that runs concurrently).  Outputs stay in the program's
 * buffers until the next infer:
 *   "para" [B,229] f32 (cam 3 | shape 10 | 24 rotation matrices, danet.py:118), "centers" [B,24,2] (stn_kps_pred),
 *   "theta", "global_para", "rot_feats", "heads", "hm", "body_iuv", "amax" (u8 [B,S,S]) and, when the plan kept the
 *   visualisation maps, "vis_u" / "vis_v" / "vis_i" [B,25,S,S], "vis_a" [B,15,S,S], "part_iuv_raw" [B*24,21,S,S].
 * ------------------------------------------------------------------------------------------ */
typedef struct danet_net* danet_net_t;
#define DANET_NET_GRAPH 1              /* flags: replay as a CUDA graph (a NULL stream is served by an internal blocking stream) */
int danet_net_load(const void* program, uint64_t bytes, danet_net_t* out);         /* program: HOST memory */
int danet_net_load_file(const char* path, danet_net_t* out);
int danet_net_destroy(danet_net_t net);
/* batch size, input [C,H,W], number of outputs, number of launch steps (any pointer may be NULL) */
int danet_net_info(danet_net_t net, int32_t* batch, int32_t* chw, int32_t* n_outputs, int32_t* n_steps);
const char* danet_net_output_name(danet_net_t net, int32_t index);                  /* NULL past the end */
/* device pointer / byte size / dims[4] / element size of a named output */
int danet_net_output(danet_net_t net, const char* name, void** dev_ptr, uint64_t* bytes, int32_t* dims,
                     int32_t* elem_bytes);
/* images: fp32 NCHW [B,C,H,W], device (or pinned host) memory; asynchronous on `stream` */
int danet_net_infer(danet_net_t net, const float* images, int32_t flags, danet_stream_t stream);
/* convenience for hosts that do not touch CUDA: pageable host images -> H2D -> steps -> synchronise (own stream) */
int danet_net_infer_host(danet_net_t net, const float* images_host, int32_t flags);
/* synchronous device -> host copy of a named output; `bytes` must equal the output's size */
int danet_net_read_output(danet_net_t net, const char* name, void* host_dst, uint64_t bytes);
/* one step of the program format (opcode, ints, floats and n_p raw pointers where a program has references; a danet_act
 * is three pointers f32, hi, lo), checked and run on the current device exactly as danet_net_infer runs it */
int danet_net_run_step(uint32_t op, int32_t n_i, const int32_t* i, int32_t n_f, const float* f, int32_t n_p,
                       void* const* p, danet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif
