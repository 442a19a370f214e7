"""The training step's target preparation on the GPU: train/trainer.py:157-212 and models/danet/danet.py:159-165, with
models/danet/smpl_regressor.py:158-162's target joints, as five launches and no host synchronisation, so that the whole
preparation can be captured in one CUDA graph.

    targets = prepare_targets(model, batch, opt_pose, opt_betas)
    input_batch.update(targets)

The reference leaves the GPU here: estimate_translation copies the joints to the host and solves one numpy problem per
image, and the boolean-mask merges and `torch.sum(has_iuv) > 0` synchronise.  Here:
  1. k_fit_merge (csrc/targets.cu): beta clamp, ground-truth merge, valid_fit, has_iuv;
  2. the SMPL forward of the merged fits (axis-angle input, the smplx Rodrigues);
  3. k_train_targets: opt_cam_t (geometry.estimate_translation's arithmetic), target_cam, target_smpl_kps, `target`;
  4. the SMPL forward of `target` (rotation matrices) for target_smpl_joints;
  5. the IUV render of target_verts with target_cam, only for the has_iuv images (the others are the zero image).
"""
import torch

from . import _args, _lib

WHERE = "danet_b200.targets.prepare_targets"
_SHAPES = {"keypoints": (49, 3), "pose": (72,), "betas": (10,), "smpl_2dkps": (24, 3)}
_FLAGS = ("has_smpl", "has_dp", "iuv_annotated")


def _check(model, batch, opt_pose, opt_betas, fit_valid, focal_length, img_res):
    smpl = getattr(getattr(model, "iuv2smpl", None), "smpl", None)
    renderer = getattr(model, "iuv_renderer", None)
    if smpl is None or renderer is None:
        raise ValueError("%s: model must have iuv2smpl.smpl and iuv_renderer (a danet_b200.DaNet)" % WHERE)
    if not isinstance(batch, dict):
        raise ValueError("%s: batch must be a dict (got %s)" % (WHERE, type(batch).__name__))
    for k in tuple(_SHAPES) + _FLAGS:
        if k not in batch:
            raise ValueError("%s: batch must have the key %r" % (WHERE, k))
    _args.tensor(WHERE, "batch['keypoints']", batch["keypoints"], dim=3)
    B = batch["keypoints"].shape[0]
    for k, shape in _SHAPES.items():
        _args.tensor(WHERE, "batch[%r]" % k, batch[k], shape=(B,) + shape)
    for k in _FLAGS:
        _args.mask(WHERE, "batch[%r]" % k, batch[k], (B,))
    _args.tensor(WHERE, "opt_pose", opt_pose, shape=(B, 72))
    _args.tensor(WHERE, "opt_betas", opt_betas, shape=(B, 10))
    if fit_valid is not None:
        _args.mask(WHERE, "fit_valid", fit_valid, (B,))
    f = _args.number(WHERE, "focal_length", focal_length)
    if isinstance(img_res, bool) or not isinstance(img_res, int) or img_res <= 0:
        raise ValueError("%s: img_res must be a positive int (got %r)" % (WHERE, img_res))
    if smpl.shapedirs.shape[-1] != 10:
        raise ValueError("%s: the SMPL model must have 10 betas (got %d)" % (WHERE, smpl.shapedirs.shape[-1]))
    if smpl.v_template.device.type != "cuda":
        raise ValueError("%s: move the model to a CUDA device (there is no CPU path)" % WHERE)
    named = [("batch[%r]" % k, batch[k]) for k in tuple(_SHAPES) + _FLAGS] + [("opt_pose", opt_pose), ("opt_betas", opt_betas)]
    if fit_valid is not None:
        named.append(("fit_valid", fit_valid))
    _args.cuda(WHERE, named, smpl.v_template.device)
    return smpl, renderer, B, f


def _u8(t):
    return t if t is None or t.dtype == torch.uint8 else t.to(torch.uint8)


@torch.no_grad()
def prepare_targets(model, batch, opt_pose, opt_betas, *, fit_valid=None, focal_length=5000., img_res=224):
    """The targets of one training step from a data batch and the SPIN fits the caller looked up.

    batch (the reference's input_batch keys): keypoints [B,49,3] (x, y in [-1,1], confidence), pose [B,72], betas [B,10],
    has_smpl, has_dp, iuv_annotated [B] (bool or uint8; iuv_annotated = dataset_name not in ['dp_coco'], trainer.py:190),
    smpl_2dkps [B,24,3].  opt_pose [B,72] / opt_betas [B,10]: the fits.  fit_valid [B]: the fits' valid state (the
    h36m_coco_itw branch of trainer.py:177-181), or None.  Every tensor is float32 (flags bool / uint8), contiguous and
    on the model's device.

    Returns a dict: opt_pose, opt_betas (merged), valid_fit, has_iuv (uint8 0 / 1), target_verts [B,V,3], opt_joints
    [B,49,3], opt_cam_t [B,3], target_smpl_kps [B,24,3], target_cam [B,3], target [B,229] (cam | betas | 24 rotation
    matrices, what smpl_losses and gcn_head_losses take), target_smpl_joints [B,24,3] (gcn_head_losses' gt_smpl_joints),
    uv_image_gt [B,3,S,S] and uvia_list [U, V, I, Ann] (iuv_img2map of uv_image_gt).

    opt_cam_t follows geometry.estimate_translation, so an image whose translation is singular (every key-point
    confidence 0) has a NaN opt_cam_t, target_cam and key points where the reference would raise; such an image is not
    rendered unless it has has_iuv.  The reference's gt_out / gt_cam_t (trainer.py:148-150,173) feed nothing the step
    consumes and are not computed."""
    smpl, renderer, B, f = _check(model, batch, opt_pose, opt_betas, fit_valid, focal_length, img_res)
    dev = smpl.v_template.device
    V = smpl.v_template.shape[0]
    S = renderer.out_size
    z = lambda *shape, dtype=torch.float32: torch.empty(*shape, dtype=dtype, device=dev)
    out = {"opt_pose": z(B, 72), "opt_betas": z(B, 10), "valid_fit": z(B, dtype=torch.uint8),
           "has_iuv": z(B, dtype=torch.uint8), "target_verts": z(B, V, 3), "opt_joints": z(B, len(smpl.joint_map), 3),
           "opt_cam_t": z(B, 3), "target_smpl_kps": z(B, 24, 3), "target_cam": z(B, 3), "target": z(B, 229),
           "target_smpl_joints": z(B, 24, 3)}
    if B == 0:                                       # empty batch: empty outputs, nothing to launch
        out["uv_image_gt"] = z(0, 3, S, S)
        out["uvia_list"] = [z(0, c, S, S) for c in (25, 25, 25, 15)]
        return out
    has_smpl, has_dp, annotated, fv = (_u8(t) for t in (batch["has_smpl"], batch["has_dp"], batch["iuv_annotated"], fit_valid))
    P = _lib.ptr
    with torch.cuda.device(dev):
        # 1. trainer.py:157-161, 177-191
        _lib.call("fit_merge", B, P(opt_pose), P(opt_betas), P(batch["pose"]), P(batch["betas"]), P(has_smpl), P(fv),
                  P(annotated), P(out["opt_pose"]), P(out["opt_betas"]), P(out["valid_fit"]), P(out["has_iuv"]))
        # 2. trainer.py:163-165: SMPL of the merged fits, axis-angle input (pose2rot=True)
        h = smpl._handle(dev)
        ws = smpl._workspace(h, B, dev)
        opt_smpl_joints = z(B, 24, 3)
        _lib.call("smpl_forward", h, B, P(out["opt_betas"]), P(out["opt_pose"]), 1, P(out["target_verts"]),
                  P(out["opt_joints"]), P(opt_smpl_joints), None, None, P(ws), 0)
        # 3. trainer.py:166-212, danet.py:159-162
        _lib.call("train_targets", B, P(out["opt_joints"]), P(opt_smpl_joints), P(batch["keypoints"]), P(out["opt_pose"]),
                  P(out["opt_betas"]), P(out["has_iuv"]), P(has_dp), P(batch["smpl_2dkps"]), f, img_res,
                  P(out["opt_cam_t"]), P(out["target_cam"]), P(out["target_smpl_kps"]), P(out["target"]))
        # 4. smpl_regressor.py:158-162: SMPL of target's betas and rotation matrices (pose2rot=False)
        rot = out["target"][:, 13:].contiguous()
        _lib.call("smpl_forward", h, B, P(out["opt_betas"]), P(rot), 0, P(z(B, V, 3)), P(z(B, len(smpl.joint_map), 3)),
                  P(out["target_smpl_joints"]), None, None, P(ws), 0)
    # 5. danet.py:163-165, 181: the has_iuv images rendered, the others the zero image; the maps of the same pass
    out["uv_image_gt"], _, out["uvia_list"] = renderer._render(out["target_verts"], out["target_cam"], want_maps=True,
                                                               select=out["has_iuv"])
    return out
