"""fp64 numpy restatement of the training targets (danet_b200.targets.prepare_targets) -- TEST INFRASTRUCTURE.

Restates train/trainer.py:157-212, models/danet/danet.py:159-165 and smpl_regressor.py:158-162 with
utils/geometry.py:94-157 (estimate_translation).  Arithmetic is fp64; values are rounded to fp32 where the reference
stores them in fp32 (the translation's `trans` array, the de-normalised key points, the SMPL outputs of the device), so
that the stages can be compared one at a time.  The one deliberate difference from the reference: a singular
translation system (numpy's LinAlgError) gives a NaN row.
"""
import numpy as np

from . import lbs as olbs


def _system(S, joints_2d, focal_length=5000., img_size=224.):
    """Per image, Q [48,3] and c [48] of utils/geometry.py:115-128 (weights already applied), fp64."""
    S = np.asarray(S, np.float32)[:, 25:].astype(np.float64)
    kp = np.asarray(joints_2d, np.float32)[:, 25:]
    w = np.sqrt(kp[..., 2]).astype(np.float64)                  # np.sqrt of the float32 confidences: fp32-rounded
    xy = kp[..., :2].astype(np.float64)
    B, J = S.shape[0], S.shape[1]
    F, O = float(focal_length), float(img_size) / 2.
    Q = np.zeros((B, J, 2, 3))
    Q[:, :, 0, 0] = F
    Q[:, :, 1, 1] = F
    Q[:, :, :, 2] = O - xy
    c = (xy - O) * S[..., 2:3] - F * S[..., :2]
    Q = Q * w[:, :, None, None]
    c = c * w[:, :, None]
    return Q.reshape(B, 2 * J, 3), c.reshape(B, 2 * J)


def estimate_translation(S, joints_2d, focal_length=5000., img_size=224.):
    """[B,3] fp64 solutions of the normal equations (NaN where singular); the reference rounds them to fp32."""
    Q, c = _system(S, joints_2d, focal_length, img_size)
    out = np.full((Q.shape[0], 3), np.nan)
    for b in range(Q.shape[0]):
        A, r = Q[b].T @ Q[b], Q[b].T @ c[b]
        try:
            out[b] = np.linalg.solve(A, r)
        except np.linalg.LinAlgError:
            pass
    return out


def translation_bound(S, joints_2d, ref, focal_length=5000., img_size=224., depth=40):
    """Componentwise bound on |got - ref| for a device translation `got` (fp32) and a reference solution `ref` (fp64)
    of the same system: 2^-24 |ref| for the final rounding, plus |A^-1| (g |Q|^T |Q| |ref| + g |Q|^T |c|), the
    first-order effect of perturbing A and b by their rounding errors, with g = 2 gamma_depth (u = 2^-53): both the
    device's sums (lane pair + a 5-level tree, the products that form Q and c, the 3x3 LU) and numpy's have errors of
    that form, and depth covers the longest chain of either."""
    Q, c = _system(S, joints_2d, focal_length, img_size)
    u = 2.0 ** -53
    g = 2 * depth * u / (1 - depth * u)
    out = np.full(ref.shape, np.inf)
    for b in range(Q.shape[0]):
        A = Q[b].T @ Q[b]
        try:
            Ai = np.abs(np.linalg.inv(A))
        except np.linalg.LinAlgError:
            continue
        aQ = np.abs(Q[b])
        pert = g * (aQ.T @ aQ) @ np.abs(ref[b]) + g * aQ.T @ np.abs(c[b])
        out[b] = 2.0 ** -24 * np.abs(ref[b]) + Ai @ pert
    return out


def fit_merge(opt_pose, opt_betas, gt_pose, gt_betas, has_smpl, iuv_annotated, fit_valid=None):
    """trainer.py:157-161 (clamp, then merge) and :177-191 (valid_fit, has_iuv)."""
    pose = np.array(opt_pose, np.float32, copy=True)
    betas = np.array(opt_betas, np.float32, copy=True)
    betas[(np.abs(betas) > 3).any(-1)] = 0.                   # NaN is not > 3
    hs = np.asarray(has_smpl).astype(bool)
    pose[hs] = np.asarray(gt_pose, np.float32)[hs]
    betas[hs] = np.asarray(gt_betas, np.float32)[hs]
    valid = hs if fit_valid is None else (hs | np.asarray(fit_valid).astype(bool))
    has_iuv = np.asarray(iuv_annotated).astype(bool) & valid
    return pose, betas, valid.astype(np.uint8), has_iuv.astype(np.uint8)


def denormalise(keypoints, img_res=224):
    """trainer.py:167-169 in fp32: 0.5 * img_res * (k + 1) on x, y; the confidence is kept."""
    kp = np.array(keypoints, np.float32, copy=True)
    kp[..., :2] = np.float32(0.5 * img_res) * (kp[..., :2] + np.float32(1))
    return kp


def cam_targets(opt_joints, smpl_joints, keypoints, opt_pose, opt_betas, has_iuv, has_dp, smpl_2dkps,
                focal_length=5000., img_res=224, cam_t=None):
    """trainer.py:166-212 and danet.py:159-162 after the SMPL forward of the merged fits: opt_cam_t (fp32-rounded),
    target_smpl_kps, target_cam and target, fp64.  `cam_t` replaces the translation (to check the later stages on a
    device's translation)."""
    B = opt_joints.shape[0]
    t = estimate_translation(opt_joints, denormalise(keypoints, img_res), focal_length, img_res).astype(np.float32)
    tt = (t if cam_t is None else np.asarray(cam_t, np.float32)).astype(np.float64)
    eye = np.broadcast_to(np.eye(3), (B, 3, 3))
    ctr = np.full((B, 2), 0.5 * img_res)
    kps = np.zeros((B, 24, 3))
    kps[:, :, :2] = olbs.perspective_projection(np.asarray(smpl_joints, np.float64), eye, tt, focal_length, ctr)
    kps[:, :, :2] = kps[:, :, :2] / (0.5 * img_res) - 1
    kps[np.asarray(has_iuv) == 1, :, 2] = 1
    dp = np.asarray(has_dp) == 1
    kps[dp] = np.asarray(smpl_2dkps, np.float64)[dp]
    cam = np.zeros((B, 3))
    cam[:, 1:] = tt[:, :2]
    cam[:, 0] = (2. * focal_length / img_res) / tt[:, 2]
    rot = olbs.batch_rodrigues_quat(np.asarray(opt_pose, np.float64).reshape(-1, 3)).reshape(B, 216)
    target = np.concatenate([cam, np.asarray(opt_betas, np.float64), rot], 1)
    return {"opt_cam_t": t, "target_smpl_kps": kps, "target_cam": cam, "target": target}


def prepare_targets(model, batch, opt_pose, opt_betas, fit_valid=None, focal_length=5000., img_res=224):
    """The whole preparation on numpy inputs (the render excepted: oracle/raster.py renders target_verts with
    target_cam for the has_iuv images).  SMPL outputs are rounded to fp32, as the device stores them."""
    pose, betas, valid, has_iuv = fit_merge(opt_pose, opt_betas, batch["pose"], batch["betas"], batch["has_smpl"],
                                            batch["iuv_annotated"], fit_valid)
    o = olbs.smpl_forward(model, betas, pose[:, 3:], pose[:, :3], pose2rot=True, dtype=np.float64)
    f32 = lambda a: np.asarray(a, np.float32)
    out = {"opt_pose": pose, "opt_betas": betas, "valid_fit": valid, "has_iuv": has_iuv,
           "target_verts": f32(o["vertices"]), "opt_joints": f32(o["joints"])}
    out.update(cam_targets(out["opt_joints"], f32(o["smpl_joints"]), batch["keypoints"], pose, betas, has_iuv,
                           batch["has_dp"], batch["smpl_2dkps"], focal_length, img_res))
    R = out["target"][:, 13:].reshape(-1, 24, 3, 3)
    out["target_smpl_joints"] = olbs.smpl_forward(model, out["target"][:, 3:13], R[:, 1:], R[:, :1], pose2rot=False,
                                                  dtype=np.float64)["smpl_joints"]
    return out
