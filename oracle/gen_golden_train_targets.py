"""Generates tests/golden/train_targets.npz with the REFERENCE'S OWN code on the CPU:

    python -m oracle.gen_golden_train_targets

utils/geometry.py (estimate_translation, estimate_translation_np, batch_rodrigues, perspective_projection) is loaded
from the reference tree that oracle/ref_import.py finds; train/trainer.py cannot be imported (torchgeometry,
torchvision, the datasets), so its lines 157-212 and danet.py:159-162 are restated below statement by statement, each
with its line.  SMPL is oracle/lbs.py on synth.make_smpl_model(0) (smplx is absent), rounded to fp32 as the
reference's SMPL returns fp32.  Two variants of one batch: `a_` without fit_valid, `b_` with it.  Plus `et_`: direct
estimate_translation cases (partial confidences, key points at and outside the image)."""
import importlib.util
import os

import numpy as np

from . import lbs as olbs, ref_import, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
B = 8
FOCAL, IMG_RES = 5000., 224


def ref_geometry():
    spec = importlib.util.spec_from_file_location("ref_utils_geometry", os.path.join(ref_import.REF, "utils", "geometry.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_batch(model, rng):
    """Mixed flags, fit rows with |beta| > 3, a ground-truth row with |beta| > 3, partial confidences (0, 0.3)."""
    def pose(n):
        p = rng.normal(0, 0.25, (n, 72))
        p[:, :3] = [np.pi, 0, 0] + rng.normal(0, 0.1, (n, 3))         # facing the camera
        return p.astype(np.float32)
    fit_pose, gt_pose = pose(B), pose(B)
    fit_betas = rng.normal(0, 1, (B, 10)).astype(np.float32)
    gt_betas = rng.normal(0, 1, (B, 10)).astype(np.float32)
    fit_betas[1, 4] = 3.5                   # extreme fit, no ground truth: zeroed
    fit_betas[2, 0] = -4.0                  # extreme fit, ground truth replaces it
    fit_betas[5, 9] = 3.0                   # exactly 3 is not > 3: kept
    gt_betas[3, 2] = 3.7                    # ground truth above 3 survives (clamp before merge)
    has_smpl = np.array([1, 0, 1, 1, 0, 0, 1, 0], np.uint8)
    has_dp = np.array([0, 1, 0, 0, 1, 0, 0, 1], np.uint8)
    iuv_annotated = np.array([1, 1, 0, 1, 1, 1, 0, 1], np.uint8)
    fit_valid = np.array([0, 1, 0, 0, 0, 1, 1, 0], np.uint8)
    # key points: the merged body's joints projected with a per-image camera, plus noise, normalised to [-1, 1]
    sel = has_smpl.astype(bool)
    mp, mb = fit_pose.copy(), np.where((np.abs(fit_betas) > 3).any(-1, keepdims=True), 0, fit_betas)
    mp[sel], mb[sel] = gt_pose[sel], gt_betas[sel]
    J = olbs.smpl_forward(model, mb, mp[:, 3:], mp[:, :3], pose2rot=True)["joints"]
    t = np.stack([rng.uniform(-0.2, 0.2, B), rng.uniform(-0.2, 0.2, B), rng.uniform(20, 60, B)], 1)
    p = J + t[:, None]
    uv = FOCAL * p[..., :2] / p[..., 2:3] / (IMG_RES / 2.) + rng.normal(0, 0.01, (B, 49, 2))
    conf = rng.choice([1.0, 1.0, 0.3, 0.0, 0.7], (B, 49))
    conf[0, 25:] = 1.0
    conf[4, 25:45] = 0.0                    # 4 joints with weight
    keypoints = np.concatenate([uv, conf[..., None]], -1).astype(np.float32)
    smpl_2dkps = rng.uniform(-1, 1, (B, 24, 3)).astype(np.float32)
    return dict(fit_pose=fit_pose, fit_betas=fit_betas, pose=gt_pose, betas=gt_betas, has_smpl=has_smpl, has_dp=has_dp,
                iuv_annotated=iuv_annotated, fit_valid=fit_valid, keypoints=keypoints, smpl_2dkps=smpl_2dkps)


def run_reference(torch, geo, model, g, with_fit_valid):
    T = lambda k: torch.from_numpy(np.array(g[k]))
    smpl = lambda betas, body_pose, global_orient, pose2rot=True: {
        k: torch.from_numpy(v.astype(np.float32)) for k, v in olbs.smpl_forward(
            model, betas.numpy(), body_pose.numpy(), global_orient.numpy(), pose2rot=pose2rot).items()
        if k in ("vertices", "joints", "smpl_joints")}
    gt_keypoints_2d, gt_pose, gt_betas = T("keypoints"), T("pose"), T("betas")
    has_smpl = T("has_smpl").byte()                                                          # trainer.py:138
    batch_size = gt_pose.shape[0]
    opt_pose, opt_betas = T("fit_pose"), T("fit_betas")                                      # :153-155
    opt_betas[(opt_betas.abs() > 3).any(dim=-1)] = 0.                                        # :158
    opt_pose[has_smpl.bool(), :] = gt_pose[has_smpl.bool(), :]                              # :160 (uint8 mask as bool)
    opt_betas[has_smpl.bool(), :] = gt_betas[has_smpl.bool(), :]                            # :161
    opt_output = smpl(betas=opt_betas, body_pose=opt_pose[:, 3:], global_orient=opt_pose[:, :3])   # :163
    opt_vertices = opt_output["vertices"]                                                    # :164
    opt_joints = opt_output["joints"]                                                        # :165
    gt_keypoints_2d_orig = gt_keypoints_2d.clone()                                           # :168
    gt_keypoints_2d_orig[:, :, :-1] = 0.5 * IMG_RES * (gt_keypoints_2d_orig[:, :, :-1] + 1)  # :169
    opt_cam_t = geo.estimate_translation(opt_joints, gt_keypoints_2d_orig, focal_length=FOCAL, img_size=IMG_RES)  # :175
    if with_fit_valid:                                                                       # :177-181
        valid_fit = T("fit_valid").bool()
        valid_fit = valid_fit | has_smpl
    else:
        valid_fit = has_smpl
    has_iuv = T("iuv_annotated").to(torch.uint8)                                             # :190
    has_iuv = has_iuv & valid_fit                                                            # :191
    has_dp = T("has_dp")                                                                     # :193
    target_smpl_kps = torch.zeros((batch_size, 24, 3))                                       # :194
    target_smpl_kps[:, :, :2] = geo.perspective_projection(                                  # :195-199
        opt_output["smpl_joints"].detach().clone(),
        rotation=torch.eye(3).unsqueeze(0).expand(batch_size, -1, -1), translation=opt_cam_t,
        focal_length=FOCAL, camera_center=torch.zeros(batch_size, 2) + (0.5 * IMG_RES))
    target_smpl_kps[:, :, :2] = target_smpl_kps[:, :, :2] / (0.5 * IMG_RES) - 1             # :200
    target_smpl_kps[has_iuv == 1, :, 2] = 1                                                  # :201
    target_smpl_kps[has_dp == 1] = T("smpl_2dkps")[has_dp == 1]                              # :202
    gt_cam_t_nr = opt_cam_t.detach().clone()                                                 # :207
    gt_camera = torch.zeros(gt_cam_t_nr.shape)                                               # :208
    gt_camera[:, 1:] = gt_cam_t_nr[:, :2]                                                    # :209
    gt_camera[:, 0] = (2. * FOCAL / IMG_RES) / gt_cam_t_nr[:, 2]                             # :210
    gt_rotmat = geo.batch_rodrigues(opt_pose.view(-1, 3)).view(-1, 24 * 3 * 3)              # danet.py:159
    target = torch.cat([gt_camera, opt_betas, gt_rotmat], dim=1)                             # danet.py:161
    gt_Rs = target[:, 13:].contiguous().view(-1, 24, 3, 3)                                   # smpl_regressor.py:159
    target_smpl_joints = smpl(betas=target[:, 3:13], body_pose=gt_Rs[:, 1:], global_orient=gt_Rs[:, 0:1],
                              pose2rot=False)["smpl_joints"]                                 # :160-162
    del opt_vertices
    return dict(opt_pose=opt_pose, opt_betas=opt_betas, valid_fit=valid_fit.to(torch.uint8), has_iuv=has_iuv,
                opt_joints=opt_joints, smpl_joints=opt_output["smpl_joints"], opt_cam_t=opt_cam_t,
                target_smpl_kps=target_smpl_kps, target_cam=gt_camera, target=target,
                target_smpl_joints=target_smpl_joints)


def translation_cases(rng, geo):
    """Images with 24 .. 2 weighted joints, depths 5 .. 100, key points at and outside the image."""
    n = 12
    S = rng.normal(0, 0.4, (n, 49, 3)).astype(np.float32)
    t = np.stack([rng.uniform(-0.3, 0.3, n), rng.uniform(-0.3, 0.3, n), np.geomspace(5, 100, n)], 1)
    p = S.astype(np.float64) + t[:, None]
    uv = FOCAL * p[..., :2] / p[..., 2:3] + IMG_RES / 2. + rng.normal(0, 1.0, (n, 49, 2))
    uv[3] += 300.0                                                # outside the image
    conf = rng.choice([1.0, 0.3, 0.0, 0.55], (n, 49))
    for i, k in enumerate(np.linspace(24, 2, n).astype(int)):     # k joints of 25..48 keep a weight
        conf[i, 25 + k:] = 0.0
        conf[i, 25:25 + k] = np.where(conf[i, 25:25 + k] == 0.0, 0.3, conf[i, 25:25 + k])
    j2d = np.concatenate([uv, conf[..., None]], -1).astype(np.float32)
    import torch
    got = geo.estimate_translation(torch.from_numpy(S), torch.from_numpy(j2d), focal_length=FOCAL, img_size=IMG_RES)
    np64 = np.stack([geo.estimate_translation_np(S[i, 25:], j2d[i, 25:, :2], j2d[i, 25:, 2], focal_length=FOCAL,
                                                 img_size=IMG_RES) for i in range(n)])
    return {"et_S": S, "et_joints_2d": j2d, "et_trans": got.numpy(), "et_trans_np": np64}


def main():
    import torch
    if not ref_import.available():
        raise SystemExit("reference tree not present")
    geo = ref_geometry()
    model = synth.make_smpl_model(0)
    rng = np.random.default_rng(4242)
    g = make_batch(model, rng)
    out = {k: v for k, v in g.items()}
    for tag, fv in (("a_", False), ("b_", True)):
        r = run_reference(torch, geo, model, g, fv)
        out.update({tag + k: v.numpy() for k, v in r.items()})
    out.update(translation_cases(rng, geo))
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "train_targets.npz"), **out)
    print("wrote", os.path.join(GOLD, "train_targets.npz"), sorted(out))


if __name__ == "__main__":
    main()
