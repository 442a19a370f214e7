"""Times the training step's target preparation at B = 16 (BASELINE config 5's per-GPU batch) and B = 64:
  - gpu: danet_b200.targets.prepare_targets (five launches, no host synchronisation);
  - reference-shaped: the same SMPL and renderer of this package driven the way train/trainer.py:157-212 and
    danet.py:159-165 drive theirs: boolean-mask merges, the translation solved per image in numpy after a D2H copy
    and copied back (oracle/train_targets.py's fp64 solve, one np.linalg.solve per image), the projection and masks as
    torch ops, and the subset render behind `torch.sum(has_iuv) > 0`.
Each is timed with CUDA events around N calls and with the host clock around N calls ending in a synchronise; the
output names the device and its power limit, read in the same run.  Prints one JSON line."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import danet_b200
from danet_b200 import geometry, iuvmap
from danet_b200.targets import prepare_targets
from oracle import train_targets as ot

dev = torch.device("cuda:0")
net = danet_b200.build_synthetic_danet(width=32, seed=0, device=dev)
smpl, rend = net.iuv2smpl.smpl, net.iuv_renderer


def inputs(B, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    r = lambda *s, sc=1.0: sc * torch.randn(*s, generator=g, device=dev)
    pose = lambda: torch.cat([torch.tensor([np.pi, 0, 0], device=dev).expand(B, 3) + r(B, 3, sc=0.1), r(B, 69, sc=0.25)], 1)
    kp = torch.cat([r(B, 49, 2, sc=0.3), (torch.rand(B, 49, 1, generator=g, device=dev) > 0.2).float()], 2)
    flag = lambda: torch.rand(B, generator=g, device=dev) < 0.5
    batch = {"keypoints": kp.contiguous(), "pose": pose(), "betas": r(B, 10), "smpl_2dkps": r(B, 24, 3, sc=0.5),
             "has_smpl": flag(), "has_dp": flag().to(torch.uint8), "iuv_annotated": flag()}
    return batch, pose(), r(B, 10, sc=1.5)


def reference_shaped(batch, fit_pose, fit_betas, f=5000., res=224):
    B = fit_pose.shape[0]
    has_smpl = batch["has_smpl"]
    opt_pose, opt_betas = fit_pose.clone(), fit_betas.clone()
    opt_betas[(opt_betas.abs() > 3).any(dim=-1)] = 0.
    opt_pose[has_smpl, :] = batch["pose"][has_smpl, :]
    opt_betas[has_smpl, :] = batch["betas"][has_smpl, :]
    o = smpl(betas=opt_betas, body_pose=opt_pose[:, 3:], global_orient=opt_pose[:, :3])
    kp = batch["keypoints"].clone()
    kp[:, :, :-1] = 0.5 * res * (kp[:, :, :-1] + 1)
    cam_t = torch.from_numpy(ot.estimate_translation(o.joints.cpu().numpy(), kp.cpu().numpy(), f, res)
                             .astype(np.float32)).to(dev)
    valid_fit = has_smpl.to(torch.uint8)
    has_iuv = batch["iuv_annotated"].to(torch.uint8) & valid_fit
    kps = torch.zeros(B, 24, 3, device=dev)
    kps[:, :, :2] = geometry.perspective_projection(o.smpl_joints, torch.eye(3, device=dev).expand(B, 3, 3), cam_t, f,
                                                    torch.zeros(B, 2, device=dev) + 0.5 * res)
    kps[:, :, :2] = kps[:, :, :2] / (0.5 * res) - 1
    kps[has_iuv == 1, :, 2] = 1
    kps[batch["has_dp"] == 1] = batch["smpl_2dkps"][batch["has_dp"] == 1]
    cam = torch.zeros(B, 3, device=dev)
    cam[:, 1:] = cam_t[:, :2]
    cam[:, 0] = (2. * f / res) / cam_t[:, 2]
    target = torch.cat([cam, opt_betas, geometry.batch_rodrigues(opt_pose.reshape(-1, 3)).reshape(B, 216)], 1)
    Rs = target[:, 13:].reshape(B, 24, 3, 3)
    tj = smpl(betas=target[:, 3:13], body_pose=Rs[:, 1:], global_orient=Rs[:, :1], pose2rot=False).smpl_joints
    uv = torch.zeros(B, 3, rend.out_size, rend.out_size, device=dev)
    sel = has_iuv.bool()
    if torch.sum(has_iuv) > 0:
        uv[sel] = rend.verts2uvimg(o.vertices[sel], cam[sel])
    return target, tj, kps, iuvmap.iuv_img2map(uv)


def timed(fn, n):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / n
    return {"device_ms": e0.elapsed_time(e1) / n, "host_ms": wall}


res = {}
n = 1 if "one" in sys.argv else 50
for B in (16, 64):
    batch, fp, fb = inputs(B)
    res["B%d" % B] = {"gpu": timed(lambda: prepare_targets(net, batch, fp, fb), n),
                      "reference_shaped": timed(lambda: reference_shaped(batch, fp, fb), n)}
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
res["device"] = q.stdout.strip() or torch.cuda.get_device_name(0)
print(json.dumps(res))
