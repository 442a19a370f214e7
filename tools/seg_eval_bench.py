"""Times the LSP scoring step (eval.py:219-266) at B = 32 on LSP-sized original images (sides 150..640 px):
  - gpu: PartRenderer, then danet_b200.seg_eval.score_renders (host crop corners, one H2D copy of the geometry, the
    table and counting launches), ending in the D2H copy of the per-image tables;
  - reference-shaped: the same render, a D2H copy of the maps, and per image the numpy uncrop with Pillow's resize
    (oracle/seg_eval.py) and the per-class numpy comparisons of eval.py:236-266.
Both start from the same vertices and cameras, and their class counts are checked against each other first.  Each is
timed with the host clock around windows of calls that end in a synchronise (three windows, each reported).  The output
names the device and its power limit, read in the same run.  Prints one JSON line."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import danet_b200
from danet_b200 import seg_eval, synthetic
from danet_b200.part_utils import PartRenderer
from oracle import seg_eval as oseg

B, N, REPS = 32, 50, 3
dev = torch.device("cuda:0")
smpl = danet_b200.SMPL(synthetic.make_smpl_model(0)).to(dev)
rend = PartRenderer(faces=smpl.faces, **synthetic.make_part_assets(0))
rng = np.random.default_rng(0)
aa = torch.from_numpy(rng.normal(0, 0.2, (B, 72)).astype(np.float32)).to(dev)
verts = smpl(betas=torch.zeros(B, 10, device=dev), body_pose=aa[:, 3:], global_orient=aa[:, :3]).vertices
cam = torch.tensor([[0.9, 0.0, 0.1]], device=dev).repeat(B, 1)
shapes = rng.integers(150, 641, (B, 2)).astype(np.int64)
center = np.stack([shapes[:, 1] / 2, shapes[:, 0] / 2], 1).astype(np.float32)
scale = (shapes.min(1) / 200.0 * rng.uniform(0.7, 1.3, B)).astype(np.float64)
off = np.concatenate([[0], np.cumsum(shapes.prod(1))])
mgt = rng.integers(0, 2, off[-1]).astype(np.uint8) * 255
pgt = rng.choice(np.array([0, 1, 2, 3, 4, 5, 6, 255], np.uint8), off[-1])
mgt_d, pgt_d = torch.from_numpy(mgt).to(dev), torch.from_numpy(pgt).to(dev)


def gpu():
    mask, parts = rend(verts, cam)
    mc, pc = seg_eval.score_renders(mask, parts, center, scale, shapes, off[:-1], mgt_d, pgt_d)
    return mc.cpu().numpy(), pc.cpu().numpy()


def reference_shaped():
    mask, parts = rend(verts, cam)
    mask, parts = mask.cpu().numpy(), parts.cpu().numpy()
    tp, fp, fn = np.zeros((2, 1)), np.zeros((2, 1)), np.zeros((2, 1))
    ptp, pfp, pfn = np.zeros((7, 1)), np.zeros((7, 1)), np.zeros((7, 1))
    acc = pacc = 0.
    for i in range(B):
        H, W = shapes[i]
        gm = mgt[off[i]:off[i + 1]].reshape(H, W) > 0
        gp = pgt[off[i]:off[i + 1]].reshape(H, W).copy()
        pm = oseg.uncrop(mask[i], center[i], scale[i], (H, W)) > 0
        acc += (gm == pm).sum()
        for c in range(2):
            cg, cp = gm == c, pm == c
            tp[c] += (cg & cp).sum(); fp[c] += (~cg & cp).sum(); fn[c] += (cg & ~cp).sum()
        pp = oseg.uncrop(parts[i].astype(np.uint8), center[i], scale[i], (H, W))
        for c in range(7):
            cg, cp = gp == c, pp == c
            cp[gp == 255] = 0
            ptp[c] += (cg & cp).sum(); pfp[c] += (~cg & cp).sum(); pfn[c] += (cg & ~cp).sum()
        gp[gp == 255] = 0
        pp[pp == 255] = 0
        pacc += (gp == pp).sum()
    return tp, ptp


def timed(fn, n=N):
    """ms per call of `REPS` windows of n calls each (after a warm-up)."""
    for _ in range(3):
        fn()
    out = []
    for _ in range(REPS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        out.append(round((time.perf_counter() - t0) / n * 1e3, 3))
    return out


mc, pc = gpu()
tp, ptp = reference_shaped()
assert (np.array([mc[:, 0, 0].sum(), mc[:, 1, 1].sum()]) == tp.ravel()).all() and (np.einsum("bcc->c", pc[:, :7]) == ptp.ravel()).all()
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
covered = int(rend(verts, cam)[0].sum())
assert covered > B * 1000, covered
print(json.dumps({"B": B, "pixels": int(off[-1]), "covered_render_pixels": covered, "gpu_ms": timed(gpu),
                  "reference_shaped_ms": timed(reference_shaped, 5),
                  "render_only_ms": timed(lambda: rend(verts, cam)[0].sum().item()),
                  "device": q.stdout.strip() or torch.cuda.get_device_name(0)}))
