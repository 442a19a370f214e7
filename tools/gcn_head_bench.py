"""Times one training step of the regressor head -- gcn_head forward + the three head losses + backward to every head
parameter, rot_feats and global_para (danet_b200.regressor, csrc/gcn_train.cu) -- at B = 16 (the reference's training
batch) and B = 64, with CUDA events after warm-up.  For scale, the same step through the oracle's torch restatement
(oracle/gcn_head.py torch_head, fp32 autograd over eager torch ops) on the same device.  Prints one JSON object with
the device name and power limit read in the same run and the number of kernel launches per step (torch.profiler).
Dev tool: `python tools/gcn_head_bench.py [--out FILE]`."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from danet_b200 import build_synthetic_danet
from danet_b200.regressor import BN_NAMES, PARAM_NAMES, gcn_head, gcn_head_losses
from oracle import gcn_head as og

dev = torch.device("cuda:0")
net = build_synthetic_danet(width=32, seed=0, device=dev).train()
mod = net.iuv2smpl.smpl_para_Outs
P = {n: mod.get_parameter(n) for n in PARAM_NAMES}
buf = {k: mod.get_buffer(k) for k in og.BUFFER_NAMES}
leaves = list(P.values())


def timed(f, n=50, warm=5):
    for _ in range(warm):
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def launches(f):
    from torch.profiler import ProfilerActivity, profile
    f()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.key.startswith(("Memcpy", "Memset")))


res = {}
for B in (16, 64):
    g = torch.Generator(device=dev).manual_seed(B)
    rot = torch.rand(B, 24, 128, device=dev, generator=g).requires_grad_()
    gp = torch.randn(B, 13, device=dev, generator=g).requires_grad_()
    target = torch.randn(B, 229, device=dev, generator=g)
    gt = torch.randn(B, 24, 3, device=dev, generator=g)
    has = (torch.rand(B, device=dev, generator=g) < 0.7).to(torch.uint8)
    G = torch.randn(B, 229, device=dev, generator=g)

    def ours():
        out = gcn_head(net, rot, gp)
        L = gcn_head_losses(out, target, gt, has)
        tot = L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"] + (out["para"] * G).sum()
        torch.autograd.grad(tot, leaves + [rot, gp])

    bn = {n: (mod.get_submodule(n).running_mean.clone(), mod.get_submodule(n).running_var.clone()) for n in BN_NAMES}
    sel = (has == 1).float()

    def torch_ref():
        para, p0, c0, c1 = og.torch_head(P, buf, bn, rot, gp, training=True)
        n = sel.sum().clamp_min(1)
        lr = og.SMPL_POSE_WEIGHTS * (((p0 - target[:, 13:]) ** 2) * sel[:, None]).sum() / (n * 216)
        lp = sum(F.l1_loss(c * sel[:, None, None], gt * sel[:, None, None], reduction="sum") / n for c in (c0, c1))
        torch.autograd.grad(lr + lp + (para * G).sum(), leaves + [rot, gp])

    res["B%d" % B] = {"ms": timed(ours), "launches": launches(ours),
                      "torch_restatement_fp32_autograd_ms": timed(torch_ref), "torch_launches": launches(torch_ref)}
try:
    res["device"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                   capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:                                    # the name alone, when nvidia-smi is not there
    res["device"] = torch.cuda.get_device_name(dev) + " (power limit not read: %s)" % e
print(json.dumps(res, indent=1))
if "--out" in sys.argv:
    with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
        json.dump(res, f, indent=1)
