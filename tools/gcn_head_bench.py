"""Times one training step of the regressor head (danet_b200.regressor, csrc/gcn_train.cu) at B = 16 (the reference's
training batch) and B = 64, with CUDA events after warm-up: the whole step, and separately its forward (gcn_head + the
three head losses) and its backward (autograd to every head parameter, rot_feats and global_para), each the mean
device time between events recorded around that half of every step.  For scale, the same step through the oracle's
torch restatement (oracle/gcn_head.py torch_head, fp32 autograd over eager torch ops) on the same device.

--compare PATH loads another build of libdanet_b200.so into the same process and times the two builds in alternating
rounds (in-tree, other, in-tree, ...), so that both see the same device, clocks and neighbours.  Prints one JSON
object with the device name and power limit read in the same run and the number of kernel launches per step
(torch.profiler).  Dev tool: `python tools/gcn_head_bench.py [--out FILE] [--compare PATH] [--rounds N]`."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from danet_b200 import _lib
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


def split(fwd, bwd, n=50, warm=5):
    """(forward ms, backward ms) per step: events before, between and after the two halves of every step"""
    for _ in range(warm):
        bwd(fwd())
    torch.cuda.synchronize()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(n)]
    for e in ev:
        e[0].record()
        o = fwd()
        e[1].record()
        bwd(o)
        e[2].record()
    torch.cuda.synchronize()
    return sum(e[0].elapsed_time(e[1]) for e in ev) / n, sum(e[1].elapsed_time(e[2]) for e in ev) / n


def launches(f):
    from torch.profiler import ProfilerActivity, profile
    f()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.key.startswith(("Memcpy", "Memset")))


def arg(name, default):
    return sys.argv[sys.argv.index(name) + 1] if name in sys.argv else default


builds = {"in_tree": _lib.load()}
if "--compare" in sys.argv:                               # a second handle: the module-level one is swapped per round
    tree_path, _lib._lib = _lib.LIB_PATH, None
    _lib.LIB_PATH = os.path.abspath(arg("--compare", None))
    builds["compare"] = _lib.load()
    res_paths = {"in_tree": tree_path, "compare": _lib.LIB_PATH}
    _lib.LIB_PATH, _lib._lib = tree_path, builds["in_tree"]
else:
    res_paths = {"in_tree": _lib.LIB_PATH}
rounds = int(arg("--rounds", 3))

res = {"builds": res_paths}
for B in (16, 64):
    g = torch.Generator(device=dev).manual_seed(B)
    rot = torch.rand(B, 24, 128, device=dev, generator=g).requires_grad_()
    gp = torch.randn(B, 13, device=dev, generator=g).requires_grad_()
    target = torch.randn(B, 229, device=dev, generator=g)
    gt = torch.randn(B, 24, 3, device=dev, generator=g)
    has = (torch.rand(B, device=dev, generator=g) < 0.7).to(torch.uint8)
    G = torch.randn(B, 229, device=dev, generator=g)

    def fwd():
        out = gcn_head(net, rot, gp)
        L = gcn_head_losses(out, target, gt, has)
        return L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"] + (out["para"] * G).sum()

    def bwd(tot):
        torch.autograd.grad(tot, leaves + [rot, gp])

    def ours():
        bwd(fwd())

    bn = {n: (mod.get_submodule(n).running_mean.clone(), mod.get_submodule(n).running_var.clone()) for n in BN_NAMES}
    sel = (has == 1).float()

    def torch_ref():
        para, p0, c0, c1 = og.torch_head(P, buf, bn, rot, gp, training=True)
        n = sel.sum().clamp_min(1)
        lr = og.SMPL_POSE_WEIGHTS * (((p0 - target[:, 13:]) ** 2) * sel[:, None]).sum() / (n * 216)
        lp = sum(F.l1_loss(c * sel[:, None, None], gt * sel[:, None, None], reduction="sum") / n for c in (c0, c1))
        torch.autograd.grad(lr + lp + (para * G).sum(), leaves + [rot, gp])

    r = {name: {"step_ms": [], "forward_ms": [], "backward_ms": []} for name in builds}
    for _ in range(rounds):
        for name, h in builds.items():
            _lib._lib = h
            r[name]["step_ms"].append(timed(ours))
            f_ms, b_ms = split(fwd, bwd)
            r[name]["forward_ms"].append(f_ms)
            r[name]["backward_ms"].append(b_ms)
    _lib._lib = builds["in_tree"]
    r["launches"] = launches(ours)
    r["torch_restatement_fp32_autograd_ms"], r["torch_launches"] = timed(torch_ref), launches(torch_ref)
    res["B%d" % B] = r
try:
    res["device"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                   capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:                                    # the name alone, when nvidia-smi is not there
    res["device"] = torch.cuda.get_device_name(dev) + " (power limit not read: %s)" % e
print(json.dumps(res, indent=1))
if "--out" in sys.argv:
    with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
        json.dump(res, f, indent=1)
