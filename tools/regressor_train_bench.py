"""Times the regressor's training path at the reference's training batch (B = 16, S = 56): forward, and forward +
backward, for body_branch, limb_branch, the GCN head and the whole predictor, next to the same graph walk in torch fp32
(oracle.regressor_train.TorchTrainOps, cuDNN and TF32 off; the head in torch is oracle.gcn_head.torch_head).  CUDA
events, median of --iters after --warmup, training mode.  Prints the card and its power limit.

    python tools/regressor_train_bench.py [--batch 16] [--size 56] [--iters 20] [--warmup 5]"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=56)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import danet_b200
    from danet_b200 import regressor as R
    from oracle import regressor_train as ort
    torch.backends.cudnn.enabled = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    net = danet_b200.build_synthetic_danet(width=32, seed=0, device=dev)
    B, S = a.batch, a.size
    body, part = (t.to(dev) for t in ort.make_inputs(B, S, 0))
    gen = torch.Generator().manual_seed(0)
    G = torch.randn(B, 229, generator=gen).to(dev)
    g_gp, g_rf = torch.randn(B, 13, generator=gen).to(dev), torch.randn(B, 24, 128, generator=gen).to(dev)
    low = R.lower_branches(net.graph)
    keys = [k for name in ("body", "limb") for op in low[name]["ops"] for k in op["keys"]]
    # torch fp32 copies of the branch state, so the two paths update separate running statistics
    tstate = {k: R._attr(net, k).detach().clone().requires_grad_(R._attr(net, k).requires_grad) for k in keys}
    tops = ort.TorchTrainOps()
    rot = torch.rand(B, 24, 128, device=dev)
    gpara = torch.randn(B, 13, device=dev)
    net.train()

    def ours_body(bwd):
        y = R.body_branch(net, body)
        if bwd:
            y.backward(g_gp)

    def ours_limb(bwd):
        y = R.limb_branch(net, part)
        if bwd:
            y.backward(g_rf)

    def ours_head(bwd):
        r, g = rot.clone().requires_grad_(bwd), gpara.clone().requires_grad_(bwd)
        out = R.gcn_head(net, r, g)
        if bwd:
            (out["para"] * G).sum().backward()

    def ours_all(bwd):
        out = R.predictor(net, body, part)
        if bwd:
            (out["para"] * G).sum().backward()

    def torch_body(bwd):
        y = R.run_branch(low["body"], tstate, body, True, tops)
        if bwd:
            y.backward(g_gp)

    def torch_limb(bwd):
        y = R.run_branch(low["limb"], tstate, part.reshape(B * 24, 21, S, S), True, tops).reshape(B, 24, 128)
        if bwd:
            y.backward(g_rf)

    def torch_all(bwd):
        y = R.run_branch(low["body"], tstate, body, True, tops)
        z = R.run_branch(low["limb"], tstate, part.reshape(B * 24, 21, S, S), True, tops).reshape(B, 24, 128)
        if bwd:
            torch.autograd.backward([y, z], [g_gp, g_rf])

    print("card: %s; B = %d, S = %d, training mode; medians of %d after %d warm-up, ms" % (card(), B, S, a.iters, a.warmup))
    print("%-26s %10s %10s %12s %12s %8s %8s" % ("", "fwd", "fwd+bwd", "torch fwd", "torch f+b", "fwd x", "f+b x"))
    rows = [("body_branch", ours_body, torch_body), ("limb_branch", ours_limb, torch_limb), ("gcn_head", ours_head, None),
            ("predictor (torch: branches)", ours_all, torch_all)]
    for name, ours, ref in rows:
        with torch.no_grad():
            f = timed(lambda: ours(False), a.iters, a.warmup)
        fb = timed(lambda: ours(True), a.iters, a.warmup)
        if ref is not None:
            with torch.no_grad():
                tf = timed(lambda: ref(False), a.iters, a.warmup)
            tfb = timed(lambda: ref(True), a.iters, a.warmup)
            print("%-26s %10.2f %10.2f %12.2f %12.2f %8.2f %8.2f" % (name, f, fb, tf, tfb, f / tf, fb / tfb))
        else:
            print("%-26s %10.2f %10.2f" % (name, f, fb))
    net.eval()


if __name__ == "__main__":
    main()
