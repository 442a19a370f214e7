"""Time the ResNet training layers (danet_b200.layers) on the GPU at every BatchNorm2d site of body_net, limb_net and
limb_reslayer and at both stem pools, at the reference's training batch (B = 16, README.md:118), forward and backward,
next to torch's own ops on the same card (F.batch_norm (+ residual) + ReLU and F.max_pool2d: cuDNN / ATen).

    python tools/bn_bench.py [--batch 16] [--iters 20] [--out FILE.json]

Times are CUDA-event medians over --iters calls after warm-up.  "bwd" is one autograd backward through the op (for
torch: through the ReLU, the residual add and the BatchNorm).  Bytes are the tensors each pass has to touch, from the
shapes: forward reads x (and the residual) and writes y; backward reads dy, x (and y under a ReLU) and writes dx (and
the residual's gradient); the pool reads x and writes y and the slots, its backward reads dy and the slots and writes
dx.  GB/s = bytes / time.  The script prints the card's name and power limit: numbers mean nothing without them."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (name, q)


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def bn_site(site, B, iters):
    from danet_b200.layers import batch_norm
    name, per, C, H, residual, relu = site
    N = B * per
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(N, C, H, H, generator=g, device="cuda").requires_grad_()
    r = torch.randn(N, C, H, H, generator=g, device="cuda").requires_grad_() if residual else None
    w = (1 + 0.1 * torch.randn(C, generator=g, device="cuda")).requires_grad_()
    b = (0.1 * torch.randn(C, generator=g, device="cuda")).requires_grad_()
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    gy = torch.randn(N, C, H, H, generator=g, device="cuda")

    def ours():
        return batch_norm(x, rm, rv, w, b, True, 0.1, 1e-5, residual=r, relu=relu)

    def theirs():
        z = F.batch_norm(x, rm, rv, w, b, True, 0.1, 1e-5)
        if r is not None:
            z = z + r
        return F.relu(z) if relu else z

    out = {"site": name, "shape": [N, C, H, H], "residual": residual, "relu": relu}
    n = N * C * H * H
    out["elements"] = n
    out["fwd_bytes"] = 4 * n * (2 + residual)
    out["bwd_bytes"] = 4 * n * (3 + relu + residual)
    for tag, f in (("ours", ours), ("torch", theirs)):
        with torch.no_grad():
            out[tag + "_fwd_ms"] = timed(f, iters)
        y = f()
        out[tag + "_bwd_ms"] = timed(lambda: torch.autograd.backward(y, gy, retain_graph=True), iters)
        del y
        x.grad = w.grad = b.grad = None
        if r is not None:
            r.grad = None
    return out


def pool(name, N, C, H, iters):
    from danet_b200.layers import max_pool2d
    g = torch.Generator(device="cuda").manual_seed(1)
    x = F.relu(torch.randn(N, C, H, H, generator=g, device="cuda")).requires_grad_()
    Ho = (H - 1) // 2 + 1
    gy = torch.randn(N, C, Ho, Ho, generator=g, device="cuda")
    n, m = N * C * H * H, N * C * Ho * Ho
    out = {"site": name, "shape": [N, C, H, H], "elements": n, "fwd_bytes": 4 * n + 5 * m, "bwd_bytes": 5 * m + 4 * n}
    for tag, f in (("ours", lambda: max_pool2d(x, 3, 2, 1)), ("torch", lambda: F.max_pool2d(x, 3, 2, 1))):
        with torch.no_grad():
            out[tag + "_fwd_ms"] = timed(f, iters)
        y = f()
        out[tag + "_bwd_ms"] = timed(lambda: torch.autograd.backward(y, gy, retain_graph=True), iters)
        del y
        x.grad = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bn_bench.py needs a CUDA device")
    from test_layers_gpu import SITES
    info = card()
    print("card:", info)
    rows = [bn_site(s, a.batch, a.iters) for s in SITES]
    rows += [pool("limb_net.maxpool", a.batch * 24, 64, 28, a.iters), pool("body_net.maxpool", a.batch, 64, 28, a.iters)]
    total = sum(r["elements"] for r in rows[:len(SITES)])
    print("BatchNorm elements per step (B = %d): %.1f M" % (a.batch, total / 1e6))
    print("%-36s %-20s %9s %9s %8s | %9s %9s %8s" % ("site", "shape", "fwd ms", "torch", "GB/s", "bwd ms", "torch", "GB/s"))
    for r in rows:
        print("%-36s %-20s %9.4f %9.4f %8.0f | %9.4f %9.4f %8.0f" % (
            r["site"], "x".join(map(str, r["shape"])), r["ours_fwd_ms"], r["torch_fwd_ms"], r["fwd_bytes"] / r["ours_fwd_ms"] / 1e6,
            r["ours_bwd_ms"], r["torch_bwd_ms"], r["bwd_bytes"] / r["ours_bwd_ms"] / 1e6))
    for part, sel in (("all BN sites", lambda r: r["site"] in {s[0] for s in SITES}),
                      ("limb_net 56x56 + 28x28", lambda r: r["site"] in ("limb_net.0.bn", "limb_net.bn1")),
                      ("pools", lambda r: r["site"].endswith("maxpool"))):
        sub = [r for r in rows if sel(r)]
        f, tf = sum(r["ours_fwd_ms"] for r in sub), sum(r["torch_fwd_ms"] for r in sub)
        bw, tb = sum(r["ours_bwd_ms"] for r in sub), sum(r["torch_bwd_ms"] for r in sub)
        print("%-26s fwd %.3f ms (torch %.3f, %.2fx)  bwd %.3f ms (torch %.3f, %.2fx)" % (part, f, tf, f / tf, bw, tb, bw / tb))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"card": info, "batch": a.batch, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
