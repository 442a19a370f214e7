"""Timing of the differentiable convolution (danet_b200.conv.conv2d, exact mode): forward + backward, and the input
gradient (dgrad) and the weight + bias gradient (wgrad) on their own, next to the same op in torch (cuDNN, fp32, TF32
off).

Shapes: the six shapes of tools/conv_bench.py and every distinct convolution of body_net, limb_net (24 B images) and
limb_reslayer (groups = 24) at B = 64.  Times are CUDA events over a window of at least --window seconds after warm-up:
  fwdbwd_ms   forward + backward to x, weight and bias
  dgrad_ms    backward to x alone (dy split, W' pack, the engine launches, the interleave)
  wgrad_ms    backward to weight and bias alone (dy split, the wgmma GEMM, the finishing sums)
  alg_tflops  2 * MACs per pass over the time (three passes for fwdbwd)
  exec_tflops tensor-pipe products issued: x3 for the split-fp16 exact mode, and for dgrad times the executed / needed
              taps of the stride-2 pieces (28 / 9 for 3x3, 81 / 49 for 7x7)
  frac_peak   exec_tflops / 989 TFLOP/s (H100 SXM dense fp16 data-sheet peak)
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi, read-only query).

    python tools/conv_bwd_bench.py [--window 0.3] [--out FILE.json] [--only SUBSTRING]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_TFLOPS = 989.0

# name, images B, groups G, per-group cin, cout, H (= W), k, stride
SHAPES = [
    ("hrnet 3x3 48", 64, 1, 48, 48, 56, 3, 1),
    ("hrnet 3x3 96", 64, 1, 96, 96, 28, 3, 1),
    ("limb stem 7x7/s2 (N=1536)", 1536, 1, 64, 64, 56, 7, 2),
    ("hrnet 3x3 192", 64, 1, 192, 192, 14, 3, 1),
    ("hrnet 3x3 384", 64, 1, 384, 384, 7, 3, 1),
    ("partial-iuv 3x3 g24 48->24 (N=1536)", 64, 24, 48, 24, 56, 3, 1),
    ("body in 1x1 75->64", 64, 1, 75, 64, 56, 1, 1),
    ("body stem 7x7/s2", 64, 1, 64, 64, 56, 7, 2),
    ("body layer1 3x3 64", 64, 1, 64, 64, 14, 3, 1),
    ("body layer2 3x3/s2 64->128", 64, 1, 64, 128, 14, 3, 2),
    ("body layer2 down 1x1/s2", 64, 1, 64, 128, 14, 1, 2),
    ("body layer2 3x3 128", 64, 1, 128, 128, 7, 3, 1),
    ("body layer3 3x3/s2 128->256", 64, 1, 128, 256, 7, 3, 2),
    ("body layer3 down 1x1/s2", 64, 1, 128, 256, 7, 1, 2),
    ("body layer3 3x3 256", 64, 1, 256, 256, 4, 3, 1),
    ("body layer4 3x3/s2 256->512", 64, 1, 256, 512, 4, 3, 2),
    ("body layer4 down 1x1/s2", 64, 1, 256, 512, 4, 1, 2),
    ("body layer4 3x3 512", 64, 1, 512, 512, 2, 3, 1),
    ("limb in 1x1 21->64 (N=1536)", 1536, 1, 21, 64, 56, 1, 1),
    ("limb layer1 3x3 64 (N=1536)", 1536, 1, 64, 64, 14, 3, 1),
    ("limb layer2 3x3/s2 64->128 (N=1536)", 1536, 1, 64, 128, 14, 3, 2),
    ("limb layer2 down 1x1/s2 (N=1536)", 1536, 1, 64, 128, 14, 1, 2),
    ("limb layer2 3x3 128 (N=1536)", 1536, 1, 128, 128, 7, 3, 1),
    ("limb layer3 3x3/s2 128->256 (N=1536)", 1536, 1, 128, 256, 7, 3, 2),
    ("limb layer3 down 1x1/s2 (N=1536)", 1536, 1, 128, 256, 7, 1, 2),
    ("limb layer3 3x3 256 (N=1536)", 1536, 1, 256, 256, 4, 3, 1),
    ("limb_reslayer 3x3/s2 g24 256->128", 64, 24, 256, 128, 4, 3, 2),
    ("limb_reslayer 3x3 g24 128", 64, 24, 128, 128, 2, 3, 1),
    ("limb_reslayer down 1x1/s2 g24", 64, 24, 256, 128, 4, 1, 2),
]


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        return {"query": "nvidia-smi unavailable"}
    return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else {}


def timed(fn, window):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    iters = max(5, int(window * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def measure(conv, x, w, b, gy, s, G, window):
    """(fwd+bwd ms, dgrad ms, wgrad ms) of one conv implementation"""
    import torch
    pad = w.shape[-1] // 2

    def fwdbwd():
        xx, ww, bb = x.requires_grad_(True), w.requires_grad_(True), b.requires_grad_(True)
        torch.autograd.grad(conv(xx, ww, bb, s, pad, 1, G), (xx, ww, bb), gy)

    x.requires_grad_(True); w.requires_grad_(False); b.requires_grad_(False)
    y = conv(x, w, b, s, pad, 1, G)
    t_d = timed(lambda: torch.autograd.grad(y, (x,), gy, retain_graph=True), window)
    x.requires_grad_(False); w.requires_grad_(True); b.requires_grad_(True)
    y = conv(x, w, b, s, pad, 1, G)
    t_w = timed(lambda: torch.autograd.grad(y, (w, b), gy, retain_graph=True), window)
    del y
    t_f = timed(fwdbwd, window)
    return t_f, t_d, t_w


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--window", type=float, default=0.3, help="seconds of timed calls per measurement")
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    ap.add_argument("--only", default=None, help="run only the shapes whose name contains this")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    import torch.nn.functional as F
    from danet_b200.conv import conv2d
    from oracle.conv_bwd import executed_taps

    if not torch.cuda.is_available():
        sys.exit("conv_bwd_bench: no CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    info = gpu_info()
    rows = []
    for (name, B, G, cin, cout, H, k, s) in SHAPES:
        if args.only and args.only not in name:
            continue
        Ho = (H - 1) // s + 1
        macs = B * G * Ho * Ho * cout * cin * k * k
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(B, G * cin, H, H, device=dev, generator=g)
        w = torch.randn(G * cout, cin, k, k, device=dev, generator=g) * (1.0 / (k * k * cin)) ** 0.5
        b = torch.randn(G * cout, device=dev, generator=g) * 0.1
        gy = torch.randn(B, G * cout, Ho, Ho, device=dev, generator=g)
        tap_x = executed_taps(k, s) / float(k * k)
        row = {"shape": name, "B": B, "groups": G, "cin": cin, "cout": cout, "H": H, "k": k, "stride": s}
        for impl, fn in (("danet", conv2d), ("torch_fp32", F.conv2d)):
            tf, td, tw = measure(fn, x, w, b, gy, s, G, args.window)
            alg = lambda ms, passes=1: passes * 2.0 * macs / (ms * 1e-3) / 1e12
            r = {"fwdbwd_ms": round(tf, 4), "dgrad_ms": round(td, 4), "wgrad_ms": round(tw, 4),
                 "fwdbwd_alg_tflops": round(alg(tf, 3), 1), "dgrad_alg_tflops": round(alg(td), 1),
                 "wgrad_alg_tflops": round(alg(tw), 1)}
            if impl == "danet":
                r["dgrad_exec_tflops"] = round(3 * tap_x * alg(td), 1)
                r["wgrad_exec_tflops"] = round(3 * alg(tw), 1)
                r["dgrad_frac_peak"] = round(3 * tap_x * alg(td) / PEAK_TFLOPS, 3)
                r["wgrad_frac_peak"] = round(3 * alg(tw) / PEAK_TFLOPS, 3)
            row[impl] = r
        rows.append(row)
        d, t = row["danet"], row["torch_fp32"]
        dg = "dgrad %8.3f ms (torch %8.3f) exec %6.1f TF/s %4.1f%%" % (
            d["dgrad_ms"], t["dgrad_ms"], d["dgrad_exec_tflops"], 100 * d["dgrad_frac_peak"])
        print("%-40s fwd+bwd %8.3f ms (torch %8.3f) | %s | wgrad %8.3f ms (torch %8.3f) exec %6.1f TF/s %4.1f%%" % (
            name, d["fwdbwd_ms"], t["fwdbwd_ms"], dg, d["wgrad_ms"], t["wgrad_ms"], d["wgrad_exec_tflops"],
            100 * d["wgrad_frac_peak"]), flush=True)
        del x, w, b, gy
        torch.cuda.empty_cache()
    res = {"gpu": info, "sm_clock_after": gpu_info().get("clocks.sm"), "rows": rows}
    print(json.dumps({"gpu": info, "sm_clock_after": res["sm_clock_after"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
