"""Per-shape timing of the wgmma convolution engine (danet_conv_tc_group) at the six convolution shapes that carry
77 % of the MACs of HRNet-W48 DaNet at batch 64, in both precisions.

Each shape runs alone in its launch, on the layouts the network plan uses: split-fp16 NHWC input planes (hi, plus lo
in exact mode), packed weights, fp32 bias, ReLU, split-fp16 output planes.  Times are CUDA events over a window of
at least --window seconds after warm-up.  Reported per shape and precision:
  ms            device time of one launch
  alg_tflops    2 * MACs / time (the convolution's own arithmetic)
  exec_tflops   tensor-pipe products actually issued: x3 in exact mode (hi*hi, hi*lo, lo*hi)
  frac_peak     exec_tflops / 989 TFLOP/s (H100 SXM dense fp16 data-sheet peak)
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi, read-only query).

    python tools/conv_bench.py [--window 0.5] [--out FILE.json] [--root TREE]

--root imports the package from another checkout of this project (to compare two builds in one run).
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

PEAK_TFLOPS = 989.0

# N, H, W, Cin, Cout, k, stride, weight sets, share of the W48 B=64 network's MACs
SHAPES = [
    (64, 56, 56, 48, 48, 3, 1, 1, "17.8%"),
    (64, 28, 28, 96, 96, 3, 1, 1, "17.8%"),
    (1536, 56, 56, 64, 64, 7, 2, 1, "16.1%"),
    (64, 14, 14, 192, 192, 3, 1, 1, "15.6%"),
    (64, 7, 7, 384, 384, 3, 1, 1, "6.7%"),
    (1536, 56, 56, 48, 24, 3, 1, 24, "3.3%"),
]


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        return {"query": "nvidia-smi unavailable"}
    return dict(zip(q.split(","), [s.strip() for s in out[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--window", type=float, default=0.5, help="seconds of timed launches per shape and precision")
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="checkout whose built package is measured")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from danet_b200 import _lib as L

    if not torch.cuda.is_available():
        sys.exit("conv_bench: no CUDA device")
    dev = torch.device("cuda:0")
    lib = L.load()
    info = gpu_info()
    rows = []
    for (N, H, W, Cin, Cout, k, s, G, share) in SHAPES:
        Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
        macs = N * Ho * Wo * Cout * Cin * k * k
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(N, H, W, Cin, device=dev, generator=g)
        w = torch.randn(G, k * k * Cin, Cout, device=dev, generator=g) * (1.0 / (k * k * Cin)) ** 0.5
        b = torch.randn(G, Cout, device=dev, generator=g) * 0.1
        for exact in (1, 0):
            d = L.ConvDesc(N, H, W, Cin, Cout, k, s, k // 2, G, 1, 4 if exact else 0)
            assert lib.danet_conv_tc_supported(ctypes.byref(d)), "shape not supported by the tensor-core path"
            xh = torch.empty(x.shape, dtype=torch.float16, device=dev)
            xl = torch.empty(x.shape, dtype=torch.float16, device=dev) if exact else None
            L.check(lib.danet_act_split(x.numel(), L.ptr(x), L.ptr(xh), L.ptr(xl), L.stream_ptr()), "act_split")
            wpk = torch.empty(int(lib.danet_conv_tc_packed_bytes(ctypes.byref(d))), dtype=torch.uint8, device=dev)
            L.check(lib.danet_conv_tc_pack(ctypes.byref(d), L.ptr(w), L.ptr(wpk), L.stream_ptr()), "conv_tc_pack")
            yh = torch.empty(N, Ho, Wo, Cout, dtype=torch.float16, device=dev)
            yl = torch.empty_like(yh) if exact else None
            p = L.ConvProblem()
            p.d = d
            p.x = L.Act(None, xh.data_ptr(), xl.data_ptr() if exact else None)
            p.res = L.Act(None, None, None)
            p.y = L.Act(None, yh.data_ptr(), yl.data_ptr() if exact else None)
            p.w_packed, p.bias = wpk.data_ptr(), b.data_ptr()
            arr = (L.ConvProblem * 1)(p)

            def launch():
                L.check(lib.danet_conv_tc_group(1, arr, L.stream_ptr()), "conv_tc_group")

            for _ in range(5):
                launch()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            torch.cuda.synchronize()
            iters = max(20, int(args.window * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
            e0.record()
            for _ in range(iters):
                launch()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            alg = 2.0 * macs / (ms * 1e-3) / 1e12
            ex = alg * (3 if exact else 1)
            rows.append({"shape": "N%d %dx%d %d->%d k%d s%d ws%d" % (N, H, W, Cin, Cout, k, s, G), "mac_share": share,
                         "precision": "exact" if exact else "fast", "ms": round(ms, 4), "iters": iters,
                         "window_s": round(ms * iters / 1e3, 3), "alg_tflops": round(alg, 1),
                         "exec_tflops": round(ex, 1), "frac_peak": round(ex / PEAK_TFLOPS, 3)})
            print("%-34s %-5s %9.4f ms  alg %6.1f  exec %6.1f TFLOP/s  %5.1f%% of %g" % (
                rows[-1]["shape"], rows[-1]["precision"], ms, alg, ex, 100 * ex / PEAK_TFLOPS, PEAK_TFLOPS), flush=True)
            del xh, xl, wpk, yh, yl
    info_after = gpu_info()
    res = {"gpu": info, "sm_clock_after": info_after.get("clocks.sm"), "root": os.path.abspath(args.root), "rows": rows}
    print(json.dumps({"gpu": info, "sm_clock_after": res["sm_clock_after"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
