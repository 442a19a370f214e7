"""Times the IUV estimator's training path at the reference's training batch (B = 16, HRNet-W48, 224 x 224 images):
forward, and forward + backward, of the network walk (danet_b200.estimator.run_estimator, the gradient of <G, outputs>)
and of the whole iuv_estimator call with its losses, next to the same walk through the torch fp32 op table
(oracle.estimator_train.TorchEstimatorOps with cuDNN on and TF32 off; its part_thetas is the CUDA one, as it carries no
gradient and the table's is a host restatement).  CUDA events, median of --iters after --warmup, training mode, the STN
noise passed in.  Prints the card, its power limit and clocks.  --profile adds one forward + backward of the walk under
torch.profiler: the forward's convolution and BatchNorm time by output map size, and the kernels with the most time.

    python tools/estimator_train_bench.py [--batch 16] [--width 48] [--iters 20] [--warmup 5] [--profile]"""
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--width", type=int, default=48)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import danet_b200
    from danet_b200 import estimator as E
    from danet_b200 import stn
    from oracle import estimator_train as oet
    torch.backends.cudnn.enabled = True
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    net = danet_b200.build_synthetic_danet(width=a.width, seed=0, device=dev)
    B = a.batch
    img = oet.make_image(B, 0).to(dev)
    iuv, kps, dp = oet.make_targets(B, 1)
    f = lambda t: torch.as_tensor(t, device=dev)
    targets = dict(iuv_image_gt=f(iuv), smpl_kps_gt=f(kps), uvia_dp_gt={k: f(v) for k, v in dp.items()},
                   has_iuv=torch.ones(B, dtype=torch.uint8, device=dev), has_dp=torch.ones(B, device=dev))
    torch.manual_seed(0)
    noise = tuple(t.to(dev) for t in E.draw_noise(B))
    low = E.lower_estimator(net.graph)
    keys = [k for op in low["ops"] for k in op["keys"]]
    from danet_b200.regressor import _attr
    state = {k: _attr(net, k) for k in keys}
    # torch fp32 copies of the state, so the two paths update separate running statistics
    tstate = {k: v.detach().clone().requires_grad_(v.requires_grad) for k, v in state.items()}

    class TorchOps(oet.TorchEstimatorOps):
        part_thetas = staticmethod(stn.part_thetas)
    tops, cops = TorchOps(), E._cuda_ops()
    S = net.graph.outputs["hm"].H
    gen = torch.Generator().manual_seed(0)
    G = {k: torch.randn(s, generator=gen).to(dev) for k, s in
         dict(u=(B, 25, S, S), v=(B, 25, S, S), index=(B, 25, S, S), ann=(B, 15, S, S),
              part_pred=(B, 24, 3, 7, S, S)).items()}
    net.train()

    def walk(st, ops, bwd):
        out = E.run_estimator(low, st, img, True, ops, noise)
        if bwd:
            sum((out[k] * g).sum() for k, g in G.items()).backward()

    def ours_call(bwd):
        out = E.iuv_estimator(net, img, **targets, center_noise=noise[0], scale_noise=noise[1])
        if bwd:
            sum(out["losses"].values()).backward()

    print("card: %s; HRNet-W%d, B = %d, 224 x 224, training mode; medians of %d after %d warm-up, ms"
          % (card(), a.width, B, a.iters, a.warmup))
    print("%-32s %10s %10s %12s %12s %8s %8s" % ("", "fwd", "fwd+bwd", "torch fwd", "torch f+b", "fwd x", "f+b x"))
    rows = [("network walk", lambda b: walk(state, cops, b), lambda b: walk(tstate, tops, b)),
            ("iuv_estimator with losses", ours_call, None)]
    for name, ours, ref in rows:
        with torch.no_grad():
            fw = timed(lambda: ours(False), a.iters, a.warmup)
        fb = timed(lambda: ours(True), a.iters, a.warmup)
        if ref is not None:
            with torch.no_grad():
                tf = timed(lambda: ref(False), a.iters, a.warmup)
            tfb = timed(lambda: ref(True), a.iters, a.warmup)
            print("%-32s %10.2f %10.2f %12.2f %12.2f %8.2f %8.2f" % (name, fw, fb, tf, tfb, fw / tf, fb / tfb))
        else:
            print("%-32s %10.2f %10.2f" % (name, fw, fb))
    if a.profile:
        profile(lambda ops: walk(state, ops, True), cops)
    net.eval()


class _Ranges(object):
    """An op table that wraps each conv2d / batch_norm call in a profiler range named by its output map size"""

    def __init__(self, ops):
        self.ops = ops

    def __getattr__(self, name):
        return getattr(self.ops, name)

    def conv2d(self, x, w, b, stride, padding, dilation, groups):
        n = (x.shape[2] - 1) // stride + 1
        with torch.profiler.record_function("fwd conv %dx%d" % (n, n)):
            return self.ops.conv2d(x, w, b, stride, padding, dilation, groups)

    def batch_norm(self, x, *args, **kw):
        with torch.profiler.record_function("fwd bn %dx%d" % (x.shape[2], x.shape[3])):
            return self.ops.batch_norm(x, *args, **kw)


def profile(step, ops):
    from torch.profiler import ProfilerActivity
    step(ops)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step(_Ranges(ops))
        torch.cuda.synchronize()
    from torch.autograd import DeviceType
    ev = prof.key_averages()
    dt = lambda e: getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
    st = lambda e: getattr(e, "self_device_time_total", getattr(e, "self_cuda_time_total", 0.0)) / 1e3
    # the CPU side of each range: device time of the kernels launched inside it
    rows = sorted((e for e in ev if e.key.startswith("fwd ") and e.device_type == DeviceType.CPU), key=lambda e: e.key)
    print("\nforward kernel time by output map size (device ms, calls):")
    for e in rows:
        print("  %-18s %8.2f  %4d" % (e.key, dt(e), e.count))
    kern = sorted((e for e in ev if e.device_type == DeviceType.CUDA and not getattr(e, "is_user_annotation", False)
                   and not e.key.startswith("fwd ") and st(e) > 0), key=st, reverse=True)
    total = sum(st(e) for e in kern)
    print("kernels of one forward + backward: %.2f device ms in all; the 12 largest:" % total)
    for e in kern[:12]:
        print("  %8.2f ms %5d x  %s" % (st(e), e.count, e.key[:90]))


if __name__ == "__main__":
    main()
