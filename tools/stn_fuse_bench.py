"""Times the training STN ops and the HRNet fuse (danet_b200.layers.hr_fuse, danet_b200.stn) against the torch
sequences they replace, at B = 16, S = 56, for HRNet-W48 and W32:

    python tools/stn_fuse_bench.py [--iters 50] [--json out.json]

- the 23 fuse outputs, forward and backward, against F.interpolate + add + relu (autograd);
- part_crops forward and backward against torch's 24-iteration affine_grid / grid_sample loop (its backward adds
  with atomics), with realistic thetas and with tiny scales (every crop pixel samples the same few input pixels: the
  gather's load-imbalance worst case);
- part_thetas against the reference's Python loop (restated here with torch ops: softmax integral, jitter, visibility,
  affine_para).
Every arm is captured once in a CUDA graph and timed by replay (CUDA-event medians after warm-up), so the figures are
GPU time without the Python / autograd host overhead of the calls.  GB/s = the bytes each op must move / time.  The script prints the card's name,
power limit and maximum SM clock: numbers mean nothing without them."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bn_bench import card, timed  # noqa: E402

B, S = 16, 56


def graphed(fn):
    """fn captured in a CUDA graph (after two warm-up calls on a side stream); returns its replay"""
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    return g.replay


def fuse_sites(width):
    from test_stn_fuse_gpu import _fuse_sites
    return _fuse_sites(width)


def bench_fuse(width, iters):
    from danet_b200.layers import hr_fuse
    g = torch.Generator(device="cuda").manual_seed(0)
    cases = []
    nbytes = 0
    for site in fuse_sites(width):
        terms = [torch.randn(B, c, h, h, generator=g, device="cuda").requires_grad_() for (c, h, f) in site[2]]
        factors = [f for (_, _, f) in site[2]]
        c, hh = site[2][0][0], site[2][0][1] * site[2][0][2]
        gy = torch.randn(B, c, hh, hh, generator=g, device="cuda")
        cases.append((terms, factors, gy))
        nbytes += sum(t.numel() for t in terms) * 4 + gy.numel() * 4          # read the terms, write y

    def ours_f():
        for terms, factors, _ in cases:
            hr_fuse(terms, factors)

    def torch_f():
        for terms, factors, _ in cases:
            y = None
            for t, f in zip(terms, factors):
                u = F.interpolate(t, scale_factor=f, mode="nearest") if f > 1 else t
                y = u if y is None else y + u
            torch.relu(y)

    def run_fb(fuse):
        def fn():
            for terms, factors, gy in cases:
                torch.autograd.grad(fuse(terms, factors), terms, gy)
        return fn

    def torch_fuse(terms, factors):
        y = None
        for t, f in zip(terms, factors):
            u = F.interpolate(t, scale_factor=f, mode="nearest") if f > 1 else t
            y = u if y is None else y + u
        return torch.relu(y)

    with torch.no_grad():
        tf_ours, tf_torch = timed(graphed(ours_f), iters), timed(graphed(torch_f), iters)
    tfb_ours, tfb_torch = timed(graphed(run_fb(hr_fuse)), iters), timed(graphed(run_fb(torch_fuse)), iters)
    # the backward reads dy and y once per term and writes every term gradient
    bwd_bytes = sum(sum(t.numel() for t in terms) * 4 + 2 * len(terms) * gy.numel() * 4 for terms, _, gy in cases)
    return {"fuse_fwd_ms": tf_ours, "fuse_fwd_torch_ms": tf_torch, "fuse_fwd_GBps": nbytes / tf_ours / 1e6,
            "fuse_fwd_bwd_ms": tfb_ours, "fuse_fwd_bwd_torch_ms": tfb_torch,
            "fuse_fwd_bwd_GBps": (nbytes + bwd_bytes) / tfb_ours / 1e6}


def bench_crops(C, iters, tiny):
    from danet_b200.stn import part_crops
    from test_stn_fuse_gpu import _realistic_thetas
    g = torch.Generator(device="cuda").manual_seed(1)
    xd = torch.randn(B, C, S, S, generator=g, device="cuda").requires_grad_()
    th = _realistic_thetas(B, 3)
    if tiny:
        th[:, :, 0, 0] = th[:, :, 1, 1] = 1e-4
    gy = torch.randn(B, 24 * C, S, S, generator=g, device="cuda")

    def torch_crops(x):
        return torch.cat([F.grid_sample(x, F.affine_grid(th[:, i], list(x.shape), align_corners=False),
                                        align_corners=False) for i in range(24)], 1)

    with torch.no_grad():
        f_ours = timed(graphed(lambda: part_crops(xd, th)), iters)
        f_torch = timed(graphed(lambda: torch_crops(xd)), iters)
    # backward = (forward + backward) - forward, both graph replays
    b_ours = timed(graphed(lambda: torch.autograd.grad(part_crops(xd, th), xd, gy)), iters) - f_ours
    b_torch = timed(graphed(lambda: torch.autograd.grad(torch_crops(xd), xd, gy)), iters) - f_torch
    crop_bytes = B * 24 * C * S * S * 4
    return {"crops_fwd_ms": f_ours, "crops_fwd_torch_ms": f_torch, "crops_bwd_ms": b_ours, "crops_bwd_torch_ms": b_torch,
            "crops_MB": crop_bytes / 1e6, "crops_fwd_GBps": crop_bytes / f_ours / 1e6,
            "crops_bwd_GBps": crop_bytes / b_ours / 1e6}


def bench_thetas(iters):
    from danet_b200.stn import part_thetas
    from oracle.net_ops import CHILDREN1, PARENTS0, SMPL2DP
    g = torch.Generator(device="cuda").manual_seed(2)
    hm = torch.randn(B, 24, S, S, generator=g, device="cuda")
    idx = torch.randn(B, 25, S, S, generator=g, device="cuda")
    ratio, off = torch.rand(24, generator=g, device="cuda"), torch.rand(24, generator=g, device="cuda") * 0.1
    cn, sn = torch.rand(B, 24, 2, generator=g, device="cuda"), torch.rand(24, 2, B, generator=g, device="cuda")

    def ref():
        p = F.softmax(10 * hm.reshape(B, 24, -1), 2).reshape(B, 24, S, S)
        ar = torch.arange(S, dtype=torch.float32, device="cuda")
        c = torch.stack([(p.sum(2) * ar).sum(2), (p.sum(3) * ar).sum(2)], -1) / (0.5 * S) - 1
        c = c + 0.1 * (cn - 0.5)
        onehot = F.one_hot(idx.argmax(1), 25).permute(0, 3, 1, 2).float()
        hidden = [torch.max(onehot[:, SMPL2DP[i]], 1)[0] for i in range(24)]
        hidden = torch.stack([F.grid_sample(hidden[i].unsqueeze(1), c[:, i].reshape(B, 1, 1, 2), align_corners=False)
                              .reshape(B) for i in range(24)]) < 0.5
        box = c.max(1)[0] - c.min(1)[0]
        sb = box.max(1)[0] / 2
        th = []
        for i in range(24):
            if i == 0:
                s = sb
            else:
                s = 2 * torch.max((c[:, CHILDREN1[i]] - c[:, i]).norm(dim=1) / 2, (c[:, PARENTS0[i]] - c[:, i]).norm(dim=1) / 2)
            s = (s * F.relu(ratio[i]) + F.relu(off[i])) * (1 + 0.2 * (sn[i, 0] - 0.5))
            if i != 0:
                s = torch.where(hidden[i], 0.8 * sb, s)
            s = s * (1 + 0.2 * (sn[i, 1] - 0.5))
            t = torch.zeros(B, 2, 3, device="cuda")
            t[:, 0, 0] = s
            t[:, 1, 1] = s
            t[:, :, -1] = c[:, i]
            th.append(t)
        return torch.stack(th, 1)

    ours = timed(graphed(lambda: part_thetas(hm, idx, ratio, off, center_noise=cn, scale_noise=sn)), iters)
    eager = timed(lambda: part_thetas(hm, idx, ratio, off, center_noise=cn, scale_noise=sn), iters)
    # the reference's loop is timed eagerly, as it runs: one_hot's range check synchronises, so it cannot be captured
    return {"thetas_ms": ours, "thetas_eager_ms": eager, "thetas_torch_eager_ms": timed(ref, iters),
            "thetas_GBps": (hm.numel() * 4) / ours / 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json")
    a = ap.parse_args()
    print(card())
    res = {"card": card()}
    for width, C in ((48, 48), (32, 32)):
        r = bench_fuse(width, a.iters)
        r.update(bench_crops(C, a.iters, False))
        r.update({k.replace("crops", "crops_tiny"): v for k, v in bench_crops(C, a.iters, True).items()})
        res["W%d" % width] = r
        print("W%d" % width, json.dumps({k: round(v, 3) for k, v in r.items()}))
    res["thetas"] = bench_thetas(a.iters)
    print("thetas", json.dumps({k: round(v, 4) for k, v in res["thetas"].items()}))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
