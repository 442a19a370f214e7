"""Times DaNet's training join on the GPU (B = 16, W48, training mode, STN noise and part dropout passed in):

    python tools/danet_train_bench.py [--B 16] [--width 48] [--iters 10]

  danet_forward        forward, and forward + backward of the sum of the losses, through the CUDA op table
  torch fp32 table     the same runner on oracle/danet_train.py's torch table in fp32 (cuDNN on, TF32 off): the
                       layers in torch, the reference's Python loops for the dropout and clean, the torch GCN head and
                       SMPL layer
  part_drop_clean      the op alone, forward and forward + backward, against the reference's loops on torch CUDA
                       (oracle/danet_train.py), and its traffic counted from shapes
Prints the card, its power limit and SM clock, then one JSON line.  CUDA events around `iters` calls after warm-up."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _time(fn, iters, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--width", type=int, default=48)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("danet_train_bench: no CUDA device")
    from danet_b200 import build_synthetic_danet, training
    from danet_b200.iuvmap import part_drop_clean
    from oracle import danet_train as odt
    from test_danet_train_gpu import _in_dict, _masks, _noise
    torch.backends.cudnn.enabled = True
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    print("card, power limit, max SM clock, SM clock:", _card())
    B = a.B
    net = build_synthetic_danet(width=a.width, seed=0, device="cuda:0")
    d = _in_dict(net, B, 1)
    noise, drop = _noise(B, 2), _masks("rate0.3", B, 3)
    from danet_b200 import synthetic
    from danet_b200.losses import STN_HM_WEIGHTS
    state = {k: v.detach().clone() for k, v in net.state_dict().items() if not k.startswith("iuv2smpl.smpl.")}
    for k, _ in net.named_parameters():
        if k in state:
            state[k].requires_grad_()
    table = odt.torch_table(state, synthetic.make_smpl_model(0), True)
    res = {"B": B, "width": a.width, "card": _card()}
    net.train()
    for tag, ops in (("cuda", None), ("torch_table", table)):
        def fwd():
            if ops is None:
                return training.danet_forward(net, d, part_drop=drop, center_noise=noise[0], scale_noise=noise[1])
            return training.run_danet(net.graph, state, d, True, ops, drop, noise, 0.3, STN_HM_WEIGHTS)

        def fwd_bwd():
            ret = fwd()
            sum(v.sum() for v in ret["losses"].values()).backward()
            net.zero_grad(set_to_none=True)
            for t in state.values():
                t.grad = None
        with torch.no_grad():
            res["%s_forward_ms" % tag] = _time(fwd, a.iters)
        res["%s_forward_backward_ms" % tag] = _time(fwd_bwd, a.iters)
    net.eval()
    S = net.graph.outputs["hm"].H
    leaves = [t.to("cuda:0").requires_grad_() for t in odt.make_leaves(B, S, 4)]
    G1, G2 = (t.to("cuda:0") for t in odt.make_probes(B, S, 5))
    G1 = torch.nan_to_num(G1)
    G2 = torch.nan_to_num(G2)
    for tag, op in (("op_cuda", part_drop_clean), ("op_torch", odt.part_drop_clean)):
        with torch.no_grad():
            res["%s_forward_ms" % tag] = _time(lambda: op(*leaves, drop), 5 * a.iters)

        def fb():
            out = op(*leaves, drop)
            torch.autograd.backward([out[0], out[1], out[4]], [G1[:, :25], G1[:, 25:50], G2])
        res["%s_forward_backward_ms" % tag] = _time(fb, 5 * a.iters)
    # traffic counted from shapes (fp32 maps, one byte per argmax), not measured
    g, p = B * 25 * S * S, B * 24 * 21 * S * S
    fwd_bytes = 4 * (3 * g + B * 15 * S * S + p) * 2 + B * 25 * S * S // 25 + B * 24 * S * S
    bwd_bytes = 4 * (2 * g * 2 + p * 14 // 21 + p) + B * 25 * S * S // 25 + B * 24 * S * S   # U, V gradients read
    res.update(op_forward_bytes=fwd_bytes, op_backward_bytes=bwd_bytes,
               op_forward_GBps=fwd_bytes / (res["op_cuda_forward_ms"] * 1e-3) / 1e9)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
