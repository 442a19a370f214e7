"""Times DaNet's whole training step (training.train_step) and its parts on the GPU: B images per GPU, W48, training mode,
STN noise and part-dropout masks drawn once and passed in.

    python tools/train_step_bench.py [--B 16] [--width 48] [--iters 10]
    torchrun --nproc-per-node N tools/train_step_bench.py          (data-parallel over N GPUs, NCCL)

  prepare_targets      the step's targets (danet_b200.targets)
  forward_backward     danet_forward, the left-fold loss sum and its backward
  all_reduce           parallel.all_reduce_gradients (more than one rank only)
  adam_*               optimizer.step() over the model's gradients: danet_b200.optim.Adam (one pass), torch.optim.Adam
                       (foreach, torch's CUDA default) and torch.optim.Adam(fused=True); the one-pass optimizer's bytes/s
                       against 28 B per stepped parameter counted from shapes, and the host time step() spends before
                       it returns (building its tables and launching)
  step                 train_step with danet_b200.optim.Adam (LRDecay, pretraining off): ms per step and images/s
Prints the card, its power limit and SM clock, then one JSON line from rank 0: per entry the median, min and max in ms of
`iters` timed calls after warm-up (CUDA events around each call)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _times(fn, iters, warm=2, barrier=False):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(iters):
        if barrier:
            dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return {"median": statistics.median(out), "min": min(out), "max": max(out)}


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
        raise SystemExit("train_step_bench: no CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from danet_b200 import build_synthetic_danet
    from danet_b200.optim import Adam
    from danet_b200.parallel import all_reduce_gradients
    from danet_b200.targets import prepare_targets
    from danet_b200.training import LRDecay, danet_forward, train_step
    from test_train_step_gpu import make_batch
    B = a.B
    net = build_synthetic_danet(width=a.width, seed=0, device=dev)
    batch, opt_pose, opt_betas, fit_valid, noise, drops = make_batch(B, 1 + rank, 1, device=dev)
    kw = dict(part_drop=drops[0], center_noise=noise[0][0], scale_noise=noise[0][1])
    res = {"B_per_gpu": B, "gpus": world, "width": a.width, "card": _card()}
    if rank == 0:
        print("card, power limit, max SM clock, SM clock:", res["card"])
    net.train()
    with torch.no_grad():
        res["prepare_targets_ms"] = _times(lambda: prepare_targets(net, batch, opt_pose, opt_betas, fit_valid=fit_valid),
                                           a.iters)
    d = dict(batch, pretrain_mode=False)
    d.update(prepare_targets(net, batch, opt_pose, opt_betas, fit_valid=fit_valid))

    def fwd_bwd():
        net.zero_grad()
        ret = danet_forward(net, d, **kw)
        total = 0
        for v in ret["losses"].values():
            total += v
        total.backward()
    res["forward_backward_ms"] = _times(fwd_bwd, a.iters)
    if world > 1:
        res["all_reduce_ms"] = _times(lambda: all_reduce_gradients(net.parameters()), a.iters, barrier=True)
    stepped = [p for p in net.parameters() if p.grad is not None]
    n = sum(p.numel() for p in stepped)
    res.update(stepped_tensors=len(stepped), stepped_parameters=n, adam_bytes_per_step=28 * n)
    # the optimizers on copies, so the model's weights stay as they are
    copies = [torch.nn.Parameter(p.detach().clone()) for p in stepped]
    for c, p in zip(copies, stepped):
        c.grad = p.grad
    for tag, make in (("adam_one_pass", lambda: Adam(copies, lr=1e-4)),
                      ("adam_torch_foreach", lambda: torch.optim.Adam(copies, lr=1e-4, foreach=True)),
                      ("adam_torch_fused", lambda: torch.optim.Adam(copies, lr=1e-4, fused=True))):
        opt = make()
        res[tag + "_ms"] = _times(opt.step, 5 * a.iters)
        if tag == "adam_one_pass":
            host = []
            for _ in range(5 * a.iters):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                opt.step()
                host.append((time.perf_counter() - t0) * 1e3)
            res["adam_one_pass_host_ms"] = {"median": statistics.median(host), "min": min(host), "max": max(host)}
        del opt
    res["adam_one_pass_GBps"] = 28 * n / (res["adam_one_pass_ms"]["median"] * 1e-3) / 1e9
    net.zero_grad()
    opt = Adam(net.parameters(), lr=1e-4)
    sched = LRDecay()
    count = [0]

    def step():
        count[0] += 1
        train_step(net, opt, batch, opt_pose, opt_betas, count[0], schedule=sched, pretr_step=0, fit_valid=fit_valid,
                   **kw)
    res["step_ms"] = _times(step, a.iters, barrier=world > 1)
    res["images_per_s"] = B * world / (res["step_ms"]["median"] * 1e-3)
    if rank == 0:
        print(json.dumps(res))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
