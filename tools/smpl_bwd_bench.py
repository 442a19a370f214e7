"""Times danet_smpl_backward (csrc/lbs.cu: dL/dbetas and dL/dR of the SMPL layer from dL/dvertices and
dL/dsmpl_joints) through the C ABI at B = 64 on the synthetic 6890-vertex model, with CUDA events after warm-up, and
one call through CUDA-graph replay.  Prints one JSON object with the device name and power limit read in the same run.
Dev tool: `python tools/smpl_bwd_bench.py [--B 64] [--iters 200]`."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import danet_b200
from danet_b200 import _lib
from oracle import lbs as olbs, synth

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=64)
ap.add_argument("--iters", type=int, default=200)
args = ap.parse_args()

dev = torch.device("cuda:0")
B = args.B
smpl = danet_b200.SMPL(synth.make_smpl_model(0)).to(dev)
rng = np.random.default_rng(0)
t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
betas = t(rng.normal(0, 1, (B, 10)))
R = t(olbs.rot6d_to_rotmat(rng.normal(0, 1, (B * 24, 6))).reshape(B, 24, 3, 3))
gv, gs = t(rng.normal(0, 1, (B, 6890, 3))), t(rng.normal(0, 1, (B, 24, 3)))
lib = _lib.load()
h = smpl._handle(dev)
ws_bytes = int(lib.danet_smpl_backward_workspace_bytes(h, B))
ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
gb, gR = torch.empty(B, 10, device=dev), torch.empty(B, 24, 3, 3, device=dev)


def call():
    _lib.check(lib.danet_smpl_backward(h, B, _lib.ptr(betas), _lib.ptr(R), _lib.ptr(gv), _lib.ptr(gs), _lib.ptr(gb),
                                       _lib.ptr(gR), _lib.ptr(ws), _lib.stream_ptr(dev)), "smpl_backward")


def timed(f, n, warm=20):
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


eager = [timed(call, args.iters) for _ in range(3)]
s = torch.cuda.Stream()
s.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(s):
    call()
torch.cuda.current_stream().wait_stream(s)
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    call()
graph = [timed(g.replay, args.iters) for _ in range(3)]
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:          # noqa: BLE001
    q = "nvidia-smi unavailable: %s" % e
print(json.dumps({"op": "danet_smpl_backward", "B": B, "device": torch.cuda.get_device_name(dev), "nvidia_smi": q,
                  "workspace_bytes": ws_bytes, "eager_ms": [round(x, 4) for x in eager],
                  "graph_ms": [round(x, 4) for x in graph]}))
