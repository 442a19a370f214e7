"""The B = 64 W48 parity block (bench.parity_block) for one configuration: python tools/parity_b64.py <simt|tc> [exact|fast]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import danet_b200
import bench

algo = sys.argv[1] if len(sys.argv) > 1 else "tc"
prec = sys.argv[2] if len(sys.argv) > 2 else "exact"
dev = torch.device("cuda:0")
net = danet_b200.build_synthetic_danet(width=48, seed=0, device=dev, conv_algo=algo, precision=prec)
p = bench.parity_block(net, dev, 48, 64)
p.pop("note", None)
print(algo, prec, json.dumps(p))
