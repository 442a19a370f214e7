"""Shared by the GCN head tests: the golden's parameters (keyed weights of danet_b200.synthetic, seed 0, with the
golden's edge_importance) and random problems for the fp64 restatement."""
import os

import numpy as np

from oracle import gcn_head as og

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RP = "iuv2smpl.smpl_para_Outs."


def param_shapes():
    shapes = {}
    for (name, i), (di, do) in zip(og.LAYERS, og.DIMS):
        shapes["%s.gc.%d.weight" % (name, i)] = (di, do)
        shapes["%s.gc.%d.bias" % (name, i)] = (do,)
        shapes["%s.act.%d.0.weight" % (name, i)] = (24,)
        shapes["%s.act.%d.0.bias" % (name, i)] = (24,)
    shapes["edge_importance"] = (1, 24, 24)
    for i in range(2):
        shapes["pose_regressors.%d.1.weight" % i] = (144, 128, 1, 1)
        shapes["pose_regressors.%d.1.bias" % i] = (144,)
        shapes["coord_regressors.%d.1.weight" % i] = (72, 128, 1, 1)
        shapes["coord_regressors.%d.1.bias" % i] = (72,)
    return shapes


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "gcn_head.npz"))


def golden_params(g):
    """(P, buf, bn) of the golden as float32 numpy arrays."""
    from danet_b200 import synthetic
    P = {}
    for k, shp in param_shapes().items():
        P[k] = synthetic.keyed_tensor(RP + k, shp, 0).numpy().astype(np.float32)
    P["edge_importance"] = g["edge_importance"]
    buf = {k: g["buf_" + k] for k in og.BUFFER_NAMES}
    bn = {n: (g["rm0_" + n], g["rv0_" + n]) for n in og.BN_NAMES}
    return P, buf, bn


def random_problem(B, has, seed):
    rng = np.random.default_rng(seed)
    rot = rng.uniform(0, 1.5, (B, 24, 128)).astype(np.float32)
    gpara = rng.normal(0, 0.3, (B, 13)).astype(np.float32)
    target = np.concatenate([rng.normal(0, 0.3, (B, 13)), rng.normal(0, 0.5, (B, 216))], 1).astype(np.float32)
    gt = rng.normal(0, 0.3, (B, 24, 3)).astype(np.float32)
    if has == "all":
        h = np.ones(B, np.uint8)
    elif has == "none":
        h = np.zeros(B, np.uint8)
    else:
        h = (rng.random(B) < 0.5).astype(np.uint8)
        h[0] = 1
        if B > 1:
            h[-1] = 0
    G = rng.normal(0, 1, (B, 229)).astype(np.float32)
    return rot, gpara, target, gt, h, G


def rel_norm(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)
