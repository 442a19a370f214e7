"""Shared by the IUV estimator training tests: the golden of the reference's IUV_Estimator
(tests/golden/estimator_train.npz, oracle/gen_golden_estimator.py) and a training step through the product's own graph
walk (danet_b200.estimator.run_estimator + estimator_losses) with any op table: the fp64 test double
(oracle.estimator_train.TorchEstimatorOps), fp32 torch, or the CUDA ops."""
import os

import numpy as np
import torch

from oracle import estimator_train as oet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EP = oet.EP
OUTPUTS = ("u", "v", "index", "ann", "hm", "part_pred")


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "estimator_train.npz"))


def golden_image(g):
    return oet.make_image(int(g["B"]), int(g["image_seed"]))


def golden_targets(g, dtype, device):
    f = lambda k: torch.as_tensor(g[k], dtype=dtype, device=device)
    dp = {k[3:]: f(k) for k in g.files if k.startswith("dp_")}
    return dict(iuv_image_gt=f("iuv_image_gt"), smpl_kps_gt=f("smpl_kps_gt"), uvia_dp_gt=dp,
                has_iuv=torch.as_tensor(g["has_iuv"], device=device), has_dp=torch.as_tensor(g["has_dp"], device=device))


def golden_noise(g, dtype, device):
    return (torch.as_tensor(g["center_noise"], dtype=dtype, device=device),
            torch.as_tensor(g["scale_noise"], dtype=dtype, device=device))


def bn_names(state):
    return sorted(k[:-len(".running_mean")] for k in state if k.endswith(".running_mean"))


def projections(B, S, seed, dtype, device):
    """fixed random upstream gradients for the raw outputs: <G_k, out_k> joins the objective (not hm, which the
    public function returns detached, as the reference does)"""
    gen = torch.Generator().manual_seed(seed)
    shapes = dict(u=(B, 25, S, S), v=(B, 25, S, S), index=(B, 25, S, S), ann=(B, 15, S, S),
                  part_pred=(B, 24, 3, 7, S, S))
    return {k: torch.randn(s, generator=gen, dtype=torch.float64).to(dtype=dtype, device=device) for k, s in shapes.items()}


class Recorder(object):
    """An op table that passes every call to `ops` and keeps every ReLU input decision (batch_norm and hr_fuse outputs)
    and every index-head argmax the thetas read"""

    def __init__(self, ops):
        self.ops, self.act, self.amax = ops, [], []

    def __getattr__(self, name):
        return getattr(self.ops, name)

    def batch_norm(self, *a, **k):
        y = self.ops.batch_norm(*a, **k)
        if k.get("relu"):
            self.act.append(y.detach())
        return y

    def hr_fuse(self, terms, factors, relu=True):
        y = self.ops.hr_fuse(terms, factors, relu)
        self.act.append(y.detach())
        return y

    def part_thetas(self, hm, index, *a, **k):
        self.amax.append(index.detach().argmax(1))
        return self.ops.part_thetas(hm, index, *a, **k)


def decision_flips(rec_a, rec_b):
    """(ReLU decisions, index argmax decisions) that differ between two recordings of the same walk"""
    relu = sum(int(((a > 0) != (b.to(a.device) > 0)).sum()) for a, b in zip(rec_a.act, rec_b.act))
    amax = sum(int((a != b.to(a.device)).sum()) for a, b in zip(rec_a.amax, rec_b.amax))
    return relu, amax


def step(state, graph, image, training, ops, targets=None, noise=(None, None), hm_weight=0.0, proj=None, scale=1.0,
         want_input_grad=True, backward=True):
    """One walk on `state` (modified in place: running statistics, num_batches_tracked) through `ops`, the losses when
    `targets` are given, and the backward of scale * (sum of the losses + sum_k <proj_k, out_k>).
    Returns (outputs {u, v, index, ann, hm, part_pred, centers, thetas, part_iuv_gt}, losses, {key: grad}, image grad)."""
    from danet_b200.estimator import estimator_losses, lower_estimator, run_estimator
    low = lower_estimator(graph)
    keys = oet.param_keys(state)
    for k in keys:
        state[k].requires_grad_(backward)
        state[k].grad = None
    x = image.detach().clone().requires_grad_(want_input_grad and backward)
    pred = run_estimator(low, state, x, training, ops, noise)
    L, part_gt = ({}, None)
    if targets is not None:
        L, part_gt = estimator_losses(pred, ops, stn_hm_weight=hm_weight, **targets)
    grads, gx = {}, None
    if backward:
        total = sum(v.sum() for v in L.values()) if L else 0
        if proj is not None:
            total = total + sum((pred[k] * proj[k]).sum() for k in proj)
        (total * scale).backward(inputs=[state[k] for k in keys] + ([x] if x.requires_grad else []))
        grads = {k: state[k].grad for k in keys}
        gx = x.grad
    for k in keys:
        state[k].requires_grad_(False)
    out = {k: v.detach() for k, v in pred.items()}
    out["part_iuv_gt"] = part_gt
    return out, {k: v.detach() for k, v in L.items()}, grads, gx
