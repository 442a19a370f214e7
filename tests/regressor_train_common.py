"""Shared by the regressor branch training tests: the golden of the reference's DecomposedPredictor
(tests/golden/regressor_train.npz, oracle/gen_golden_regressor.py) and the fp64 test double driven through the
product's own graph walk (danet_b200.regressor.run_branch with oracle.regressor_train.TorchTrainOps)."""
import os

import numpy as np
import torch

from oracle import regressor_train as ort

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RP = ort.RP
BRANCH_PREFIXES = tuple(RP + p for p in ("body_net.", "limb_net.", "limb_reslayer."))


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "regressor_train.npz"))


def golden_inputs(g):
    return ort.make_inputs(int(g["B"]), int(g["S"]), int(g["input_seed"]))


def branch_param_keys(state):
    """the 128 trainable tensors of the three branches (conv weights, BatchNorm weights and biases, final_layer)"""
    return [k for k, v in state.items() if k.startswith(BRANCH_PREFIXES) and v.is_floating_point()
            and not k.endswith(("running_mean", "running_var"))]


def bn2d_names(state):
    return sorted(k[:-len(".running_mean")] for k in state if k.startswith(BRANCH_PREFIXES) and k.endswith(".running_mean"))


class Recorder(object):
    """An op table that passes every call to `ops` and keeps each batch_norm output (after residual and ReLU)"""

    def __init__(self, ops):
        self.ops, self.bn = ops, []

    def __getattr__(self, name):
        return getattr(self.ops, name)

    def batch_norm(self, *a, **k):
        y = self.ops.batch_norm(*a, **k)
        self.bn.append(y.detach())
        return y


def relu_flips(bn_a, bn_b):
    """elements whose ReLU decision differs between two recordings of the same walk"""
    return sum(int(((a > 0) != (b.to(a.device) > 0)).sum()) for a, b in zip(bn_a, bn_b))


def double_step(state, graph, body, part, training, g_gp=None, g_rf=None, want_input_grad=True, ops=None):
    """Both branches in the test double on `state` (modified in place: running statistics, num_batches_tracked);
    backward with upstream gradients g_gp [B,13] and g_rf [B,24,128] when given.  Returns (global_para, rot_feats,
    {key: grad}) with the input gradients under 'body_iuv' / 'part_iuv'."""
    from danet_b200.regressor import lower_branches, run_branch
    low = lower_branches(graph)
    ops = ops if ops is not None else ort.TorchTrainOps()
    dt = next(v for v in state.values() if v.is_floating_point()).dtype
    keys = branch_param_keys(state)
    for k in keys:
        state[k].requires_grad_(True)
        state[k].grad = None
    B, S = part.shape[0], part.shape[-1]
    b = body.detach().to(dt).clone().requires_grad_(want_input_grad)
    p = part.detach().to(dt).clone().requires_grad_(want_input_grad)
    gp = run_branch(low["body"], state, b, training, ops)
    rf = run_branch(low["limb"], state, p.reshape(B * 24, 21, S, S), training, ops).reshape(B, 24, 128)
    grads = {}
    if g_gp is not None:
        torch.autograd.backward([gp, rf], [torch.as_tensor(g_gp, dtype=dt, device=gp.device),
                                           torch.as_tensor(g_rf, dtype=dt, device=gp.device)])
        grads = {k: state[k].grad for k in keys}
        if want_input_grad:
            grads["body_iuv"], grads["part_iuv"] = b.grad, p.grad
    for k in keys:
        state[k].requires_grad_(False)
    return gp.detach(), rf.detach(), grads
