"""Part dropout and iuvmap_clean as the reference's own torch expressions (models/danet/danet.py:194-205, 265-283, with
utils/iuvmap.py's iuvmap_clean imported through oracle/ref_import.py), differentiable by torch autograd.

TEST INFRASTRUCTURE.  `part_drop_clean` has the signature of danet_b200.iuvmap.part_drop_clean and runs on any device
and dtype, so it is both the bit-exact reference of the CUDA op and the op-table entry of the join's tests.  The
inputs are cloned first: the reference's in-place products then act on the clones, and autograd sees the same graph
as in DaNet._forward."""
import functools
import os
import sys
import types
import warnings

import torch

from oracle import ref_import

_CLEAN = []


def _ref_iuvmap_clean():
    """The reference's iuvmap_clean, loaded once through ref_import.load() with the process state that load() changes
    put back afterwards: working directory, sys.path, torch.Tensor.cuda, torch.cuda.comm.broadcast, yaml.load, the
    warning filters and the stub and reference modules in sys.modules."""
    if not _CLEAN and "ns" in ref_import._loaded:         # loaded (and its state kept) by someone else
        _CLEAN.append(ref_import._loaded["ns"].iuvmap.iuvmap_clean)
    if not _CLEAN:
        import torch.cuda.comm as comm
        import yaml
        saved = (os.getcwd(), list(sys.path), torch.Tensor.cuda, comm.broadcast, yaml.load, set(sys.modules))
        try:
            with warnings.catch_warnings():
                _CLEAN.append(ref_import.load().iuvmap.iuvmap_clean)
        finally:
            os.chdir(saved[0])
            sys.path[:] = saved[1]
            torch.Tensor.cuda, comm.broadcast, yaml.load = saved[2:5]
            for name in set(sys.modules) - saved[5]:
                f = getattr(sys.modules[name], "__file__", None)
                if f is None or os.path.abspath(f).startswith(ref_import.REF + os.sep):
                    del sys.modules[name]
            ref_import._loaded.pop("ns", None)           # a later load() sets its state up afresh
    return _CLEAN[0]


def zero_idxs(part_drop):
    """bool [B,24] -> the reference's zero_idxs: per image, the dropped DensePose parts 1..24 in increasing order"""
    return [[int(i) + 1 for i in torch.nonzero(row.cpu())] for row in part_drop]


def crop_channels(dp2smpl_mapping, part):
    """the (crop, channel) pairs the reference zeroes for DensePose part `part` (danet.py:269-271)"""
    return [(i, m_i + 1) for i, mapping in enumerate(dp2smpl_mapping) for m_i, map_idx in enumerate(mapping)
            if map_idx == part]


def part_drop_clean(u, v, index, ann, part_iuv_pred, part_drop=None):
    from danet_b200 import constants
    clean = _ref_iuvmap_clean()
    u_pred, v_pred, index_pred, part = (t.clone() for t in (u, v, index, part_iuv_pred))
    zero = zero_idxs(part_drop) if part_drop is not None else None
    if zero is not None:
        for bs in range(len(zero)):
            u_pred[bs, zero[bs]] *= 0
            v_pred[bs, zero[bs]] *= 0
            index_pred[bs, zero[bs]] *= 0
    u_cl, v_cl, index_cl, ann_cl = clean(u_pred, v_pred, index_pred, ann)
    if zero is not None:
        for bs in range(len(zero)):
            ch = [c for z in zero[bs] for c in crop_channels(constants.DP2SMPL_MAPPING, z)]
            part[bs, [c[0] for c in ch], :, [c[1] for c in ch]] *= 0
    maps = []
    for p in range(part.size(1)):
        pu, pv, pi_, _ = clean(part[:, p, 0], part[:, p, 1], part[:, p, 2])
        maps.append(torch.stack([pu, pv, pi_], dim=1))
    return u_cl, v_cl, index_cl, ann_cl, torch.stack(maps, dim=1)


def make_leaves(B, S, seed):
    """Seeded raw estimator maps with the values that decide the reference's corner cases: pixels whose Index logits
    are all negative (a dropped part's 0 wins), exact 0.0 / -0.0 ties, NaN and +-inf.
    Returns (u, v, index [B,25,S,S], ann [B,15,S,S], part_iuv_pred [B,24,3,7,S,S]) fp32 on the CPU."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    u, v, idx, ann, parts = r(B, 25, S, S), r(B, 25, S, S), r(B, 25, S, S), r(B, 15, S, S), r(B, 24, 3, 7, S, S)
    idx[:, :, 0, :] = -idx[:, :, 0, :].abs() - 0.01                  # row 0: negative-only logits
    parts[:, :, 2, :, 0, :] = -parts[:, :, 2, :, 0, :].abs() - 0.01
    idx[:, :, 1, 0] = 0.0                                             # exact ties of 0.0 and -0.0
    idx[:, 1::2, 1, 0] = -0.0
    idx[:, :, 1, 1] = -1.0
    idx[:, 3, 1, 1] = -0.0
    idx[:, 7, 1, 1] = 0.0
    parts[:, :, 2, :, 1, 0] = 0.0
    parts[:, :, 2, ::2, 1, 1] = -0.0
    ann[:, :, 1, 0] = 0.0
    for t, vals in ((u, (float("nan"), float("inf"), -float("inf"), -0.0)), (v, (float("nan"), -float("inf"))),
                    (idx, (float("nan"), float("inf"), -float("inf"))), (parts, (float("nan"), float("inf"), -0.0)),
                    (ann, (float("nan"),))):
        flat = t.view(-1)
        pos = torch.randint(0, flat.numel(), (4 * B * len(vals),), generator=g)
        for k, p in enumerate(pos.tolist()):
            flat[p] = vals[k % len(vals)]
    return u, v, idx, ann, parts


def make_probes(B, S, seed):
    """Upstream gradients G1 [B,75,S,S] (of cat[u_cl, v_cl, index_cl]) and G2 [B,24,3,7,S,S] (of the part maps), with
    -0.0 and +-inf entries"""
    g = torch.Generator().manual_seed(seed)
    G1, G2 = torch.randn(B, 75, S, S, generator=g), torch.randn(B, 24, 3, 7, S, S, generator=g)
    for t in (G1, G2):
        t[t > 1.2] = -0.0
        flat = t.view(-1)
        pos = torch.randint(0, flat.numel(), (4 * B,), generator=g)
        for k, p in enumerate(pos.tolist()):
            flat[p] = float("inf") if k % 2 else -float("inf")
    return G1, G2


def bits_equal(a, b):
    """the same fp32 bits everywhere, where NaN matches NaN (payloads differ between CPU and GPU arithmetic)"""
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    if a.shape != b.shape:
        return False
    same = (a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))
    return bool(same.all())


# ---------------------------------------------------------------------------------------------------------------------
# the op table of danet_b200.training.run_danet in torch (fp64 or fp32), with this file's part_drop_clean
# ---------------------------------------------------------------------------------------------------------------------
HEAD = "iuv2smpl.smpl_para_Outs."


def gcn_head_losses(out, target, gt_smpl_joints, has_smpl, rot_w=60.0, pos_w=1.0):
    """smpl_regressor.py:147-166 in torch (oracle/gcn_head.py's losses): rot_w * MSE over the selected images,
    pos_w * L1 sum / #selected for both coordinate outputs"""
    sel = (has_smpl == 1).to(target.dtype)
    n = sel.sum()
    pose0 = out["joint_rotation"][0]
    L = {"joint_rotation0": rot_w * (((pose0 - target[:, 13:]) * sel[:, None]) ** 2).sum() / (n * 216)}
    for k, c in enumerate(out["joint_position"]):
        L["joint_position%d" % k] = pos_w * ((c - gt_smpl_joints) * sel[:, None, None]).abs().sum() / n
    return L


class TorchSmpl(object):
    """SMPL forward in torch (oracle/lbs_grad.smpl_layer) with the call signature smpl_losses uses"""

    def __init__(self, model):
        self.model = model

    def __call__(self, betas, body_pose, global_orient, pose2rot=False):
        from oracle import lbs_grad
        assert not pose2rot
        R = torch.cat([global_orient, body_pose], 1)
        verts, _, joints = lbs_grad.smpl_layer(self.model, betas, R)
        return types.SimpleNamespace(vertices=verts, joints=joints)


def torch_table(state, smpl_model, training):
    """The op table of run_danet over `state` (the model's state_dict keys as torch tensors of one dtype; BatchNorm
    statistics updated in place): the estimator's ops of oracle/estimator_train.py, the branches' of
    oracle/regressor_train.py, part_drop_clean above, oracle/gcn_head.py's torch_head and losses, and smpl_losses over
    the torch SMPL layer of `smpl_model` (the model's numpy arrays)."""
    from danet_b200 import smpl as psmpl
    from danet_b200.iuvmap import draw_part_drop
    from oracle import gcn_head as og
    from oracle.estimator_train import TorchEstimatorOps
    ops = TorchEstimatorOps()
    P = {n: state[HEAD + n] for n in og.PARAM_NAMES}
    buf = {k: state[HEAD + k] for k in og.BUFFER_NAMES}
    bn = {n: (state[HEAD + n + ".running_mean"], state[HEAD + n + ".running_var"]) for n in og.BN_NAMES}

    def gcn_head(rot_feats, global_para):
        para, pose0, c0, c1 = og.torch_head(P, buf, bn, rot_feats, global_para, training)
        if not training:
            return {"para": para, "joint_rotation": [], "joint_position": []}
        with torch.no_grad():
            for n in og.BN_NAMES:
                state[HEAD + n + ".num_batches_tracked"].add_(1)
        return {"para": para, "joint_rotation": [pose0], "joint_position": [c0, c1]}
    ops.gcn_head = gcn_head
    ops.gcn_head_losses = gcn_head_losses
    ops.smpl_losses = functools.partial(psmpl.smpl_losses, TorchSmpl(smpl_model))
    ops.part_drop_clean = part_drop_clean
    ops.draw_part_drop = draw_part_drop
    return ops
