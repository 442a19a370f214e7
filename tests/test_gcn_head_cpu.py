"""CPU tests of the regressor head's training path: the fp64 restatement (oracle/gcn_head.py) against the golden the
reference's own DecomposedPredictor.forward produced under autograd (oracle/gen_golden_gcn_head.py), and the exports
of the library built here."""
import ctypes
import os

import numpy as np
import pytest

from oracle import gcn_head as og
from gcn_head_common import ROOT, golden, golden_params, rel_norm


@pytest.fixture(scope="module")
def gold():
    return golden()


def _oracle_step(g, P, buf, bn):
    out, sv = og.forward(P, buf, bn, g["rot_feats"], g["global_para"], training=True)
    L, (gp0, gc0, gc1) = og.losses(out["pose0"], out["coord0"], out["coord1"], g["target"], g["gt_joints"], g["has_smpl"])
    grads = og.backward(P, sv, {"para": g["G"], "pose0": gp0, "coord0": gc0, "coord1": gc1}, training=True)
    return out, L, grads


def test_golden_records_every_parameter_gradient(gold):
    names = {k[2:] for k in gold.files if k.startswith("g_")}
    assert names == set(og.PARAM_NAMES) | {"rot_feats", "global_para"}
    assert len(og.PARAM_NAMES) == 29
    assert sum(gold["g_" + n].size for n in og.PARAM_NAMES) == 221280
    assert (gold["edge_importance"] < 0).sum() >= 12
    assert list(gold["has_smpl"]) == [1, 0, 1, 1]


def test_restatement_reproduces_reference_golden(gold):
    g = gold
    P, buf, bn = golden_params(g)
    out, L, grads = _oracle_step(g, P, buf, bn)
    for k in ("para", "pose0", "coord0", "coord1"):
        np.testing.assert_allclose(out[k], g[k], atol=2e-5, rtol=1e-5, err_msg=k)
    np.testing.assert_allclose(L, [g["L_joint_rotation0"], g["L_joint_position0"], g["L_joint_position1"]], rtol=2e-6)
    for n in og.PARAM_NAMES + ["rot_feats", "global_para"]:
        assert grads[n].shape == g["g_" + n].shape, n
        assert rel_norm(grads[n], g["g_" + n]) < 2e-5, (n, rel_norm(grads[n], g["g_" + n]))
    for n in og.BN_NAMES:
        np.testing.assert_allclose(out["bn"][n][0], g["rm1_" + n], atol=1e-6)
        np.testing.assert_allclose(out["bn"][n][1], g["rv1_" + n], atol=1e-6)
        assert int(g["nbt_" + n]) == 1


def test_restatement_eval_mode_and_no_selection_against_torch_fp64(gold):
    """Eval mode (frozen BatchNorm) and the all-deselected losses, where the reference itself raises: the fp64 numpy
    backward against torch autograd over the fp64 torch restatement."""
    import torch
    g = gold
    P, buf, bn = golden_params(g)
    for training in (False, True):
        out, sv = og.forward(P, buf, bn, g["rot_feats"], g["global_para"], training=training)
        grads_in = {"para": g["G"]}
        if training:
            L, (gp0, gc0, gc1) = og.losses(out["pose0"], out["coord0"], out["coord1"], g["target"], g["gt_joints"],
                                           np.zeros(4))
            assert not L.any() and not any(x.any() for x in (gp0, gc0, gc1))
            rng = np.random.default_rng(5)
            grads_in.update(pose0=rng.normal(0, 1, (4, 216)), coord0=rng.normal(0, 1, (4, 24, 3)),
                            coord1=rng.normal(0, 1, (4, 24, 3)))
        G = og.backward(P, sv, grads_in, training=training)
        t = lambda x: torch.tensor(np.asarray(x, np.float64))
        Pt = {k: t(v).requires_grad_() for k, v in P.items()}
        bnt = {k: (t(v[0]), t(v[1])) for k, v in bn.items()}
        rot, gp = t(g["rot_feats"]).requires_grad_(), t(g["global_para"]).requires_grad_()
        para, p0, c0, c1 = og.torch_head(Pt, {k: t(v) for k, v in buf.items()}, bnt, rot, gp, training)
        np.testing.assert_allclose(para.detach().numpy(), out["para"], atol=1e-12)
        tot = (para * t(g["G"])).sum()
        if training:
            tot = tot + (p0 * t(grads_in["pose0"])).sum() + (c0 * t(grads_in["coord0"])).sum() + (c1 * t(grads_in["coord1"])).sum()
        names = [n for n in og.PARAM_NAMES if training or not n.startswith(("pose_regressors.0", "coord_regressors"))]
        ref = torch.autograd.grad(tot, [Pt[n] for n in names] + [rot, gp])
        for n, r in zip(names + ["rot_feats", "global_para"], ref):
            assert rel_norm(G[n], r.numpy()) < 1e-10, (training, n)


def test_library_exports_training_entries():
    lib_path = os.path.join(ROOT, "danet-densepose2smpl_b200", "libdanet_b200.so")
    if not os.path.exists(lib_path):
        pytest.skip("library not built")
    lib = ctypes.CDLL(lib_path)
    for sym in ("danet_gcn_head_train_forward", "danet_gcn_head_train_backward", "danet_gcn_head_train_workspace_bytes",
                "danet_gcn_head_losses"):
        assert hasattr(lib, sym), sym
    from danet_b200 import _lib
    for sym in ("danet_gcn_head_train_forward", "danet_gcn_head_train_backward", "danet_gcn_head_train_workspace_bytes",
                "danet_gcn_head_losses"):
        assert sym in _lib.SIGNATURES
    lib.danet_gcn_head_train_workspace_bytes.restype = ctypes.c_int64
    lib.danet_gcn_head_train_workspace_bytes.argtypes = [ctypes.c_int32]
    assert lib.danet_gcn_head_train_workspace_bytes(16) > lib.danet_gcn_head_train_workspace_bytes(1) > 0
