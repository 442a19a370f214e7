"""The regressor branch drivers without a GPU: the graph walk, driven through the fp64 test double, reproduces the
reference's DecomposedPredictor (outputs, running statistics, every gradient sketch); the lowered op list consumes every
branch key exactly once; the new C entries refuse bad arguments before any launch; and the new layers and public
functions refuse what they do not support with ValueError."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import regressor_train as ort
from regressor_train_common import (BRANCH_PREFIXES, RP, branch_param_keys, bn2d_names, double_step, golden,
                                    golden_inputs)

TOL = 1e-9


@pytest.fixture(scope="module")
def gold():
    return golden()


@pytest.fixture(scope="module")
def keyed():
    return ort.keyed_state(0)


def test_golden_layout(gold, keyed):
    state, _ = keyed
    body, part = golden_inputs(gold)
    np.testing.assert_allclose(ort.input_checksum(body), gold["checksum_body_iuv"], rtol=1e-12)
    np.testing.assert_allclose(ort.input_checksum(part), gold["checksum_part_iuv"], rtol=1e-12)
    assert tuple(body.shape) == (2, 75, 56, 56) and tuple(part.shape) == (2, 24, 3, 7, 56, 56)
    sk = {k[3:] for k in gold.files if k.startswith("sk_")}
    branch = set(branch_param_keys(state))
    assert len(branch) == 128
    from danet_b200.regressor import PARAM_NAMES
    assert sk == branch | {RP + n for n in PARAM_NAMES} | {"body_iuv", "part_iuv"}
    bn = {k[4:] for k in gold.files if k.startswith("nbt_")}
    assert len(bn) == 47 and set(bn2d_names(state)) <= bn and len(bn2d_names(state)) == 42
    assert all(int(gold["nbt_" + n]) == 1 for n in bn)
    assert os.path.getsize(os.path.join(os.path.dirname(__file__), "golden", "regressor_train.npz")) < 4 << 20


def test_double_walk_reproduces_reference_golden(gold, keyed):
    """fp64 torch ops through the product's lowering and walk against the reference's own modules"""
    state = {k: v.clone() for k, v in keyed[0].items()}
    for n in bn2d_names(state):
        np.testing.assert_array_equal(state[n + ".running_mean"].numpy(), gold["rm0_" + n])
        np.testing.assert_array_equal(state[n + ".running_var"].numpy(), gold["rv0_" + n])
    body, part = golden_inputs(gold)
    gp, rf, grads = double_step(state, keyed[1], body, part, True, gold["g_global_para"], gold["g_rot_feats"])
    assert ort.rel_norm(gp, gold["global_para"]) < TOL
    assert ort.rel_norm(rf, gold["rot_feats"]) < TOL
    assert len(grads) == 130
    worst = max((ort.sketch_error(ort.sketch(k, g), gold["sk_" + k], g.numel()), k) for k, g in grads.items())
    assert worst[0] < TOL, worst
    for n in bn2d_names(state):
        assert ort.rel_norm(state[n + ".running_mean"], gold["rm1_" + n]) < TOL, n
        assert ort.rel_norm(state[n + ".running_var"], gold["rv1_" + n]) < TOL, n
        assert int(state[n + ".num_batches_tracked"]) == int(gold["nbt_" + n])


def test_lowered_ops_consume_every_branch_key_once(keyed):
    from danet_b200 import netgraph
    from danet_b200.regressor import lower_branches
    g = netgraph.danet_graph(48)
    low = lower_branches(g)
    assert lower_branches(g) is low                        # lowered once per graph
    ops = low["body"]["ops"] + low["limb"]["ops"]
    kinds = [op["op"] for op in ops]
    assert {k: kinds.count(k) for k in set(kinds)} == {"conv2d": 42, "batch_norm": 42, "max_pool2d": 2, "linear": 1,
                                                       "adaptive_avg_pool2d": 2}
    used = [k for op in ops for k in op["keys"]]
    branch_keys = sorted(k for k in g.params if k.startswith(BRANCH_PREFIXES))
    assert len(used) == len(set(used))
    assert sorted(k for k in used if k.startswith(BRANCH_PREFIXES)) == branch_keys
    assert [k for k in used if not k.startswith(BRANCH_PREFIXES)] == [RP + "mean_cam_shape"]     # the linear's add term
    # layout: limb_reslayer's grouped ops take [B, 24C, H, W]; limb_net and body_net stay per image
    for op in ops:
        if "groups" in op:
            assert op["groups"] == (24 if ".limb_reslayer." in (op.get("weight") or op.get("bn")) else 1), op
    bn = {op["bn"]: op for op in ops if op["op"] == "batch_norm"}
    assert bn[RP + "limb_net.1"]["groups"] == 1 and bn[RP + "limb_reslayer.layer4.0.bn2"]["groups"] == 24
    assert bn[RP + "limb_reslayer.layer4.0.bn2"]["res"] is not None and bn[RP + "limb_reslayer.layer4.0.bn2"]["relu"]
    assert not bn[RP + "limb_reslayer.layer4.0.downsample.1"]["relu"]


def test_eval_mode_walk_leaves_statistics(keyed):
    state = {k: v.clone() for k, v in keyed[0].items()}
    body, part = ort.make_inputs(1, 24, 5)
    double_step(state, keyed[1], body, part, False)
    for k, v in keyed[0].items():
        assert torch.equal(state[k], v), k


@pytest.fixture(scope="module")
def lib():
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "danet-densepose2smpl_b200",
                      "libdanet_b200.so")
    if not os.path.exists(so):
        import __graft_entry__
        __graft_entry__.build()
    from danet_b200 import _lib
    return _lib.load()


def _err(lib):
    return lib.danet_last_error().decode()


def _fake(n):
    return [ctypes.c_void_p(0x100000 * (i + 1)) for i in range(n)]


def test_library_exports_the_tail_backward_entries(lib):
    from danet_b200 import _lib
    for sym in ("danet_global_avgpool_backward", "danet_linear_backward"):
        assert hasattr(lib, sym) and sym in _lib.SIGNATURES, sym


def test_avgpool_backward_host_checks(lib):
    dy, dx = _fake(2)
    for args, msg in [((0, 4, dy, dx), "bad sizes"), ((4, 0, dy, dx), "bad sizes"), ((1 << 16, 1 << 15, dy, dx), "bad sizes"),
                      ((4, 4, None, dx), "non-null"), ((4, 4, dy, None), "non-null")]:
        assert lib.danet_global_avgpool_backward(*args, None) < 0, args
        assert msg in _err(lib), (args, _err(lib))


def test_linear_backward_host_checks(lib):
    x, w, dy, dx, dw, db = _fake(6)

    def call(N=2, In=512, Out=13, x=x, w=w, dy=dy, dx=dx, dw=dw, db=db):
        return lib.danet_linear_backward(N, In, Out, x, w, dy, dx, dw, db, None)
    for bad, msg in [(dict(N=0), "bad sizes"), (dict(In=-1), "bad sizes"), (dict(Out=0), "bad sizes"),
                     (dict(N=1 << 16, In=1 << 15), "bad sizes"), (dict(dy=None), "dy must be non-null"),
                     (dict(w=None), "dx needs the weight"), (dict(x=None), "dw needs the input")]:
        assert call(**bad) < 0, bad
        assert msg in _err(lib), (bad, _err(lib))
    assert call(dx=None, dw=None, db=None) == 0              # nothing asked: nothing launched


def test_tail_layers_refuse_unsupported_inputs():
    from danet_b200.layers import adaptive_avg_pool2d, linear
    x = torch.randn(2, 3, 4, 4)
    with pytest.raises(ValueError, match="CUDA tensor"):
        adaptive_avg_pool2d(x, 1)
    with pytest.raises(ValueError, match="output_size=1"):
        adaptive_avg_pool2d(x, 2)
    with pytest.raises(ValueError, match="float32"):
        adaptive_avg_pool2d(x.double(), 1)
    with pytest.raises(ValueError, match="4-D"):
        adaptive_avg_pool2d(x.view(2, 3, 16), (1, 1))
    with pytest.raises(ValueError, match="contiguous"):
        adaptive_avg_pool2d(x.transpose(2, 3), 1)
    a, w, b = torch.randn(2, 5), torch.randn(3, 5), torch.randn(3)
    with pytest.raises(ValueError, match="CUDA tensor"):
        linear(a, w, b)
    with pytest.raises(ValueError, match="weight must be"):
        linear(a, w[:, :4].contiguous(), b)
    with pytest.raises(ValueError, match="2-D"):
        linear(a.view(2, 5, 1), w, b)
    with pytest.raises(ValueError, match="shape"):
        linear(a, w, b[:2])
    with pytest.raises(ValueError, match="shape"):
        linear(a, w, b, add=torch.zeros(4))
    with pytest.raises(ValueError, match="float32"):
        linear(a, w, b.double())
