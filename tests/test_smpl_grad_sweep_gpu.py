"""GPU half of the SMPL backward sweep (tests/smpl_grad_sweep_common.py): every case's dbeta and dR, through
SMPL.backward_lbs and through autograd, held element by element to the bound against the fp64 reference of
oracle/lbs_grad.py; and the backward's determinism: bit-for-bit repeats, batch independence, CUDA-graph replay,
outputs written in full whatever the buffers held, and exact zeros from a zero gradient."""
import functools

import numpy as np
import pytest
import torch

from oracle import lbs as olbs
import fp64_bound as fb
import smpl_grad_sweep_common as sc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@functools.lru_cache(maxsize=None)
def _smpl(name):
    import danet_b200
    return danet_b200.SMPL(sc.model(name)).to(DEV)


def _d(t):
    return None if t is None else t.to(DEV)


def _backward_lbs(smpl, mdl, inp):
    gv, gs = sc.fold(mdl, inp)
    return smpl.backward_lbs(_d(inp.betas), _d(inp.R), _d(gv), _d(gs))


def _autograd(smpl, inp):
    b = _d(inp.betas).requires_grad_(True)
    R = _d(inp.R).requires_grad_(True)
    out = smpl(betas=b, body_pose=R[:, 1:], global_orient=R[:, :1], transl=_d(inp.transl), pose2rot=False)
    ys, gs = [], []
    for g, y in ((inp.gv, out.vertices), (inp.gs, out.smpl_joints), (inp.gj, out.joints)):
        if g is not None:
            ys.append(y)
            gs.append(_d(g))
    torch.autograd.backward(ys, gs)
    return b.grad, R.grad


@pytest.mark.parametrize("case", sc.CASES, ids=sc.case_id)
def test_case_meets_the_bound(case):
    mdl, smpl = sc.model(case.model), _smpl(case.model)
    inp = sc.make_inputs(case)
    idx = sc.bodies(case)
    ref = sc.reference(mdl, sc.subset(inp, idx), device=DEV)
    for route, got in (("backward_lbs", _backward_lbs(smpl, mdl, inp)), ("autograd", _autograd(smpl, inp))):
        got = [g[idx] for g in got]
        q = max(fb.worst(g, r, fb.U24 * M, fb.U24 * r.abs() + fb.TINY)[0] for g, (r, M) in zip(got, ref))
        e = max(fb.err_ratio(g, r, fb.U24 * M) for g, (r, M) in zip(got, ref))
        print("%s %s: worst |err| / (2^-24 M) = %.3g (C = %d)" % (sc.case_id(case), route, e, sc.C))
        assert q <= sc.C, (route, q)


def _b64():
    c = sc.Case("packed", 64, "both", "rot6d", "normal", 1.0)
    return sc.model("packed"), _smpl("packed"), sc.make_inputs(c)


def test_backward_lbs_is_bit_repeatable():
    mdl, smpl, inp = _b64()
    first = _backward_lbs(smpl, mdl, inp)
    for _ in range(3):
        again = _backward_lbs(smpl, mdl, inp)
        assert torch.equal(again[0], first[0]) and torch.equal(again[1], first[1])


def test_smpl_losses_gradient_is_bit_repeatable():
    from danet_b200.smpl import smpl_losses
    B = 64
    rng = np.random.default_rng(5)
    R = olbs.rot6d_to_rotmat(rng.normal(0, 1, (B * 24, 6))).reshape(B, 216)
    para = np.concatenate([np.stack([rng.uniform(0.6, 1.1, B), rng.normal(0, .05, B), rng.normal(0, .05, B)], 1),
                           rng.normal(0, 1, (B, 10)), R + rng.normal(0, 0.02, (B, 216))], 1)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32)).to(DEV)
    args = [t(para + rng.normal(0, 0.1, para.shape)),
            t(np.concatenate([rng.uniform(-1, 1, (B, 49, 2)), rng.uniform(0, 1, (B, 49, 1))], -1)),
            t(np.concatenate([rng.normal(0, .3, (B, 24, 3)), rng.uniform(0, 1, (B, 24, 1))], -1)),
            t(rng.normal(0, .5, (B, 6890, 3))), t(rng.integers(0, 2, B)), t(rng.integers(0, 2, B))]
    w = {"smpl_verts": 60.0}

    def grad():
        p = t(para).requires_grad_(True)
        sum(smpl_losses(_smpl("packed"), p, *args, weights=w).values()).backward()
        return p.grad
    first = grad()
    assert torch.isfinite(first).all()
    for _ in range(2):
        assert torch.equal(grad(), first)


def test_batch_independence():
    """body i's gradient inside a batch of 65 (three CTAs of the chain kernel) is the gradient of body i alone"""
    c = sc.Case("packed", 65, "both", "noisy", "pm5", 1.0)
    mdl, smpl = sc.model("packed"), _smpl("packed")
    inp = sc.make_inputs(c)
    gb, gR = _backward_lbs(smpl, mdl, inp)
    for i in range(c.B):
        b1, R1 = _backward_lbs(smpl, mdl, sc.subset(inp, [i]))
        assert torch.equal(b1[0], gb[i]) and torch.equal(R1[0], gR[i]), i


def _abi_call(smpl, B, betas, R, gv, gs, gb, gR, ws):
    from danet_b200 import _lib
    lib = _lib.load()
    h = smpl._handle(DEV)
    _lib.check(lib.danet_smpl_backward(h, B, _lib.ptr(betas), _lib.ptr(R), _lib.ptr(gv), _lib.ptr(gs), _lib.ptr(gb),
                                       _lib.ptr(gR), _lib.ptr(ws), _lib.stream_ptr(DEV)), "smpl_backward")


def _ws_bytes(smpl, B):
    from danet_b200 import _lib
    return int(_lib.load().danet_smpl_backward_workspace_bytes(smpl._handle(DEV), B))


def test_cuda_graph_replay_matches_eager():
    mdl, smpl, inp = _b64()
    B = inp.betas.shape[0]
    eager = _backward_lbs(smpl, mdl, inp)                   # creates the handle
    gv, gs = sc.fold(mdl, inp)
    betas, R, gv, gs = _d(inp.betas), _d(inp.R), _d(gv), _d(gs)
    ws = torch.empty(_ws_bytes(smpl, B), dtype=torch.uint8, device=DEV)
    gb = torch.empty(B, betas.shape[1], device=DEV)
    gR = torch.empty(B, 24, 3, 3, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _abi_call(smpl, B, betas, R, gv, gs, gb, gR, ws)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _abi_call(smpl, B, betas, R, gv, gs, gb, gR, ws)
    gb.fill_(float("nan"))
    gR.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gb, eager[0]) and torch.equal(gR, eager[1])


@pytest.mark.parametrize("name,B", [("packed", 33), ("nv129", 3), ("dense", 2)])
def test_outputs_fully_written(name, B):
    """workspace and outputs pre-filled with NaN: the results equal a normal call"""
    c = sc.Case(name, B, "both", "rot6d", "normal", 1.0)
    mdl, smpl = sc.model(name), _smpl(name)
    inp = sc.make_inputs(c)
    want = _backward_lbs(smpl, mdl, inp)
    gv, gs = sc.fold(mdl, inp)
    ws = torch.full((_ws_bytes(smpl, B),), 0xFF, dtype=torch.uint8, device=DEV)     # every float in it is a NaN
    gb = torch.full((B, inp.betas.shape[1]), float("nan"), device=DEV)
    gR = torch.full((B, 24, 3, 3), float("nan"), device=DEV)
    _abi_call(smpl, B, _d(inp.betas), _d(inp.R), _d(gv), _d(gs), gb, gR, ws)
    torch.cuda.synchronize()
    assert torch.equal(gb, want[0]) and torch.equal(gR, want[1])


@pytest.mark.parametrize("with_joints", [True, False])
def test_zero_gradient_gives_exact_zeros(with_joints):
    c = sc.Case("packed", 33, "both", "gaussian", "pm5", 1.0)
    smpl, inp = _smpl("packed"), sc.make_inputs(c)
    gb, gR = smpl.backward_lbs(_d(inp.betas), _d(inp.R), torch.zeros(33, 6890, 3, device=DEV),
                               torch.zeros(33, 24, 3, device=DEV) if with_joints else None)
    assert (gb == 0).all() and (gR == 0).all()
