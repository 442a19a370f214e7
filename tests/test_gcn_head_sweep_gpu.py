"""GPU half of the regressor head sweep (tests/gcn_head_sweep_common.py): every case through the C entries of
csrc/gcn_train.cu with every stage held to its per-element bound against fp64 computed from the values the kernels were
fed; the same bits from the autograd ops (gcn_head + gcn_head_losses), from a repeat and from NaN-prefilled outputs
and workspace; and the NaN policy against torch fp32 on the non-finite cases."""
import ctypes

import pytest
import torch

import fp64_bound as fb
import gcn_head_sweep_common as gs
from oracle import gcn_head as og

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _dev(inp):
    t = lambda x: None if x is None else x.to(DEV).contiguous()
    out = {k: t(v) for k, v in inp.items() if k not in ("P", "buf", "bn")}
    out["P"] = {k: t(v) for k, v in inp["P"].items()}
    out["buf"] = {k: t(v) for k, v in inp["buf"].items()}
    out["bn"] = {k: (t(a), t(b)) for k, (a, b) in inp["bn"].items()}
    return out


def run_c(c, di, fill):
    """forward, losses and backward through the C entries into outputs and a workspace prefilled with `fill`; returns
    {stage name: fp32 tensor}"""
    from danet_b200 import _lib
    from danet_b200.regressor import _pack
    lib = _lib.load()
    B, tr = c.B, int(c.train)
    e = lambda *s: torch.full(s, fill, device=DEV)
    P = di["P"]
    params = [P[n] for n in og.PARAM_NAMES]
    bufs = [di["bn"][n][0] for n in og.BN_NAMES] + [di["bn"][n][1] for n in og.BN_NAMES] + \
        [di["buf"][k] for k in ("r2p_A", "p2r_A", "I_n", "A_mask", "mean_pose")]
    train_only = ("pose_regressors.0", "coord_regressors")
    grads = [None if (not c.train and n.startswith(train_only)) else e(*P[n].shape) for n in og.PARAM_NAMES]
    nbytes = lib.danet_gcn_head_train_workspace_bytes(B)
    ws = e(nbytes // 4)
    para, stats = e(B, 229), e(2, 5, 24)
    pose0, c0, c1 = (e(B, 216), e(B, 24, 3), e(B, 24, 3)) if c.train else (None, None, None)
    ptr, st = _lib.ptr, _lib.stream_ptr(DEV)
    p = _pack(params, bufs)
    _lib.check(lib.danet_gcn_head_train_forward(B, ctypes.byref(p), tr, ptr(di["rot"]), ptr(di["gpara"]), ptr(para),
                                                ptr(pose0), ptr(c0), ptr(c1), ptr(stats if c.train else None), ptr(ws), st),
               "forward")
    got = {}
    if c.train:
        losses, gl = e(3), (e(B, 216), e(B, 24, 3), e(B, 24, 3))
        has = di["has"].to(torch.uint8)
        _lib.check(lib.danet_gcn_head_losses(B, ptr(pose0), ptr(c0), ptr(c1), ptr(di["target"]), ptr(di["gt"]), ptr(has),
                                             gs.ROT_W, gs.POS_W, ptr(losses), *map(ptr, gl), st), "losses")
        got.update(loss0=losses[0], loss1=losses[1], loss2=losses[2], g_pose0_loss=gl[0], g_coord0_loss=gl[1],
                   g_coord1_loss=gl[2], pose0=pose0, coord0=c0, coord1=c1)
        for l in range(5):
            got["rm%d" % l], got["rv%d" % l] = stats[0, l], stats[1, l]
    g_rot, g_gp = e(B, 24, 128), e(B, 13)
    pg = _pack(params, bufs, grads)
    _lib.check(lib.danet_gcn_head_train_backward(B, ctypes.byref(pg), tr, ptr(di["rot"]), ptr(di["g_para"]),
                                                 ptr(di["g_pose0"]), ptr(di["g_coord0"]), ptr(di["g_coord1"]), ptr(g_rot),
                                                 ptr(g_gp), ptr(ws), st), "backward")
    torch.cuda.synchronize()
    R = gs.regions(ws, B)
    skip = ("dA", "sums") if c.train else ("dA", "sums", "p6_0", "dp6_0")     # eval has no pose0 head
    got.update({k: v for k, v in R.items() if k not in skip})
    for l in (1, 2, 3):
        got["dA%d" % l] = R["dA"][l - 1]
    got.update(paraglob=para[:, :13], pararot=para[:, 13:], g_rot_feats=g_rot, g_global_para=g_gp)
    for n, g in zip(og.PARAM_NAMES, grads):
        if g is not None:
            from test_gcn_head_sweep_cpu import grad_stage
            got[grad_stage(n)] = g
    return got


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("c", gs.CASES, ids=gs.case_id)
def test_case_stages_and_bits(c):
    inp = gs.make_case(c)
    di = _dev(inp)
    got = run_c(c, di, float("nan"))
    S = gs.stages(c, inp, got, device=DEV)
    worst = {n: fb.err_ratio(got[n], st.r, gs.bound(st)[0]) for n, st in S.items() if not n.startswith("_") and n in got}
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("%s worst |err|/(2^-24 M): %s" % (gs.case_id(c), ", ".join("%s %.3g" % kv for kv in top)))
    bad = gs.check(got, S)
    assert not bad, bad
    # a repeat into zero-filled outputs and workspace gives the same bits (no stage reads what it did not write)
    again = run_c(c, di, 0.0)
    diff = [k for k in got if not _same_bits(got[k], again[k])]
    assert not diff, diff


def _net():
    from danet_b200 import build_synthetic_danet
    return build_synthetic_danet(width=32, seed=0, device=DEV)


@pytest.fixture(scope="module")
def net():
    return _net()


@pytest.mark.parametrize("c", gs.CASES, ids=gs.case_id)
def test_autograd_ops_give_the_c_entries_bits(net, c):
    from danet_b200.regressor import PARAM_NAMES, TRAINING_ONLY, gcn_head, gcn_head_losses
    inp = gs.make_case(c)
    di = _dev(inp)
    ref = run_c(c, di, float("nan"))
    mod = net.iuv2smpl.smpl_para_Outs
    with torch.no_grad():
        for n in PARAM_NAMES:
            mod.get_parameter(n).copy_(di["P"][n])
        for k in ("r2p_A", "p2r_A", "I_n", "A_mask", "mean_pose"):
            b = mod.get_buffer(k)
            b.copy_(di["buf"][k].view(b.shape))
        for n, (rm, rv) in di["bn"].items():
            m = mod.get_submodule(n)
            m.running_mean.copy_(rm)
            m.running_var.copy_(rv)
    net.train(c.train)
    try:
        rot, gp = di["rot"].clone().requires_grad_(), di["gpara"].clone().requires_grad_()
        out = gcn_head(net, rot, gp)
        tot = (out["para"] * di["g_para"]).sum()
        names = [n for n in PARAM_NAMES if c.train or n not in TRAINING_ONLY]
        checks = {"pararot": out["para"][:, 13:], "paraglob": out["para"][:, :13]}
        if c.train:
            L = gcn_head_losses(out, di["target"], di["gt"], di["has"])
            p0, (c0, c1) = out["joint_rotation"][0], out["joint_position"]
            checks.update(pose0=p0, coord0=c0, coord1=c1, loss0=L["joint_rotation0"], loss1=L["joint_position0"],
                          loss2=L["joint_position1"])
            for l, n in enumerate(og.BN_NAMES):
                checks["rm%d" % l] = mod.get_submodule(n).running_mean
                checks["rv%d" % l] = mod.get_submodule(n).running_var
            tot = tot + (p0 * di["g_pose0"]).sum() + (c0 * di["g_coord0"]).sum() + (c1 * di["g_coord1"]).sum()
        g = torch.autograd.grad(tot, [mod.get_parameter(n) for n in names] + [rot, gp])
    finally:
        net.eval()
    from test_gcn_head_sweep_cpu import grad_stage
    for n, t in zip(names + ["rot_feats", "global_para"], g):
        checks[grad_stage(n)] = t
    diff = [k for k, v in checks.items() if not _same_bits(v.detach().reshape(ref[k].shape), ref[k])]
    assert not diff, diff


NONFINITE = [c for c in gs.CASES if c.nonfinite or c.adj == "nan"]


@pytest.mark.parametrize("c", NONFINITE, ids=gs.case_id)
def test_nan_reaches_where_torch_sends_it(c):
    inp = gs.make_case(c)
    di = _dev(inp)
    got = run_c(c, di, 0.0)
    P = {k: v.clone().requires_grad_() for k, v in di["P"].items()}
    buf = {k: v.view(1, 144) if k == "mean_pose" else v.view(1, 24, 24) for k, v in di["buf"].items()}
    bn = {k: (a.clone(), b.clone()) for k, (a, b) in di["bn"].items()}
    rot, gp = di["rot"].clone().requires_grad_(), di["gpara"].clone().requires_grad_()
    para, p0, c0, c1 = og.torch_head(P, buf, bn, rot, gp, training=c.train)
    tot = (para * di["g_para"]).sum()
    if c.train:
        tot = tot + (p0 * di["g_pose0"]).sum() + (c0 * di["g_coord0"]).sum() + (c1 * di["g_coord1"]).sum()
    names = [n for n in og.PARAM_NAMES if c.train or not n.startswith(("pose_regressors.0", "coord_regressors"))]
    g = torch.autograd.grad(tot, [P[n] for n in names] + [rot, gp], allow_unused=True)
    from test_gcn_head_sweep_cpu import grad_stage
    want = {"pararot": para[:, 13:], "paraglob": para[:, :13]}
    want.update({grad_stage(n): t for n, t in zip(names + ["rot_feats", "global_para"], g) if t is not None})
    assert any(bool(torch.isnan(t).any()) for t in want.values())
    diff = [k for k, t in want.items() if not torch.equal(torch.isnan(t.detach()).reshape(got[k].shape), torch.isnan(got[k]))]
    assert not diff, diff


def test_oversized_batch_raises_before_allocating(net):
    from danet_b200.regressor import gcn_head
    B = 174761                                            # expanded views: no storage behind the batch
    rot = torch.zeros(1, 24, 128, device=DEV).expand(B, 24, 128)
    gp = torch.zeros(1, 13, device=DEV).expand(B, 13)
    before = torch.cuda.memory_allocated(DEV)
    with pytest.raises(ValueError, match="batch size"):
        gcn_head(net, rot, gp)
    assert torch.cuda.memory_allocated(DEV) == before
