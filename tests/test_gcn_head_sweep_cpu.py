"""CPU half of the regressor head sweep (tests/gcn_head_sweep_common.py): coverage, the per-stage fp64 references
composed end to end against torch fp64 autograd over oracle/gcn_head.py's torch_head, the workspace mirror against the
library, the batch-size refusal, and fp32 emulations that show the bound catches a set of wrong kernels and passes
the right ones."""
import ctypes
import os

import pytest
import torch

import fp64_bound as fb
import gcn_head_sweep_common as gs
from oracle import gcn_head as og

LIB = os.path.join(gs.ROOT, "danet-densepose2smpl_b200", "libdanet_b200.so")
# finite cases; at |mean| / std = 2^20 torch's own fp64 batch_norm (an unshifted variance) loses more than 1e-10
COMPOSE = [c for c in gs.CASES if c.B <= 16 and not c.nonfinite and c.adj != "nan" and c.bn != "ratio20"]


def test_every_class_has_a_case():
    assert fb.uncovered(gs.CASES, gs.CLASSES) == []


def _autograd(c, inp):
    """torch fp64 autograd over og.torch_head: outputs, new running statistics and every gradient"""
    d = lambda t: t.double().clone()
    P = {k: d(v).requires_grad_() for k, v in inp["P"].items()}
    buf = {k: d(v).view(1, 144) if k == "mean_pose" else d(v).view(1, 24, 24) for k, v in inp["buf"].items()}
    bn = {k: (d(a), d(b)) for k, (a, b) in inp["bn"].items()}
    rot, gp = d(inp["rot"]).requires_grad_(), d(inp["gpara"]).requires_grad_()
    para, p0, c0, c1 = og.torch_head(P, buf, bn, rot, gp, training=c.train)
    tot = (para * d(inp["g_para"])).sum()
    if c.train:
        tot = tot + (p0 * d(inp["g_pose0"])).sum() + (c0 * d(inp["g_coord0"])).sum() + (c1 * d(inp["g_coord1"])).sum()
    names = [n for n in og.PARAM_NAMES if c.train or not n.startswith(("pose_regressors.0", "coord_regressors"))]
    g = torch.autograd.grad(tot, [P[n] for n in names] + [rot, gp], allow_unused=True)
    G = dict(zip(names + ["rot_feats", "global_para"], g))
    return dict(para=para.detach(), pose0=p0, coord0=c0, coord1=c1, bn=bn), G


def grad_stage(name):
    """the stage that holds the gradient of parameter `name`"""
    for l, (n, i) in enumerate(og.LAYERS):
        for suffix, st in ((".gc.%d.weight" % i, "gW%d"), (".gc.%d.bias" % i, "gb%d"), (".act.%d.0.weight" % i, "g_bn_weight%d"),
                           (".act.%d.0.bias" % i, "g_bn_bias%d")):
            if name == n + suffix:
                return st % l
    m = {"edge_importance": "g_edge_importance", "rot_feats": "g_rot_feats", "global_para": "g_global_para"}
    for k in range(2):
        m["pose_regressors.%d.1.weight" % k], m["pose_regressors.%d.1.bias" % k] = "g_pose%d_w" % k, "g_pose%d_b" % k
        m["coord_regressors.%d.1.weight" % k], m["coord_regressors.%d.1.bias" % k] = "g_coord%d_w" % k, "g_coord%d_b" % k
    return m[name]


def _close(a, b, what):
    a, b = a.double().reshape(b.shape), b.double()
    tol = 1e-10 * max(float(b.abs().max()), 1e-300)
    assert float((a - b).abs().max()) <= tol, (what, float((a - b).abs().max()), tol)


@pytest.mark.parametrize("c", COMPOSE, ids=gs.case_id)
def test_composed_reference_matches_torch_autograd(c):
    inp = gs.make_case(c)
    S = gs.stages(c, inp)
    out, G = _autograd(c, inp)
    _close(torch.cat([S["paraglob"].r, S["pararot"].r], 1), out["para"], "para")
    if c.train:
        _close(S["pose0"].r, out["pose0"].detach(), "pose0")
        _close(S["coord0"].r, out["coord0"].detach(), "coord0")
        _close(S["coord1"].r, out["coord1"].detach(), "coord1")
        for l, n in enumerate(og.BN_NAMES):
            _close(S["rm%d" % l].r, out["bn"][n][0], "rm%d" % l)
            _close(S["rv%d" % l].r, out["bn"][n][1], "rv%d" % l)
        ref = og.forward({k: v.double().numpy() for k, v in inp["P"].items()},
                         gs.np_buffers(inp["buf"]),
                         {k: (a.double().numpy(), b.double().numpy()) for k, (a, b) in inp["bn"].items()},
                         inp["rot"].double().numpy(), inp["gpara"].double().numpy())[0]
        L, (gp0, gc0, gc1) = og.losses(ref["pose0"], ref["coord0"], ref["coord1"], inp["target"].numpy(),
                                       inp["gt"].numpy(), inp["has"].numpy())
        for k in range(3):
            _close(S["loss%d" % k].r, torch.tensor(L[k]), "loss%d" % k)
        _close(S["g_pose0_loss"].r, torch.from_numpy(gp0), "g_pose0_loss")
    for n, g in G.items():
        st = S[grad_stage(n)].r
        _close(st, g if g is not None else torch.zeros_like(st), n)


# ----------------------------------------------------------------------------------------------------------------------
# the library's workspace size and batch-size refusal (no device work: these run without a GPU)
# ----------------------------------------------------------------------------------------------------------------------
def _lib():
    if not os.path.exists(LIB):
        pytest.skip("libdanet_b200.so is not built")
    from danet_b200 import _lib as L
    try:
        return L.load()
    except OSError as e:                                  # no CUDA runtime to load it against
        pytest.skip("libdanet_b200.so does not load here: %s" % e)


def test_workspace_mirror_matches_library():
    lib = _lib()
    for B in range(1, 601):
        assert gs.layout(B)[1] * 4 == lib.danet_gcn_head_train_workspace_bytes(B), B
    assert lib.danet_gcn_head_train_workspace_bytes(174760) == gs.layout(174760)[1] * 4
    assert lib.danet_gcn_head_train_workspace_bytes(174761) == 0
    assert lib.danet_gcn_head_train_workspace_bytes(0) == 0


def test_oversized_batch_is_refused_before_any_launch():
    lib = _lib()
    from danet_b200 import _lib as L
    p = L.GcnTrainParams()                                # null pointers: the batch check comes first
    junk = ctypes.c_void_p(16)
    for B in (174761, 349526, 2 ** 31 - 1):
        rc = lib.danet_gcn_head_train_forward(B, ctypes.byref(p), 1, *([junk] * 8), None)
        assert rc != 0 and b"batch size" in lib.danet_last_error(), B
        rc = lib.danet_gcn_head_train_backward(B, ctypes.byref(p), 1, *([junk] * 8), None)
        assert rc != 0 and b"batch size" in lib.danet_last_error(), B


# ----------------------------------------------------------------------------------------------------------------------
# fp32 emulations: the clean one stays well inside the bound, each seeded defect breaks it
# ----------------------------------------------------------------------------------------------------------------------
def emulate(c, inp, defect=None):
    """fp32 stage outputs: every stage computed in fp32 (torch's own order) from the fp32 outputs of the stages before
    it, with `defect` applied to one stage"""
    S = gs.stages(c, inp, dtype=torch.float32, defect=defect)
    return {k: v.r.float() for k, v in S.items() if not k.startswith("_")}


DEFECTS = {
    "gemm K tail dropped (dW)": ("gW2", dict(B=5)),
    "M-tail row skipped (forward gemm)": ("Y1", dict(B=5)),
    "A in place of A^T in the backward adj_mul": ("gH1", dict(B=3)),
    "residual share missing in g_H[0]": ("gH0", dict(B=3)),
    "N in place of N - 1 in the running variance": ("rv0", dict(B=2)),
    "batch statistics in eval mode": ("invstd0", dict(B=3, train=False)),
    "rot6d backward without -dd gu": ("dp6_1", dict(B=2)),
    "k_adj_bwd without the degree term": ("g_edge_importance", dict(B=3)),
    "k_colsum over 24 B - 1 rows": ("gb3", dict(B=3)),
    "losses divided by B": ("loss1", dict(B=5, has="some")),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_bound_catches_defect(defect):
    stage, kw = DEFECTS[defect]
    c = gs.case(**kw)
    inp = gs.make_case(c)
    got = emulate(c, inp, defect)
    bad = [b[0] for b in gs.check(got, gs.stages(c, inp, got))]
    assert stage in bad, (defect, bad)


@pytest.mark.parametrize("c", [gs.case(5), gs.case(3, False), gs.case(2, has="some", r6="par10"),
                               gs.case(8, bn="ratio20")], ids=gs.case_id)
def test_clean_emulation_stays_well_inside(c):
    inp = gs.make_case(c)
    got = emulate(c, inp)
    S = gs.stages(c, inp, got)
    for name, st in S.items():
        if name.startswith("_") or st.kind == "exact":
            continue
        scale, floor, lim = gs.bound(st)
        lim = lim / (2 if st.kind == "rel" or st.C <= 7 else 4)
        x = fb.worst(got[name], st.r, scale, floor)[0]
        assert x <= lim, (name, x, lim)
