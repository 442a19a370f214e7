"""GPU half of the loss sweep (tests/loss_sweep_common.py): every case through the C entries, with outputs and
workspace prefilled with NaN, held to the per-element bound and the non-finite policy against the fp64 reference;
repeats bit-identical; the autograd ops give the C entries' bits.  Each case prints its worst error / bound per output."""
import numpy as np
import pytest
import torch

import fp64_bound as fb
import loss_sweep_common as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _nan(shape):
    return torch.full(shape, float("nan"), device=DEV)


def _ws(nbytes):
    return torch.full((max(int(nbytes), 16),), 0xFF, dtype=torch.uint8, device=DEV)


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def report(name, ratios):
    print("%s  %s" % (name, "  ".join("%s %.3f" % kv for kv in ratios.items())))


def hold(name, got, ref):
    out = {}
    for k, val in got.items():
        r, M, C = ref[k]
        out[k] = fb.worst(val.cpu(), r, *S.bound(r, M, C))[0]
        assert out[k] <= 1.0, "%s %s: error %.3g of the bound" % (name, k, out[k])
    report(name, out)


def c_body(c, p):
    from danet_b200 import _lib
    N, C, HW = c.N, c.C, c.H * c.W
    L = p["pred"].shape[2]
    pred, gt, ann, A, has = (_dev(p[k]) for k in ("pred", "gt", "ann", "A", "has"))
    grads = _nan((N, 3, L))
    ga = _nan(ann.shape) if c.Cann and "a" in c.need else None
    losses = _nan((4,))
    ws = _ws(_lib.load().danet_body_uv_losses_workspace_bytes(N, HW))
    base, gbase, tb = pred.data_ptr(), grads.data_ptr(), gt.data_ptr()
    off = lambda b, k: b + 4 * k * L
    gp = [off(gbase, k) if "uvi"[k] in c.need else 0 for k in range(3)]
    _lib.call("body_uv_losses", N, C, c.Cann, HW, 3 * L, 3 * L, *map(_lib.ptr, (off(base, 0), off(base, 1), off(base, 2),
              ann, off(tb, 0), off(tb, 1), off(tb, 2), A, has)), float(N), S.PW, _lib.ptr(losses),
              *map(_lib.ptr, gp), _lib.ptr(ga), _lib.ptr(ws), device=DEV)
    torch.cuda.synchronize()
    out = {"losses": losses}
    for k, name in enumerate(("gu", "gv", "gi")):
        if "uvi"[k] in c.need:
            out[name] = grads[:, k, :C * HW].reshape(N, C, HW)
            assert bool(torch.isnan(grads[:, k, C * HW:]).all()), "padding written"
    if ga is not None:
        out["ga"] = ga.view(N, c.Cann, HW)
    return out


def op_body(c, p):
    """the same case through body_uv_losses / part_iuv_losses (contiguous or part layout), when they express it"""
    from danet_b200 import losses as Lm
    N, C, H, W = c.N, c.C, c.H, c.W
    HW = H * W
    if c.pad:
        return None
    if c.part:
        B = N // 24
        pred = _dev(p["pred"]).view(B, 24, 3, C, H, W).requires_grad_()
        gt = _dev(p["gt"]).view(B, 24, 3, C, H, W)
        has = None if p["has"] is None else _dev(p["has"]).view(B, 24)[:, 0]
        L = Lm.part_iuv_losses(pred, gt, has, S.PW)
        torch.autograd.backward(list(L), [torch.ones((), device=DEV)] * 3)
        g = pred.grad.view(N, 3, C, HW)
        return {"losses": torch.stack(list(L) + [torch.zeros((), device=DEV)]),
                "gu": g[:, 0], "gv": g[:, 1], "gi": g[:, 2]}
    x = [_dev(p["pred"][:, k, :C * HW]).view(N, C, H, W).requires_grad_("uvi"[k] in c.need) for k in range(3)]
    t = [_dev(p["gt"][:, k, :C * HW]).view(N, C, H, W) for k in range(3)]
    a = _dev(p["ann"]).view(N, c.Cann, H, W).requires_grad_("a" in c.need) if c.Cann else None
    A = _dev(p["A"]).view(N, c.Cann, H, W) if c.Cann else None
    L = Lm.body_uv_losses(*x, a, [*t, A], _dev(p["has"]), S.PW)
    ins = [v for v in x + [a] if v is not None and v.requires_grad]
    if ins:
        torch.autograd.backward([l for l in L if l is not None and l.requires_grad],
                                [torch.ones((), device=DEV)] * sum(1 for l in L if l is not None and l.requires_grad))
    out = {"losses": torch.stack([l if l is not None else torch.zeros((), device=DEV) for l in L]).detach()}
    for k, name in enumerate(("gu", "gv", "gi")):
        if "uvi"[k] in c.need:
            out[name] = x[k].grad.view(N, C, HW)
    if a is not None and "a" in c.need:
        out["ga"] = a.grad.view(N, c.Cann, HW)
    return out


def same_bits(a, b, what):
    a, b = a.detach().contiguous(), b.detach().contiguous()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what


@pytest.mark.parametrize("c", S.BODY_CASES, ids=lambda c: S.body_id(c))
def test_body(c):
    p = S.make_body(c)
    got = c_body(c, p)
    hold(S.body_id(c), got, S.body_reference(c, p))
    again = c_body(c, p)
    for k in got:
        same_bits(got[k], again[k], "repeat " + k)
    full = c_body(c._replace(need="uvia" if c.Cann else "uvi"), p)
    for k in got:
        same_bits(got[k], full[k], "needs-grad subset changes " + k)
    op = op_body(c, p)
    if op is not None:
        for k in got:
            if k == "losses" and c.part:
                same_bits(got[k][:3], op[k][:3], "op " + k)
            else:
                same_bits(got[k], op[k], "op " + k)


def c_dp(c, p, need=None):
    from danet_b200 import _lib
    need = c.need if need is None else need
    N, Sz = c.N, c.S
    arrs = [_dev(p[k]) for k in ("u", "v", "idx", "ann", "X", "Y", "I", "Up", "Vp", "W", "A")]
    gr = [_nan(a.shape) if ch in need else None for a, ch in zip(arrs[:4], "uvia")]
    L = _nan((4,))
    ws = _ws(_lib.load().danet_dp_uvia_losses_workspace_bytes(N, Sz * Sz))
    _lib.call("dp_uvia_losses", N, Sz, c.Cann, c.P, *map(_lib.ptr, arrs), _lib.ptr(_dev(p["has"])), int(c.align), S.PW,
              S.PART_W, S.INDEX_W, _lib.ptr(L), *map(_lib.ptr, gr), _lib.ptr(ws), device=DEV)
    torch.cuda.synchronize()
    out = {"losses": L}
    for g, name in zip(gr, ("gu", "gv", "gi", "ga")):
        if g is not None:
            out[name] = g
    return out


@pytest.mark.parametrize("c", S.DP_CASES, ids=lambda c: S.dp_id(c))
def test_dp(c):
    p = S.make_dp(c)
    got = c_dp(c, p)
    hold(S.dp_id(c), got, S.dp_reference(c, p))
    again, full = c_dp(c, p), c_dp(c, p, "uvia")
    for k in got:
        same_bits(got[k], again[k], "repeat " + k)
        same_bits(got[k], full[k], "needs-grad subset changes " + k)
    if c.nonfinite:
        return
    from danet_b200 import losses as Lm
    x = [_dev(p[k]).requires_grad_(ch in c.need) for k, ch in zip(("u", "v", "idx", "ann"), "uvia")]
    t = lambda k: _dev(p[k])
    L = Lm.dp_uvia_losses(*x, t("X"), t("Y"), t("I"), t("I"), t("Up"), t("Vp"), t("W"), t("A"),
                          has_dp=_dev(p["has"]), align_corners=c.align, point_weight=S.PW, part_weight=S.PART_W,
                          index_weight=S.INDEX_W, check_labels=False)
    same_bits(torch.stack(L).detach(), got["losses"], "op losses")
    for k, (xx, name) in enumerate(zip(x, ("gu", "gv", "gi", "ga"))):
        if xx.requires_grad:
            g, = torch.autograd.grad(L[k], xx, retain_graph=True)
            same_bits(g, got[name], "op " + name)


def c_stn(c, p):
    from danet_b200 import _lib
    hm, kps = _dev(p["hm"]), _dev(p["kps"])
    B, J, Sz = hm.shape[:3]
    L = _nan((2,))
    groi = _nan(hm.shape)
    ghm = groi if c.alias else _nan(hm.shape)
    ws = _ws(_lib.load().danet_stn_kps_losses_workspace_bytes(B, J))
    _lib.call("stn_kps_losses", B, J, Sz, _lib.ptr(hm), _lib.ptr(kps), c.cols, c.kw, c.hw, _lib.ptr(L), _lib.ptr(groi),
              _lib.ptr(ghm), _lib.ptr(ws), device=DEV)
    torch.cuda.synchronize()
    return {"losses": L, "g": groi} if c.alias else {"losses": L, "groi": groi, "ghm": ghm}


@pytest.mark.parametrize("c", S.STN_CASES, ids=lambda c: S.stn_id(c))
def test_stn(c):
    p = S.make_stn(c)
    got = c_stn(c, p)
    hold(S.stn_id(c), got, S.stn_reference(c, p))
    again = c_stn(c, p)
    for k in got:
        same_bits(got[k], again[k], "repeat " + k)


@pytest.mark.parametrize("c", S.PART_CASES, ids=lambda c: S.part_id(c))
def test_part(c):
    from danet_b200 import _lib
    from danet_b200 import losses as Lm
    p = S.make_part(c)
    U, V, I, th = (_dev(p[k]) for k in ("U", "V", "I", "theta"))
    out = _nan((c.B, 24, 3, 7, c.S, c.S))
    _lib.call("part_iuv_targets", c.B, c.S, c.C, *map(_lib.ptr, (U, V, I, th)), int(c.align), _lib.ptr(out), device=DEV)
    torch.cuda.synchronize()
    r, M, C, flips, worst = S.part_reference(c, p)
    assert worst <= 1.0
    q = fb.worst(out.cpu(), r, *S.bound(r, M, C))[0]
    report(S.part_id(c), {"out": q, "bg flips": flips})
    assert q <= 1.0
    same_bits(out, Lm.part_iuv_targets([U, V, I], th, align_corners=c.align), "op")
