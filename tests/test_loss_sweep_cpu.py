"""CPU half of the loss sweep (tests/loss_sweep_common.py): coverage of the case tables, the fp64 reference against
torch's own ops, the kernels' own arithmetic (csrc/losses.cu and csrc/iuv_train.cu compiled with
DANET_LOSSES_HOST_CHECK and walked on the host) against the bound and the non-finite policy, and fp32 emulations with
seeded defects that the bound catches while the clean emulation stays well inside it."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fp64_bound as fb
import loss_sweep_common as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_class_is_covered():
    missing = fb.uncovered(S.CASES, S.CLASSES)
    assert not missing, "classes with no case: %s" % ", ".join(missing)


# ----------------------------------------------------------------------------------------------------------------------
# the reference against torch's own ops, in fp64
# ----------------------------------------------------------------------------------------------------------------------
def _cap_body(c):
    if c.part:
        return c._replace(N=24 * max(1, min(c.N // 24, 2)))
    per = c.C * c.H * c.W
    return c._replace(N=max(1, min(c.N, 600000 // per)) if per <= 600000 else c.N)


FINITE_BODY = [c for c in S.BODY_CASES if not c.nonfinite and c.H * c.W <= 4096]


@pytest.mark.parametrize("c", FINITE_BODY[:12] + [c for c in S.BODY_CASES if c.nonfinite],
                         ids=lambda c: S.body_id(c))
def test_body_reference_against_torch(c):
    c = _cap_body(c)
    p = S.make_body(c)
    ref = S.body_reference(c, p)
    (u, v, i), (Um, Vm, Im) = S._views(c, p)
    N, C, HW = c.N, c.C, c.H * c.W
    has = torch.ones(N, dtype=torch.bool) if p["has"] is None else torch.from_numpy(p["has"]) != 0
    nsel = int(has.sum())
    xs = [t.double().requires_grad_() for t in (u, v, i)]
    lu = lv = li = torch.zeros((), dtype=torch.float64)
    if nsel:
        m = (Im > 0) & has.view(-1, 1, 1)
        lu = F.smooth_l1_loss(xs[0][m], Um.double()[m], reduction="sum") * S.PW / N
        lv = F.smooth_l1_loss(xs[1][m], Vm.double()[m], reduction="sum") * S.PW / N
        lab = S.target_argmax(Im)
        li = F.cross_entropy(xs[2][has], lab[has], reduction="mean")
    for k, (got, name) in enumerate(((lu, "gu"), (lv, "gv"), (li, "gi"))):
        r = ref["losses"][0][k]
        assert torch.equal(torch.isnan(got), torch.isnan(r)), name
        if torch.isfinite(got):
            assert abs(float(got.detach()) - float(r)) <= 1e-10 * (1 + abs(float(r))), name
        if nsel and got.requires_grad:
            g, = torch.autograd.grad(got, xs[k], allow_unused=True)
            g = torch.zeros_like(xs[k]) if g is None else g
            rr = ref[name][0]
            fin = torch.isfinite(g)
            assert torch.equal(torch.isnan(g), torch.isnan(rr)), name
            assert torch.allclose(g[fin], rr[fin], rtol=1e-10, atol=1e-14), name


def _dp_torch(c, p):
    """torch's own grid_sample, smooth_l1_loss and cross_entropy on the restated fp32 grid: the four losses"""
    N, Sz, P = c.N, c.S, c.P
    t = lambda k: torch.from_numpy(p[k])
    hs, sc = torch.tensor(0.5 * Sz, dtype=torch.float32), torch.tensor(2.0 / Sz, dtype=torch.float32)
    gx, gy = (t("X") - hs) * sc, (t("Y") - hs) * sc
    # the fp32 source coordinates the kernel samples at, handed to grid_sample as fp64 grid values it maps back to them
    ix, iy = (S.grid_unnormalize32(g, Sz, c.align).double() for g in (gx, gy))
    norm = (lambda a: a * 2 / (Sz - 1) - 1) if c.align else (lambda a: (2 * a + 1) / Sz - 1)
    grid = torch.stack([norm(ix), norm(iy)], -1).view(N, 1, P, 2)
    has = torch.ones(N, dtype=torch.bool) if p["has"] is None else t("has") != 0
    L = []
    W = t("W").double().view(N, 25, P)
    for k, tg in (("u", "Up"), ("v", "Vp")):
        s = F.grid_sample(t(k).double(), grid, align_corners=c.align).view(N, 25, P)
        d = W * (s - t(tg).double().view(N, 25, P))
        L.append((W * F.smooth_l1_loss(d, torch.zeros_like(d), reduction="none"))[has].sum() * S.PW)
    s = F.grid_sample(t("idx").double(), grid, align_corners=c.align).view(N, 25, P)
    lab = t("I").trunc().long()
    L.append(F.cross_entropy(s[has], lab[has], reduction="mean") * S.PART_W)
    a = t("ann").double().view(N, c.Cann, -1)
    L.append(F.cross_entropy(a[has], t("A").trunc().long()[has], reduction="mean") * S.INDEX_W)
    return torch.stack(L)


@pytest.mark.parametrize("c", [c for c in S.DP_CASES if c.N <= 3 and not c.nonfinite and c.has != "zero"][:10],
                         ids=lambda c: S.dp_id(c))
def test_dp_reference_against_torch(c):
    p = S.make_dp(c)
    got = _dp_torch(c, p)
    r = S.dp_reference(c, p)["losses"][0]
    # grid_sample unnormalizes in fp64 again: a point it does not map back exactly onto the kernel's coordinate can
    # move to the neighbouring taps at an integer coordinate, with weights of 1e-16 against 0
    assert torch.allclose(got, r, rtol=1e-7, atol=1e-12), (got, r)


def test_stn_and_part_references_against_torch():
    for c in [c for c in S.STN_CASES if c.S <= 20 and not c.nonfinite and not c.alias][:6]:
        p = S.make_stn(c)
        ref = S.stn_reference(c, p)
        hm = torch.from_numpy(p["hm"]).double().requires_grad_()
        kps = torch.from_numpy(p["kps"]).double()
        B, J, Sz = c.B, c.J, c.S
        pr = torch.softmax(10 * hm.view(B, J, -1), -1)
        col = (torch.arange(Sz * Sz) % Sz).double()
        row = (torch.arange(Sz * Sz) // Sz).double()
        cx, cy = (pr * col).sum(-1) / (0.5 * Sz) - 1, (pr * row).sum(-1) / (0.5 * Sz) - 1
        if c.cols == 3 and c.kw:
            w = kps[..., 2]
            l = w * (F.smooth_l1_loss(cx, kps[..., 0], reduction="none") + F.smooth_l1_loss(cy, kps[..., 1], reduction="none"))
            roi = l.sum() * c.kw / B
            assert abs(float(roi) - float(ref["losses"][0][0])) <= 1e-10 * (1 + abs(float(roi)))
            g, = torch.autograd.grad(roi, hm)
            rg = ref["groi"][0] if "groi" in ref else None
            if rg is not None:
                assert torch.allclose(g, rg, rtol=1e-9, atol=1e-14)
    # general (sheared) thetas are held by the host walk and the GPU sweep only: grid_sample does not reproduce the
    # reference to 1e-10 on them even where the coordinates round-trip exactly
    for c in [c for c in S.PART_CASES if c.S <= 12 and c.theta != "general"]:
        p = S.make_part(c)
        r = S.part_reference(c, p)[0]
        B, Sz = c.B, c.S
        base = S.affine_base32(Sz, c.align)
        th = torch.from_numpy(p["theta"]).view(B * 24, 2, 3)
        xb, yb = base.repeat(Sz), base.repeat_interleave(Sz)
        gx = (th[:, 0, 0:1] * xb + th[:, 0, 1:2] * yb) + th[:, 0, 2:3]
        gy = (th[:, 1, 0:1] * xb + th[:, 1, 1:2] * yb) + th[:, 1, 2:3]
        ix, iy = (S.grid_unnormalize32(g, Sz, c.align).double() for g in (gx, gy))
        norm = (lambda a: a * 2 / (Sz - 1) - 1) if c.align else (lambda a: (2 * a + 1) / Sz - 1)
        grid = torch.stack([norm(ix), norm(iy)], -1).view(B * 24, Sz, Sz, 2)
        mp = torch.tensor(S.DP2SMPL)
        Um, Vm, Im = (torch.from_numpy(p[k]).double() for k in ("U", "V", "I"))
        Isel = Im[:, mp]
        isum = torch.zeros(B, 24, Sz, Sz)
        for k in range(6):
            isum = isum + torch.from_numpy(p["I"])[:, mp][:, :, k]
        z = torch.zeros(B, 24, 1, Sz, Sz, dtype=torch.float64)
        src = torch.cat([z, Um[:, mp], z, Vm[:, mp], (isum < 0.5).double().unsqueeze(2), Isel], 2).view(B * 24, 21, Sz, Sz)
        got = F.grid_sample(src, grid, align_corners=c.align).view(B, 24, 3, 7, Sz, Sz)
        # pixels whose coordinates grid_sample's own fp64 unnormalize does not map back exactly can change taps
        unn = (lambda g: (g + 1) / 2 * (Sz - 1)) if c.align else (lambda g: ((g + 1) * Sz - 1) / 2)
        same = ((unn(grid[..., 0]) == ix.view(B * 24, Sz, Sz)) & (unn(grid[..., 1]) == iy.view(B * 24, Sz, Sz)))
        same = same.view(B, 24, 1, 1, Sz, Sz).expand_as(r)
        assert bool(same.any())
        assert torch.allclose(got[same], r[same], rtol=1e-10, atol=1e-12), S.part_id(c)


# ----------------------------------------------------------------------------------------------------------------------
# the kernels' own arithmetic, walked on the host
# ----------------------------------------------------------------------------------------------------------------------
def _compile(tmp, src, name):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    out = str(tmp / name)
    csrc = os.path.join(ROOT, "danet-densepose2smpl_b200", "csrc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
                           "-DDANET_LOSSES_HOST_CHECK", "-shared", os.path.join(csrc, src), os.path.join(csrc, "api.cu"),
                           "-o", out])
    return ctypes.CDLL(out)


@pytest.fixture(scope="module")
def hostlibs(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("loss_sweep_host")
    lo, it = _compile(tmp, "losses.cu", "liblosses.so"), _compile(tmp, "iuv_train.cu", "libiuv.so")
    p, i32, i64, f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float
    lo.danet_test_body_uv_losses_host.argtypes = [i32, i32, i32, i32, i64, i64] + [p] * 9 + [f, f] + [p] * 5
    it.danet_test_dp_uvia_losses_host.argtypes = [i32] * 4 + [p] * 12 + [i32, f, f, f] + [p] * 5
    it.danet_test_stn_kps_losses_host.argtypes = [i32, i32, i32, p, p, i32, f, f, p, p, p]
    it.danet_test_part_iuv_targets_host.argtypes = [i32, i32, i32, p, p, p, p, i32, p]
    return lo, it


def _P(x):
    return None if x is None else x.ctypes.data_as(ctypes.c_void_p)


def host_body(lib, c, p):
    N, C, HW = c.N, c.C, c.H * c.W
    L = p["pred"].shape[2]
    pred, gt = p["pred"].reshape(N, -1), p["gt"].reshape(N, -1)
    grads = np.full((N, 3, L), np.nan, np.float32)
    ga = np.full_like(p["ann"], np.nan) if c.Cann else None
    off = lambda a, k: a[:, k * L:].ctypes.data_as(ctypes.c_void_p) if a is not None else None
    gp = [off(grads.reshape(N, -1), k) if "uvi"[k] in c.need else None for k in range(3)]
    losses = np.full(4, np.nan, np.float32)
    assert lib.danet_test_body_uv_losses_host(
        N, C, c.Cann, HW, 3 * L, 3 * L, off(pred, 0), off(pred, 1), off(pred, 2), _P(p["ann"]), off(gt, 0), off(gt, 1),
        off(gt, 2), _P(p["A"]), _P(p["has"]), float(N), S.PW, _P(losses), *gp, _P(ga) if "a" in c.need else None) == 0
    out = {"losses": losses}
    for k, name in enumerate(("gu", "gv", "gi")):
        if "uvi"[k] in c.need:
            out[name] = grads[:, k, :C * HW].reshape(N, C, HW)
            assert np.isnan(grads[:, k, C * HW:]).all(), "padding written"
    if c.Cann and "a" in c.need:
        out["ga"] = ga.reshape(N, c.Cann, HW)
    return out


def check_all(got, ref, where):
    worst = {}
    for k, val in got.items():
        r, M, C = ref[k]
        worst[k] = fb.worst(torch.from_numpy(np.asarray(val)), r, *S.bound(r, M, C))[0]
        assert worst[k] <= 1.0, "%s %s: error %.3g of the bound" % (where, k, worst[k])
    return worst


@pytest.mark.parametrize("c", S.BODY_CASES, ids=lambda c: S.body_id(c))
def test_body_host_walk_within_bound(hostlibs, c):
    c = _cap_body(c)
    p = S.make_body(c)
    check_all(host_body(hostlibs[0], c, p), S.body_reference(c, p), S.body_id(c))


def host_dp(lib, c, p):
    N, Sz = c.N, c.S
    arrs = [p[k] for k in ("u", "v", "idx", "ann", "X", "Y", "I", "Up", "Vp", "W", "A")]
    gr = [np.full_like(a, np.nan) if ch in c.need else None for a, ch in zip(arrs[:4], "uvia")]
    L = np.full(4, np.nan, np.float32)
    assert lib.danet_test_dp_uvia_losses_host(N, Sz, c.Cann, c.P, *map(_P, arrs), _P(p["has"]), int(c.align), S.PW,
                                              S.PART_W, S.INDEX_W, _P(L), *map(_P, gr)) == 0
    out = {"losses": L}
    for g, name in zip(gr, ("gu", "gv", "gi", "ga")):
        if g is not None:
            out[name] = g
    return out


@pytest.mark.parametrize("c", S.DP_CASES, ids=lambda c: S.dp_id(c))
def test_dp_host_walk_within_bound(hostlibs, c):
    p = S.make_dp(c)
    check_all(host_dp(hostlibs[1], c, p), S.dp_reference(c, p), S.dp_id(c))


def host_stn(lib, c, p):
    hm, kps = p["hm"], p["kps"]
    B, J, Sz = hm.shape[:3]
    L = np.full(2, np.nan, np.float32)
    groi = np.full_like(hm, np.nan)
    ghm = groi if c.alias else np.full_like(hm, np.nan)
    assert lib.danet_test_stn_kps_losses_host(B, J, Sz, _P(hm), _P(kps), c.cols, c.kw, c.hw, _P(L), _P(groi), _P(ghm)) == 0
    return {"losses": L, "g": groi} if c.alias else {"losses": L, "groi": groi, "ghm": ghm}


@pytest.mark.parametrize("c", S.STN_CASES, ids=lambda c: S.stn_id(c))
def test_stn_host_walk_within_bound(hostlibs, c):
    p = S.make_stn(c)
    check_all(host_stn(hostlibs[1], c, p), S.stn_reference(c, p), S.stn_id(c))


def host_part(lib, c, p):
    B, Sz = c.B, c.S
    out = np.full((B, 24, 3, 7, Sz, Sz), np.nan, np.float32)
    assert lib.danet_test_part_iuv_targets_host(B, Sz, c.C, _P(p["U"]), _P(p["V"]), _P(p["I"]), _P(p["theta"]),
                                                int(c.align), _P(out)) == 0
    return out


@pytest.mark.parametrize("c", S.PART_CASES, ids=lambda c: S.part_id(c))
def test_part_host_walk_within_bound(hostlibs, c):
    p = S.make_part(c)
    r, M, C, flips, worst = S.part_reference(c, p)
    assert worst <= 1.0, "a background decision differs from fp64 away from 0.5"
    q = fb.worst(torch.from_numpy(host_part(hostlibs[1], c, p)), r, *S.bound(r, M, C))[0]
    assert q <= 1.0
    if c.theta == "out":
        assert float(r.abs().max()) == 0.0


def test_issue_pixel_nan_and_leading_minus_inf(hostlibs):
    """one pixel, C = 4, I one-hot at 1, u = [0, NaN, 0, 0], index = [-inf, 0.5, 0.2, 0.1]: loss_U and g_u[1] NaN,
    loss_IndexUV 0.8801 and g_index [0, -0.585, 0.307, 0.278] as torch gives"""
    c = S.body(1, 4, 1, 1)
    pred = np.zeros((1, 3, 4), np.float32)
    pred[0, 0] = [0, np.nan, 0, 0]
    pred[0, 2] = [-np.inf, 0.5, 0.2, 0.1]
    gt = np.zeros((1, 3, 4), np.float32)
    gt[0, 2, 1] = 1
    got = host_body(hostlibs[0], c, dict(pred=pred, gt=gt, ann=None, A=None, has=None))
    assert np.isnan(got["losses"][0]) and np.isnan(got["gu"][0, 1, 0])
    assert abs(got["losses"][2] - 0.8801) < 1e-4
    np.testing.assert_allclose(got["gi"][0, :, 0], [0, -0.585, 0.307, 0.278], atol=1e-3)


# ----------------------------------------------------------------------------------------------------------------------
# seeded defects: fp32 emulations (the reference's arithmetic in float32) caught by the bound
# ----------------------------------------------------------------------------------------------------------------------
def _emu_ratio(kind, c, defect):
    """worst over outputs of error / bound-without-C: the fraction of C the emulation uses, and C"""
    if kind == "body":
        c = _cap_body(c)
        p = S.make_body(c)
        ref, emu = S.body_reference(c, p), S.body_reference(c, p, S.F32, defect)
    elif kind == "dp":
        p = S.make_dp(c)
        ref, emu = S.dp_reference(c, p), S.dp_reference(c, p, S.F32, defect)
    elif kind == "stn":
        p = S.make_stn(c)
        ref, emu = S.stn_reference(c, p), S.stn_reference(c, p, S.F32, defect)
    else:
        p = S.make_part(c)
        r, M, C = S.part_reference(c, p)[:3]
        ref, emu = {"out": (r, M, C)}, {"out": (S.part_reference(c, p, S.F32, defect)[0], None, None)}
    worst = []
    for k, (r, M, C) in ref.items():
        got = emu[k][0].to(S.F64)
        fin = torch.isfinite(r)
        if not bool(fin.any()):
            continue
        Ct = torch.as_tensor(C, dtype=S.F64).expand_as(r)
        if bool((torch.isfinite(got) != fin).any()) or bool((torch.isnan(got) != torch.isnan(r)).any()):
            worst.append((float("inf"), 1.0))
            continue
        e = ((got - r).abs() - fb.U24 * r.abs() - fb.TINY).clamp(min=0) / (fb.U24 * torch.as_tensor(M).to(S.F64).expand_as(r))
        e = torch.where(fin, e.nan_to_num(0, float("inf"), 0), torch.zeros((), dtype=S.F64))
        k_ = int(e.argmax())
        worst.append((float(e.view(-1)[k_]), float(Ct.reshape(-1)[k_])))
    return worst


EMU = {
    "body": [c for c in S.BODY_CASES if not c.nonfinite and c.C * c.H * c.W * c.N <= 400000][7:30],
    "dp": [c for c in S.DP_CASES if not c.nonfinite and c.N <= 3][:10],
    "stn": [c for c in S.STN_CASES if not c.nonfinite and c.S <= 20],
    "part": [c for c in S.PART_CASES if c.S <= 12],
}


def test_clean_emulations_within_a_quarter_of_the_bound():
    for kind, cases in EMU.items():
        for c in cases:
            for q, C in _emu_ratio(kind, c, None):
                assert q <= (C / 2 if C <= 7 else C / 4), "%s %s: clean fp32 emulation at %.3g of C = %g" % (kind, c, q, C)


DEFECTS = [("body", "no_max_rescale"), ("body", "ce_over_n"), ("body", "sl1_over_nsel"), ("body", "last_tie"),
           ("dp", "drop_last"), ("dp", "index_over_hw"), ("dp", "other_align"), ("part", "swap_taps"),
           ("stn", "xy_swapped"), ("stn", "round_centre"), ("part", "bg_of_5")]


@pytest.mark.parametrize("kind,defect", DEFECTS)
def test_bound_catches_seeded_defect(kind, defect):
    caught = [c for c in EMU[kind] if any(q > C for q, C in _emu_ratio(kind, c, defect))]
    assert caught, "%s: no case catches it" % defect
