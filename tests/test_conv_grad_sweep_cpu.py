"""The differentiable convolution's sweep without a GPU (tests/conv_grad_sweep_common.py): the case table covers every
coverage class, the restated weight-gradient geometry is the library's own, and the per-element bound separates a
split that scales its operand by a power of two from one that does not."""
import ctypes

import pytest
import torch

import conv_grad_sweep_common as S
import fp64_bound as fb


def test_every_class_has_a_case():
    cov = S.coverage()
    missing = [name for name, cases in cov.items() if not cases]
    assert not missing, "coverage classes without a case:\n  " + "\n  ".join(missing)


@pytest.mark.parametrize("drop", [1, 2, 7, 14])
def test_the_classes_notice_a_missing_case(drop):
    """the table has no slack in the classes these cases alone cover: deleting one turns its class red"""
    full, less = S.coverage(), S.coverage(S.CASES[:drop] + S.CASES[drop + 1:])
    only = [name for name in full if full[name] == [drop]]
    assert only, "case %d is not the only case of any class: pick another" % drop
    assert all(not less[name] for name in only)


def test_cases_are_distinct_and_supported():
    assert len(set(S.CASES)) == len(S.CASES)
    for c in S.CASES:
        B, cin, cout, H, W, k, s, G, bias = c
        assert (k, s) in ((1, 1), (3, 1), (1, 2), (3, 2), (7, 2)) and min(B, cin, cout, H, W, G) >= 1 and bias in (0, 1), c
        assert S.wgrad_geo(c)["nchunk"] >= 1


def _lib_nchunk(N, H, W, Cin, Cout, k, s, pad, wsets):
    """nchunk as the library sizes it: one chunk of partials is wsets * taps * Cout * Cin floats, at least 256 bytes, so
    the 256-byte rounding of the workspace adds less than one chunk"""
    from danet_b200 import _lib as L
    d = L.ConvDesc(N, H, W, Cin, Cout, k, s, pad, wsets, 0, 4)
    nbytes = int(L.load().danet_conv_wgrad_workspace_bytes(ctypes.byref(d)))
    return nbytes // (wsets * k * k * Cout * Cin * 4) if nbytes else 0


def test_wgrad_geometry_is_the_librarys():
    for c in S.CASES:
        assert _lib_nchunk(*S.desc_fields(c)) == S.wgrad_geo(c)["nchunk"], c
    n = 0
    for k, s in ((1, 1), (3, 1), (1, 2), (3, 2), (7, 2)):
        for H, W in ((1, 1), (7, 9), (16, 16), (33, 17), (56, 56), (120, 200)):
            for N, G in ((1, 1), (3, 1), (16, 1), (48, 24), (64, 1)):
                for Cin, Cout in ((8, 8), (64, 136), (256, 512)):
                    g = S.make_geo(N, H, W, Cin, Cout, k, s, k // 2, G)
                    assert _lib_nchunk(N, H, W, Cin, Cout, k, s, k // 2, G) == g["nchunk"], (N, H, W, Cin, Cout, k, s, G, g)
                    n += g["nchunk"] > 1
    assert n > 100


def test_refused_shapes_have_no_workspace():
    for args in [(2, 8, 8, 12, 8, 3, 1, 1, 1), (2, 8, 8, 8, 12, 3, 1, 1, 1), (2, 8, 8, 8, 8, 5, 1, 2, 1),
                 (2, 8, 8, 8, 8, 3, 3, 1, 1), (2, 8, 8, 8, 8, 3, 1, 0, 1), (3, 8, 8, 8, 8, 3, 1, 1, 2),
                 (1, 1 << 15, 1 << 15, 8, 8, 1, 1, 0, 1)]:
        assert S.make_geo(*args) is None, args
        assert _lib_nchunk(*args) == 0, args


# ----------------------------------------------------------------------------------------------------------------------
# the bound on an emulation of the split: hi = rn_f16(v * 2^s), lo = rn_f16(v * 2^s - hi), three products in fp64
# ----------------------------------------------------------------------------------------------------------------------
def _split(v, scaled):
    """(hi, lo) in fp64, scale removed.  Unscaled: s = 0 and the fp16 conversion saturates, as the unscaled planes do."""
    s = S.split_exp(v) if scaled else 0
    vs = v * 2.0 ** s
    hi = vs.clamp(-65504, 65504).half().float()
    lo = (vs - hi).clamp(-65504, 65504).half().float()
    return hi.double() * 2.0 ** -s, lo.double() * 2.0 ** -s


def _emulate(case, x, w, b, dy, scaled_x):
    op = S.Ops(case, x.shape, w.shape)
    xh, xl = _split(x, scaled_x)
    wh, wl = _split(w, True)
    dh, dl = _split(dy, True)
    y = op.C(xh, wh) + op.C(xh, wl) + op.C(xl, wh) + b.double()[None, :, None, None]
    dx = op.Ct(dh, wh) + op.Ct(dh, wl) + op.Ct(dl, wh)
    dW = op.Wg(xh, dh) + op.Wg(xh, dl) + op.Wg(xl, dh)
    return {"y": y, "dx": dx, "dW": dW}


EMU_CASES = [(2, 5, 7, 9, 8, 3, 2, 1, 1), (2, 16, 24, 11, 10, 3, 1, 1, 1), (1, 8, 16, 12, 9, 7, 2, 1, 1)]


@pytest.mark.parametrize("ex,ew,edy", S.RANGE)
def test_bound_holds_for_the_scaled_split(ex, ew, edy):
    for j, case in enumerate(EMU_CASES):
        x, w, b, dy = S.make_inputs(case, seed=50 + j)
        x, w, b, dy = S.scaled(x, w, b, dy, ex, ew, edy)
        got, bnd = _emulate(case, x, w, b, dy, True), S.bounds(case, x, w, b, dy)
        for name in got:
            q, at = fb.worst(got[name], *bnd[name])
            assert q <= 1.0, (name, q, at, case, (ex, ew, edy))


@pytest.mark.parametrize("ex", [-16, 17])
def test_bound_breaks_for_the_unscaled_split(ex):
    """x * 2^-16: the lo halves are fp16 subnormals or zero; x * 2^17: the hi halves saturate at 65504"""
    for j, case in enumerate(EMU_CASES):
        x, w, b, dy = S.make_inputs(case, seed=50 + j)
        x, w, b, dy = S.scaled(x, w, b, dy, ex, 0, 0)
        got, bnd = _emulate(case, x, w, b, dy, False), S.bounds(case, x, w, b, dy)
        for name in ("y", "dW"):
            q, _ = fb.worst(got[name], *bnd[name])
            assert q > 4.0, (name, q, case, ex)
        ok = _emulate(case, x, w, b, dy, True)
        assert fb.worst(ok["y"], *bnd["y"])[0] <= 1.0


def test_split_exponent():
    assert S.split_exp(torch.tensor([1.0, -3.0])) == 12                 # 3 * 2^12 in [2^13, 2^14)
    assert S.split_exp(torch.tensor([2.0 ** -130, 0.0])) == 126         # clamped: 2^-126 stays a normal fp32 number
    assert S.split_exp(torch.tensor([3e38, float("inf")])) == -114      # the largest finite value decides
    assert S.split_exp(torch.tensor([0.0, float("nan")])) == 0
