"""The covering sweep of the differentiable convolution (danet_b200.conv.conv2d) on the GPU: y, dx, dW and db of every
case of tests/conv_grad_sweep_common.py (tests/test_conv_grad_sweep_cpu.py proves the table covers every class), held
element by element to the scale-free bound stated there against fp64 torch autograd of F.conv2d on the device; then
operands far from 1, mixed magnitudes inside one tensor, exact zeros, non-finite values and input layouts.

The constant C of the bound is calibrated, not derived: on an NVIDIA H100 80GB HBM3 (700 W power limit) the worst ratio
|error - floor| / (u A + phi terms) over every test of this file was 0.87 for y, 2.87 for dx and 2.25 for dW (db never
left its floor); C is 9.0.  The largest ratios come from test_mixed_magnitudes' one dy element 2^20 above the rest: the
tensor core truncates its accumulator inside a K segment, so once that product is in a running sum each later step can
drop an ulp of it.  Without that test the worst was 1.93 (dW, network rows)."""
import math

import pytest
import torch

import conv_grad_sweep_common as S
import fp64_bound as fb

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
C = 9.0
OUTS = ("y", "dx", "dW", "db")


def run(case, x, w, b, dy, need=(True, True, True)):
    """conv2d forward and backward on the device: (y, dx, dW, db), None where not asked for or without a bias"""
    from danet_b200.conv import conv2d
    x = x.to(DEV).detach().clone().requires_grad_(need[0])          # clone keeps the memory format and the strides
    w = w.to(DEV).detach().clone().requires_grad_(need[1])
    b = b.to(DEV).detach().clone().requires_grad_(need[2]) if b is not None else None
    y = conv2d(x, w, b, case[6], case[5] // 2, 1, case[7])
    y.backward(dy.to(DEV))
    return y.detach(), x.grad, w.grad, (b.grad if b is not None else None)


def check(case, x, w, b, dy, what="", got=None, select=None):
    """hold every output (or the parts select[name] picks) to the bound; returns {output: worst ratio}"""
    x, w, b, dy = (t.to(DEV) if t is not None else None for t in (x, w, b, dy))
    got = dict(zip(OUTS, run(case, x, w, b, dy) if got is None else got))
    bnd = S.bounds(case, x, w, b, dy)
    worst = {}
    for name, (r, base, floor) in bnd.items():
        g = got[name]
        assert g is not None and g.shape == r.shape and g.dtype == torch.float32, (name, case)
        if select is not None:
            if name not in select:
                continue
            g, r, base, floor = (select[name](t) for t in (g, r, base, floor))
        assert torch.isfinite(g).all(), "%s has NaN / inf at %s: %s %s" % (
            name, tuple(int(v) for v in (~torch.isfinite(g)).nonzero()[0]), what, case)
        assert torch.isfinite(r).all(), (name, "a non-finite reference", what, case)
        q, at = fb.worst(g, r, base, floor)
        print("RATIO %s %.4f %s %s" % (name, q, what, case))
        assert q <= C, "%s off by %.3g x the bound at %s (got %r, want %r): %s %s" % (
            name, q / C, at, float(g[at]), float(r[at]), what, case)
        worst[name] = q
    return worst


# ----------------------------------------------------------------------------------------------------------------------
# a. the sweep
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(S.CASES)), ids=lambda i: "%d-%s" % (i, "x".join(str(v) for v in S.CASES[i])))
def test_sweep(i):
    case = S.CASES[i]
    check(case, *S.make_inputs(case, seed=2000 + i), what="sweep")


# ----------------------------------------------------------------------------------------------------------------------
# b. operand range: one case per (k, s), a grouped one and one with padded channels
# ----------------------------------------------------------------------------------------------------------------------
RANGE_CASES = [
    (2, 16, 24, 9, 8, 1, 1, 1, 1),
    (2, 24, 16, 10, 9, 3, 1, 1, 1),
    (2, 16, 24, 9, 10, 1, 2, 1, 1),
    (2, 24, 40, 11, 10, 3, 2, 1, 1),
    (2, 16, 16, 13, 12, 7, 2, 1, 1),
    (2, 16, 24, 7, 6, 3, 2, 3, 1),
    (2, 5, 25, 9, 7, 3, 1, 1, 1),
]


@pytest.mark.parametrize("ex,ew,edy", S.RANGE, ids=lambda v: str(v))
def test_operand_range(ex, ew, edy):
    for j, case in enumerate(RANGE_CASES):
        x, w, b, dy = S.scaled(*S.make_inputs(case, seed=3000 + j), ex, ew, edy)
        for name, r in zip(OUTS, S.reference(case, x.to(DEV), w.to(DEV), b.to(DEV), dy.to(DEV))):
            assert torch.isfinite(r).all() and r.abs().max() <= 3.4028234663852886e38, (name, case)   # the test's own inputs
        check(case, x, w, b, dy, what="x*2^%d w*2^%d dy*2^%d" % (ex, ew, edy))


# ----------------------------------------------------------------------------------------------------------------------
# c. mixed magnitudes inside one tensor: the bound's floors cover them
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [RANGE_CASES[1], RANGE_CASES[4], RANGE_CASES[5]], ids=lambda c: "x".join(map(str, c)))
def test_mixed_magnitudes(case):
    x, w, b, dy = S.make_inputs(case, seed=3100)
    xm = x.clone()
    xm[:, 1::2] *= 2.0 ** -12                                     # every other channel at 2^-12 of the rest
    check(case, xm, w, b, dy, what="x channels at 2^-12")
    dym = dy.clone()
    dym[0, 0, dy.shape[2] // 2, dy.shape[3] // 2] *= 2.0 ** 20    # one gradient 2^20 above the rest
    check(case, x, w, b, dym, what="one dy element * 2^20")


# ----------------------------------------------------------------------------------------------------------------------
# d. exact zeros (pow2_scale's path without a finite nonzero value)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("zero", [0.0, -0.0], ids=["+0", "-0"])
def test_exact_zeros(zero):
    for j, case in enumerate(RANGE_CASES):
        x, w, b, dy = S.make_inputs(case, seed=3200 + j)
        bb = b.to(DEV)[None, :, None, None]
        y, dx, dW, db = run(case, x, w, b, torch.full_like(dy, zero))
        assert (dx == 0).all() and (dW == 0).all() and (db == 0).all(), case
        y, dx, dW, db = run(case, torch.full_like(x, zero), w, b, dy)
        assert torch.equal(y, bb.expand_as(y)) and (dW == 0).all(), case
        y, dx, dW, db = run(case, x, torch.full_like(w, zero), b, dy)
        assert torch.equal(y, bb.expand_as(y)) and (dx == 0).all(), case


# ----------------------------------------------------------------------------------------------------------------------
# e. non-finite values stay non-finite
# ----------------------------------------------------------------------------------------------------------------------
NONFINITE_CASES = [RANGE_CASES[1], RANGE_CASES[3], RANGE_CASES[4], RANGE_CASES[5]]


@pytest.mark.parametrize("val", [math.nan, math.inf, -math.inf], ids=["nan", "+inf", "-inf"])
@pytest.mark.parametrize("where", ["x", "dy", "w"])
def test_non_finite_values(where, val):
    """Every element the fp64 reference makes non-finite is non-finite.  The masks need not be equal: the dgrad pieces
    and the forward's tap groups multiply structural zero taps and wgrad multiplies patch overhang rows, so 0 * inf can
    add NaNs beside the reference's.  What the poisoned element cannot reach stays finite and within the bound."""
    for j, case in enumerate(NONFINITE_CASES):
        x, w, b, dy = S.make_inputs(case, seed=3300 + j)
        if where == "x":
            x[0, 1, x.shape[2] // 2, x.shape[3] // 2] = val
        elif where == "dy":
            dy[0, 1, dy.shape[2] // 2, dy.shape[3] // 2] = val
        else:
            w[1, 0, case[5] // 2, case[5] // 2] = val
        got = run(case, x, w, b, dy)
        ref = S.reference(case, x.to(DEV), w.to(DEV), b.to(DEV), dy.to(DEV))
        for name, g, r in zip(OUTS, got, ref):
            bad = ~torch.isfinite(r)
            assert bad.any() or name in {"x": ("dx", "db"), "dy": ("y",), "w": ("dW", "db")}[where], (name, case)
            assert not torch.isfinite(g[bad]).any(), "%s: %d of the reference's %d non-finite elements are finite: %s=%r %s" % (
                name, int(torch.isfinite(g[bad]).sum()), int(bad.sum()), where, val, case)
        if where in ("x", "dy"):
            rest = lambda t: t[1:]
            check(case, x, w, b, dy, what="%s=%r in image 0" % (where, val), got=got, select={"y": rest, "dx": rest})
        else:
            others = torch.arange(w.shape[0]) != 1
            check(case, x, w, b, dy, what="w=%r" % val, got=got, select={"y": lambda t: t[:, others], "dW": lambda t: t})


# ----------------------------------------------------------------------------------------------------------------------
# f. layouts: the same bits as the contiguous run
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [RANGE_CASES[1], RANGE_CASES[4], RANGE_CASES[5]], ids=lambda c: "x".join(map(str, c)))
def test_layouts(case):
    from danet_b200.conv import conv2d
    x, w, b, dy = (t.to(DEV) for t in S.make_inputs(case, seed=3400))
    base = run(case, x, w, b, dy)

    def same(got, what):
        for name, a, c in zip(OUTS, got, base):
            assert torch.equal(a, c), (name, what, case)

    same(run(case, x.to(memory_format=torch.channels_last), w, b, dy), "channels_last x")
    wv = torch.empty(w.shape[::-1], device=DEV).permute(3, 2, 1, 0)
    wv.copy_(w)
    assert not wv.is_contiguous()
    same(run(case, x, wv, b, dy), "non-contiguous weight view")
    dyt = dy.transpose(2, 3).contiguous().transpose(2, 3)
    assert not dyt.is_contiguous()
    same(run(case, x, w, b, dyt), "transposed dy")
    # the stride-0 gradient of y.sum() against the same ones, materialised
    ones = run(case, x, w, b, torch.ones_like(dy))
    xs, ws, bs = x.clone().requires_grad_(), w.clone().requires_grad_(), b.clone().requires_grad_()
    y = conv2d(xs, ws, bs, case[6], case[5] // 2, 1, case[7])
    y.sum().backward()
    for name, a, c in zip(OUTS[1:], (xs.grad, ws.grad, bs.grad), ones[1:]):
        assert torch.equal(a, c), (name, "y.sum().backward()", case)
    ex = run(case, x, w, b, torch.ones(1, 1, 1, 1, device=DEV).expand_as(dy))
    for name, a, c in zip(OUTS, ex, ones):
        assert torch.equal(a, c), (name, "expanded dy", case)
