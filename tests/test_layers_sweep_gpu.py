"""The covering sweep of danet_b200.layers on the GPU (tests/layers_sweep_common.py): every case of batch_norm,
max_pool2d, adaptive_avg_pool2d, linear and hr_fuse through the autograd ops, each output element held to the
per-element bound against the fp64 reference (exact outputs to equality); the non-finite policy of the ReLU; bit-for-bit
repeats; and the C entries with outputs and workspace prefilled with NaN, which must give the autograd call's bits.
Each case prints its worst |err| / (2^-24 M) per output."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import fp64_bound as fb
import layers_sweep_common as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def at_offset(t, grad=False):
    """(view, base): t's values in a contiguous view 4 bytes into a fresh buffer (base requires grad when asked; the
    view's gradient is base.grad[1:])"""
    base = torch.empty(t.numel() + 1, device=DEV)
    base[1:].copy_(t.reshape(-1).to(DEV))
    if grad:
        base.requires_grad_()
    return base[1:].view(t.shape), base


def leaf(t, offset, grad):
    """(input, grad getter): t on the device, at a 4-byte offset when asked, requiring grad when asked"""
    if offset:
        v, base = at_offset(t, grad)
        return v, (lambda: base.grad[1:].view(t.shape) if base.grad is not None else None)
    x = t.to(DEV).clone().requires_grad_(grad)
    return x, (lambda: x.grad)


def report(name, ratios):
    print("%s  %s" % (name, "  ".join("%s %.2f" % kv for kv in ratios.items())))


def hold(name, got, r, M, C, tiny=fb.TINY, finiteness_only=False):
    q = fb.worst(got, r, fb.U24 * M, fb.U24 * r.abs() + tiny, finiteness_only)[0]
    assert q <= C, "%s: worst excess %.3g units of 2^-24 M over the bound's %d" % (name, q, C)
    return fb.err_ratio(got, r, fb.U24 * M)


# ----------------------------------------------------------------------------------------------------------------------
# batch_norm
# ----------------------------------------------------------------------------------------------------------------------
def run_bn(c, p):
    from danet_b200.layers import batch_norm
    x, gx = leaf(p["x"], "x" in c.offset, "x" in c.need)
    w, gw = leaf(p["w"], False, "w" in c.need)
    b, gb = leaf(p["b"], False, "b" in c.need)
    r, gr = (leaf(p["r"], "r" in c.offset, "r" in c.need) if p["r"] is not None else (None, lambda: None))
    rm, rv = p["rm"].to(DEV).clone(), p["rv"].to(DEV).clone()
    y = batch_norm(x, rm, rv, w, b, c.train, S.MOM, S.EPS, residual=r, relu=c.form in ("relu", "res_relu"))
    out = {"y": y.detach().clone(), "rm": rm, "rv": rv}
    if c.need:
        dy = at_offset(p["dy"])[0] if "d" in c.offset else p["dy"].to(DEV)
        y.backward(dy)
        for k, get in (("dx", gx), ("dw", gw), ("db", gb), ("dr", gr)):
            if k[1] in c.need:
                out[k] = get()
    return out


@pytest.mark.parametrize("c", S.BN_CASES, ids=[S.bn_id(c) for c in S.BN_CASES])
def test_batch_norm(c):
    p = S.make_bn(c)
    got = run_bn(c, p)
    relu = c.form in ("relu", "res_relu")
    mask = S.relu_mask(got["y"]) if relu else None
    ref, z = S.bn_reference(c, p, mask, device=DEV)
    if relu:
        # NaN stays NaN (torch's relu), and the op's mask differs from the sign of the fp64 pre-activation only near 0
        assert torch.equal(torch.isnan(got["y"]), torch.isnan(z)), "ReLU output: NaN pattern differs from relu(z)"
        flips = (mask != (z > 0)) & ~torch.isnan(z)
        r_y, M_y, _ = ref["y"]
        assert bool((z[flips].abs() <= 2 * S.C_BN_Y * fb.U24 * M_y[flips] + fb.TINY).all()), "ReLU mask flips away from 0"
    ratios = {}
    for k, (r, M, tiny) in ref.items():
        assert got[k] is not None and got[k].dtype == torch.float32 and got[k].shape == r.shape, k
        if k == "dr":
            fin = torch.isfinite(r)
            assert torch.equal(got[k][fin].double(), r[fin]) and torch.equal(torch.isnan(got[k]), torch.isnan(r)), k
            continue
        # a channel whose x holds +inf: the reference's correction pass makes its mean inf - inf = NaN, while the op
        # keeps the +inf torch's batch_norm gives in the running mean (N4C3_7x7_train_relu_m1_s1_nonfinitex)
        ratios[k] = hold(k, got[k], r, M, S.BN_C[k], tiny, finiteness_only=k == "rm")
    for k in ("dx", "dw", "db", "dr"):
        if k not in ref:
            assert k not in got or got[k] is None, k
    if not c.train:
        assert torch.equal(got["rm"], p["rm"].to(DEV)) and torch.equal(got["rv"], p["rv"].to(DEV))
    report(S.bn_id(c), ratios)


# ----------------------------------------------------------------------------------------------------------------------
# max pool
# ----------------------------------------------------------------------------------------------------------------------
def _slot_index(slot, H, W):
    N, C, Ho, Wo = slot.shape
    s = slot.long()
    oh = torch.arange(Ho, device=DEV).view(1, 1, Ho, 1)
    ow = torch.arange(Wo, device=DEV).view(1, 1, 1, Wo)
    return (2 * oh - 1 + s // 3) * W + (2 * ow - 1 + s % 3)


@pytest.mark.parametrize("c", S.POOL_CASES, ids=[S.pool_id(c) for c in S.POOL_CASES])
def test_max_pool(c):
    from danet_b200.layers import max_pool2d, max_pool_forward
    x, dy = S.make_pool(c)
    x, gx = leaf(x, c.offset, True)
    y_t, idx_t = F.max_pool2d(x.detach(), 3, 2, 1, return_indices=True)
    y0, slot = max_pool_forward(x.detach())
    assert torch.equal(y0.view(torch.int32), y_t.view(torch.int32))
    assert torch.equal(_slot_index(slot, c.H, c.W), idx_t)
    y = max_pool2d(x, 3, 2, 1)
    assert torch.equal(y.detach().view(torch.int32), y_t.view(torch.int32))
    y.backward(dy.to(DEV))
    r, M, cnt = S.pool_backward_reference(idx_t, dy.to(DEV), c.H, c.W)
    dx = gx()
    one = cnt <= 1
    assert torch.equal(dx[one].double(), r[one]), "pool dx: a pixel one window chose is not bit-equal"
    report(S.pool_id(c), {"dx": hold("dx", dx, r, M, S.C_POOL_DX)})


# ----------------------------------------------------------------------------------------------------------------------
# adaptive average pool
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", S.AVG_CASES, ids=[S.avg_id(c) for c in S.AVG_CASES])
def test_adaptive_avg_pool(c):
    from danet_b200.layers import adaptive_avg_pool2d
    x, dy = S.make_avg(c)
    xi, gx = leaf(x, c.offset, True)
    y = adaptive_avg_pool2d(xi, 1)
    xd = x.to(DEV).double()
    HW = c.H * c.W
    ratios = {"y": hold("y", y.detach(), xd.mean((2, 3), keepdim=True), xd.abs().mean((2, 3), keepdim=True),
                        S.c_avg_y(HW))}
    y.backward(dy.to(DEV))
    r = (dy.to(DEV).double() / HW).expand(c.N, c.C, c.H, c.W)
    ratios["dx"] = hold("dx", gx(), r, r.abs(), S.C_AVG_DX)
    report(S.avg_id(c), ratios)


# ----------------------------------------------------------------------------------------------------------------------
# linear
# ----------------------------------------------------------------------------------------------------------------------
def run_lin(c, x, w, b, a, dy):
    from danet_b200.layers import linear
    xi = x.to(DEV).requires_grad_("x" in c.need)
    wi = w.to(DEV).requires_grad_("w" in c.need)
    bi = b.to(DEV).requires_grad_("b" in c.need) if b is not None else None
    y = linear(xi, wi, bi, add=a.to(DEV) if a is not None else None)
    out = {"y": y.detach()}
    if c.need:
        y.backward(dy.to(DEV))
    out.update({"dx": xi.grad, "dw": wi.grad, "db": bi.grad if bi is not None else None})
    return out


@pytest.mark.parametrize("c", S.LIN_CASES, ids=[S.lin_id(c) for c in S.LIN_CASES])
def test_linear(c):
    x, w, b, a, dy = S.make_lin(c)
    got = run_lin(c, x, w, b, a, dy)
    ref = S.lin_reference(*(t.to(DEV) if t is not None else None for t in (x, w, b, a, dy)))
    ratios = {"y": hold("y", got["y"], *ref["y"], S.c_lin_y(c.In))}
    for k in ("dx", "dw", "db"):
        if k[1] in c.need and (k != "db" or c.bias):
            ratios[k] = hold(k, got[k], *ref[k], S.C_SUM)
        else:
            assert got[k] is None, k
    report(S.lin_id(c), ratios)


# ----------------------------------------------------------------------------------------------------------------------
# hr_fuse
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", S.FUSE_CASES, ids=[S.fuse_id(c) for c in S.FUSE_CASES])
def test_hr_fuse(c):
    from danet_b200.layers import hr_fuse
    terms, dy = S.make_fuse(c)
    ins = [leaf(t, "t" in c.offset and j == len(terms) - 1, True) for j, t in enumerate(terms)]
    y = hr_fuse([t for t, _ in ins], list(c.factors), relu=c.relu)
    want = S.fuse_forward_reference([t.to(DEV) for t in terms], c.factors, c.relu)
    assert torch.equal(y.detach().view(torch.int32), want.view(torch.int32)), "hr_fuse forward is not the fp32 chain"
    dyd = at_offset(dy)[0] if "d" in c.offset else dy.to(DEV)
    y.backward(dyd)
    dz = torch.where(S.relu_mask(want), dy.to(DEV), torch.zeros_like(want)) if c.relu else dy.to(DEV)
    ratios = {}
    for j, ((_, get), f) in enumerate(zip(ins, c.factors)):
        r, M = S.fuse_backward_reference(dz, f)
        g = get()
        if f == 1:
            assert torch.equal(g.double(), r), "dterm %d at factor 1 is not the masked dy" % j
        ratios["dt%d(f%d)" % (j, f)] = hold("dterm %d" % j, g, r, M, S.c_fuse_dx(f))
    report(S.fuse_id(c), ratios)


# ----------------------------------------------------------------------------------------------------------------------
# the ReLU's non-finite policy against torch's own ops
# ----------------------------------------------------------------------------------------------------------------------
def test_relu_nan_policy_matches_torch():
    """relu(bn(x)) with NaN and +-inf in x (eval mode: per-element) and a NaN fuse term: the outputs are NaN where
    torch's are, and the gradients pass dy at a NaN output as torch's threshold_backward does"""
    from danet_b200.layers import batch_norm, hr_fuse
    c = S.bn(4, 3, 7, 7, False, "relu", nonfinite="x")
    p = S.make_bn(c)
    outs = []
    for ours in (True, False):
        x = p["x"].to(DEV).clone().requires_grad_()
        args = (p["rm"].to(DEV), p["rv"].to(DEV), p["w"].to(DEV), p["b"].to(DEV), False, S.MOM, S.EPS)
        y = batch_norm(x, *args, relu=True) if ours else F.relu(F.batch_norm(x, *args))
        y.backward(p["dy"].to(DEV))
        outs.append((y.detach(), x.grad))
    (y, dx), (yt, dxt) = outs
    assert bool(torch.isnan(yt).any()) and torch.equal(torch.isnan(y), torch.isnan(yt))
    assert torch.equal(torch.isnan(dx), torch.isnan(dxt)) and torch.equal(dx == 0, dxt == 0)
    t = torch.randn(1, 2, 4, 4, device=DEV)
    t[0, 0, 1, 1] = float("nan")
    tt = t.clone().requires_grad_()
    to = t.clone().requires_grad_()
    gy = torch.randn(1, 2, 4, 4, device=DEV)
    hr_fuse([to], [1]).backward(gy)
    torch.relu(tt).backward(gy)
    assert torch.equal(to.grad, tt.grad)


# ----------------------------------------------------------------------------------------------------------------------
# bit-for-bit repeats
# ----------------------------------------------------------------------------------------------------------------------
REPEAT_BN = [c for c in S.BN_CASES if (c.N, c.C, c.H, c.W) in ((16, 64, 7, 7), (3, 3, 128, 129), (700, 3, 7, 7))]


@pytest.mark.parametrize("c", REPEAT_BN, ids=[S.bn_id(c) for c in REPEAT_BN])
def test_batch_norm_repeats_bits(c):
    p = S.make_bn(c)
    a, b = run_bn(c, p), run_bn(c, p)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_pool_linear_fuse_repeat_bits():
    from danet_b200.layers import adaptive_avg_pool2d, hr_fuse, max_pool2d
    c = S.LIN_CASES[4]
    x, w, b, a, dy = S.make_lin(c)
    r1, r2 = run_lin(c, x, w, b, a, dy), run_lin(c, x, w, b, a, dy)
    for k in r1:
        assert (r1[k] is None and r2[k] is None) or torch.equal(r1[k], r2[k]), k
    for op, shape in ((lambda t: max_pool2d(t, 3, 2, 1), (8, 64, 56, 56)), (lambda t: adaptive_avg_pool2d(t, 1), (2, 64, 56, 56)),
                      (lambda t: hr_fuse([t, t[:, :, ::2, ::2].contiguous()], [1, 2]), (2, 8, 56, 56))):
        x = torch.randn(*shape, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
        res = []
        for _ in range(2):
            xi = x.clone().requires_grad_()
            y = op(xi)
            y.backward(torch.ones_like(y) * 0.37)
            res.append((y.detach(), xi.grad))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


# ----------------------------------------------------------------------------------------------------------------------
# the C entries with NaN-prefilled outputs and workspace give the autograd call's bits
# ----------------------------------------------------------------------------------------------------------------------
def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


PREFILL_BN = [S.bn(16, 64, 7, 7, True, "res_relu"), S.bn(16, 64, 7, 7, False, "res_relu"),
              S.bn(700, 3, 7, 7, True, "relu"), S.bn(5, 3, 1, 1, False, "res")]


@pytest.mark.parametrize("c", PREFILL_BN, ids=[S.bn_id(c) for c in PREFILL_BN])
def test_batch_norm_c_entries_prefilled_nan(c):
    from danet_b200 import _lib
    lib = _lib.load()
    p = S.make_bn(c)
    want = run_bn(c, p)
    N, C, H, W = c.N, c.C, c.H, c.W
    d = {k: (v.to(DEV) if v is not None else None) for k, v in p.items()}
    nb = int(lib.danet_bn2d_workspace_bytes(N, C, H * W))
    ws = torch.full((nb // 4 + 4,), float("nan"), device=DEV)
    y, save, nr = _nan(N, C, H, W), _nan(2, C, dtype=torch.float64), _nan(2, C)
    relu = c.form in ("relu", "res_relu")
    _lib.call("bn2d_forward", N, C, H * W, _lib.ptr(d["x"]), _lib.ptr(d["w"]), _lib.ptr(d["b"]), _lib.ptr(d["rm"]),
              _lib.ptr(d["rv"]), int(c.train), S.MOM, S.EPS, _lib.ptr(d["r"]), int(relu), _lib.ptr(y), _lib.ptr(save),
              _lib.ptr(nr if c.train else None), _lib.ptr(ws), device=DEV)
    assert torch.equal(y, want["y"])
    if c.train:
        assert torch.equal(nr[0], want["rm"]) and torch.equal(nr[1], want["rv"])
    ws.fill_(float("nan"))
    dx, dw, db = _nan(N, C, H, W), _nan(C), _nan(C)
    dr = _nan(N, C, H, W) if d["r"] is not None else None
    _lib.call("bn2d_backward", N, C, H * W, _lib.ptr(d["x"]), _lib.ptr(y if relu else None), _lib.ptr(d["dy"]),
              _lib.ptr(d["w"]), _lib.ptr(save), int(c.train), int(relu), _lib.ptr(dx), _lib.ptr(dw), _lib.ptr(db),
              _lib.ptr(dr), _lib.ptr(ws), device=DEV)
    for k, t in (("dx", dx), ("dw", dw), ("db", db), ("dr", dr)):
        if t is not None:
            assert torch.equal(t, want[k]), k


def test_other_c_entries_prefilled_nan():
    from danet_b200 import _lib
    from danet_b200.layers import adaptive_avg_pool2d, hr_fuse, max_pool2d
    g = torch.Generator(device=DEV).manual_seed(3)
    # linear, forward and backward
    c = S.LIN_CASES[4]
    x, w, b, a, dy = (t.to(DEV) if t is not None else None for t in S.make_lin(c))
    want = run_lin(c, x, w, b, a, dy)
    y, dx, dw, db = _nan(c.N, c.Out), _nan(c.N, c.In), _nan(c.Out, c.In), _nan(c.Out)
    _lib.call("linear", c.N, c.In, c.Out, _lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(a), _lib.ptr(y), device=DEV)
    _lib.call("linear_backward", c.N, c.In, c.Out, _lib.ptr(x), _lib.ptr(w), _lib.ptr(dy), _lib.ptr(dx), _lib.ptr(dw),
              _lib.ptr(db), device=DEV)
    for k, t in (("y", y), ("dx", dx), ("dw", dw), ("db", db)):
        assert torch.equal(t, want[k]), k
    # max pool
    x = torch.randn(2, 5, 9, 7, generator=g, device=DEV)
    gy = torch.randn(2, 5, 5, 4, generator=g, device=DEV)
    xi = x.clone().requires_grad_()
    yo = max_pool2d(xi, 3, 2, 1)
    yo.backward(gy)
    y, slot, dx = _nan(2, 5, 5, 4), torch.full((2, 5, 5, 4), 255, dtype=torch.uint8, device=DEV), _nan(2, 5, 9, 7)
    _lib.call("maxpool3x3s2_nchw_forward", 2, 5, 9, 7, _lib.ptr(x), _lib.ptr(y), _lib.ptr(slot), device=DEV)
    _lib.call("maxpool3x3s2_nchw_backward", 2, 5, 9, 7, _lib.ptr(gy), _lib.ptr(slot), _lib.ptr(dx), device=DEV)
    assert torch.equal(y, yo.detach()) and torch.equal(dx, xi.grad)
    # average pool
    x = torch.randn(3, 5, 7, 7, generator=g, device=DEV)
    gy = torch.randn(3, 5, 1, 1, generator=g, device=DEV)
    xi = x.clone().requires_grad_()
    yo = adaptive_avg_pool2d(xi, 1)
    yo.backward(gy)
    y, dx = _nan(3, 5, 1, 1), _nan(3, 5, 7, 7)
    act = _lib.Act(x.data_ptr(), None, None)
    _lib.call("global_avgpool", 15, 49, 1, ctypes.byref(act), _lib.ptr(y), device=DEV)
    _lib.call("global_avgpool_backward", 15, 49, _lib.ptr(gy), _lib.ptr(dx), device=DEV)
    assert torch.equal(y, yo.detach()) and torch.equal(dx, xi.grad)
    # hr_fuse
    t0, t1 = torch.randn(2, 3, 8, 8, generator=g, device=DEV), torch.randn(2, 3, 4, 4, generator=g, device=DEV)
    gy = torch.randn(2, 3, 8, 8, generator=g, device=DEV)
    a0, a1 = t0.clone().requires_grad_(), t1.clone().requires_grad_()
    yo = hr_fuse([a0, a1], [1, 2])
    yo.backward(gy)
    y, d0, d1 = _nan(2, 3, 8, 8), _nan(2, 3, 8, 8), _nan(2, 3, 4, 4)
    ptrs = (ctypes.c_void_p * 4)(t0.data_ptr(), t1.data_ptr(), 0, 0)
    facs = (ctypes.c_int32 * 4)(1, 2, 0, 0)
    _lib.call("hr_fuse_forward", 2, 3, 8, 8, 2, ptrs, facs, 1, _lib.ptr(y), device=DEV)
    _lib.call("hr_fuse_backward", 2, 3, 8, 8, 1, _lib.ptr(gy), _lib.ptr(y), _lib.ptr(d0), device=DEV)
    _lib.call("hr_fuse_backward", 2, 3, 8, 8, 2, _lib.ptr(gy), _lib.ptr(y), _lib.ptr(d1), device=DEV)
    assert torch.equal(y, yo.detach()) and torch.equal(d0, a0.grad) and torch.equal(d1, a1.grad)


def test_linear_past_2_27_outputs_fills_every_output():
    """N * Out > 2^27 through the C entry into a NaN-prefilled y: every output is written and within the bound"""
    from danet_b200 import _lib
    c = S.BIG_LIN
    x, w, b, _, _ = (t.to(DEV) if t is not None else None for t in S.make_lin(c))
    y = _nan(c.N, c.Out)
    _lib.call("linear", c.N, c.In, c.Out, _lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(None), _lib.ptr(y), device=DEV)
    assert not bool(torch.isnan(y).any()), "outputs left unwritten"
    r = x.double() @ w.double().t() + b.double()
    M = x.double().abs() @ w.double().abs().t() + b.double().abs()
    hold("y", y, r, M, S.c_lin_y(c.In))
