"""CPU side of the training-layer sweep (tests/layers_sweep_common.py): every coverage class has a case; the fp64
reference formulas agree with torch's own ops in fp64; and the bound is tight enough: fp32 emulations of the kernels'
arithmetic (torch CPU float32, one rounding per operation, and the kernels' summation orders) stay within C / 4 of it
where C counts a long serial sum (avgpool y, linear y) and within C / 2 for the short chains (C <= 7, where a few
roundings of one element can line up), while each emulation seeded with one defect fails it on at least one case."""
import math

import pytest
import torch
import torch.nn.functional as F

import fp64_bound as fb
import layers_sweep_common as S

SMALL = 200000                       # cases up to this many elements are emulated on the CPU


def test_every_class_is_covered():
    missing = ["%s: %s" % (op, name) for op, (cases, classes) in S.TABLES.items() for name in fb.uncovered(cases, classes)]
    assert not missing, "uncovered classes: " + "; ".join(missing)


# ----------------------------------------------------------------------------------------------------------------------
# the reference against torch
# ----------------------------------------------------------------------------------------------------------------------
def _close(a, b, what, M=None):
    """a within 1e-12 of b, relative to the largest |b| or, where the result cancels, to the magnitude M"""
    a, b = a.double(), b.double()
    scale = float(b.abs().max()) if M is None else float(torch.as_tensor(M).double().max())
    assert float((a - b).abs().max()) <= 1e-12 * max(scale, 1e-300), what


# torch's own fp64 batch_norm loses about 2^-53 (|mean| / std)^2 of the variance, 3e-11 at 2^20: that ratio is left out
BN_REF_CASES = [c for c in S.BN_CASES if not c.nonfinite and c.N * c.C * c.H * c.W <= 20000 and c.scale == 1.0
                and c.ratio <= 2.0 ** 10]


@pytest.mark.parametrize("c", BN_REF_CASES, ids=[S.bn_id(c) for c in BN_REF_CASES])
def test_bn_reference_against_torch(c):
    p = S.make_bn(c)
    d = {k: (v.double() if v is not None else None) for k, v in p.items()}
    x, w, b = (d[k].clone().requires_grad_() for k in ("x", "w", "b"))
    r = d["r"].clone().requires_grad_() if d["r"] is not None else None
    rm, rv = d["rm"].clone(), d["rv"].clone()
    z = F.batch_norm(x, rm, rv, w, b, c.train, S.MOM, S.EPS)
    if r is not None:
        z = z + r
    relu = c.form in ("relu", "res_relu")
    y = F.relu(z) if relu else z
    y.backward(d["dy"])
    ref, _ = S.bn_reference(c, p, S.relu_mask(y.detach()) if relu else None)
    _close(ref["y"][0], y.detach(), "y", ref["y"][1])
    want = {"dx": x.grad, "dw": w.grad, "db": b.grad, "dr": r.grad if r is not None else None}
    if c.train:
        _close(ref["rm"][0], rm, "rm")
        _close(ref["rv"][0], rv, "rv")
    for k in ("dx", "dw", "db", "dr"):
        if k in ref:
            _close(ref[k][0], want[k], k, ref[k][1])


def test_pool_avg_linear_fuse_references_against_torch():
    for c in S.POOL_CASES[:16]:
        x, dy = S.make_pool(c)
        if c.kind == "nonfinite":
            continue
        xd = x.double().requires_grad_()
        y, idx = F.max_pool2d(xd, 3, 2, 1, return_indices=True)
        y.backward(dy.double())
        _close(S.pool_backward_reference(idx, dy, c.H, c.W)[0], xd.grad, "pool dx " + S.pool_id(c))
    for c in S.AVG_CASES:
        x, dy = S.make_avg(c)
        xd = x.double().requires_grad_()
        y = F.adaptive_avg_pool2d(xd, 1)
        _close(x.double().mean((2, 3), keepdim=True), y.detach(), "avg y")
        y.backward(dy.double())
        _close((dy.double() / (c.H * c.W)).expand_as(xd), xd.grad, "avg dx")
    for c in S.LIN_CASES[:-1]:
        x, w, b, a, dy = S.make_lin(c)
        ref = S.lin_reference(x, w, b, a, dy)
        xd, wd = x.double().requires_grad_(), w.double().requires_grad_()
        bd = b.double().requires_grad_() if b is not None else None
        y = F.linear(xd, wd, bd) + (a.double() if a is not None else 0)
        y.backward(dy.double())
        _close(ref["y"][0], y.detach(), "linear y")
        _close(ref["dx"][0], xd.grad, "linear dx")
        _close(ref["dw"][0], wd.grad, "linear dw")
        if bd is not None:
            _close(ref["db"][0], bd.grad, "linear db")
    for c in S.FUSE_CASES:
        terms, dy = S.make_fuse(c)
        if c.kind == "nan":
            continue
        td = [t.double().requires_grad_() for t in terms]
        y = S.fuse_forward_reference(td, c.factors, False)
        z = F.relu(y) if c.relu else y
        z.backward(dy.double())
        dz = torch.where(S.relu_mask(z.detach()), dy.double(), torch.zeros_like(y)) if c.relu else dy.double()
        for t, f in zip(td, c.factors):
            _close(S.fuse_backward_reference(dz, f)[0], t.grad, "fuse dterm " + S.fuse_id(c))


# ----------------------------------------------------------------------------------------------------------------------
# fp32 emulations of the kernels, each with optional defects
# ----------------------------------------------------------------------------------------------------------------------
def _kernel_sums(a, b, N, HW, drop_last=False):
    """k_db_partial's order in double: per chunk of ipc images, 256 threads add their pixels q = t, t + 256, ... image
    after image, a halving tree adds the threads, then the chunks add in order.  a, b: [N, C, HW] float64 (the values
    after the shift); returns (sum a, sum a * b) per channel"""
    C = a.shape[1]
    ipc = max(1, 16384 // HW)
    nch = -(-N // ipc)
    tot1, tot2 = torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64)
    for j in range(nch - 1 if drop_last and nch > 1 else nch):
        acc1, acc2 = torch.zeros(C, 256, dtype=torch.float64), torch.zeros(C, 256, dtype=torch.float64)
        for n in range(j * ipc, min(N, (j + 1) * ipc)):
            for q0 in range(0, HW, 256):
                blk, bb = a[n, :, q0:q0 + 256], b[n, :, q0:q0 + 256]
                acc1[:, :blk.shape[1]] += blk
                acc2[:, :blk.shape[1]] += blk * bb
        o = 128
        while o:
            acc1[:, :o] += acc1[:, o:2 * o]
            acc2[:, :o] += acc2[:, o:2 * o]
            o //= 2
        tot1 += acc1[:, 0]
        tot2 += acc2[:, 0]
    return tot1, tot2


def _f(t):
    return t.to(torch.float32)


def emulate_bn(c, p, defect=None):
    """{name: got} of the forward and backward kernels in fp32 (torch CPU), with one defect when asked:
    'straddle' (a float4 group that straddles planes takes its first element's channel), 'last_chunk' (the statistics
    drop the last image chunk), 'unshifted_var' (var = sum x^2 / n - mean^2 of unshifted sums), 'biased_running_var'"""
    x, w, b, rm, rv, r, dy = (p[k] for k in ("x", "w", "b", "rm", "rv", "r", "dy"))
    N, C, H, W = x.shape
    HW, n = H * W, N * H * W
    x3 = x.double().reshape(N, C, HW)
    if c.train:
        K = x3[0, :, 0] if defect != "unshifted_var" else torch.zeros(C, dtype=torch.float64)
        s1, s2 = _kernel_sums(x3 - K.view(1, C, 1), x3 - K.view(1, C, 1), N, HW, drop_last=defect == "last_chunk")
        dm = s1 / n
        mean = K + dm
        var = torch.clamp(s2 / n - dm * dm, min=0.0)
        invstd = 1.0 / torch.sqrt(var + S.EPS)
        m = S.MOM
        unb = 1.0 if defect == "biased_running_var" else n / (n - 1)
        new_rm = _f((1 - m) * rm.double() + m * mean)
        new_rv = _f((1 - m) * rv.double() + m * var * unb)
    else:
        mean, invstd = rm.double(), 1.0 / torch.sqrt(rv.double() + S.EPS)
    m_hi = _f(mean)
    m_lo = _f(mean - m_hi.double())
    k = _f(w.double() * invstd)
    # channel of each flat element, as the apply pass looks it up
    total = N * C * HW
    e = torch.arange(total)
    ch = (e // HW) % C
    if defect == "straddle":
        g0 = (e // 4) * 4
        straddle = (g0 // HW) != ((torch.clamp(g0 + 3, max=total - 1)) // HW)
        vec_ok = g0 + 3 < total
        ch = torch.where(straddle & vec_ok, (g0 // HW) % C, ch)
    xf = x.reshape(-1)
    v = ((xf - m_hi[ch]) - m_lo[ch]) * k[ch] + b[ch]
    if r is not None:
        v = v + r.reshape(-1)
    relu = c.form in ("relu", "res_relu")
    if relu:
        v = torch.where((v > 0) | torch.isnan(v), v, torch.zeros_like(v))
    out = {"y": v.view(N, C, H, W)}
    if c.train:
        out["rm"], out["rv"] = new_rm, new_rv
    yv = v
    dz = torch.where(S.relu_mask(yv), dy.reshape(-1), torch.zeros_like(yv)) if relu else dy.reshape(-1)
    dz3 = dz.double().view(N, C, HW)
    sdz = dz3.sum((0, 2))
    sdzx = (dz3 * (x3 - mean.view(1, C, 1))).sum((0, 2))
    if "b" in c.need:
        out["db"] = _f(sdz)
    if "w" in c.need:
        out["dw"] = _f(sdzx * invstd)
    if "x" in c.need:
        kk = _f(w.double() * invstd)
        if c.train:
            c1, c2 = _f(sdz / n), _f(sdzx * invstd * invstd / n)
            dx = (dz - c1[ch] - ((xf - m_hi[ch]) - m_lo[ch]) * c2[ch]) * kk[ch]
        else:
            dx = dz * kk[ch]
        out["dx"] = dx.view(N, C, H, W)
    if "r" in c.need:
        out["dr"] = dz.view(N, C, H, W)
    return out


def emulate_pool_dx(x, dy, skip_fourth=False):
    """k_maxpool3x3s2_bwd: each pixel adds, from 0 in fp32 and in row-major window order, the dy of the windows whose
    first maximum (NaN first) it is; skip_fourth leaves out the fourth window"""
    N, C, H, W = x.shape
    Ho, Wo = dy.shape[2:]
    _, idx = F.max_pool2d(x.double(), 3, 2, 1, return_indices=True)
    dx = torch.zeros(N, C, H * W, dtype=torch.float32)
    count = torch.zeros(N, C, H * W, dtype=torch.int64)
    flat_idx, flat_dy = idx.view(N, C, -1), dy.view(N, C, -1)
    for o in range(Ho * Wo):                      # row-major window order
        i = flat_idx[:, :, o:o + 1]
        cnt = count.gather(2, i)
        add = flat_dy[:, :, o:o + 1]
        if skip_fourth:
            add = torch.where(cnt >= 3, torch.zeros_like(add), add)
        dx.scatter_(2, i, dx.gather(2, i) + add)
        count.scatter_(2, i, cnt + 1)
    return dx.view(N, C, H, W), idx


def emulate_avg(x, dy, bad_divisor=False):
    N, C, H, W = x.shape
    HW = H * W
    xs = x.reshape(N, C, HW)
    s = torch.zeros(N, C, dtype=torch.float32)
    for q in range(HW):
        s = s + xs[:, :, q]
    y = (s / float(HW)).view(N, C, 1, 1)
    dx = (dy / float(HW - 1 if bad_divisor else HW)).expand(N, C, H, W)
    return y, dx


def emulate_linear_y(x, w, b, a, drop_tail=False):
    """k_linear: lane l FMAs x[i] w[i] for i = l, l + 32, ... (fp32, an FMA rounds once); a 5-step xor shuffle tree;
    lane 0 adds b, then add.  drop_tail leaves out the last, partial lane group"""
    N, In = x.shape
    end = (In // 32) * 32 if drop_tail else In
    lanes = torch.zeros(N, w.shape[0], 32, dtype=torch.float32)
    for i in range(end):
        prod = x[:, i].double().view(N, 1) * w[:, i].double().view(1, -1)
        lanes[:, :, i % 32] = _f(lanes[:, :, i % 32].double() + prod)
    ar = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, :, ar ^ o]
    y = lanes[:, :, 0]
    y = y + (b if b is not None else 0.0)
    y = y + (a if a is not None else 0.0)
    return y


def emulate_fuse_dt(dz, f, bad_stride=False):
    """k_hr_fuse_bwd: a dterm element adds its f x f block of the masked dy in row-major order, from 0 in fp32;
    bad_stride steps the block's rows by W / f instead of W"""
    N, C, H, W = dz.shape
    flat = dz.reshape(-1)
    Hj, Wj = H // f, W // f
    i = torch.arange(N * C * Hj * Wj)
    row, wj = i // Wj, i % Wj
    stride = Wj if bad_stride else W
    acc = torch.zeros(i.shape[0], dtype=torch.float32)
    for rr in range(f):
        for q in range(f):
            e = (row * f + rr) * stride + wj * f + q if not bad_stride else row * f * W + rr * stride + wj * f + q
            acc = acc + flat[e.clamp(max=flat.numel() - 1)]
    return acc.view(N, C, Hj, Wj)


# ----------------------------------------------------------------------------------------------------------------------
# the bound against the emulations
# ----------------------------------------------------------------------------------------------------------------------
BN_EMU = [c for c in S.BN_CASES if c.N * c.C * c.H * c.W <= SMALL and not c.nonfinite]


def _worst(got, r, M, tiny=fb.TINY):
    """the excess over the floor in units of 2^-24 M: <= C passes"""
    return fb.worst(got, r, fb.U24 * M, fb.U24 * r.abs() + tiny)[0]


def _bn_ratios(c, defect=None):
    p = S.make_bn(c)
    got = emulate_bn(c, p, defect)
    relu = c.form in ("relu", "res_relu")
    ref, _ = S.bn_reference(c, p, S.relu_mask(got["y"]) if relu else None)
    out = {}
    for k, (r, M, tiny) in ref.items():
        if k != "dr":
            out[k] = (_worst(got[k], r, M, tiny), S.BN_C[k])
    return out


def test_bn_emulation_within_half_the_bound():
    worst = {}
    for c in BN_EMU:
        for k, (q, C) in _bn_ratios(c).items():
            assert q <= C / 2, (S.bn_id(c), k, q, C)
            worst[k] = max(worst.get(k, -math.inf), q)
    print("batch_norm emulation, worst excess over the floor in units of 2^-24 M:", worst)


@pytest.mark.parametrize("defect", ["straddle", "last_chunk", "unshifted_var", "biased_running_var"])
def test_bn_bound_catches(defect):
    cases = [c for c in BN_EMU if defect != "unshifted_var" or c.ratio == 2.0 ** 20]
    if defect == "last_chunk":
        cases = [c for c in S.BN_CASES if c.train and S.chan_chunks(c.N, c.H * c.W) >= 2 and not c.nonfinite]
    failed = [S.bn_id(c) for c in cases if c.train or defect == "straddle"
              if any(q > C for q, C in _bn_ratios(c, defect).values())]
    assert failed, "no case fails the bound with the %s defect" % defect
    print(defect, "fails on", len(failed), "cases, e.g.", failed[:3])


def _pool_case_ratio(c, skip_fourth):
    x, dy = S.make_pool(c)
    dx, idx = emulate_pool_dx(x, dy, skip_fourth)
    r, M, _ = S.pool_backward_reference(idx, dy, c.H, c.W)
    return _worst(dx, r, M)


def _avg_ratios(c, bad):
    x, dy = S.make_avg(c)
    y, dx = emulate_avg(x, dy, bad)
    HW = c.H * c.W
    xd = x.double()
    r = (dy.double() / HW).expand_as(xd)
    return (_worst(y, xd.mean((2, 3), keepdim=True), xd.abs().mean((2, 3), keepdim=True)),
            _worst(dx, r, r.abs()))


def _lin_ratio(c, drop):
    x, w, b, a, dy = S.make_lin(c)
    r, M = S.lin_reference(x, w, b, a, dy)["y"]
    return _worst(emulate_linear_y(x, w, b, a, drop), r, M)


def _fuse_ratios(c, bad):
    terms, dy = S.make_fuse(c)
    y = S.fuse_forward_reference(terms, c.factors, c.relu)
    dz = torch.where(S.relu_mask(y), dy, torch.zeros_like(dy)) if c.relu else dy
    out = []
    for f in c.factors:
        r, M = S.fuse_backward_reference(dz, f)
        out.append((_worst(emulate_fuse_dt(dz, f, bad), r, M), S.c_fuse_dx(f)))
    return out


POOL_EMU = [c for c in S.POOL_CASES if c.N * c.C * c.H * c.W <= 20000]
AVG_EMU = [c for c in S.AVG_CASES if c.N * c.C * c.H * c.W <= SMALL]
LIN_EMU = [c for c in S.LIN_CASES if c.N * c.Out * c.In <= 3000000]
FUSE_EMU = [c for c in S.FUSE_CASES if c.N * c.C * c.H * c.W <= 20000]


def test_other_emulations_well_within_the_bound():
    for c in POOL_EMU:
        q = _pool_case_ratio(c, False)
        assert q <= S.C_POOL_DX / 2, (S.pool_id(c), q)
    for c in AVG_EMU:
        qy, qd = _avg_ratios(c, False)
        assert qy <= S.c_avg_y(c.H * c.W) / 4 and qd <= S.C_AVG_DX / 2, (S.avg_id(c), qy, qd)
    for c in LIN_EMU:
        q = _lin_ratio(c, False)
        assert q <= S.c_lin_y(c.In) / 4, (S.lin_id(c), q)
    for c in FUSE_EMU:
        if c.kind == "nan":
            continue
        for q, C in _fuse_ratios(c, False):
            assert q <= C / 2, (S.fuse_id(c), q, C)


def test_bound_catches_the_fourth_pool_window_skipped():
    assert any(_pool_case_ratio(c, True) > S.C_POOL_DX for c in POOL_EMU if c.kind != "nonfinite")


def test_bound_catches_avgpool_backward_over_hw_minus_1():
    assert any(_avg_ratios(c, True)[1] > S.C_AVG_DX for c in AVG_EMU)


def test_bound_catches_linear_dropping_the_last_partial_lane_group():
    assert any(_lin_ratio(c, True) > S.c_lin_y(c.In) for c in LIN_EMU if c.In % 32)


def test_bound_catches_the_wrong_fuse_row_stride():
    assert any(q > C for c in FUSE_EMU if c.kind != "nan" for q, C in _fuse_ratios(c, True))
