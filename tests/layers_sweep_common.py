"""The covering sweep of the training layers of danet_b200.layers (csrc/bn_train.cu, and k_linear / k_global_avgpool
of csrc/glue.cu): batch_norm, max_pool2d, adaptive_avg_pool2d, linear and hr_fuse, forward and backward.  This file
holds the case tables, the coverage classes, the inputs, the fp64 reference and the per-element bound.
tests/test_layers_sweep_cpu.py fails with the names of uncovered classes, checks the reference against torch's own ops
and shows that the bound catches a set of wrong kernels (numpy emulations); tests/test_layers_sweep_gpu.py runs every
case on the GPU.

The bound: each output element against its fp64 reference r,

    |got - r| <= C * 2^-24 * M + 2^-24 * |r| + tiny

with M the element's magnitude, computed from absolute values (reference() below), and tiny the subnormal floor:
2^-149, times 1 + |w| invstd where a BatchNorm result multiplies an fp32 difference by w * invstd.  A rounded fp32
operation moves a term of the exact result by at most 2^-24 of that term, so C is the longest chain of rounded fp32
operations a term of the result passes through in the kernel; the 2^-24 |r| term is the final rounding.  Sums in double
add at most (terms) * 2^-53 relative, far below one fp32 unit at every size here, and count as nothing.

    BatchNorm y         ((x - m_hi) - m_lo) * k + b (+ r): the two subtractions, k = fl(w invstd), the product, + b,
                        + r: C_BN_Y = 6.  mean and invstd come from double sums.  The variance is
                        sum (x - K)^2 / n - (mean - K)^2 with K a data element, so it cancels at most n - 1 < 2^21 of
                        the double sums: 2^-32 relative at most.
    BatchNorm dx        train: (dz - c1 - ((x - m_hi) - m_lo) * c2) * k, c1 = fl(sum dz / n),
                        c2 = fl(invstd^2 sum dz (x - mean) / n): the x-hat term passes the two subtractions, c2's
                        rounding, the product, the subtraction from dz - c1, k's rounding and the last product:
                        C_BN_DX = 7; eval: dz * k, 2.
    dweight, dbias,     one rounding of a double sum: C_SUM = 1.
    running statistics
    max pool dx         a pixel adds the dy of at most four windows from 0 in fp32: C_POOL_DX = 3 (1 chooser: exact).
    avgpool y           HW - 1 serial fp32 additions, then / HW (its rounding is the |r| term): C = HW - 1.
    avgpool dx          dy / HW, one rounding: C_AVG_DX = 1.
    linear y            a lane's ceil(In / 32) FMAs, 5 shuffle additions, + b, + add: C = ceil(In / 32) + 7.
    linear dx, dW, db   one rounding of a double sum: C_SUM = 1.
    hr_fuse dterm       a thread adds the f x f masked dy of its block from 0 in fp32: C = f^2 - 1 (f = 1: exact).

Exact results are held to equality instead: the max-pool forward and slots (to torch's CUDA max_pool2d), the pool
backward where one window chose the pixel, the hr_fuse forward (to the fp32 torch chain) and d residual.

The ReLU policy (NaN and +-inf stay non-finite): relu(NaN) = NaN, and the backward passes dy except where y <= 0, so
a NaN output passes dy, as torch's threshold_backward does.  The reference takes its ReLU mask from the op under test
(not y <= 0); the sweep checks that the mask differs from the fp64 pre-activation's sign only near zero.
"""
import collections
import itertools
import math

import torch
import torch.nn.functional as F

from fp64_bound import TINY
MOM, EPS = 0.1, 1e-5

C_BN_Y = 6
C_BN_DX = 7
C_SUM = 1
C_POOL_DX = 3
C_AVG_DX = 1


def c_avg_y(HW):
    return max(HW - 1, 0)


def c_lin_y(In):
    return -(-In // 32) + 7


def c_fuse_dx(f):
    return f * f - 1


def chan_chunks(N, HW):
    """chan_sums_chunks of csrc/conv_wgrad.cu: images per chunk max(1, 16384 // HW)"""
    ipc = max(1, 16384 // HW)
    return -(-N // ipc)


# ----------------------------------------------------------------------------------------------------------------------
# batch_norm cases
# ----------------------------------------------------------------------------------------------------------------------
BN = collections.namedtuple("BN", ["N", "C", "H", "W", "train", "form", "ratio", "scale", "w", "dy", "const", "offset",
                                   "need", "nonfinite"])
FORMS = ("bn", "relu", "res_relu", "res")
RATIOS = (0.0, 1.0, 2.0 ** 10, 2.0 ** 20)


def bn(N, C, H, W, train=True, form="res_relu", ratio=1.0, scale=1.0, w="normal", dy="normal", const=False, offset="",
       need="xwbr", nonfinite=""):
    if "r" in need and not form.startswith("res"):
        need = need.replace("r", "")
    return BN(N, C, H, W, train, form, ratio, scale, w, dy, const, offset, need, nonfinite)


BN_CASES = [
    # forms, train and eval, at the network's shapes
    bn(2, 64, 28, 28, True, "relu"), bn(2, 64, 28, 28, False, "relu"),
    bn(16, 64, 7, 7, True, "res_relu"), bn(16, 64, 7, 7, False, "res_relu"),
    bn(4, 128, 7, 7, True, "bn"), bn(4, 128, 7, 7, False, "bn"),
    bn(2, 32, 14, 14, True, "res"), bn(2, 32, 14, 14, False, "res"),
    bn(1, 3072, 2, 2, True, "res_relu"), bn(2, 3072, 2, 2, False, "relu"),
    bn(4, 3072, 7, 7, True, "relu", ratio=2.0 ** 10),
    bn(16, 64, 56, 56, True, "relu"),
    # planes that straddle float4 groups, and N * C * HW % 4 != 0
    bn(2, 3, 1, 1, True, "res_relu"), bn(3, 1, 1, 1, True, "relu"), bn(5, 3, 1, 1, False, "res"),
    bn(1, 3, 1, 2, True, "res_relu"), bn(3, 3, 1, 2, False, "relu"), bn(2, 1, 1, 2, True, "bn"),
    bn(3, 3, 1, 3, True, "res_relu"), bn(2, 5, 3, 1, False, "res_relu"),
    bn(3, 3, 1, 5, True, "relu"), bn(2, 7, 5, 1, True, "res"),
    bn(3, 5, 7, 7, True, "res_relu"), bn(3, 5, 7, 7, False, "bn"),
    # one image per chunk (HW >= 16384), and three or more chunks
    bn(3, 3, 128, 129, True, "res_relu"), bn(2, 1, 130, 130, False, "relu"),
    bn(700, 3, 7, 7, True, "res_relu"), bn(1000, 1, 7, 7, True, "relu", ratio=2.0 ** 20),
    # |mean| / std
    bn(4, 3, 28, 28, True, "res_relu", ratio=0.0), bn(4, 3, 28, 28, True, "relu", ratio=2.0 ** 10),
    bn(4, 3, 28, 28, True, "relu", ratio=2.0 ** 20), bn(16, 3, 56, 56, True, "bn", ratio=2.0 ** 20),
    bn(2, 3, 1, 1, True, "res", ratio=2.0 ** 20), bn(4, 3, 28, 28, False, "res_relu", ratio=2.0 ** 20),
    bn(4, 3072, 2, 2, True, "res_relu", ratio=2.0 ** 20),
    # operand scales
    bn(4, 3, 14, 14, True, "res_relu", scale=2.0 ** -120), bn(4, 3, 14, 14, False, "relu", scale=2.0 ** -120),
    bn(4, 3, 14, 14, True, "res_relu", scale=2.0 ** 60), bn(4, 3, 14, 14, False, "bn", scale=2.0 ** 60),
    # constant channel, weights
    bn(4, 3, 14, 14, True, "relu", const=True), bn(4, 3, 5, 5, True, "res_relu", const=True),
    bn(4, 3, 14, 14, False, "relu", const=True),
    bn(4, 3, 14, 14, True, "res_relu", w="zero"), bn(4, 3, 14, 14, True, "relu", w="neg"),
    bn(4, 3, 14, 14, False, "res", w="neg"),
    # upstream gradients
    bn(4, 3, 14, 14, True, "res_relu", dy="tiny"), bn(4, 3, 14, 14, False, "relu", dy="tiny"),
    bn(4, 3, 14, 14, True, "res_relu", dy="huge"), bn(4, 3, 14, 14, True, "bn", dy="spike"),
    bn(16, 64, 7, 7, False, "res_relu", dy="spike"),
    # storage offsets: the scalar apply paths
    bn(3, 3, 1, 5, True, "res_relu", offset="x"), bn(4, 3, 7, 7, True, "res_relu", offset="r"),
    bn(4, 3, 7, 7, True, "res_relu", offset="d"), bn(2, 5, 3, 1, False, "res_relu", offset="xd"),
    bn(4, 3, 7, 7, True, "relu", offset="xrd"), bn(2, 64, 28, 28, True, "relu", offset="d"),
    # non-finite values
    bn(4, 3, 7, 7, True, "relu", nonfinite="x"), bn(4, 3, 7, 7, False, "relu", nonfinite="x"),
    bn(4, 3, 7, 7, False, "res_relu", nonfinite="r"), bn(4, 3, 7, 7, True, "res_relu", nonfinite="r"),
    bn(4, 3, 7, 7, True, "res_relu", nonfinite="d"), bn(4, 3, 7, 7, False, "bn", nonfinite="d"),
]
# every needs_input_grad subset, training and eval
for _k, _sub in enumerate(s for n in range(1, 5) for s in itertools.combinations("xwbr", n)):
    for _train in (True, False):
        BN_CASES.append(bn(2, 3, 5, 5, _train, "res_relu", need="".join(_sub)))
BN_CASES.append(bn(2, 3, 5, 5, False, "relu", need="x"))


def bn_id(c):
    s = "N%dC%d_%dx%d_%s_%s_m%g_s%g" % (c.N, c.C, c.H, c.W, "train" if c.train else "eval", c.form, c.ratio, c.scale)
    for k in ("w", "dy"):
        if getattr(c, k) != "normal":
            s += "_%s%s" % (k, getattr(c, k))
    if c.const:
        s += "_const"
    if c.offset:
        s += "_off" + c.offset
    if c.need != "xwbr" and c.need != "xwb":
        s += "_need" + c.need
    if c.nonfinite:
        s += "_nonfinite" + c.nonfinite
    return s


def _bn_classes():
    cl = []
    for f in FORMS:
        cl.append(("train " + f, lambda c, f=f: c.train and c.form == f))
        cl.append(("eval " + f, lambda c, f=f: not c.train and c.form == f))
    for C in (1, 3, 3072):
        cl.append(("C = %d" % C, lambda c, C=C: c.C == C))
    cl.append(("HW = 1, N >= 2", lambda c: c.H * c.W == 1 and c.N >= 2))
    for HW in (2, 3, 5, 49, 4, 3136):
        cl.append(("HW = %d" % HW, lambda c, HW=HW: c.H * c.W == HW))
    cl.append(("HW >= 16384 (one image per chunk)", lambda c: c.H * c.W >= 16384))
    cl.append(("three or more chunks", lambda c: chan_chunks(c.N, c.H * c.W) >= 3))
    cl.append(("N*C*HW % 4 != 0", lambda c: (c.N * c.C * c.H * c.W) % 4 != 0))
    cl.append(("N*HW = 2", lambda c: c.N * c.H * c.W == 2))
    cl.append(("x offset alone", lambda c: c.offset == "x"))
    cl.append(("residual offset alone", lambda c: c.offset == "r"))
    cl.append(("dy offset alone", lambda c: c.offset == "d"))
    cl.append(("mixed offsets", lambda c: len(c.offset) >= 2))
    for r in RATIOS:
        cl.append(("|mean|/std = %g" % r, lambda c, r=r: c.ratio == r and not c.const))
    for s in (2.0 ** -120, 2.0 ** 60):
        cl.append(("scale %g" % s, lambda c, s=s: c.scale == s))
    cl.append(("constant channel, train", lambda c: c.const and c.train))
    cl.append(("constant channel, eval", lambda c: c.const and not c.train))
    cl.append(("w = 0", lambda c: c.w == "zero"))
    cl.append(("w < 0", lambda c: c.w == "neg"))
    for d in ("tiny", "huge", "spike"):
        cl.append(("dy " + d, lambda c, d=d: c.dy == d))
    for n in range(1, 5):
        for sub in itertools.combinations("xwbr", n):
            s = "".join(sub)
            cl.append(("needs %s" % s, lambda c, s=s: c.need == s))
    cl.append(("eval dx only (no sums)", lambda c: not c.train and c.need == "x"))
    cl.append(("d residual only (no sums)", lambda c: c.need == "r"))
    for t in ("x", "r", "d"):
        cl.append(("non-finite in " + t, lambda c, t=t: c.nonfinite == t))
    return cl


BN_CLASSES = _bn_classes()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def make_bn(c, seed=0):
    """fp32 CPU tensors of a case: x, w, b, rm, rv, r (or None), dy"""
    g = _gen(1000 + seed + (BN_CASES.index(c) if c in BN_CASES else 0))
    N, C, H, W = c.N, c.C, c.H, c.W
    rn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    sd = c.scale * (0.5 + torch.rand(C, generator=g, dtype=torch.float64))
    mu = c.ratio * sd * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0).double() + 0.3 * sd * rn(C)
    x = rn(N, C, H, W) * sd.view(1, C, 1, 1) + mu.view(1, C, 1, 1)
    b = 0.3 * rn(C)
    if c.const:
        x[:, 0] = 3.0
        b[0] = 0.0                                            # y = 0 exactly: exact-zero ReLU inputs
    w = {"normal": 1 + 0.3 * rn(C), "zero": torch.zeros(C, dtype=torch.float64),
         "neg": -(1 + 0.3 * rn(C).abs())}[c.w]
    if c.w == "normal" and C >= 3:
        w[1] = -w[1].abs()                                   # one negative weight in every case
    xf = x.float()
    bm, bv = xf.double().mean((0, 2, 3)), xf.double().var((0, 2, 3), unbiased=False)
    rm = bm + 0.1 * sd * rn(C)
    rv = torch.where(bv > 0, bv * (0.8 + 0.4 * torch.rand(C, generator=g, dtype=torch.float64)), sd * sd)
    r = rn(N, C, H, W) if c.form.startswith("res") else None
    dy = rn(N, C, H, W)
    if c.dy == "tiny":
        dy = dy * 2.0 ** -120
    elif c.dy == "huge":
        dy = dy * 2.0 ** 60
    elif c.dy == "spike":
        dy.view(-1)[dy.numel() // 3] = 2.0 ** 20
    out = {"x": xf, "w": w.float(), "b": b.float(), "rm": rm.float(), "rv": rv.float(),
           "r": None if r is None else r.float(), "dy": dy.float()}
    if c.nonfinite:
        t = out[{"x": "x", "r": "r", "d": "dy"}[c.nonfinite]]
        t[0, 0, 0, 1] = float("nan")
        t[1, 1, 0, 0] = float("inf")
        t[2, 1, 1, 2] = float("-inf")
        t[3, 2, 0, 0] = float("inf")
    return out


def bn_reference(c, p, mask=None, device="cpu"):
    """{name: (r, M, tiny)} in fp64 for y, rm, rv and the gradients the case needs; mask (bool, the op's y > 0 or NaN)
    is the ReLU's, None without ReLU.  Two-pass mean and variance."""
    d = lambda t: None if t is None else t.to(device=device, dtype=torch.float64)
    x, w, b, rm, rv, r, dy = (d(p[k]) for k in ("x", "w", "b", "rm", "rv", "r", "dy"))
    N, C, H, W = x.shape
    n = N * H * W
    v = lambda t: t.view(1, C, 1, 1)
    if c.train:
        mean = x.sum((0, 2, 3)) / n                       # then one correction pass: exact enough at any |mean| / std
        mean = mean + (x - v(mean)).sum((0, 2, 3)) / n
        var = ((x - v(mean)) ** 2).sum((0, 2, 3)) / n
    else:
        mean, var = rm, rv
    invstd = 1.0 / torch.sqrt(var + EPS)
    xh = (x - v(mean)) * v(invstd)
    z = xh * v(w) + v(b)
    if r is not None:
        z = z + r
    relu = c.form in ("relu", "res_relu")
    y = torch.where(mask, z, torch.zeros_like(z)) if relu else z
    wi = w.abs() * invstd
    out = {"y": (y, (x - v(mean)).abs() * v(wi) + v(b.abs()) + (0 if r is None else r.abs()),
                 TINY * (1 + 2 * v(wi)).expand_as(x))}
    if c.train:
        m = MOM
        out["rm"] = ((1 - m) * rm + m * mean, (1 - m) * rm.abs() + m * mean.abs(), TINY)
        vu = var * n / (n - 1)
        out["rv"] = ((1 - m) * rv + m * vu, (1 - m) * rv.abs() + m * vu, TINY)
    dz = torch.where(mask, dy, torch.zeros_like(dy)) if relu else dy
    adz = dz.abs()
    sdz, sdzxh = dz.sum((0, 2, 3)), (dz * xh).sum((0, 2, 3))
    asdz, asdzxh = adz.sum((0, 2, 3)), (adz * xh.abs()).sum((0, 2, 3))
    if "x" in c.need:
        if c.train:
            dx = v(w * invstd) * (dz - v(sdz / n) - xh * v(sdzxh / n))
            M = v(wi) * (adz + v(asdz / n) + xh.abs() * v(asdzxh / n))
            tiny = TINY * (1 + v(wi) * (4 + 2 * v(invstd * asdzxh / n)))
        else:
            dx, M, tiny = v(w * invstd) * dz, v(wi) * adz, TINY * (1 + 2 * v(wi))
        out["dx"] = (dx, M, tiny.expand_as(dx))
    if "w" in c.need:
        out["dw"] = (sdzxh, asdzxh, TINY)
    if "b" in c.need:
        out["db"] = (sdz, asdz, TINY)
    if "r" in c.need:
        out["dr"] = (dz, adz, 0.0)
    return out, z


BN_C = {"y": C_BN_Y, "rm": C_SUM, "rv": C_SUM, "dx": C_BN_DX, "dw": C_SUM, "db": C_SUM, "dr": 0}

# ----------------------------------------------------------------------------------------------------------------------
# max pool 3 x 3 / 2 / 1
# ----------------------------------------------------------------------------------------------------------------------
Pool = collections.namedtuple("Pool", ["N", "C", "H", "W", "kind", "offset"])
POOL_KINDS = ("normal", "ties", "nonfinite")
POOL_CASES = [Pool(2, 3, H, W, k, False) for H, W, k in [
    (1, 1, "normal"), (1, 2, "ties"), (2, 1, "normal"), (2, 3, "ties"), (3, 2, "normal"), (3, 4, "nonfinite"),
    (4, 5, "ties"), (5, 4, "normal"), (5, 9, "nonfinite"), (9, 5, "ties"), (9, 9, "normal"), (4, 4, "ties"),
    (1, 9, "normal"), (9, 1, "ties"), (3, 3, "nonfinite"), (5, 5, "ties")]] + [
    Pool(2, 3, 9, 9, "ties", True), Pool(3, 5, 5, 4, "nonfinite", True), Pool(1, 1, 1, 1, "normal", True),
    Pool(8, 64, 56, 56, "ties", False), Pool(8, 64, 56, 56, "normal", False), Pool(16, 64, 28, 28, "ties", False)]


def pool_id(c):
    return "N%dC%d_%dx%d_%s%s" % (c.N, c.C, c.H, c.W, c.kind, "_off" if c.offset else "")


WAVE = 132 * 2048           # threads that one wave of 256-thread blocks holds on an H100 (132 SMs x 2048)


def _pool_classes():
    cl = []
    for v in (1, 2, 3, 4, 5, 9):
        cl.append(("H = %d" % v, lambda c, v=v: c.H == v))
        cl.append(("W = %d" % v, lambda c, v=v: c.W == v))
    cl.append(("non-square", lambda c: c.H != c.W))
    for k in POOL_KINDS:
        cl.append((k, lambda c, k=k: c.kind == k))
    cl.append(("windows all -inf", lambda c: c.kind == "nonfinite" and c.H >= 3 and c.W >= 3))
    cl.append(("offset input", lambda c: c.offset))
    cl.append(("forward more than one wave", lambda c: c.N * c.C * ((c.H + 1) // 2) * ((c.W + 1) // 2) > WAVE))
    cl.append(("backward more than one wave", lambda c: c.N * c.C * c.H * c.W > WAVE))
    cl.append(("a pixel chosen by four windows", lambda c: c.kind == "ties" and c.H >= 4 and c.W >= 4))
    return cl


POOL_CLASSES = _pool_classes()


def make_pool(c, seed=0):
    g = _gen(2000 + seed + (POOL_CASES.index(c) if c in POOL_CASES else 0))
    N, C, H, W = c.N, c.C, c.H, c.W
    if c.kind == "ties":
        x = torch.randint(-2, 3, (N, C, H, W), generator=g).float().clamp_min(0)
        x[:, :, 1::4, 1::4] = 10.0          # odd-odd pixels: the maximum of all four of their windows
    else:
        x = torch.randn(N, C, H, W, generator=g)
    if c.kind == "nonfinite":
        x[0, 0, 0, 0] = float("nan")
        x[0, 1].view(-1)[-1] = float("inf")
        x[1, 0].view(-1)[x[1, 0].numel() // 2] = float("nan")
        x[1, 1] = float("-inf")             # every window of the plane is -inf
        x[1, 2, 0, 0] = float("-inf")
    dy = torch.randn(N, C, (H + 1) // 2, (W + 1) // 2, generator=g)
    return x, dy


def pool_backward_reference(idx, dy, H, W):
    """(dx, M, count) in fp64 from the flat window indices idx (torch's): dx adds dy over the windows that chose a
    pixel, M adds |dy|, count is the number of windows"""
    N, C = dy.shape[:2]
    flat = lambda t: t.reshape(N * C, -1)
    i = flat(idx.long())
    z = torch.zeros(N * C, H * W, dtype=torch.float64, device=dy.device)
    dx = z.clone().scatter_add_(1, i, flat(dy.double())).view(N, C, H, W)
    M = z.clone().scatter_add_(1, i, flat(dy.double().abs())).view(N, C, H, W)
    cnt = z.clone().scatter_add_(1, i, torch.ones_like(flat(dy.double()))).view(N, C, H, W)
    return dx, M, cnt


# ----------------------------------------------------------------------------------------------------------------------
# adaptive average pool (output 1)
# ----------------------------------------------------------------------------------------------------------------------
Avg = collections.namedtuple("Avg", ["N", "C", "H", "W", "kind", "offset"])
AVG_CASES = [Avg(3, 5, 1, 1, "normal", False), Avg(1, 3, 1, 2, "mixed", False), Avg(3, 7, 7, 7, "normal", False),
             Avg(2, 64, 56, 56, "mixed", False), Avg(1, 3, 129, 129, "normal", False), Avg(1, 3, 129, 129, "mixed", False),
             Avg(16, 512, 7, 7, "normal", False), Avg(3, 5, 7, 7, "mixed", True), Avg(1, 1, 1, 1, "normal", True)]


def avg_id(c):
    return "N%dC%d_%dx%d_%s%s" % (c.N, c.C, c.H, c.W, c.kind, "_off" if c.offset else "")


AVG_CLASSES = [("HW = %d" % v, lambda c, v=v: c.H * c.W == v) for v in (1, 2, 49, 3136, 16641)] + [
    ("odd N*C", lambda c: (c.N * c.C) % 2 == 1), ("mixed magnitudes", lambda c: c.kind == "mixed"),
    ("offset input", lambda c: c.offset)]


def make_avg(c, seed=0):
    g = _gen(3000 + seed + (AVG_CASES.index(c) if c in AVG_CASES else 0))
    x = torch.randn(c.N, c.C, c.H, c.W, generator=g, dtype=torch.float64)
    if c.kind == "mixed":                   # magnitudes 2^-40 .. 2^40 within a plane
        x = x * torch.exp2(torch.randint(-40, 41, x.shape, generator=g).double())
    dy = torch.randn(c.N, c.C, 1, 1, generator=g)
    return x.float(), dy


# ----------------------------------------------------------------------------------------------------------------------
# linear
# ----------------------------------------------------------------------------------------------------------------------
Lin = collections.namedtuple("Lin", ["N", "In", "Out", "bias", "add", "need"])
BIG_LIN = Lin(131073, 1, 1024, True, False, "xwb")          # N * Out = 2^27 + 1024
LIN_CASES = [Lin(N, In, Out, b, a, nd) for N, In, Out, b, a, nd in [
    (1, 1, 1, False, False, "xwb"), (2, 31, 13, True, False, "xwb"), (65, 32, 85, True, True, "xwb"),
    (2, 33, 1024, False, True, "xw"), (65, 2049, 85, True, True, "xwb"), (1, 2049, 13, True, False, "w"),
    (65, 1, 1024, False, False, "x"), (2, 33, 85, True, True, "b"), (1, 31, 1, True, True, "wb"),
    (65, 2049, 1, False, True, "xb"), (2, 32, 13, False, False, ""), (65, 33, 13, True, True, "xwb"),
    (16, 2048, 85, True, True, "xwb"), (16, 512, 1024, True, False, "xwb")]] + [BIG_LIN]


def lin_id(c):
    return "N%d_In%d_Out%d%s%s_need%s" % (c.N, c.In, c.Out, "_b" if c.bias else "", "_add" if c.add else "", c.need or "-")


LIN_CLASSES = ([("In = %d" % v, lambda c, v=v: c.In == v) for v in (1, 31, 32, 33, 2049)] +
               [("Out = %d" % v, lambda c, v=v: c.Out == v) for v in (1, 13, 85, 1024)] +
               [("N = %d" % v, lambda c, v=v: c.N == v) for v in (1, 2, 65)] +
               [("bias %s, add %s" % (b, a), lambda c, b=b, a=a: c.bias == b and c.add == a)
                for b in (False, True) for a in (False, True)] +
               [("needs %s" % (s or "nothing"), lambda c, s=s: c.need == s)
                for s in ("", "x", "w", "b", "xw", "xb", "wb", "xwb")] +
               [("N*Out > 2^27", lambda c: c.N * c.Out > 2 ** 27)])


def make_lin(c, seed=0):
    g = _gen(4000 + seed + (LIN_CASES.index(c) if c in LIN_CASES else 0))
    x = torch.randn(c.N, c.In, generator=g)
    w = torch.randn(c.Out, c.In, generator=g) / math.sqrt(c.In)
    b = torch.randn(c.Out, generator=g) if c.bias else None
    a = torch.randn(c.Out, generator=g) * 4 if c.add else None
    dy = torch.randn(c.N, c.Out, generator=g)
    return x, w, b, a, dy


def lin_reference(x, w, b, a, dy):
    """{name: (r, M)} in fp64"""
    x, w, dy = x.double(), w.double(), dy.double()
    y, M = x @ w.t(), x.abs() @ w.abs().t()
    for t in (b, a):
        if t is not None:
            y, M = y + t.double(), M + t.double().abs()
    return {"y": (y, M), "dx": (dy @ w, dy.abs() @ w.abs()), "dw": (dy.t() @ x, dy.abs().t() @ x.abs()),
            "db": (dy.sum(0), dy.abs().sum(0))}


# ----------------------------------------------------------------------------------------------------------------------
# hr_fuse
# ----------------------------------------------------------------------------------------------------------------------
Fuse = collections.namedtuple("Fuse", ["N", "C", "H", "W", "factors", "relu", "kind", "offset"])
FUSE_CASES = [Fuse(2, 3, H, W, f, r, k, o) for H, W, f, r, k, o in [
    (8, 8, (1,), True, "normal", ""), (8, 16, (1, 2), True, "normal", ""), (16, 8, (2, 1), False, "normal", ""),
    (16, 16, (1, 2, 4, 8), True, "normal", ""), (16, 16, (8, 4, 2, 1), True, "normal", ""),
    (16, 24, (4, 1, 8), True, "zero", ""), (6, 6, (1, 2), True, "normal", ""), (6, 10, (1,), False, "normal", ""),
    (6, 6, (2, 1), True, "zero", ""), (16, 16, (1, 2, 4), True, "normal", "t"), (16, 16, (2, 1, 8), True, "normal", "d"),
    (8, 8, (1, 4), False, "normal", "td"), (16, 16, (1, 2, 8), True, "nan", ""), (12, 12, (1, 2, 4), True, "nan", "d"),
    (8, 8, (2, 4), False, "nan", ""), (56, 56, (1, 2, 4, 8), True, "normal", "")]]


def fuse_id(c):
    return "N%dC%d_%dx%d_f%s_%s_%s%s" % (c.N, c.C, c.H, c.W, "".join(map(str, c.factors)), "relu" if c.relu else "norelu",
                                          c.kind, "_off" + c.offset if c.offset else "")


def _fuse_classes():
    cl = [("%d terms" % n, lambda c, n=n: len(c.factors) == n) for n in (1, 2, 3, 4)]
    cl += [("factor %d" % f, lambda c, f=f: f in c.factors) for f in (1, 2, 4, 8)]
    cl.append(("upsampled first term", lambda c: c.factors[0] != 1))
    cl.append(("W % 4 != 0 at f = 1", lambda c: 1 in c.factors and c.W % 4 != 0))
    cl.append(("offset term", lambda c: "t" in c.offset))
    cl.append(("offset dy", lambda c: "d" in c.offset))
    cl.append(("relu", lambda c: c.relu))
    cl.append(("no relu", lambda c: not c.relu))
    cl.append(("NaN", lambda c: c.kind == "nan"))
    cl.append(("NaN with relu", lambda c: c.kind == "nan" and c.relu))
    cl.append(("exact-zero sums", lambda c: c.kind == "zero"))
    return cl


FUSE_CLASSES = _fuse_classes()


def make_fuse(c, seed=0):
    g = _gen(5000 + seed + (FUSE_CASES.index(c) if c in FUSE_CASES else 0))
    N, C, H, W = c.N, c.C, c.H, c.W
    terms = [torch.randn(N, C, H // f, W // f, generator=g) for f in c.factors]
    if c.kind == "zero":                     # integer terms whose sum is exactly 0 at many pixels
        terms = [torch.randint(-2, 3, t.shape, generator=g).float() for t in terms]
    if c.kind == "nan":
        terms[0][0, 0, 0, 0] = float("nan")
        terms[-1][1, 1, -1, -1] = float("nan")
        terms[-1][1, 2, 0, 0] = float("inf")
    dy = torch.randn(N, C, H, W, generator=g)
    return terms, dy


def fuse_forward_reference(terms, factors, relu):
    """the fp32 torch chain: y = up(t0); y = y + up(t); relu"""
    y = None
    for t, f in zip(terms, factors):
        u = F.interpolate(t, scale_factor=f, mode="nearest") if f > 1 else t
        y = u.clone() if y is None else y + u
    return torch.relu(y) if relu else y


def fuse_backward_reference(dz, f):
    """(dterm, M) in fp64 for a term upsampled by f from the masked dy dz"""
    N, C, H, W = dz.shape
    d = dz.double().view(N, C, H // f, f, W // f, f)
    return d.sum((3, 5)), d.abs().sum((3, 5))


def relu_mask(y):
    """the ReLU's backward mask on its output: pass where not y <= 0 (NaN passes)"""
    return ~(y <= 0)


# ----------------------------------------------------------------------------------------------------------------------
# coverage
# ----------------------------------------------------------------------------------------------------------------------
TABLES = {"batch_norm": (BN_CASES, BN_CLASSES), "max_pool2d": (POOL_CASES, POOL_CLASSES),
          "adaptive_avg_pool2d": (AVG_CASES, AVG_CLASSES), "linear": (LIN_CASES, LIN_CLASSES),
          "hr_fuse": (FUSE_CASES, FUSE_CLASSES)}
