"""The covering sweep of the regressor head's training path (csrc/gcn_train.cu): the GCN layers, BatchNorm1d(24) on
batch statistics, ReLU, the residual, the pose and coord heads, rot6d, the adjacency normalisation, the head losses
and the backward of all of it.  This file holds the case table, the coverage classes, the inputs, a mirror of the
workspace layout, and the fp64 per-stage references with their magnitudes M and the bound.
tests/test_gcn_head_sweep_cpu.py fails with the names of uncovered classes, composes the per-stage references end to
end against torch fp64 autograd and shows that the bound catches a set of wrong kernels (fp32 emulations);
tests/test_gcn_head_sweep_gpu.py runs every case on the GPU.

Per-stage isolation.  The forward keeps every intermediate in the workspace, and the backward writes each of its
intermediates (the full gradient gH[l] of every layer output, dY[l], d(AX)[l]) to a region of its own.  Each stage is
checked against fp64 computed from the fp32 values the kernel was fed, read back from the workspace, so each kernel
gets a bound of its own, with no running-error analysis through five train-mode BatchNorms.

The bound: each element of a stage output against its fp64 reference r,

    |got - r| <= C * 2^-24 * M + 2^-24 * |r| + tiny

M is the element's magnitude, computed from absolute values; C is the longest chain of rounded fp32 operations a term
of the result passes through in the kernel; 2^-24 |r| is the final rounding; tiny = C * 2^-139 is the subnormal floor
(TINY_HEAD).

    k_adj_fwd      M = I + mask * relu(E): 2.  d = 1 / sqrt(colsum): 23 adds, sqrt, divide, and its relative error
                   amplified by sum |M| / |sum M|: held relatively.  A_hat = d_i M_ij d_j: 2.
    k_adj_mul      24 FMAs, + 1 with an addend: 24 / 25.
    k_gemm         K FMAs, then + bias: K + 1 (K = Fin forward, Fout for d(AX), 24 B for dW).
    k_bn_stats     mean: y - K, ceil(N / 256) serial adds, 5 shuffle levels, 8 warp sums, / N, + K: C_RED + 3 against
                   M = sum |y - K| / N (the shift K = Y[0, n, 0], 0 if that is not finite, keeps the error
                   relative to the spread).
                   invstd and the running variance: relative bounds C * 2^-24 * r.  The variance passes y - K, - dm, the
                   FMA chain of the reduction and / N: C_VAR = C_RED + 3; dm's own error enters squared (the centred
                   terms sum to ~0), far below one unit.  invstd = 1 / sqrt(var + eps): C_VAR / 2 + 3.  The running
                   variance adds * N, / (N - 1), the momentum products and the sum: C_VAR + 5.  Running mean: 4.
    k_bn_act       (y - mean) * invstd * g + b (+ res): 4 / 5.
    k_group_head   128 FMAs, + bias, + add: 130.
    rot6d          an absolute-value restatement that keeps the real fp64 norms as divisors (nearly parallel pairs
                   get a large M through 1 / |u|); C_R6 = 17 forward, C_R6B = 36 backward (their op chains).
    k_head_losses  the rotation loss: d, its square, ceil(216 B / 256) FMAs, 13 reduction levels, * rot_w, * inv and
                   inv's rounding; the position losses likewise over 72 B; g_pose0: 4 (relative).
    k_bn_bwd       d gamma, d beta: C_RED + 2 / C_RED; dY: C_RED + 8 (train), 2 (eval).
    k_colsum       24 B - 1 adds.
    k_dadj         ceil(B Fin / 256) FMAs + 13 reduction levels.
    k_head_bwd_w   B FMAs (dW) and B adds (db); k_head_bwd_x: K FMAs (+ 1 with an addend).
    k_adj_bwd      3 partial sums, 48 FMAs of two products, -0.5 d^3 (3 products) and the last FMA: 56.

Exact results are held to equality: para[:, :13] against global_para and g_global_para against g_para[:, :13], the
zeros of has = none, the coord L1 gradients +-pos_w / n, and the gradients where a ReLU is off (the reference is 0
there, so the bound's floor is 0).

The ReLU policy: relu(NaN) = NaN, and the backward passes dy except where the input is <= 0, so a NaN passes dy, as
torch's threshold_backward does.  Per stage, the backward reference takes its ReLU mask from the kernel's own
pre-activation, restated exactly: k_bn_act, k_bn_bwd_reduce and k_bn_bwd_dy all compute z = fma(fl(fl(y - mean) *
invstd), g, b) (FADD, FMUL, FFMA in their SASS), and the sign of an FMA's rounded result is that of its exact one, so
t = fl(fl(y - mean) * invstd) in fp32 and then t * g + b in fp64 (exact product, sign-exact sum) give the kernel's
mask bit for bit, with or without the residual of layer 3.  Composed end to end, the mask is the fp64 sign.

The shift K of the BatchNorm statistics is Y[0, n, 0] when that is finite and 0 otherwise, so an infinite first
element gives the infinite mean torch gives rather than NaN.
"""
import collections
import math
import os

import numpy as np
import torch

import fp64_bound as fb
from oracle import gcn_head as og

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the head's own subnormal floor per rounded operation, 2^10 TINY: a rounding in fp32's subnormal range (TINY) can be
# scaled up by a later factor of its chain, such as invstd <= eps^-1/2 < 2^9 in the BatchNorm kernels
TINY_HEAD = 2.0 ** 10 * fb.TINY
EPS, MOM = 1e-5, 0.1
KDI = [128, 128, 256, 256, 128]
KDO = [128, 256, 256, 128, 128]
ROT_W, POS_W = og.SMPL_POSE_WEIGHTS, og.JOINT_POSITION_WEIGHTS
C_R6, C_R6B = 17, 36
C_ADJ_BWD = 56


def c_red(n):
    """a CTA reduction of n terms over 256 threads: ceil(n / 256) serial steps, 5 shuffle levels, 8 warp sums"""
    return -(-n // 256) + 13


# ----------------------------------------------------------------------------------------------------------------------
# workspace layout (floats), the mirror of layout() in csrc/gcn_train.cu
# ----------------------------------------------------------------------------------------------------------------------
def layout(B):
    off = [0]
    L = {}

    def take(key, n):
        L[key] = off[0]
        off[0] += (n + 63) // 64 * 64

    R = 24 * B
    take("M", 576), take("Ahat", 576), take("d", 24)
    for l in range(5):
        take("AX%d" % l, R * KDI[l]), take("Y%d" % l, R * KDO[l]), take("H%d" % l, R * KDO[l])
        take("mean%d" % l, 24), take("invstd%d" % l, 24)
    for k in range(2):
        take("p6_%d" % k, B * 144), take("dp6_%d" % k, B * 144)
    for l in range(5):
        take("gH%d" % l, R * KDO[l]), take("dY%d" % l, R * KDO[l]), take("dAX%d" % l, R * KDI[l])
    take("dA", 3 * 576), take("sums", 48)
    return L, off[0]


def region_shapes(B):
    s = {"M": (24, 24), "Ahat": (24, 24), "d": (24,), "dA": (3, 24, 24)}
    for l in range(5):
        s["AX%d" % l] = s["dAX%d" % l] = (B, 24, KDI[l])
        s["Y%d" % l] = s["H%d" % l] = s["gH%d" % l] = s["dY%d" % l] = (B, 24, KDO[l])
        s["mean%d" % l] = s["invstd%d" % l] = (24,)
    for k in range(2):
        s["p6_%d" % k] = s["dp6_%d" % k] = (B, 24, 6)
    return s


def regions(ws, B):
    """{name: view} of a float32 workspace tensor"""
    L, _ = layout(B)
    out = {}
    for k, shp in region_shapes(B).items():
        n = int(np.prod(shp))
        out[k] = ws[L[k]:L[k] + n].view(shp)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
Case = collections.namedtuple("Case", ["B", "train", "has", "src", "up", "bn", "adj", "r6", "nonfinite"])
BS = (1, 2, 3, 5, 8, 16, 33, 64, 65, 257, 520)
SRCS = ("para", "pose0", "coord0", "coord1", "all")
UPS = ("normal", "tiny", "huge", "spike", "zero")
BNS = ("normal", "ratio0", "ratio10", "ratio20", "const", "gamma0", "gammaneg", "betaoff")
ADJS = ("normal", "negzero", "big", "nan")
R6S = ("normal", "generic", "par10", "par20", "a1zero", "uzero", "big30", "small30")
NONFINITE = ("", "rotnan", "rotinf", "rotinf0", "gnan")


def case(B, train=True, has="all", src="all", up="normal", bn="normal", adj="normal", r6="normal", nonfinite=""):
    if not train:
        src = "para"
    return Case(B, train, has, src, up, bn, adj, r6, nonfinite)


CASES = [case(B) for B in BS] + [
    case(3, False), case(16, False), case(65, False, bn="ratio20"), case(520, False), case(1, False, has="none"),
    case(2, has="some"), case(16, has="some"), case(65, has="some"), case(3, has="none"), case(64, has="none"),
    case(5, src="para"), case(8, src="pose0"), case(33, src="coord0"), case(16, src="coord1"), case(2, src="coord1"),
    case(8, up="tiny"), case(16, up="huge"), case(5, up="spike"), case(3, up="zero"), case(16, False, up="huge"),
    case(16, bn="ratio0"), case(16, bn="ratio10"), case(16, bn="ratio20"), case(1, bn="ratio20"), case(257, bn="ratio20"),
    case(5, bn="ratio10"), case(8, bn="const"), case(8, False, bn="const"), case(16, bn="gamma0"), case(5, bn="gammaneg"),
    case(16, bn="betaoff"),
    case(16, adj="negzero"), case(3, adj="negzero"), case(16, adj="big"), case(8, adj="nan"),
    case(16, r6="generic"), case(16, r6="par10"), case(8, r6="par20"), case(16, r6="a1zero"), case(5, r6="uzero"),
    case(8, r6="big30"), case(8, r6="small30"), case(8, False, r6="par20"),
    case(16, nonfinite="rotnan"), case(8, nonfinite="rotinf"), case(5, nonfinite="rotinf0"),
    case(16, nonfinite="gnan"),
    case(8, False, nonfinite="rotnan"),
]


def case_id(c):
    s = "B%d_%s_has%s_src%s" % (c.B, "train" if c.train else "eval", c.has, c.src)
    for k, d in (("up", "normal"), ("bn", "normal"), ("adj", "normal"), ("r6", "normal"), ("nonfinite", "")):
        if getattr(c, k) != d:
            s += "_%s%s" % (k, getattr(c, k))
    return s


def _classes():
    cl = [("B = %d" % B, lambda c, B=B: c.B == B) for B in BS]
    cl += [("24 B % 64 != 0 (M tail)", lambda c: (24 * c.B) % 64 != 0),
           ("odd B > 1 (dW K tail)", lambda c: c.B > 1 and c.B % 2 == 1),
           ("B F < 256", lambda c: c.B * 128 < 256), ("B F = 256", lambda c: c.B * 128 == 256),
           ("B F > 256", lambda c: c.B * 128 > 256),
           ("odd B, F = 128, unequal thread counts", lambda c: c.B % 2 == 1 and (c.B * 128) % 256 != 0 and c.B > 2)]
    cl += [("training", lambda c: c.train), ("eval", lambda c: not c.train)]
    cl += [("has %s" % h, lambda c, h=h: c.has == h) for h in ("all", "some", "none")]
    cl += [("gradient source %s" % s, lambda c, s=s: c.train and c.src == s) for s in SRCS]
    cl += [("upstream %s" % u, lambda c, u=u: c.up == u) for u in UPS]
    cl += [("BatchNorm %s" % b, lambda c, b=b: c.bn == b) for b in BNS[1:]]
    cl += [("adjacency %s" % a, lambda c, a=a: c.adj == a) for a in ADJS[1:]]
    cl += [("rot6d %s" % r, lambda c, r=r: c.r6 == r) for r in R6S[1:]]
    cl += [("non-finite %s" % n, lambda c, n=n: c.nonfinite == n) for n in NONFINITE[1:]]
    return cl


CLASSES = _classes()


# ----------------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------------
def _buffers():
    g = np.load(os.path.join(ROOT, "tests", "golden", "gcn_head.npz"))
    return {k: torch.from_numpy(np.ascontiguousarray(g["buf_" + k].reshape(-1))).float() for k in og.BUFFER_NAMES}


def np_buffers(buf):
    """the flat buffers of make_case in oracle/gcn_head.py's shapes ([1,24,24], mean_pose [1,144]), fp64"""
    return {k: v.double().numpy().reshape((1, 144) if k == "mean_pose" else (1, 24, 24)) for k, v in buf.items()}


def _rot6d_pairs(kind, rng):
    """[24, 6] 6d vectors (a1 = x[0::2], a2 = x[1::2]) of one rot6d class"""
    def unit(n):
        v = rng.normal(size=(n, 3))
        return v / np.linalg.norm(v, axis=1, keepdims=True)
    a1 = unit(24) * rng.uniform(0.5, 2, (24, 1))
    b1 = a1 / np.linalg.norm(a1, axis=1, keepdims=True)
    perp = np.cross(b1, unit(24))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    a2 = unit(24) * rng.uniform(0.5, 2, (24, 1))
    if kind in ("par10", "par20"):
        t = 2.0 ** (-10 if kind == "par10" else -20)
        a2 = b1 * rng.uniform(0.5, 2, (24, 1)) + t * perp
    elif kind == "a1zero":
        a1[::2] = 0.0
    elif kind == "uzero":
        a1[::2] = np.array([1.0, 0.0, 0.0])
        a2[::2] = np.array([2.0, 0.0, 0.0])
        a1[1::4] = np.array([0.0, -3.0, 0.0])
        a2[1::4] = np.array([0.0, 1.5, 0.0])
    elif kind in ("big30", "small30"):
        s = 2.0 ** (30 if kind == "big30" else -30)
        a1, a2 = a1 * s, a2 * s
    x = np.empty((24, 6))
    x[:, 0::2], x[:, 1::2] = a1, a2
    return torch.from_numpy(x).float()


def make_case(c, seed=0):
    """fp32 CPU tensors: P (the 29 parameters by name), buf, bn {name: (rm, rv)}, rot, gpara, target, gt, has, and the
    upstream gradients g_para, g_pose0, g_coord0, g_coord1 (None in eval mode)"""
    idx = CASES.index(c) if c in CASES else 997
    rng = np.random.default_rng(7000 + 31 * seed + idx)
    B = c.B
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).float()
    P = {}
    for l, ((name, i), (di, do)) in enumerate(zip(og.LAYERS, og.DIMS)):
        P["%s.gc.%d.weight" % (name, i)] = t(rng.normal(0, 1 / math.sqrt(di), (di, do)))
        P["%s.gc.%d.bias" % (name, i)] = t(rng.normal(0, 0.1, do))
        w = 1 + 0.3 * rng.normal(size=24)
        w[5] = -abs(w[5])                                            # one negative gamma in every case
        P["%s.act.%d.0.weight" % (name, i)] = t(w)
        P["%s.act.%d.0.bias" % (name, i)] = t(0.3 * rng.normal(size=24))
    buf = _buffers()
    E = 1 + 0.1 * rng.normal(size=(24, 24))
    if c.adj == "negzero":
        E = rng.normal(size=(24, 24))
        E[rng.random((24, 24)) < 0.25] = 0.0
    elif c.adj == "big":
        E = 1024.0 * np.where(rng.random((24, 24)) < 0.7, 1.0, -1.0)
    P["edge_importance"] = t(E[None])
    if c.adj == "nan":
        m = buf["A_mask"].view(24, 24).nonzero()[3]
        P["edge_importance"][0, m[0], m[1]] = float("nan")
    for k in range(2):
        P["pose_regressors.%d.1.weight" % k] = t(rng.normal(0, 0.02, (144, 128, 1, 1)))
        P["pose_regressors.%d.1.bias" % k] = t(rng.normal(0, 0.02, 144))
        P["coord_regressors.%d.1.weight" % k] = t(rng.normal(0, 0.05, (72, 128, 1, 1)))
        P["coord_regressors.%d.1.bias" % k] = t(rng.normal(0, 0.1, 72))
    if c.r6 != "normal":                    # p6 = 0 . x + 0 + mean_pose exactly: the chosen 6d pairs reach rot6d
        for k in range(2):
            P["pose_regressors.%d.1.weight" % k].zero_()
            P["pose_regressors.%d.1.bias" % k].zero_()
        buf["mean_pose"] = _rot6d_pairs(c.r6, rng).reshape(-1)
    rot = t(rng.uniform(0, 1.5, (B, 24, 128)))
    bn = {n: (t(0.1 * rng.normal(size=24)), t(rng.uniform(0.5, 1.5, 24))) for n in og.BN_NAMES}
    if c.bn in ("ratio0", "ratio10", "ratio20"):          # a constant gc bias sets |mean| / std per layer
        r = {"ratio0": 0.0, "ratio10": 2.0 ** 10, "ratio20": 2.0 ** 20}[c.bn]
        f = lambda x: {k: v.double().numpy() for k, v in x.items()}
        _, sv = og.forward(f(P), np_buffers(buf), {k: (a.double().numpy(), b.double().numpy()) for k, (a, b) in bn.items()},
                           rot.double().numpy(), np.zeros((B, 13)), training=True)
        for l, (name, i) in enumerate(og.LAYERS):
            xh, Z = sv["layers"][l]["xh"], sv["layers"][l]["Z"]
            Y = sv["layers"][l]["AX"] @ f(P)["%s.gc.%d.weight" % (name, i)] + f(P)["%s.gc.%d.bias" % (name, i)]
            mu, sd = Y.mean(axis=(0, 2)), Y.std(axis=(0, 2))
            P["%s.gc.%d.bias" % (name, i)] = t(f(P)["%s.gc.%d.bias" % (name, i)] - mu.mean() + r * sd.mean())
            if c.train is False:                           # eval: running statistics near the batch's
                bn[og.BN_NAMES[l]] = (t(mu - mu.mean() + r * sd.mean()), t(sd ** 2))
    elif c.bn == "const":                                  # refine_gcn.gc.1: W = 0, constant bias: every node constant
        P["refine_gcn.gc.1.weight"].zero_()
        P["refine_gcn.gc.1.bias"].fill_(0.7)
    elif c.bn == "gamma0":
        P["refine_gcn.act.1.0.weight"].zero_()
    elif c.bn == "gammaneg":
        for name, i in og.LAYERS:
            P["%s.act.%d.0.weight" % (name, i)] = -P["%s.act.%d.0.weight" % (name, i)].abs()
    elif c.bn == "betaoff":
        for name, i in og.LAYERS:
            P["%s.act.%d.0.bias" % (name, i)].fill_(-2.0)
    gpara = t(rng.normal(0, 0.3, (B, 13)))
    target = t(np.concatenate([rng.normal(0, 0.3, (B, 13)), rng.normal(0, 0.5, (B, 216))], 1))
    gt = t(rng.normal(0, 0.3, (B, 24, 3)))
    if c.has == "all":
        has = np.ones(B, np.uint8)
    elif c.has == "none":
        has = np.zeros(B, np.uint8)
    else:
        has = (rng.random(B) < 0.5).astype(np.uint8)
        has[0] = 1
        if B > 1:
            has[-1] = 0
    scale = {"tiny": 2.0 ** -100, "huge": 2.0 ** 60}.get(c.up, 1.0)
    ups = {"para": t(rng.normal(size=(B, 229)) * scale)}
    if c.train:
        ups.update(pose0=t(rng.normal(size=(B, 216)) * scale), coord0=t(rng.normal(size=(B, 24, 3)) * scale),
                   coord1=t(rng.normal(size=(B, 24, 3)) * scale))
    for k in ups:
        if c.up == "zero" or (c.src != "all" and k != c.src):
            ups[k].zero_()
    if c.up == "spike":
        ups[c.src if c.src != "all" else "para"].view(-1)[ups["para"].numel() // 3 % ups[
            c.src if c.src != "all" else "para"].numel()] = 2.0 ** 20
    if c.nonfinite == "rotnan":
        rot[B // 2, 3, 17] = float("nan")
    elif c.nonfinite == "rotinf0":                        # image 0: the BatchNorm shift K = Y[0, n, 0] is infinite
        rot[0, 3, 17] = float("inf")
    elif c.nonfinite == "rotinf":
        rot[B - 1, 11, 5] = float("inf")
    elif c.nonfinite == "gnan":
        ups["para"][B // 2, 40] = float("nan")
    return dict(P=P, buf=buf, bn=bn, rot=rot, gpara=gpara, target=target, gt=gt, has=torch.from_numpy(has),
                g_para=ups["para"], g_pose0=ups.get("pose0"), g_coord0=ups.get("coord0"), g_coord1=ups.get("coord1"))


# ----------------------------------------------------------------------------------------------------------------------
# fp64 per-stage references
# ----------------------------------------------------------------------------------------------------------------------
def _relu(z):
    return torch.where(z <= 0, torch.zeros_like(z), z)


def _cross_abs(a, b):
    """|a| x |b| componentwise magnitude of a cross product"""
    return torch.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                        a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], -1)


def _cross(a, b):
    return torch.linalg.cross(a, b, dim=-1)


def _rot6d_state(x):
    """x [..., 6] fp64 -> value and magnitude of every intermediate (the absolute-value restatement with real norms)"""
    a1, a2 = x[..., 0::2], x[..., 1::2]
    Ma1, Ma2 = a1.abs(), a2.abs()
    n1r = a1.norm(dim=-1, keepdim=True)
    n1 = n1r.clamp_min(1e-12)
    Mn1 = torch.where(n1r > 1e-12, n1r, torch.zeros_like(n1r))
    b1 = a1 / n1
    Mb1 = Ma1 / n1 + a1.abs() * Mn1 / n1 ** 2
    dd = (b1 * a2).sum(-1, keepdim=True)
    Mdd = (Mb1 * Ma2 + b1.abs() * Ma2).sum(-1, keepdim=True)
    u = a2 - dd * b1
    Mu = Ma2 + Mdd * b1.abs() + dd.abs() * Mb1
    n2r = u.norm(dim=-1, keepdim=True)
    n2 = n2r.clamp_min(1e-12)
    Mn2 = torch.where(n2r > 1e-12, (u.abs() * Mu).sum(-1, keepdim=True) / n2, torch.zeros_like(n2))
    b2 = u / n2
    Mb2 = Mu / n2 + u.abs() * Mn2 / n2 ** 2
    return dict(a1=a1, a2=a2, Ma2=Ma2, n1r=n1r, n1=n1, Mn1=Mn1, b1=b1, Mb1=Mb1, dd=dd, Mdd=Mdd, u=u, Mu=Mu, n2r=n2r,
                n2=n2, Mn2=Mn2, b2=b2, Mb2=Mb2)


def rot6d_ref(x):
    """x [..., 6] -> (R [..., 9], M [..., 9])"""
    s = _rot6d_state(x)
    b3, Mb3 = _cross(s["b1"], s["b2"]), _cross_abs(s["Mb1"], s["b2"].abs()) + _cross_abs(s["b1"].abs(), s["Mb2"])
    R = torch.stack([s["b1"], s["b2"], b3], -1).flatten(-2)
    M = torch.stack([s["Mb1"], s["Mb2"], Mb3], -1).flatten(-2)
    return R, M


def _normalize_bwd(nr, n, Mn, b, Mb, g, Mg):
    big = nr > 1e-12
    bg = (b * g).sum(-1, keepdim=True)
    Mbg = (Mb * Mg).sum(-1, keepdim=True)
    num = torch.where(big, g - b * bg, g)
    Mnum = torch.where(big, Mg + Mb * Mbg, Mg)
    return num / n, Mnum / n + num.abs() * Mn / n ** 2


def rot6d_bwd_ref(x, gR, drop_dd=False):
    """x [..., 6], gR [..., 9] -> (dx [..., 6], M); drop_dd leaves out the -dd gu term (a seeded defect)"""
    s = _rot6d_state(x)
    g = gR.reshape(gR.shape[:-1] + (3, 3))
    g1, g2, g3 = g[..., 0], g[..., 1], g[..., 2]
    gb1 = g1 + _cross(s["b2"], g3)
    Mgb1 = g1.abs() + _cross_abs(s["Mb2"], g3.abs())
    gb2 = g2 + _cross(g3, s["b1"])
    Mgb2 = g2.abs() + _cross_abs(g3.abs(), s["Mb1"])
    gu, Mgu = _normalize_bwd(s["n2r"], s["n2"], s["Mn2"], s["b2"], s["Mb2"], gb2, Mgb2)
    gub1 = (gu * s["b1"]).sum(-1, keepdim=True)
    Mgub1 = (Mgu * s["Mb1"]).sum(-1, keepdim=True)
    ga2, Mga2 = gu - s["b1"] * gub1, Mgu + s["Mb1"] * Mgub1
    gb1 = gb1 - s["a2"] * gub1 - (0 if drop_dd else s["dd"] * gu)
    Mgb1 = Mgb1 + s["Ma2"] * Mgub1 + s["Mdd"] * Mgu + s["dd"].abs() * Mgu
    ga1, Mga1 = _normalize_bwd(s["n1r"], s["n1"], s["Mn1"], s["b1"], s["Mb1"], gb1, Mgb1)
    out, M = torch.empty(x.shape, dtype=x.dtype, device=x.device), torch.empty(x.shape, dtype=x.dtype, device=x.device)
    out[..., 0::2], out[..., 1::2] = ga1, ga2
    M[..., 0::2], M[..., 1::2] = Mga1, Mga2
    return out, M


Stage = collections.namedtuple("Stage", ["r", "M", "C", "kind"])      # kind: "abs", "rel" or "exact"


def stages(c, inp, got=None, device="cpu", dtype=torch.float64, defect=None):
    """{stage: Stage} in fp64.  With `got` (the kernel's fp32 outputs and workspace regions, by stage name), every stage
    is computed from the values the kernel fed it; without, the stages compose end to end.  dtype=float32 with a
    `defect` (a key of test_gcn_head_sweep_cpu.DEFECTS) makes it an fp32 emulation with one wrong stage."""
    d = lambda x: None if x is None else x.to(device=device, dtype=dtype)
    B, train = c.B, c.train
    P = {k: d(v) for k, v in inp["P"].items()}
    buf = {k: d(v) for k, v in inp["buf"].items()}
    S = {}

    def put(name, r, M, C, kind="abs"):
        S[name] = Stage(r, M, C, kind)
        return r

    def val(name):
        return d(got[name]) if got is not None else S[name].r

    dfx = lambda name: defect is not None and defect.startswith(name)

    W = lambda l: P["%s.gc.%d.weight" % og.LAYERS[l]]
    bgc = lambda l: P["%s.gc.%d.bias" % og.LAYERS[l]]
    gam = lambda l: P["%s.act.%d.0.weight" % og.LAYERS[l]]
    bet = lambda l: P["%s.act.%d.0.bias" % og.LAYERS[l]]
    rot = d(inp["rot"])
    # adjacency
    E = P["edge_importance"].view(24, 24)
    mask, I = buf["A_mask"].view(24, 24), buf["I_n"].view(24, 24)
    Mm = put("M", I + mask * _relu(E), I.abs() + (mask * _relu(E)).abs(), 2)
    Mg = val("M")
    s = Mg.sum(0)
    tiny_s = torch.finfo(dtype).tiny
    dvec = torch.where(s > 0, s.clamp_min(tiny_s) ** -0.5, torch.zeros_like(s))
    put("d", dvec, dvec * (11.5 * Mg.abs().sum(0) / s.abs().clamp_min(tiny_s) + 2), 1, "rel")
    dg = val("d")
    put("Ahat", dg[:, None] * Mg * dg[None, :], (dg[:, None] * Mg * dg[None, :]).abs(), 2)
    adjs = [buf["r2p_A"].view(24, 24), val("Ahat"), val("Ahat"), val("Ahat"), buf["p2r_A"].view(24, 24)]
    mp = buf["mean_pose"].view(24, 6)

    def head(key, X, K, add=None):
        Wk = P[key + ".weight"].reshape(24, K, 128)
        r = torch.einsum("jkf,bjf->bjk", Wk, X) + P[key + ".bias"].view(24, K)
        M = torch.einsum("jkf,bjf->bjk", Wk.abs(), X.abs()) + P[key + ".bias"].view(24, K).abs()
        if add is not None:
            r, M = r + add, M + add.abs()
        return r, M

    if train:
        r, M = head("pose_regressors.0.1", rot, 6, mp)
        put("p6_0", r, M, 130)
        R, M = rot6d_ref(val("p6_0"))
        put("pose0", R.reshape(B, 216), M.reshape(B, 216), C_R6)
    X = rot
    for l in range(5):
        Fo = KDO[l]
        N = B * Fo
        put("AX%d" % l, torch.einsum("nk,bkf->bnf", adjs[l], X), torch.einsum("nk,bkf->bnf", adjs[l].abs(), X.abs()), 24)
        AX = val("AX%d" % l)
        Yr = AX @ W(l) + bgc(l)
        if l == 1 and dfx("M-tail row skipped"):
            Yr = Yr.clone()
            Yr[-1, -1] = 0
        put("Y%d" % l, Yr, AX.abs() @ W(l).abs() + bgc(l).abs(), KDI[l] + 1)
        Y = val("Y%d" % l)
        rm, rv = (d(t) for t in inp["bn"][og.BN_NAMES[l]])
        if train or (l == 0 and dfx("batch statistics in eval")):
            K = torch.where(torch.isfinite(Y[0, :, 0]), Y[0, :, 0], torch.zeros_like(Y[0, :, 0]))
            yk = Y - K[None, :, None]
            dm = yk.sum((0, 2)) / N
            dm = dm + (yk - dm[None, :, None]).sum((0, 2)) / N          # one correction pass
            mean = K + dm
            var = ((yk - dm[None, :, None]) ** 2).sum((0, 2)) / N
            put("mean%d" % l, mean, yk.abs().sum((0, 2)) / N, c_red(N) + 3)
            cvar = c_red(N) + 3
            invstd = 1 / torch.sqrt(var + EPS)
            put("invstd%d" % l, invstd, invstd * (cvar / 2 * var / (var + EPS) + 3), 1, "rel")
            put("rm%d" % l, (1 - MOM) * rm + MOM * val("mean%d" % l), (1 - MOM) * rm.abs() + MOM * val("mean%d" % l).abs(), 4)
            vu = var * N / (N if dfx("N in place of N - 1") else N - 1)
            rvn = (1 - MOM) * rv + MOM * vu
            put("rv%d" % l, rvn, rvn * (cvar + 5), 1, "rel")
        else:
            put("mean%d" % l, rm, torch.zeros_like(rm), 0, "exact")
            invstd = 1 / torch.sqrt(rv + EPS)
            put("invstd%d" % l, invstd, invstd * 3, 1, "rel")
        mu, ist = val("mean%d" % l), val("invstd%d" % l)
        v = lambda t: t[None, :, None]
        z = (Y - v(mu)) * v(ist) * v(gam(l)) + v(bet(l))
        Mz = (Y - v(mu)).abs() * v(ist) * v(gam(l).abs()) + v(bet(l).abs())
        h, Mh = _relu(z), Mz
        if l == 3:
            h, Mh = h + val("H0"), Mh + val("H0").abs()
        put("H%d" % l, h, Mh, 5 if l == 3 else 4)
        S["_z%d" % l] = (z, Mz)
        if train and l in (0, 3):
            k = 0 if l == 0 else 1
            r, M = head("coord_regressors.%d.1" % k, val("H%d" % l), 3)
            put("coord%d" % k, r, M, 129)
        X = val("H%d" % l)
    r, M = head("pose_regressors.1.1", X, 6, mp)
    put("p6_1", r, M, 130)
    R, M = rot6d_ref(val("p6_1"))
    put("pararot", R.reshape(B, 216), M.reshape(B, 216), C_R6)
    put("paraglob", d(inp["gpara"]), None, 0, "exact")
    # losses
    if train:
        sel = (inp["has"].to(device) == 1).double()
        n = float(sel.sum())
        inv = 1 / n if n > 0 else 0.0
        inv1 = 1 / B if dfx("losses divided by B") else inv
        p0, c0, c1 = val("pose0"), val("coord0").reshape(B, 72), val("coord1").reshape(B, 72)
        tgt, gtj = d(inp["target"])[:, 13:], d(inp["gt"]).reshape(B, 72)
        dr = (p0 - tgt) * sel[:, None]
        L0 = ROT_W * (dr ** 2).sum() * inv / 216
        put("loss0", L0, L0.abs(), 2 + -(-216 * B // 256) + 13 + 3)
        put("g_pose0_loss", ROT_W * 2 * dr * inv / 216, (ROT_W * 2 * dr * inv / 216).abs(), 4)
        for k, cc in ((0, c0), (1, c1)):
            dc = (cc - gtj) * sel[:, None]
            Lk = POS_W * dc.abs().sum() * (inv1 if k == 0 else inv)
            put("loss%d" % (k + 1), Lk, Lk.abs(), 1 + -(-72 * B // 256) + 13 + 3)
            f32inv = torch.tensor(inv, dtype=torch.float32)
            dc32 = (cc.float() - gtj.float()) * sel[:, None].float()
            g = (POS_W * torch.sign(dc32) * f32inv.to(device)).reshape(B, 24, 3)  # pos_w * sign(d) * fl(1 / n) in fp32
            put("g_coord%d_loss" % k, d(g), None, 0, "exact")
    # ---------------------------------------------------------------- backward
    gp = d(inp["g_para"])
    put("g_global_para", gp[:, :13], None, 0, "exact")
    r, M = rot6d_bwd_ref(val("p6_1"), gp[:, 13:].reshape(B, 24, 9), drop_dd=dfx("rot6d backward without"))
    put("dp6_1", r, M, C_R6B)

    def head_bwd(name, key, K, X, dp, dp_M=None):
        Wk = P[key + ".weight"].reshape(24, K, 128)
        put("g_%s_w" % name, torch.einsum("bjk,bjf->jkf", dp, X).reshape(P[key + ".weight"].shape),
            torch.einsum("bjk,bjf->jkf", dp.abs(), X.abs()).reshape(P[key + ".weight"].shape), B)
        put("g_%s_b" % name, dp.sum(0).reshape(-1), dp.abs().sum(0).reshape(-1), B)
        return torch.einsum("jkf,bjk->bjf", Wk, dp), torch.einsum("jkf,bjk->bjf", Wk.abs(), dp.abs())

    dx, Mx = head_bwd("pose1", "pose_regressors.1.1", 6, val("H4"), val("dp6_1"))
    put("gH4", dx, Mx, 6)
    gc = {k: (d(inp["g_coord%d" % k]) if train else None) for k in range(2)}
    hx = {}
    if train:
        hx[1] = head_bwd("coord1", "coord_regressors.1.1", 3, val("H3"), gc[1])
        hx[0] = head_bwd("coord0", "coord_regressors.0.1", 3, val("H0"), gc[0])
    dA = {}
    for l in range(4, -1, -1):
        Fi, Fo = KDI[l], KDO[l]
        N = B * Fo
        dH = val("gH%d" % l)
        Y, mu, ist = val("Y%d" % l), val("mean%d" % l), val("invstd%d" % l)
        v = lambda t: t[None, :, None]
        z, Mz = S["_z%d" % l]
        on = ~(z <= 0)
        if got is not None:                 # the kernel's own z: fma(fl(fl(y - mean) * invstd), g, b), sign-exact
            f = lambda t: t.to(torch.float32)
            t32 = ((f(Y) - f(v(mu))) * f(v(ist))).to(torch.float64)
            on = ~(t32 * v(gam(l)) + v(bet(l)) <= 0)
        S["_on%d" % l] = on
        dz = torch.where(on, dH, torch.zeros_like(dH))
        xh = (Y - v(mu)) * v(ist)
        sdz, sdzxh = dz.sum((0, 2)), (dz * xh).sum((0, 2))
        asdz, asdzxh = dz.abs().sum((0, 2)), (dz.abs() * xh.abs()).sum((0, 2))
        put("g_bn_weight%d" % l, sdzxh, asdzxh, c_red(N) + 2)
        put("g_bn_bias%d" % l, sdz, asdz, c_red(N))
        g = gam(l)
        if train:
            dY = v(ist) / N * (N * dz * v(g) - v(g * sdz) - xh * v(g * sdzxh))
            MdY = v(ist) / N * (N * dz.abs() * v(g.abs()) + v(g.abs() * asdz) + xh.abs() * v(g.abs() * asdzxh))
            put("dY%d" % l, dY, MdY, c_red(N) + 8)
        else:
            put("dY%d" % l, dz * v(g * ist), (dz * v(g * ist)).abs(), 2)
        dYg = val("dY%d" % l)
        AX = val("AX%d" % l)
        rows = dYg.reshape(24 * B, -1)
        gbr = rows[:-1].sum(0) if l == 3 and dfx("k_colsum over") else rows.sum(0)
        put("gb%d" % l, gbr, dYg.abs().sum((0, 1)), max(24 * B - 1, 0))
        keep = 24 * B - (24 * B) % 16 if l == 2 and dfx("gemm K tail dropped") else 24 * B
        put("gW%d" % l, AX.reshape(24 * B, -1)[:keep].t() @ rows[:keep],
            torch.einsum("bni,bno->io", AX.abs(), dYg.abs()), 24 * B)
        put("dAX%d" % l, dYg @ W(l).t(), dYg.abs() @ W(l).abs().t(), Fo)
        dAXg = val("dAX%d" % l)
        if 1 <= l <= 3:
            Xin = val("H%d" % (l - 1))
            put("dA%d" % l, torch.einsum("bnf,bkf->nk", dAXg, Xin), torch.einsum("bnf,bkf->nk", dAXg.abs(), Xin.abs()),
                c_red(B * Fi))
        At = adjs[l].t() if l == 2 and dfx("A in place of A^T") else adjs[l]
        r = torch.einsum("nk,bnf->bkf", At, dAXg)
        M = torch.einsum("nk,bnf->bkf", adjs[l].abs(), dAXg.abs())
        C = 24
        if l == 4 and train:
            r, M, C = r + hx[1][0], M + hx[1][1], 25
        if l == 1:
            r, M, C = (r if dfx("residual share missing") else r + val("gH3")), M + val("gH3").abs(), 25
            if train:
                r, M, C = r + hx[0][0], M + hx[0][1], 26
        if l == 0:
            if train:
                rr, MM = rot6d_bwd_ref(val("p6_0"), d(inp["g_pose0"]).reshape(B, 24, 9))
                put("dp6_0", rr, MM, C_R6B)
                dx0, Mx0 = head_bwd("pose0", "pose_regressors.0.1", 6, rot, val("dp6_0"))
                r, M, C = r + dx0, M + Mx0, 25
            put("g_rot_feats", r, M, C)
        else:
            put("gH%d" % (l - 1), r, M, C)
    # d A_hat -> d edge_importance
    dAs = [val("dA%d" % l) for l in (1, 2, 3)]
    sG = (dAs[0] + dAs[1]) + dAs[2]
    MsG = dAs[0].abs() + dAs[1].abs() + dAs[2].abs()
    Mm, dd_ = val("M"), val("d")
    gd = (sG * Mm * dd_[None, :]).sum(1) + (sG * Mm * dd_[:, None]).sum(0)
    Mgd = (MsG * Mm.abs() * dd_[None, :]).sum(1) + (MsG * Mm.abs() * dd_[:, None]).sum(0)
    gs = torch.where(dd_ > 0, -0.5 * dd_ ** 3 * gd, torch.zeros_like(gd))
    if dfx("k_adj_bwd without"):
        gs = torch.zeros_like(gs)
    Mgs = torch.where(dd_ > 0, 0.5 * dd_ ** 3 * Mgd, torch.zeros_like(gd))
    dM = sG * dd_[:, None] * dd_[None, :] + gs[None, :]
    MdM = MsG * dd_[:, None] * dd_[None, :] + Mgs[None, :]
    onE = ~(E <= 0)
    put("g_edge_importance", torch.where(onE, dM * mask, torch.zeros_like(dM)),
        torch.where(onE, MdM * mask.abs(), torch.zeros_like(dM)), C_ADJ_BWD)
    return S


# ----------------------------------------------------------------------------------------------------------------------
# the bound
# ----------------------------------------------------------------------------------------------------------------------
def bound(st):
    """(scale, floor, limit) of a stage for fp64_bound.worst: an 'abs' stage passes at C units of 2^-24 M, a 'rel' one
    (M already holds C r) at 1, and an 'exact' one only at equality"""
    if st.kind == "exact":
        return 0.0, 0.0, 0.0
    scale, floor = fb.U24 * st.M.reshape(st.r.shape), fb.U24 * st.r.abs() + TINY_HEAD * max(st.C, 1)
    return scale, floor, 1.0 if st.kind == "rel" else float(st.C)


def check(got, S, skip=()):
    """[(stage, worst, limit)] of the failing stages"""
    bad = []
    for name, st in S.items():
        if name.startswith("_") or name in skip or name not in got:
            continue
        scale, floor, lim = bound(st)
        q = fb.worst(got[name], st.r, scale, floor)[0]
        if not q <= lim:
            bad.append((name, q, lim))
    return bad
