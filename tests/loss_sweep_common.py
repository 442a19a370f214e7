"""The covering sweep of the IUV-branch losses: body_uv_losses and part_iuv_losses (csrc/losses.cu, one kernel with
strided rows), and dp_uvia_losses, stn_kps_losses and part_iuv_targets (csrc/iuv_train.cu).  This file holds the case
tables, the coverage classes, the seeded inputs, the fp64 reference and the per-element bound.
tests/test_loss_sweep_cpu.py fails with the names of uncovered classes, checks the reference against torch's own ops,
runs the kernels' own arithmetic (the DANET_LOSSES_HOST_CHECK host walks) against the bound and shows that the bound
catches a set of wrong kernels (fp32 emulations); tests/test_loss_sweep_gpu.py runs every case on the GPU.

The reference is computed in fp64 from the fp32 values the kernel was given.  The decisions the kernel makes in fp32
are restated exactly in fp32 first: the point grid (X - S/2) * 2/S and its unnormalize, floor and the tap fraction
t = ix - floor(ix), the affine_grid base and crop coordinate, the heat-map window centre int(k * S + 0.5), label
truncation and the target argmax (first maximum, NaN counting as maximal, as torch.argmax).  Everything after them is
fp64.  part_iuv_targets' background decision sum(I) < 0.5 takes the kernel's fp32 sum in its order; the decisions that
differ from fp64 are counted and each must lie within the bound of 0.5.

The bound, per output element against its reference r:

    |got - r| <= C * 2^-24 * M + 2^-24 * |r| + tiny

M is built from absolute values, C is the longest chain of fp32 roundings a term passes through, and the 2^-24 |r|
term is the final rounding; (C + 1) 2^-149 covers the roundings that fall in the subnormal range, where the error is
absolute.  CUDA's expf is within 2 ulp and logf within 1 ulp (EXP_ULP); sums in
double count as nothing.

    smooth-L1 gradient     clamp(fl(a - b)) * fl(pw / B): C_SL1_G = 2, M = |r|.
    smooth-L1 loss         a term 0.5 d^2 or |d| - 0.5 carries 3 roundings relative to itself (d's rounding doubles
                           in d^2); per pixel C - 1 serial additions, 5 shuffle levels, nw - 1 serial warp partials
                           (nw = block / 32), one rounding of the scale: C = 3 + (C - 1) + 5 + (nw - 1) + 1.
    softmax gradient       p = expf(fl(x - m)) * fl(1 / s): fl(x - m) turns into |x - m| 2^-24 relative in p, expf
                           EXP_ULP, the reciprocal and the product one each, and s carries at most
                           C (EXP_ULP + 2) + D with D = m - min x over the finite logits (one rounding per channel,
                           and the online rescales s * expf(m_old - x) add |m_old - x| in all); then - onehot and
                           * scale (2 roundings in the scale).  M = scale (p (1 + |x - m| + C + D) + |p - onehot|),
                           C_CE_G = EXP_ULP + 4.
    cross-entropy loss     (m + logf(s)) - x_t cancels: M_pix = |m| + |x_t| + |log s| + C + D + |loss|,
                           C_CE_PIX = EXP_ULP + 2; the sum adds 5 + (nw - 1).
    dp samples             four taps of fp32 weights (1 - tx)(1 - ty) (3 roundings), products and 3 additions:
                           C_SAMP = 7 on M_samp = sum |pred| w.  U / V: d = fl(w fl(sample - t)), coef =
                           pw w w sl1'(d) (3 roundings); the gather adds the K points that cover a pixel serially:
                           C = C_SAMP + 5 + K on M = sum_p w_p pw w^2 (|sl1'| + [|d| <= 1] w (M_samp + |sample - t|)).
                           The index term adds 2 C_SAMP max M_samp per point to the softmax M.
    stn soft-argmax        e_k = expf(fl(10 h_k) - m): eps_k = |z_k| + |m| + |z_k - m| + EXP_ULP (units of 2^-24,
                           relative); se, sx, sy are fp32 sums of ceil(HW / 256) terms per thread, 5 shuffle levels
                           and 7 warp partials: cx = sx / se is off by at most
                           Mcx = sum p_k (x_k + cx) (eps_k + K_t + 12) + cx.  The centre's error reaches g_roi through
                           x - cx and through dx = c - kp, so M carries |c| + |kp|.
    part targets           four taps with FMAs: C_PART = 7 on M = sum |v| w.

Exact results are held to equality (M = 0 leaves only the subnormal floor): masked zeros, deselected images, pixels no point or
crop tap reaches, crops whose taps all fall outside the map, and the losses when no image is selected.

The non-finite policy (csrc/loss_common.cuh): a NaN difference gives a NaN smooth-L1 loss and gradient; a -inf logit
adds nothing to its row's log-sum-exp; a row with a NaN or +inf logit, or only -inf logits, has a NaN loss and NaN
gradients; a -inf target logit gives a +inf loss.  The target of an all-NaN or all--inf target pixel is channel 0,
for the loss and the gradient alike.
"""
import collections
import math
import zlib

import numpy as np
import torch

import fp64_bound as fb
from fp64_bound import TINY, U24
EXP_ULP = 2
C_SL1_G = 2
C_CE_G = EXP_ULP + 4
C_CE_PIX = EXP_ULP + 2
C_SAMP = 7
C_PART = 7
PW, PART_W, INDEX_W = 0.5, 0.3, 2.0
F32 = torch.float32
F64 = torch.float64

DP2SMPL = [[7, 8, 9, 10, 1, 2], [1, 2, 8, 10, 12, 14], [1, 2, 7, 9, 11, 13], [7, 8, 9, 10, 1, 2],
           [1, 2, 8, 10, 12, 14], [1, 2, 7, 9, 11, 13], [7, 8, 9, 10, 1, 2], [8, 10, 12, 14, 5, 5],
           [7, 9, 11, 13, 6, 6], [7, 8, 9, 10, 1, 2], [8, 10, 12, 14, 5, 5], [7, 9, 11, 13, 6, 6],
           [1, 2, 23, 24, 23, 24], [1, 2, 15, 17, 19, 21], [1, 2, 16, 18, 20, 22], [1, 2, 23, 24, 23, 24],
           [1, 2, 15, 17, 19, 21], [1, 2, 16, 18, 20, 22], [1, 2, 15, 17, 19, 21], [1, 2, 16, 18, 20, 22],
           [15, 17, 19, 21, 4, 4], [16, 18, 20, 22, 3, 3], [15, 17, 19, 21, 4, 4], [16, 18, 20, 22, 3, 3]]


def rng_for(case):
    return np.random.default_rng(zlib.crc32(repr(case).encode()))


def f32(x):
    return np.asarray(x, np.float32)


def block_threads(total):
    """danet_body_uv_losses' block size for N * HW pixels"""
    return 256 if total >= 132 * 2048 * 2 else (128 if total >= 132 * 2048 // 2 else 64)


def bound(r, M, C):
    """(scale, floor) of the bound C 2^-24 M + 2^-24 |r| + (C + 1) 2^-149 for fp64_bound.worst, which passes at <= 1:
    C differs from element to element here, so it goes into the scale"""
    C = torch.as_tensor(C, dtype=F64, device=r.device)
    return C * U24 * torch.as_tensor(M, dtype=F64, device=r.device), U24 * r.abs() + (C + 1) * TINY


# ----------------------------------------------------------------------------------------------------------------------
# body_uv_losses / part_iuv_losses
# ----------------------------------------------------------------------------------------------------------------------
Body = collections.namedtuple("Body", ["N", "C", "Cann", "H", "W", "pad", "part", "has", "I", "scale", "offset",
                                       "nonfinite", "need"])


def body(N, C, H, W, Cann=0, pad=0, part=False, has="all", I="onehot", scale=0, offset=False, nonfinite="", need="uvia"):
    if not Cann:
        need = need.replace("a", "")
    return Body(N, C, Cann, H, W, pad, part, has, I, scale, offset, nonfinite, need)


def body_id(c):
    return "N%dC%dx%d_%dx%d%s%s_%s_%s%s%s%s_%s" % (
        c.N, c.C, c.Cann, c.H, c.W, "_pad%d" % c.pad if c.pad else "", "_part" if c.part else "", c.has, c.I,
        "_s%d" % c.scale if c.scale else "", "_off" if c.offset else "", "_" + c.nonfinite if c.nonfinite else "", c.need)


BODY_CASES = [
    # the 64 / 128 / 256-thread blocks on both sides of each threshold, and the training shapes
    body(1, 1, 1, 135167), body(1, 1, 1, 135168), body(1, 1, 1, 540671), body(4, 1, 1, 135168),
    body(16, 25, 56, 56, Cann=15, has="some"), body(64, 25, 56, 56, Cann=15, has="some"),
    body(16 * 24, 7, 56, 56, part=True, has="some"),
    # channels, annotation heads, strided rows
    body(3, 1, 5, 7), body(2, 7, 9, 9), body(3, 25, 7, 3, Cann=15), body(2, 25, 4, 4, Cann=1), body(2, 7, 3, 5, Cann=15),
    body(3, 7, 6, 6, pad=13), body(2, 25, 5, 5, Cann=15, pad=7), body(2 * 24, 7, 6, 6, part=True),
    # selections
    body(4, 25, 6, 6, Cann=15, has="none"), body(4, 25, 6, 6, Cann=15, has="some"), body(4, 25, 6, 6, Cann=15, has="one"),
    body(4, 25, 6, 6, Cann=15, has="zero"), body(3 * 24, 7, 5, 5, part=True, has="one"),
    body(2 * 24, 7, 5, 5, part=True, has="zero"),
    # target maps
    body(3, 25, 8, 8, Cann=15, I="soft"), body(3, 25, 8, 8, Cann=15, I="tie"), body(3, 7, 8, 8, I="tie", has="some"),
    # logit magnitudes: 2^0 ... 2^10, offset 2^14
    *[body(2, 25, 6, 6, Cann=15, scale=s, offset=o) for s in (0, 4, 10) for o in (False, True)],
    body(3, 7, 6, 6, scale=2, offset=True, I="soft"),
    # non-finite values
    body(3, 25, 6, 6, Cann=15, nonfinite="nan"), body(3, 25, 6, 6, Cann=15, nonfinite="inf"),
    body(3, 25, 6, 6, Cann=15, nonfinite="lead_ninf"), body(3, 25, 6, 6, Cann=15, nonfinite="tgt_nan"),
    body(3, 25, 6, 6, Cann=15, nonfinite="tgt_ninf"), body(2, 7, 5, 5, Cann=1, nonfinite="lead_ninf", has="some"),
]
for _k, _sub in enumerate(["u", "v", "i", "a", "uv", "ia", "uia", "va", ""]):
    BODY_CASES.append(body(2 + _k % 2, 25, 5, 6, Cann=15, has=("some", "all")[_k % 2], need=_sub))


def make_body(c):
    """seeded inputs: pred [N,3,L] and gt [N,3,L] (u / v / index and U / V / I groups of each row, L = C*HW + pad),
    ann / A [N,Cann*HW] or None, has [N] uint8 or None"""
    rng = rng_for(c)
    N, C, HW, L = c.N, c.C, c.H * c.W, c.C * c.H * c.W + c.pad
    pred = rng.normal(0.5, 0.7, (N, 3, L))
    pred[:, 2] = rng.normal(0, 1.0, (N, L)) * 2.0 ** c.scale + (2.0 ** 14 if c.offset else 0.0)
    gt = rng.uniform(0, 1, (N, 3, L))
    lab = rng.integers(0, C, (N, HW))
    I = np.zeros((N, C, HW))
    if c.I == "soft":
        I = np.maximum(rng.normal(0, 1, (N, C, HW)), 0)
    else:
        np.put_along_axis(I, lab[:, None], 1.0, 1)
        I *= rng.choice([0.0, 1.0, 2.0], (N, 1, HW), p=[0.2, 0.5, 0.3])    # background pixels, and weights 2
        if c.I == "tie" and C > 1:
            I[:, min(2, C - 1)] = I.max(1)                                     # ties with the one-hot channel
            I[:, 0] = I.max(1)                                                 # channel 0 first: the argmax keeps it
    gt[:, 2, :C * HW] = I.reshape(N, -1)
    ann = A = None
    if c.Cann:
        ann = rng.normal(0, 1.5, (N, c.Cann * HW)) * 2.0 ** c.scale + (2.0 ** 14 if c.offset else 0.0)
        A = np.zeros((N, c.Cann, HW))
        np.put_along_axis(A, rng.integers(0, c.Cann, (N, HW))[:, None], 1.0, 1)
        A = A.reshape(N, -1)
    B = N // 24 if c.part else N
    has = {"none": None, "all": np.ones(B), "zero": np.zeros(B)}.get(c.has)
    if c.has == "some":
        has = (rng.random(B) > 0.5).astype(np.float64)
        has[0], has[-1] = 1, 0
    elif c.has == "one":
        has = np.zeros(B)
        has[B // 2] = 1
    if has is not None and c.part:
        has = np.repeat(has, 24)
    if c.nonfinite:
        n = 0 if has is None else int(np.nonzero(has)[0][0])
        pv = pred[n].reshape(3, -1)
        iv = gt[n, 2, :C * HW].reshape(C, HW)
        if c.nonfinite in ("nan", "inf"):
            iv[:, 3] = 0
            iv[1, 3] = 1                                                        # target channel 1 at pixel 3
            bad = np.nan if c.nonfinite == "nan" else np.inf
            pv[0, 1 * HW + 3] = bad                                             # u at the target: masked in
            pv[1, 1 * HW + 3] = -bad if c.nonfinite == "inf" else 0.3
            pv[2, 2 * HW + 5] = bad                                             # a logit of pixel 5
            pv[2, 4 * HW + 6] = -np.inf                                         # a -inf logit, not the target
            if ann is not None:
                ann[n, 2 * HW + 7] = bad
        elif c.nonfinite == "lead_ninf":
            for p in (0, 1, 4):
                iv[:, p] = 0
                iv[min(1, C - 1), p] = 1
                pv[2, p] = -np.inf                                              # channel 0 first, not the target
            pv[2, 1 * HW + 4] = -np.inf                                         # -inf target logit: loss +inf
            if ann is not None:
                ann[n, 0:HW:2] = -np.inf
            pv[2, 2:C * HW:HW] = [-np.inf] * C                                  # pixel 2: every logit -inf
        elif c.nonfinite == "tgt_nan":
            iv[:, 2] = np.nan                                                   # all NaN: channel 0
            iv[:, 3] = 0.5
            iv[3, 3] = np.nan                                                   # first NaN wins
            iv[5, 3] = np.nan
        elif c.nonfinite == "tgt_ninf":
            iv[:, 2] = -np.inf                                                  # all -inf: channel 0
        gt[n, 2, :C * HW] = iv.reshape(-1)
        pred[n] = pv.reshape(3, -1)
    return dict(pred=f32(pred), gt=f32(gt), ann=None if ann is None else f32(ann), A=None if A is None else f32(A),
                has=None if has is None else has.astype(np.uint8))


def _views(c, p):
    N, C, HW = c.N, c.C, c.H * c.W
    g = lambda a, k: torch.from_numpy(a[:, k, :C * HW].reshape(N, C, HW).copy())
    return [g(p["pred"], k) for k in range(3)], [g(p["gt"], k) for k in range(3)]


def target_argmax(I, last=False):
    """torch.argmax of the target map over dim 1, in fp32: first maximum (last, for the seeded defect), NaN maximal"""
    nan = torch.isnan(I)
    mx = torch.where(nan, torch.full_like(I, -math.inf), I).amax(1, keepdim=True)
    hit = torch.where(nan.any(1, keepdim=True), nan, I == mx)
    idx = torch.arange(I.shape[1]).view(1, -1, 1).expand_as(I)
    if last:
        return torch.where(hit, idx, -1).amax(1)
    return torch.where(hit, idx, I.shape[1]).amin(1)


def softmax_terms(x, lab, valid, dt):
    """rows over dim 1: loss, p - onehot, and the bound's M for the gradient (without the scale) and the loss.
    `valid` [N, n] masks rows; lab [N, n] in [0, C)."""
    m = x.amax(1, keepdim=True)
    e = torch.exp(x - m)
    s = e.sum(1, keepdim=True)
    p = e / s
    oh = torch.zeros_like(x).scatter_(1, lab.unsqueeze(1), 1.0)
    xt = x.gather(1, lab.unsqueeze(1))
    loss = (m + torch.log(s) - xt).squeeze(1)
    fin = torch.isfinite(x)
    D = (m - torch.where(fin, x, m).amin(1, keepdim=True)).abs()
    Cn = x.shape[1]
    Mg = p.abs() * (1 + (x - m).abs().nan_to_num(0, 0, 0) + Cn + D) + (p - oh).abs()
    Ml = (m.abs() + xt.abs() + torch.log(s).abs() + Cn + D).squeeze(1) + loss.abs()
    v = valid.unsqueeze(1)
    return (torch.where(valid, loss, torch.zeros((), dtype=dt)), torch.where(v, p - oh, torch.zeros((), dtype=dt)),
            torch.where(v, Mg, torch.zeros((), dtype=dt)), torch.where(valid, Ml.nan_to_num(0, 0, 0), torch.zeros((), dtype=dt)))


def sl1(d):
    a = d.abs()
    return torch.where(a < 1, 0.5 * d * d, a - 0.5)


def sl1_grad(d):
    return torch.where(torch.isnan(d), d, d.clamp(-1, 1))


def body_reference(c, p, dt=F64, defect=None):
    """{output: (r, M, C)} for u / v / index / ann gradients [N,C,HW] and the four losses.  dt = float32 with a
    `defect` is the fp32 emulation the seeded-defect tests use."""
    (u, v, i), (Um, Vm, Im) = _views(c, p)
    N, C, HW = c.N, c.C, c.H * c.W
    has = None if p["has"] is None else torch.from_numpy(p["has"]) != 0
    sel = torch.ones(N, dtype=torch.bool) if has is None else has
    nsel = int(sel.sum())
    on = sel & (nsel > 0)
    nw = block_threads(N * HW) // 32
    sc = PW / (max(nsel, 1) if defect == "sl1_over_nsel" else N)
    out = {}
    losses = []
    for name, x, t in (("u", u, Um), ("v", v, Vm)):
        d = x.to(dt) - t.to(dt)
        mask = (Im > 0) & on.view(-1, 1, 1)
        z = torch.zeros((), dtype=dt)
        g = torch.where(mask, sl1_grad(d) * sc, z)
        out["g" + name] = (g, g.abs(), C_SL1_G)
        l = torch.where(mask, sl1(d), z)
        losses.append((l.sum() * sc, l.abs().sum() * sc, 3 + (C - 1) + 5 + (nw - 1) + 1))
    lab = target_argmax(Im, last=defect == "last_tie")
    cs = 1.0 / ((N if defect == "ce_over_n" else nsel) * HW) if nsel else 0.0
    valid = on.view(-1, 1).expand(N, HW)
    xi = i.to(dt)
    if defect == "no_max_rescale":
        xi = xi                                                                 # handled below
    loss, g, Mg, Ml = softmax_terms(xi, lab, valid, dt)
    if defect == "no_max_rescale":
        e = torch.exp(xi)
        s = e.sum(1, keepdim=True)
        g = torch.where(valid.unsqueeze(1), e / s - torch.zeros_like(xi).scatter_(1, lab.unsqueeze(1), 1.0), g * 0)
        loss = torch.where(valid, (torch.log(s) - xi.gather(1, lab.unsqueeze(1))).squeeze(1), loss * 0)
    out["gi"] = (g * cs, Mg * cs, C_CE_G)
    losses.append((loss.sum() * cs, Ml.sum() * cs, C_CE_PIX + 5 + (nw - 1)))
    if c.Cann:
        a = torch.from_numpy(p["ann"]).view(N, c.Cann, HW).to(dt)
        A = torch.from_numpy(p["A"]).view(N, c.Cann, HW)
        loss, g, Mg, Ml = softmax_terms(a, target_argmax(A, last=defect == "last_tie"), valid, dt)
        out["ga"] = (g * cs, Mg * cs, C_CE_G)
        losses.append((loss.sum() * cs, Ml.sum() * cs, C_CE_PIX + 5 + (nw - 1)))
    else:
        losses.append((torch.zeros((), dtype=dt), torch.zeros((), dtype=dt), 0))
    if nsel == 0:
        losses = [(torch.zeros((), dtype=dt), torch.zeros((), dtype=dt), 0)] * 4
    out["losses"] = (torch.stack([l[0] for l in losses]), torch.stack([l[1] for l in losses]),
                     torch.tensor([float(l[2]) for l in losses], dtype=F64))
    return out


# ----------------------------------------------------------------------------------------------------------------------
# dp_uvia_losses
# ----------------------------------------------------------------------------------------------------------------------
Dp = collections.namedtuple("Dp", ["N", "S", "P", "Cann", "align", "has", "pts", "nonfinite", "need"])


def dp(N, S, P, Cann=15, align=False, has="all", pts="mixed", nonfinite="", need="uvia"):
    return Dp(N, S, P, Cann, align, has, pts, nonfinite, need)


def dp_id(c):
    return "N%dS%dP%dA%d%s_%s_%s%s_%s" % (c.N, c.S, c.P, c.Cann, "_ac" if c.align else "", c.has, c.pts,
                                         "_" + c.nonfinite if c.nonfinite else "", c.need)


DP_CASES = [
    dp(16, 56, 196, has="some"), dp(3, 9, 196), dp(2, 9, 196, align=True),
    dp(3, 5, 1), dp(2, 17, 31, align=True), dp(2, 7, 256), dp(2, 8, 256, pts="pile"), dp(2, 8, 256, pts="pile", align=True),
    dp(2, 12, 31, pts="edge"), dp(2, 12, 31, pts="edge", align=True), dp(2, 10, 40, pts="outside"),
    dp(2, 6, 20, pts="centre"), dp(3, 16, 31), dp(2, 16, 31, align=True),                     # HW = 256: one full tile
    dp(3, 9, 31, has="some"), dp(3, 9, 31, has="one"), dp(3, 9, 31, has="zero"), dp(3, 9, 31, has="none"),
    dp(2, 8, 31, Cann=1), dp(2, 8, 31, nonfinite="nan"), dp(2, 8, 31, nonfinite="inf"),
    dp(2, 8, 31, nonfinite="lead_ninf"), dp(2, 8, 31, nonfinite="coords"),
]
for _k, _sub in enumerate(["u", "v", "i", "a", "uv", "ia", "uia", ""]):
    DP_CASES.append(dp(2 + _k % 2, 7, 31, has=("some", "all")[_k % 2], align=bool(_k % 3 == 0), need=_sub))


def make_dp(c):
    rng = rng_for(c)
    N, S, P, HW = c.N, c.S, c.P, c.S * c.S
    u, v = rng.normal(0.5, 0.6, (N, 25, HW)), rng.normal(0.5, 0.6, (N, 25, HW))
    idx, ann = rng.normal(0, 2, (N, 25, HW)), rng.normal(0, 2, (N, c.Cann, HW))
    X, Y = rng.uniform(-1.5, S + 0.5, (N, P)), rng.uniform(-1.5, S + 0.5, (N, P))
    end = S if c.align else S - 0.5                                             # the last row / column under align
    specials = {"centre": [(k + 0.5, (3 * k) % S + 0.5) for k in range(S)],
                "edge": [(end, 2.5), (1.5, end), (end, end), (0.0 if c.align else 0.5, end), (end - 0.25, end)],
                "outside": [(-3.0, 2.0), (S + 5.0, 1.0), (2.0, -2.5), (1e9, -1e9), (-1.0, -1.0), (S + 0.9, S + 0.9)]}
    if c.pts == "pile":
        X[:], Y[:] = 3.5, 2.5                                                   # every point on one pixel centre
    if c.pts == "mixed":
        sp = specials["centre"][:2] + specials["edge"][:2] + specials["outside"][:3]
    else:
        sp = specials.get(c.pts, [])
    for k, (x, y) in enumerate(sp[:P]):
        X[:, k], Y[:, k] = x, y
    I = rng.integers(0, 25, (N, P)) + rng.choice([0.0, 0.25, 0.75, 0.999], (N, P))
    I[:, 0], I[:, -1] = 0.0, 24.0
    if P > 2:
        I[:, 1] = 24.9
    W = rng.choice([0.0, 1.0, 2.0], (N, 25, P))
    Up, Vp = rng.uniform(0, 1, (N, 25, P)), rng.uniform(0, 1, (N, 25, P))
    A = rng.integers(0, c.Cann, (N, HW)) + rng.choice([0.0, 0.5], (N, HW))
    has = {"none": None, "all": np.ones(N), "zero": np.zeros(N)}.get(c.has)
    if c.has == "some":
        has = (rng.random(N) > 0.5).astype(np.float64)
        has[0], has[-1] = 1, 0
    elif c.has == "one":
        has = np.zeros(N)
        has[N - 1] = 1
    if c.nonfinite == "nan":
        u[0, 3, :] = np.nan                                                     # every sample of channel 3 is NaN
        idx[0, 5, 2 * S + 2] = np.nan
        ann[0, 1, 4] = np.nan
    elif c.nonfinite == "inf":
        v[0, 2, :] = np.inf
        idx[0, 7, :] = -np.inf                                                  # a -inf channel everywhere
        ann[0, 2, 5] = np.inf
    elif c.nonfinite == "lead_ninf":
        idx[0, 0, :] = -np.inf
        ann[0, 0, :] = -np.inf
        I[0, 2:5] = 0.0                                                         # a -inf target logit
    elif c.nonfinite == "coords":
        X[0, 2], Y[0, 3], X[0, 4] = np.nan, np.inf, -np.inf
    return dict(u=f32(u.reshape(N, 25, S, S)), v=f32(v.reshape(N, 25, S, S)), idx=f32(idx.reshape(N, 25, S, S)),
                ann=f32(ann.reshape(N, c.Cann, S, S)), X=f32(X), Y=f32(Y), I=f32(I), Up=f32(Up.reshape(N, -1)),
                Vp=f32(Vp.reshape(N, -1)), W=f32(W.reshape(N, -1)), A=f32(A),
                has=None if has is None else has.astype(np.uint8))


def grid_unnormalize32(g, S, align):
    """fp32, one rounding per operation (csrc/stn_common.cuh grid_unnormalize)"""
    one, half = torch.tensor(1.0, dtype=F32), torch.tensor(0.5, dtype=F32)
    if align:
        return ((g + one) * half) * torch.tensor(float(S - 1), dtype=F32)
    return ((g + one) * torch.tensor(float(S), dtype=F32) - one) * half


def foot(ix, iy, S):
    """the kernels' make_foot, restated in fp32: (x0, y0 int64, valid, [4] fp64 weights) with torch.floor and
    t = ix - floor(ix) in fp32; invalid points (all corners outside, or NaN) get weights 0"""
    fx, fy = torch.floor(ix), torch.floor(iy)
    ok = (fx > -2) & (fx < S) & (fy > -2) & (fy < S)
    tx, ty = (ix - fx).to(F64), (iy - fy).to(F64)
    w = [(1 - tx) * (1 - ty), tx * (1 - ty), (1 - tx) * ty, tx * ty]
    w = [torch.where(ok, wk, torch.zeros((), dtype=F64)).nan_to_num(0, 0, 0) for wk in w]
    x0 = torch.where(ok, fx, torch.full_like(fx, -2)).to(torch.int64)
    y0 = torch.where(ok, fy, torch.full_like(fy, -2)).to(torch.int64)
    return x0, y0, ok, w


def taps(x0, y0, S):
    for k in range(4):
        xx, yy = x0 + (k & 1), y0 + (k >> 1)
        inb = (xx >= 0) & (xx < S) & (yy >= 0) & (yy < S)
        yield k, inb, torch.where(inb, yy * S + xx, torch.zeros_like(xx))


def dp_reference(c, p, dt=F64, defect=None):
    N, S, P, HW = c.N, c.S, c.P, c.S * c.S
    t = lambda k: torch.from_numpy(p[k])
    has = None if p["has"] is None else t("has") != 0
    sel = torch.ones(N, dtype=torch.bool) if has is None else has
    nsel = int(sel.sum())
    on = sel & (nsel > 0)
    hs, scl = torch.tensor(0.5 * S, dtype=F32), torch.tensor(2.0 / S, dtype=F32)
    align = (not c.align) if defect == "other_align" else c.align
    gx, gy = (t("X") - hs) * scl, (t("Y") - hs) * scl
    x0, y0, ok, fw = foot(grid_unnormalize32(gx, S, align), grid_unnormalize32(gy, S, align), S)
    tap = list(taps(x0, y0, S))
    z = torch.zeros((), dtype=dt)

    def sample(pred):                                                           # [N,C,HW] -> [N,C,P], and M
        s = torch.zeros(N, pred.shape[1], P, dtype=dt)
        Ms = torch.zeros(N, pred.shape[1], P, dtype=F64)
        for k, inb, q in tap:
            val = pred.to(dt).gather(2, q.unsqueeze(1).expand(-1, pred.shape[1], -1))
            s = s + torch.where(inb.unsqueeze(1), val * fw[k].to(dt).unsqueeze(1), z)
            Ms = Ms + torch.where(inb.unsqueeze(1), val.to(F64).abs() * fw[k].unsqueeze(1), torch.zeros((), dtype=F64))
        return s, Ms.nan_to_num(0, 0, 0)

    # the pixels each point covers with a non-zero weight, the per-pixel count K and (for a defect) the last point
    cover = [(k, inb & (fw[k] != 0) & on.view(-1, 1), q) for k, inb, q in tap]
    K = torch.zeros(N, HW, dtype=F64)
    last = torch.full((N, HW), -1, dtype=torch.int64)
    pidx = torch.arange(P).view(1, -1).expand(N, -1)
    for k, cv, q in cover:
        K.scatter_add_(1, q, cv.to(F64))
        last.scatter_reduce_(1, q, torch.where(cv, pidx, -1), "amax")

    def gather(coef, Mc, C):                                                    # [N,C,P] -> grads [N,C,HW]
        g = torch.zeros(N, C, HW, dtype=dt)
        M = torch.zeros(N, C, HW, dtype=F64)
        for k, cv, q in cover:
            if defect == "drop_last":
                cv = cv & (last.gather(1, q) != pidx)
            qq = q.unsqueeze(1).expand(-1, C, -1)
            g.scatter_add_(2, qq, torch.where(cv.unsqueeze(1), coef * fw[k].to(dt).unsqueeze(1), z))
            M.scatter_add_(2, qq, torch.where(cv.unsqueeze(1), Mc * fw[k].unsqueeze(1), torch.zeros((), dtype=F64)))
        return g, M.nan_to_num(0, 0, 0)

    out, losses = {}, []
    Wp = t("W").view(N, 25, P).to(dt)
    onp = on.view(-1, 1, 1)
    for name, tg in (("u", "Up"), ("v", "Vp")):
        s, Ms = sample(t(name).view(N, 25, HW))
        diff = s - t(tg).view(N, 25, P).to(dt)
        d = Wp * diff
        gl = sl1_grad(d)
        coef = torch.where(onp, PW * Wp * Wp * gl, z)
        lin = torch.where(d.abs() <= 1, Wp.to(F64) * (Ms + diff.to(F64).abs()), torch.zeros((), dtype=F64))
        Mc = (PW * Wp * Wp).to(F64) * (gl.to(F64).abs() + lin)
        Mc = torch.where(onp, Mc.nan_to_num(0, 0, 0), torch.zeros((), dtype=F64))
        g, M = gather(coef, Mc, 25)
        out["g" + name] = (g, M, C_SAMP + 5 + K.unsqueeze(1))
        l = torch.where(onp, Wp * sl1(d), z)
        Ml = torch.where(onp, (Wp * sl1(d)).to(F64).abs() + Mc / PW, torch.zeros((), dtype=F64)).nan_to_num(0, 0, 0)
        losses.append((l.sum() * PW, Ml.sum() * PW, 4 + C_SAMP + 24 + 5 + 7 + 1))
    # index: cross-entropy of the 25 samples against the truncated label
    Ilab = t("I")
    lab = torch.where((Ilab > -1) & (Ilab < 25), Ilab.trunc(), torch.full_like(Ilab, -1)).to(torch.int64)
    x, Ms = sample(t("idx").view(N, 25, HW))
    valid = on.view(-1, 1) & (lab >= 0)
    loss, g, Mg, Mpix = softmax_terms(x, lab.clamp(min=0), valid, dt)
    Msx = Ms.amax(1, keepdim=True)
    Mg = Mg + torch.where(valid.unsqueeze(1), 2 * C_SAMP * g.abs().to(F64).new_ones(()) * Msx, torch.zeros((), dtype=F64))
    npts = nsel * (HW if defect == "index_over_hw" else P)
    sc = PART_W / npts if nsel else 0.0
    gi, M = gather(g * sc, Mg * sc, 25)
    out["gi"] = (gi, M, C_CE_G + 5 + K.unsqueeze(1))
    Mpix = Mpix + torch.where(valid, 2 * C_SAMP * Msx.squeeze(1), torch.zeros((), dtype=F64))
    losses.append((loss.sum() * (PART_W / (nsel * P) if nsel else 0.0), Mpix.sum() * (PART_W / (nsel * P) if nsel else 0.0),
                   C_CE_PIX + 5 + 7 + 1))
    # annotation: per-pixel cross-entropy over Cann against the truncated label
    Al = t("A")
    alab = torch.where((Al > -1) & (Al < c.Cann), Al.trunc(), torch.full_like(Al, -1)).to(torch.int64)
    avalid = on.view(-1, 1) & (alab >= 0)
    loss, g, Mg, Mpix = softmax_terms(t("ann").view(N, c.Cann, HW).to(dt), alab.clamp(min=0), avalid, dt)
    cs = INDEX_W / (nsel * HW) if nsel else 0.0
    out["ga"] = (g * cs, Mg * cs, C_CE_G + 1)
    losses.append((loss.sum() * cs, Mpix.sum() * cs, C_CE_PIX + 5 + 7 + 1))
    if nsel == 0:
        losses = [(torch.zeros((), dtype=dt), torch.zeros((), dtype=F64), 0)] * 4
    out["losses"] = (torch.stack([l[0] for l in losses]), torch.stack([l[1].to(F64) for l in losses]),
                     torch.tensor([float(l[2]) for l in losses], dtype=F64))
    for k in ("gu", "gv", "gi", "ga"):
        r, M, C = out[k]
        out[k] = (r.view(N, -1, S, S), M.view(N, -1, S, S), C.view(N, 1, S, S) if torch.is_tensor(C) else C)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# stn_kps_losses
# ----------------------------------------------------------------------------------------------------------------------
Stn = collections.namedtuple("Stn", ["B", "J", "S", "cols", "kw", "hw", "hm", "nonfinite", "alias"])


def stn(B, J, S, cols=3, kw=1.0, hw=0.7, hm="normal", nonfinite="", alias=False):
    return Stn(B, J, S, cols, kw, hw, hm, nonfinite, alias)


def stn_id(c):
    return "B%dJ%dS%d_c%d_k%g_h%g_%s%s%s" % (c.B, c.J, c.S, c.cols, c.kw, c.hw, c.hm,
                                              "_" + c.nonfinite if c.nonfinite else "", "_alias" if c.alias else "")


STN_CASES = [
    stn(16, 24, 56), stn(2, 24, 12), stn(3, 24, 15), stn(2, 5, 17), stn(2, 24, 12, cols=2), stn(2, 24, 20, cols=2, kw=0.0),
    stn(2, 24, 12, kw=0.0), stn(2, 24, 12, hw=0.0), stn(2, 24, 12, kw=2.0, hw=0.0, alias=True),
    stn(2, 24, 12, alias=True), stn(2, 24, 12, hm="peaked"), stn(2, 24, 20, hm="peaked"), stn(2, 24, 12, hm="const"),
    stn(2, 24, 12, hm="offset"), stn(2, 24, 18, hm="offset", cols=2),
    stn(2, 24, 12, nonfinite="nan"), stn(2, 24, 12, nonfinite="inf"), stn(2, 24, 12, nonfinite="ninf"),
]


def make_stn(c):
    rng = rng_for(c)
    B, J, S = c.B, c.J, c.S
    hm = rng.normal(0, 0.1, (B, J, S, S))
    if c.hm == "peaked":
        hm = rng.normal(0, 4.0, (B, J, S, S))                                   # 10 hm spread > 100
    elif c.hm == "const":
        hm[:] = 0.3
    elif c.hm == "offset":
        hm = hm + 2.0 ** 10
    kps = rng.uniform(-1.2, 1.2, (B, J, 3))
    kps[..., 2] = rng.choice([0.0, 1.0, 2.0], (B, J))
    left = -2.0 / S - 1.0 + 0.3 / S                                             # k S + 0.5 in (-1, 0): truncated to 0
    edge = [(-1.0, 0.0), (1.0, 0.2), (0.0, -1.0), (0.3, 1.0), (left, 0.1), (0.1, left), (40.0, 0.0), (0.0, -40.0),
            (1e12, 0.0), (-1.0 - 8.0 / S, 0.0)]
    for k, (x, y) in enumerate(edge[:J]):
        kps[0, k, :2] = x, y
    kps[-1, 0, :2] = 1.0 + 3.5 / S, -1.0 - 3.5 / S                              # the window's last row / column on
    if c.nonfinite == "nan":
        hm[0, 1, 2, 3] = np.nan
    elif c.nonfinite == "inf":
        hm[0, 2, 4, 4] = np.inf
        hm[1, 3, 0, 0] = -np.inf
    elif c.nonfinite == "ninf":
        hm[0, 2, :2, :] = -np.inf
    return dict(hm=f32(hm), kps=f32(kps[..., :c.cols]))


def hm_window(kps, S):
    """fp32 restatement of hm_window: (mx, my int64, on) per joint"""
    half = torch.tensor(0.5, dtype=F32)
    k = kps[..., :2] * half + half
    tt = k * torch.tensor(float(S), dtype=F32) + half
    lim = 1073741824.0
    on = ((tt > -lim) & (tt < lim)).all(-1)
    m = torch.where(on.unsqueeze(-1), tt, torch.zeros_like(tt)).trunc().to(torch.int64)
    mx, my = m[..., 0], m[..., 1]
    on = on & ~((mx - 3 >= S) | (my - 3 >= S) | (mx + 4 < 0) | (my + 4 < 0))
    return mx, my, on


def stn_reference(c, p, dt=F64, defect=None):
    B, J, S, HW = c.B, c.J, c.S, c.S * c.S
    h = torch.from_numpy(p["hm"]).view(B, J, HW)
    kps = torch.from_numpy(p["kps"])
    z = 10 * h.to(dt)
    m = z.amax(-1, keepdim=True)
    e = torch.exp(z - m)
    se = e.sum(-1, keepdim=True)
    pr = e / se
    col = (torch.arange(HW) % S).to(dt)
    row = (torch.arange(HW) // S).to(dt)
    if defect == "xy_swapped":
        col, row = row, col
    cx, cy = (pr * col).sum(-1), (pr * row).sum(-1)
    hS = 0.5 * S
    c_x, c_y = cx / hS - 1, cy / hS - 1
    # error of the soft-argmax (units of 2^-24): eps_k per term, then K_t + 12 summation roundings
    Kt = -(-HW // 256)
    z64, m64, p64 = z.to(F64), m.to(F64), pr.to(F64)
    eps = (z64.abs() + m64.abs() + (z64 - m64).abs() + EXP_ULP + Kt + 12).nan_to_num(0, 0, 0)
    col64, row64 = col.to(F64), row.to(F64)
    Mcx = (p64 * (col64 + cx.to(F64).unsqueeze(-1)) * eps).sum(-1) + cx.to(F64).abs() + 2 * cx.to(F64).abs()
    Mcy = (p64 * (row64 + cy.to(F64).unsqueeze(-1)) * eps).sum(-1) + cy.to(F64).abs() + 2 * cy.to(F64).abs()
    zz = torch.zeros((), dtype=dt)
    out = {}
    gcx = gcy = torch.zeros(B, J, dtype=dt)
    roi = torch.zeros((), dtype=dt)
    Mroi = torch.zeros((), dtype=F64)
    Mgcx = Mgcy = torch.zeros(B, J, dtype=F64)
    if c.cols == 3 and c.kw != 0:
        w = kps[..., 2].to(dt)
        onj = w != 0
        dx, dy = c_x - kps[..., 0].to(dt), c_y - kps[..., 1].to(dt)
        s = c.kw / B * w
        gcx = torch.where(onj, s * sl1_grad(dx), zz)
        gcy = torch.where(onj, s * sl1_grad(dy), zz)
        lj = torch.where(onj, w * (sl1(dx) + sl1(dy)), zz)
        roi = lj.sum() * (c.kw / B)
        Mdx = (Mcx / hS + 2 * cx.to(F64).abs() / hS + c_x.to(F64).abs() + kps[..., 0].to(F64).abs() + dx.to(F64).abs())
        Mdy = (Mcy / hS + 2 * cy.to(F64).abs() / hS + c_y.to(F64).abs() + kps[..., 1].to(F64).abs() + dy.to(F64).abs())
        gx64, gy64 = sl1_grad(dx).to(F64).abs(), sl1_grad(dy).to(F64).abs()
        w64 = w.to(F64).abs()
        Mj = w64 * (gx64 * Mdx + gy64 * Mdy + (sl1(dx) + sl1(dy)).to(F64).abs())
        Mroi = torch.where(onj, Mj, torch.zeros((), dtype=F64)).nan_to_num(0, 0, 0).sum() * (c.kw / B)
        lin = lambda d: (d.abs() <= 1).to(F64)
        s64 = (c.kw / B) * w64
        Mgcx = torch.where(onj, s64 * (3 * gx64 + lin(dx) * Mdx), torch.zeros((), dtype=F64)).nan_to_num(0, 0, 0)
        Mgcy = torch.where(onj, s64 * (3 * gy64 + lin(dy) * Mdy), torch.zeros((), dtype=F64)).nan_to_num(0, 0, 0)
    ex, ey = col - cx.unsqueeze(-1), row - cy.unsqueeze(-1)
    groi = 10 * pr * (gcx.unsqueeze(-1) * ex + gcy.unsqueeze(-1) * ey) / hS
    ex64, ey64 = ex.to(F64).abs(), ey.to(F64).abs()
    a64 = gcx.to(F64).abs().unsqueeze(-1) * ex64 + gcy.to(F64).abs().unsqueeze(-1) * ey64
    Mgroi = 10 * p64 / hS * ((eps + 6) * a64 + Mgcx.unsqueeze(-1) * ex64 + Mgcy.unsqueeze(-1) * ey64
                             + gcx.to(F64).abs().unsqueeze(-1) * (Mcx.unsqueeze(-1) + ex64)
                             + gcy.to(F64).abs().unsqueeze(-1) * (Mcy.unsqueeze(-1) + ey64))
    # e_k below 2^-126 keeps an absolute error of 2^-149, which the rest of the chain scales by 10 a / (S / 2)
    Mgroi = (Mgroi + 4 * 10 / hS * a64 * 2.0 ** -125).nan_to_num(0, 0, 0)
    # heat-map loss against the Gaussian target
    mx, my, won = hm_window(kps, S)
    if defect == "round_centre":
        half = torch.tensor(0.5, dtype=F32)
        tt = (kps[..., :2] * half + half) * torch.tensor(float(S), dtype=F32) + half
        mm = torch.where(won.unsqueeze(-1), torch.floor(tt + 0.5), torch.zeros_like(tt)).to(torch.int64)
        mx, my = mm[..., 0], mm[..., 1]
    ddx = (torch.arange(HW) % S).view(1, 1, -1) - mx.unsqueeze(-1)
    ddy = (torch.arange(HW) // S).view(1, 1, -1) - my.unsqueeze(-1)
    inwin = won.unsqueeze(-1) & (ddx.abs() <= 3) & (ddy.abs() <= 3)
    tgt = torch.where(inwin, torch.exp(-(ddx * ddx + ddy * ddy).to(dt) / 2), zz)
    ghmv = torch.zeros(B, J, HW, dtype=dt)
    stnhm = torch.zeros((), dtype=dt)
    Mghm = torch.zeros(B, J, HW, dtype=F64)
    Mstnhm = torch.zeros((), dtype=F64)
    if c.hw != 0:
        d = h.to(dt) - tgt
        sc = c.hw / (B * J * HW)
        ghmv = sc * sl1_grad(d)
        stnhm = sl1(d).sum() * sc
        g64 = sl1_grad(d).to(F64).abs()
        Mghm = (sc * (g64 + (d.abs() <= 1).to(F64) * (d.to(F64).abs() + tgt.to(F64)))).nan_to_num(0, 0, 0)
        Mstnhm = ((sl1(d).to(F64) + g64 * tgt.to(F64)).nan_to_num(0, 0, 0)).sum() * sc
    C_groi = 4
    C_ghm = EXP_ULP + 3
    if c.alias:
        out["g"] = ((groi + ghmv).view(B, J, S, S), (Mgroi + Mghm).view(B, J, S, S), max(C_groi, C_ghm) + 1)
    else:
        out["groi"] = (groi.view(B, J, S, S), Mgroi.view(B, J, S, S), C_groi)
        out["ghm"] = (ghmv.view(B, J, S, S), Mghm.view(B, J, S, S), C_ghm)
    out["losses"] = (torch.stack([roi, stnhm]), torch.stack([Mroi, Mstnhm]),
                     torch.tensor([5.0, C_ghm + Kt + 12 + 1], dtype=F64))
    return out


# ----------------------------------------------------------------------------------------------------------------------
# part_iuv_targets
# ----------------------------------------------------------------------------------------------------------------------
Part = collections.namedtuple("Part", ["B", "S", "C", "align", "theta", "half"])


def part(B, S, C=25, align=False, theta="near", half=False):
    return Part(B, S, C, align, theta, half)


def part_id(c):
    return "B%dS%dC%d%s_%s%s" % (c.B, c.S, c.C, "_ac" if c.align else "", c.theta, "_half" if c.half else "")


PART_CASES = [
    part(16, 56), part(16, 56, align=True), part(2, 2), part(2, 2, align=True), part(2, 9, theta="general"),
    part(2, 9, align=True, theta="general"), part(2, 8, theta="zero"), part(2, 8, align=True, theta="neg"),
    part(2, 8, theta="neg"), part(2, 8, theta="out"), part(2, 8, align=True, theta="out"), part(2, 12, C=27),
    part(2, 10, half=True), part(2, 10, align=True, half=True, theta="general"),
]


def make_part(c):
    rng = rng_for(c)
    B, S, C = c.B, c.S, c.C
    Um, Vm = rng.uniform(0, 1, (B, C, S, S)), rng.uniform(0, 1, (B, C, S, S))
    Im = rng.uniform(0, 0.4, (B, C, S, S)) * (rng.random((B, C, S, S)) > 0.5)
    if c.half:                                                                  # sum of the mapped I at 0.5 and one ulp off
        q = np.float32(0.25)
        for k, val in enumerate((q, np.nextafter(q, np.float32(0)), np.nextafter(q, np.float32(1)))):
            Im[:, :, k, :] = 0
            Im[:, 1, k, :] = q
            Im[:, 2, k, :] = val
    th = np.zeros((B, 24, 2, 3))
    if c.theta == "near":
        s = rng.uniform(0.2, 0.6, (B, 24))
        th[..., 0, 0], th[..., 1, 1] = s, s
        th[..., :, 2] = rng.uniform(-0.6, 0.6, (B, 24, 2))
    elif c.theta == "general":
        th = rng.normal(0, 0.7, (B, 24, 2, 3))
    elif c.theta == "zero":
        th[..., :, 2] = rng.uniform(-0.9, 0.9, (B, 24, 2))
    elif c.theta == "neg":
        s = -rng.uniform(0.2, 1.2, (B, 24))
        th[..., 0, 0], th[..., 1, 1] = s, s * rng.choice([1, -1], (B, 24))
        th[..., :, 2] = rng.uniform(-0.3, 0.3, (B, 24, 2))
    elif c.theta == "out":
        th[..., 0, 0], th[..., 1, 1] = 0.3, 0.3
        th[..., 0, 2] = rng.choice([4.0, -4.0], (B, 24))
    return dict(U=f32(Um), V=f32(Vm), I=f32(Im), theta=f32(th))


def affine_base32(S, align):
    step = torch.tensor(2.0 / (S - 1), dtype=F32)
    i = torch.arange(S)
    lo = torch.tensor(-1.0, dtype=F32) + step * i.to(F32)
    hi = torch.tensor(1.0, dtype=F32) - step * (S - 1 - i).to(F32)
    v = torch.where(i < S // 2, lo, hi)
    if not align:
        v = (v * torch.tensor(float(S - 1), dtype=F32)) / torch.tensor(float(S), dtype=F32)
    return v


def part_reference(c, p, dt=F64, defect=None):
    """(r [B,24,3,7,S,S], M, C, background decisions that differ from fp64, the worst |sum64 - 0.5| / bound among them)"""
    B, S, HW = c.B, c.S, c.S * c.S
    Um, Vm, Im = (torch.from_numpy(p[k]).view(B, -1, HW) for k in ("U", "V", "I"))
    th = torch.from_numpy(p["theta"]).view(B, 24, 6)
    base = affine_base32(S, c.align)
    xb, yb = base.repeat(S), base.repeat_interleave(S)
    t = lambda k: th[..., k].unsqueeze(-1)
    gx = (t(0) * xb + t(1) * yb) + t(2)
    gy = (t(3) * xb + t(4) * yb) + t(5)
    x0, y0, ok, fw = foot(grid_unnormalize32(gx, S, c.align), grid_unnormalize32(gy, S, c.align), S)
    if defect == "swap_taps":
        fw = [fw[1], fw[0], fw[2], fw[3]]
    mp = torch.tensor(DP2SMPL)
    r = torch.zeros(B, 24, 3, 7, HW, dtype=dt)
    M = torch.zeros(B, 24, 3, 7, HW, dtype=F64)
    Isel = Im[:, mp]                                                            # [B,24,6,HW]
    isum32 = torch.zeros(B, 24, HW, dtype=F32)
    for k in range(5 if defect == "bg_of_5" else 6):
        isum32 = isum32 + Isel[:, :, k]
    isum64 = Isel.to(F64).sum(2)
    bg = (isum32 < 0.5).to(F64)
    flips = (isum32 < 0.5) != (isum64 < 0.5)
    worst = float(((isum64 - 0.5).abs() / (5 * U24 * Isel.to(F64).abs().sum(2) + TINY))[flips].max()) if bool(flips.any()) else 0.0
    src = [Um[:, mp].to(F64), Vm[:, mp].to(F64), Isel.to(F64)]
    for k, inb, q in taps(x0, y0, S):
        w = torch.where(inb, fw[k], torch.zeros((), dtype=F64))                # [B,24,HW]
        g = lambda a: a.gather(-1, q.unsqueeze(2).expand(-1, -1, a.shape[2], -1))
        for m in range(3):
            val = g(src[m])
            r[:, :, m, 1:] += (val * w.unsqueeze(2)).to(dt)
            M[:, :, m, 1:] += val.abs() * w.unsqueeze(2)
        bgv = bg.gather(-1, q)
        r[:, :, 2, 0] += (bgv * w).to(dt)
        M[:, :, 2, 0] += bgv * w
    return r.view(B, 24, 3, 7, S, S), M.view(B, 24, 3, 7, S, S), C_PART, int(flips.sum()), worst


# ----------------------------------------------------------------------------------------------------------------------
# coverage
# ----------------------------------------------------------------------------------------------------------------------
def _classes():
    """[(name, predicate)] over CASES: each table's classes see only that table's cases"""
    b, d, s, q = [], [], [], []
    hw = lambda c: c.N * c.H * c.W
    b += [("body N*HW = %d" % n, lambda c, n=n: hw(c) == n) for n in (135167, 135168, 540671, 540672)]
    b += [("body B = 64 global heads", lambda c: c.N == 64 and c.C == 25 and c.H == 56 and c.Cann == 15),
          ("body 128-thread block", lambda c: block_threads(hw(c)) == 128),
          ("body C = 1", lambda c: c.C == 1), ("body C = 7", lambda c: c.C == 7),
          ("body C = 25", lambda c: c.C == 25), ("body ann absent", lambda c: not c.Cann),
          ("body Cann = 1", lambda c: c.Cann == 1), ("body Cann = 15", lambda c: c.Cann == 15),
          ("body strided rows", lambda c: c.pad or c.part), ("body part layout", lambda c: c.part)]
    b += [("body has %s" % h, lambda c, h=h: c.has == h) for h in ("none", "all", "some", "one", "zero")]
    b += [("body soft I", lambda c: c.I == "soft"), ("body one-hot I", lambda c: c.I == "onehot"),
          ("body target ties", lambda c: c.I == "tie")]
    b += [("body logits 2^%d" % e, lambda c, e=e: c.scale == e) for e in (0, 4, 10)]
    b += [("body logit offset 2^14", lambda c: c.offset),
          ("body NaN predictions", lambda c: c.nonfinite == "nan"),
          ("body +-inf predictions", lambda c: c.nonfinite == "inf"),
          ("body leading -inf", lambda c: c.nonfinite == "lead_ninf"),
          ("body all-NaN target pixel", lambda c: c.nonfinite == "tgt_nan"),
          ("body all--inf target pixel", lambda c: c.nonfinite == "tgt_ninf")]
    d += [("dp P = %d" % P, lambda c, P=P: c.P == P) for P in (1, 31, 196, 256)]
    d += [("dp HW < 256", lambda c: c.S * c.S < 256), ("dp HW % 256 != 0, > 256", lambda c: c.S * c.S > 256 and c.S * c.S % 256),
          ("dp points on pixel centres", lambda c: c.pts in ("centre", "mixed", "pile") and not c.align),
          ("dp last row / column, align False", lambda c: c.pts in ("edge", "mixed") and not c.align),
          ("dp last row / column, align True", lambda c: c.pts in ("edge", "mixed") and c.align),
          ("dp points outside", lambda c: c.pts in ("outside", "mixed")),
          ("dp 256 points on one pixel", lambda c: c.pts == "pile" and c.P == 256),
          ("dp point weights 0 / 1 / 2", lambda c: True), ("dp fractional labels, 0 and 24", lambda c: True)]
    d += [("dp has %s" % h, lambda c, h=h: c.has == h) for h in ("none", "all", "some", "one", "zero")]
    d += [("dp Cann = 1", lambda c: c.Cann == 1)]
    d += [("dp %s" % k, lambda c, k=k: c.nonfinite == k) for k in ("nan", "inf", "lead_ninf", "coords")]
    s += [("stn HW < 256", lambda c: c.S * c.S < 256), ("stn HW > 256", lambda c: c.S * c.S > 256),
          ("stn kps_cols 2", lambda c: c.cols == 2), ("stn kps_cols 3", lambda c: c.cols == 3),
          ("stn kps_weight 0", lambda c: c.kw == 0 and c.cols == 3), ("stn hm_weight 0", lambda c: c.hw == 0),
          ("stn joints on / left of / far outside the border", lambda c: True)]
    s += [("stn hm %s" % k, lambda c, k=k: c.hm == k) for k in ("peaked", "const", "offset")]
    s += [("stn %s hm" % k, lambda c, k=k: c.nonfinite == k) for k in ("nan", "inf", "ninf")]
    s += [("stn grad_roi == grad_hm", lambda c: c.alias)]
    q += [("part S = 2", lambda c: c.S == 2), ("part S = 56", lambda c: c.S == 56),
          ("part align False", lambda c: not c.align), ("part align True", lambda c: c.align),
          ("part general theta", lambda c: c.theta == "general"), ("part scale 0", lambda c: c.theta == "zero"),
          ("part negative scales", lambda c: c.theta == "neg"), ("part all outside", lambda c: c.theta == "out"),
          ("part sum I at 0.5 and one ulp off", lambda c: c.half)]
    b += [("body needs-grad '%s'" % n, lambda c, n=n: c.need == n) for n in ("u", "v", "i", "a", "uv", "ia", "uia", "va", "")]
    d += [("dp needs-grad '%s'" % n, lambda c, n=n: c.need == n) for n in ("u", "v", "i", "a", "uv", "ia", "uia", "")]
    return [(name, lambda c, t=t, fn=fn: type(c) is t and fn(c))
            for t, cl in ((Body, b), (Dp, d), (Stn, s), (Part, q)) for name, fn in cl]


CASES = BODY_CASES + DP_CASES + STN_CASES + PART_CASES
CLASSES = _classes()
