"""fp64 numpy restatement of the training STN ops and the HRNet fuse (csrc/stn_train.cu, csrc/bn_train.cu) --
TEST INFRASTRUCTURE: the checker of danet_b200.stn and danet_b200.layers.hr_fuse, held to the golden the reference's
own code produced (tests/golden/stn_train.npz, oracle/gen_golden_stn_train.py)."""
import numpy as np

from oracle.net_ops import CHILDREN1, PARENTS0, SMPL2DP

f32 = np.float32


def part_thetas(hm, index_pred, ratio, offset, vis_score=0.5, center_noise=None, center_jitter=0.1, scale_noise=None,
                scale_jitter=0.2, align_corners=False):
    """iuv_estimator.py:137-140,172-191,262-301 in fp64.  hm [B,24,S,S], index_pred [B,25,Si,Si], center_noise
    [B,24,2], scale_noise [24,2,B].  Returns (centres [B,24,2] (jittered), thetas [B,24,2,3], scores [B,24] (the
    visibility samples, NaN for part 0 or without the check))."""
    hm = np.asarray(hm, np.float64)
    B, J, S = hm.shape[:3]
    h = (10.0 * hm).reshape(B, J, -1)
    e = np.exp(h - h.max(2, keepdims=True))
    p = (e / e.sum(2, keepdims=True)).reshape(B, J, S, S)
    ar = np.arange(S, dtype=np.float64)
    c = np.stack([(p.sum(2) * ar).sum(2), (p.sum(3) * ar).sum(2)], -1) / (0.5 * S) - 1.0
    if center_noise is not None:
        c = c + center_jitter * (np.asarray(center_noise, np.float64) - 0.5)
    box = c.max(1) - c.min(1)
    scale_box = box.max(1) / 2.0
    amax = np.argmax(np.asarray(index_pred), axis=1)             # first maximum, like torch.argmax
    Si = amax.shape[1]
    scores = np.full((B, 24), np.nan)
    th = np.zeros((B, 24, 2, 3))
    for i in range(24):
        if i == 0:
            s = scale_box.copy()
        else:
            sc = np.linalg.norm(c[:, CHILDREN1[i]] - c[:, i], axis=1) / 2.0
            sp = np.linalg.norm(c[:, PARENTS0[i]] - c[:, i], axis=1) / 2.0
            s = 2.0 * np.maximum(sc, sp)
        s = s * max(float(ratio[i]), 0.0) + max(float(offset[i]), 0.0)
        if scale_noise is not None:
            s = s * (1.0 + scale_jitter * (np.asarray(scale_noise[i, 0], np.float64) - 0.5))
        if i != 0 and vis_score > 0:
            m = np.isin(amax, SMPL2DP[i]).astype(np.float64)
            scores[:, i] = [bilinear(m[b], c[b, i, 0], c[b, i, 1], Si, align_corners) for b in range(B)]
            s = np.where(scores[:, i] < vis_score, 0.8 * scale_box, s)
        if scale_noise is not None:
            s = s * (1.0 + scale_jitter * (np.asarray(scale_noise[i, 1], np.float64) - 0.5))
        th[:, i, 0, 0] = th[:, i, 1, 1] = s
        th[:, i, :, 2] = c[:, i]
    return c, th, scores


def unnormalize(g, S, align_corners):
    return (g + 1.0) * 0.5 * (S - 1) if align_corners else ((g + 1.0) * S - 1.0) * 0.5


def bilinear(plane, gx, gy, S, align_corners):
    """F.grid_sample (bilinear, zeros) of one [S, S] plane at one grid point"""
    ix, iy = unnormalize(gx, S, align_corners), unnormalize(gy, S, align_corners)
    x0, y0 = int(np.floor(ix)), int(np.floor(iy))
    tx, ty = ix - x0, iy - y0
    acc = 0.0
    for dy in (0, 1):
        for dx in (0, 1):
            xx, yy = x0 + dx, y0 + dy
            if 0 <= xx < S and 0 <= yy < S:
                acc += plane[yy, xx] * (tx if dx else 1 - tx) * (ty if dy else 1 - ty)
    return acc


def affine_base(S, align_corners):
    """affine_grid's base coordinates in fp32, rounded like torch's (csrc/stn_common.cuh affine_base)"""
    step = f32(2.0) / f32(S - 1)
    i = np.arange(S)
    lo = f32(-1.0) + step * i.astype(f32)
    hi = f32(1.0) - step * (S - 1 - i).astype(f32)
    v = np.where(i < S // 2, lo, hi).astype(f32)
    if not align_corners:
        v = (v * f32(S - 1)) / f32(S)
    return v.astype(f32)


def crop_coords(S, s, c, align_corners):
    """fp32 source coordinates of the S crop pixels along one axis (scale s, centre c), every product and sum rounded
    on its own: the kernel's crop_coord, bit for bit"""
    g = f32(s) * affine_base(S, align_corners) + f32(c)
    if align_corners:
        return ((g + f32(1.0)) * f32(0.5)) * f32(S - 1)
    return ((g + f32(1.0)) * f32(S) + f32(-1.0)) * f32(0.5)


def crop_taps(S, s, c, align_corners):
    """per crop pixel along one axis: (i0, w0, w1) of the kernel's crop_tap (fp32 weights); i0 = -2: no tap"""
    with np.errstate(invalid="ignore", over="ignore"):
        ix = crop_coords(S, s, c, align_corners)
        f = np.floor(ix)
        ok = (f > -2) & (f < S)
        w1 = np.where(ok, ix - f, 0).astype(f32)
        w0 = np.where(ok, f32(1.0) - w1, 0).astype(f32)
        i0 = np.where(ok, f, -2).astype(np.int64)
    return i0, w0, w1


def part_crops(xd, thetas, align_corners=False, dcrops=None):
    """fp64 forward (and, with dcrops, the adjoint w.r.t. xd) over the kernel's fp32 coordinates and 2-D weights
    fp32(w_x * w_y).  xd [B,C,S,S], thetas [B,24,2,3].  Returns crops [B,24C,S,S], dxd, and the per-element scales
    sum |w x| of the forward and sum |w dcrops| of the backward."""
    xd = np.asarray(xd, np.float64)
    B, C, S = xd.shape[:3]
    th = np.asarray(thetas, np.float32)
    out = np.zeros((B, 24, C, S, S))
    out_abs = np.zeros_like(out)
    g = None if dcrops is None else np.asarray(dcrops, np.float64).reshape(B, 24, C, S, S)
    dxd = None if g is None else np.zeros((B, C, S * S))
    dabs = None if g is None else np.zeros((B, C, S * S))
    for b in range(B):
        flat = xd[b].reshape(C, S * S)
        for i in range(24):
            tx = crop_taps(S, th[b, i, 0, 0], th[b, i, 0, 2], align_corners)
            ty = crop_taps(S, th[b, i, 1, 1], th[b, i, 1, 2], align_corners)
            for dy in (0, 1):
                for dx in (0, 1):
                    yy, wy = ty[0] + dy, ty[1 + dy]
                    xx, wx = tx[0] + dx, tx[1 + dx]
                    W = (wy[:, None] * wx[None, :]).astype(f32).astype(np.float64)          # [py, px]
                    ok = ((yy >= 0) & (yy < S))[:, None] & ((xx >= 0) & (xx < S))[None, :]
                    src = (np.clip(yy, 0, S - 1)[:, None] * S + np.clip(xx, 0, S - 1)[None, :])
                    Wm = np.where(ok, W, 0.0)
                    v = flat[:, src]                                                          # [C, py, px]
                    out[b, i] += Wm * v
                    out_abs[b, i] += np.abs(Wm * v)
                    if g is not None:
                        contrib = (Wm * g[b, i])[:, ok]                                       # [C, taps]
                        np.add.at(dxd[b], (slice(None), src[ok]), contrib)
                        np.add.at(dabs[b], (slice(None), src[ok]), np.abs(contrib))
    shape = (B, C, S, S)
    return (out.reshape(B, 24 * C, S, S), None if g is None else dxd.reshape(shape), out_abs.reshape(B, 24 * C, S, S),
            None if g is None else dabs.reshape(shape))


def hr_fuse(terms, factors, relu=True, dy=None):
    """fp64 relu(sum_j up(t_j)) and, with dy, the term gradients (dy * [y > 0] summed over each f x f block)"""
    y = None
    for t, f in zip(terms, factors):
        u = np.asarray(t, np.float64).repeat(f, 2).repeat(f, 3)
        y = u if y is None else y + u
    if relu:
        y = np.maximum(y, 0.0)
    if dy is None:
        return y
    g = np.asarray(dy, np.float64) * ((y > 0) if relu else 1.0)
    grads = []
    for t, f in zip(terms, factors):
        N, C, h, w = np.shape(t)
        grads.append(g.reshape(N, C, h, f, w, f).sum((3, 5)))
    return y, grads
