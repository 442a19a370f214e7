"""fp64 torch test double of the IUV estimator's training ops -- TEST INFRASTRUCTURE (oracle/__init__.py).

danet_b200.estimator.run_estimator / estimator_losses walk the lowered network graph through a table of ops;
TorchEstimatorOps is that table in the inputs' dtype: conv2d and batch_norm from oracle.regressor_train.TorchTrainOps,
hr_fuse as nearest upsampling + sum + ReLU, part_crops as the reference's F.affine_grid + F.grid_sample per part,
part_thetas from oracle.stn_train, the losses and targets from oracle.losses / oracle.iuv_train (numpy fp64, their
gradients handed to autograd).  Driven by the product's own walk in float64 it reproduces the reference's
IUV_Estimator (tests/golden/estimator_train.npz, oracle/gen_golden_estimator.py); the GPU tests then use it as the
oracle at the batch sizes and widths the golden does not cover."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import iuv_train as oiu
from oracle import losses as olo
from oracle import raster as ora
from oracle import stn_train as ost
from oracle.regressor_train import TorchTrainOps

EP = "img2iuv."


def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else (None if t is None else np.asarray(t))


class _NumpyLosses(torch.autograd.Function):
    """losses [K] = fn(*preds as numpy) with fn returning (losses, grads): grads[k][j] = d losses[k] / d preds[j] (an
    array or None); the backward sums them with the incoming gradients."""

    @staticmethod
    def forward(ctx, fn, *preds):
        L, G = fn(*[_np(p) for p in preds])
        ref = preds[0]
        ctx.G = [[None if g is None else torch.as_tensor(g, dtype=ref.dtype, device=ref.device) for g in row] for row in G]
        ctx.n = len(preds)
        return torch.as_tensor(np.asarray(L, np.float64), dtype=ref.dtype, device=ref.device)

    @staticmethod
    def backward(ctx, g):
        out = []
        for j in range(ctx.n):
            acc = None
            for k, row in enumerate(ctx.G):
                if row[j] is not None:
                    acc = row[j] * g[k] if acc is None else acc + row[j] * g[k]
            out.append(acc)
        return (None, *out)


class TorchEstimatorOps(TorchTrainOps):
    """Same interface as the CUDA op table of danet_b200.estimator."""

    @staticmethod
    def hr_fuse(terms, factors, relu=True):
        y = None
        for t, f in zip(terms, factors):
            u = t if f == 1 else t.repeat_interleave(f, 2).repeat_interleave(f, 3)
            y = u if y is None else y + u
        return torch.relu(y) if relu else y

    @staticmethod
    def part_thetas(hm, index_pred, learned_ratio, learned_offset, *, vis_score=0.5, center_noise=None,
                    center_jitter=0.1, scale_noise=None, scale_jitter=0.2):
        c, th, _ = ost.part_thetas(_np(hm), _np(index_pred), _np(learned_ratio), _np(learned_offset), vis_score,
                                   _np(center_noise), center_jitter, _np(scale_noise), scale_jitter)
        f = lambda a: torch.as_tensor(a, dtype=hm.dtype, device=hm.device)
        return f(c), f(th)

    @staticmethod
    def part_crops(xd, thetas):
        outs = []
        for i in range(thetas.shape[1]):
            grid = F.affine_grid(thetas[:, i].detach(), list(xd.shape), align_corners=False)
            outs.append(F.grid_sample(xd, grid, align_corners=False))
        return torch.cat(outs, 1)

    @staticmethod
    def iuv_img2map(img):
        maps = ora.iuv_img2map(_np(img).astype(np.float32))
        return tuple(torch.as_tensor(np.asarray(m), dtype=torch.float64, device=img.device) for m in maps)

    @staticmethod
    def body_uv_losses(u, v, idx, ann, uvia, has_iuv=None):
        has = None if has_iuv is None else _np(has_iuv).astype(bool)
        maps = [_np(m) for m in uvia]

        def fn(u_, v_, i_, a_):
            L, g = olo.body_uv_losses(u_, v_, i_, a_, maps, has)
            return L, [[g["u"], None, None, None], [None, g["v"], None, None], [None, None, g["index"], None],
                       [None, None, None, g["ann"]]]
        L = _NumpyLosses.apply(fn, u, v, idx, ann)
        return L[0], L[1], L[2], L[3]

    @staticmethod
    def dp_uvia_losses(u, v, idx, ann, body_uv_X_points, body_uv_Y_points, body_uv_I_points, body_uv_Ind_points,
                       body_uv_U_points, body_uv_V_points, body_uv_point_weights, body_uv_ann_labels,
                       body_uv_ann_weights=None, has_dp=None):
        pts = [_np(t) for t in (body_uv_X_points, body_uv_Y_points, body_uv_I_points, body_uv_U_points,
                                body_uv_V_points, body_uv_point_weights, body_uv_ann_labels)]
        has = None if has_dp is None else _np(has_dp)

        def fn(u_, v_, i_, a_):
            L, g = oiu.dp_uvia_losses(u_, v_, i_, a_, *pts, has_dp=has)
            return L, [[g["u"], None, None, None], [None, g["v"], None, None], [None, None, g["index"], None],
                       [None, None, None, g["ann"]]]
        L = _NumpyLosses.apply(fn, u, v, idx, ann)
        return L[0], L[1], L[2], L[3]

    @staticmethod
    def stn_kps_losses(hm, kps, kps_weight=1.0, hm_weight=0.0):
        k = _np(kps)
        roi_on, hm_on = kps_weight > 0 and k.shape[2] == 3, hm_weight > 0

        def fn(h):
            roi, stnhm, groi, ghm = oiu.stn_kps_losses(h, k, kps_weight, hm_weight)
            return [roi or 0.0, stnhm or 0.0], [[groi], [ghm]]
        L = _NumpyLosses.apply(fn, hm)
        return (L[0] if roi_on else None), (L[1] if hm_on else None)

    @staticmethod
    def part_iuv_targets(uvia, thetas):
        U, V, I = (_np(m) for m in uvia[:3])
        return torch.as_tensor(oiu.part_iuv_targets(U, V, I, _np(thetas)), dtype=thetas.dtype, device=thetas.device)

    @staticmethod
    def part_iuv_losses(pred, gt, has_iuv=None):
        has = None if has_iuv is None else _np(has_iuv).astype(bool)
        g_ = _np(gt)

        def fn(p):
            L, g = olo.part_iuv_losses(p, g_, has)
            # each part loss k reads only its own group k of a row
            rows = []
            for k in range(3):
                gk = np.zeros_like(g)
                gk[:, :, k] = g[:, :, k]
                rows.append([gk])
            return L, rows
        L = _NumpyLosses.apply(fn, pred)
        return L[0], L[1], L[2]


def keyed_state(width, seed=0, dtype=torch.float64):
    """The keyed state of the IUV estimator (danet_b200.synthetic.keyed_state_dict over the graph's img2iuv.* keys) and
    the graph: what build_synthetic_danet loads, and the golden's weights."""
    from danet_b200 import constants, netgraph, synthetic
    g = netgraph.danet_graph(width)
    template = {k: torch.zeros(s.shape, dtype=torch.long if s.init == "long0" else torch.float32)
                for k, s in g.params.items() if k.startswith(EP)}
    # kept from the template, as DaNet initialises them (the reference's learned_ratio.pkl)
    template[EP + "learned_ratio"] = torch.from_numpy(constants.LEARNED_RATIO.copy()).float()
    template[EP + "learned_offset"] = torch.from_numpy(constants.LEARNED_OFFSET.copy()).float()
    sd = synthetic.keyed_state_dict(template, seed)
    return {k: (v.to(dtype) if v.is_floating_point() else v.clone()) for k, v in sd.items()}, g


def param_keys(state):
    """the trainable tensors of the estimator (every img2iuv.iuv_est.* float tensor but the running statistics)"""
    return [k for k, v in state.items() if k.startswith(EP + "iuv_est.") and v.is_floating_point()
            and not k.endswith(("running_mean", "running_var"))]


def make_image(B, seed, size=224):
    g = torch.Generator().manual_seed(seed)
    f32 = dict(generator=g, dtype=torch.float32)
    low = torch.randn(B, 3, 7, 7, **f32)
    return (F.interpolate(low, size=size, mode="bilinear", align_corners=False) * 2
            + 0.3 * torch.randn(B, 3, size, size, **f32)).contiguous()


def make_targets(B, seed, S=56, npts=196):
    """fp32 numpy targets of one batch: the IUV image [B,3,S,S] (part index / 24, U, V; background rows), key points
    [B,24,3] (weights 0, 1, 2) and the DensePose blobs of datasets/base_dataset.py:228-232"""
    rng = np.random.default_rng(seed)
    part = rng.integers(0, 25, (B, S, S)).astype(np.float32)
    part[:, :6, :] = 0
    img = np.stack([part / 24.0, rng.uniform(0, 1, (B, S, S)), rng.uniform(0, 1, (B, S, S))], 1).astype(np.float32)
    img[:, 1:] *= (part > 0)[:, None]
    kps = np.concatenate([rng.uniform(-0.8, 0.8, (B, 24, 2)), rng.choice([0.0, 1.0, 1.0, 2.0], (B, 24, 1))], 2)
    X, Y = rng.uniform(0, S, (B, npts)), rng.uniform(0, S, (B, npts))
    I = rng.integers(1, 25, (B, npts)).astype(np.float64)
    U, V, W = np.zeros((B, 25, npts)), np.zeros((B, 25, npts)), np.zeros((B, 25, npts))
    for n in range(B):
        for p in range(npts):
            c = int(I[n, p])
            U[n, c, p], V[n, c, p], W[n, c, p] = rng.uniform(), rng.uniform(), 1.0
    f = lambda a: np.asarray(a, np.float32)
    dp = {"body_uv_X_points": f(X), "body_uv_Y_points": f(Y), "body_uv_I_points": f(I),
          "body_uv_Ind_points": f(np.repeat(np.arange(B)[:, None], npts, 1)), "body_uv_U_points": f(U.reshape(B, -1)),
          "body_uv_V_points": f(V.reshape(B, -1)), "body_uv_point_weights": f(W.reshape(B, -1)),
          "body_uv_ann_labels": f(rng.integers(0, 15, (B, S * S))), "body_uv_ann_weights": f(np.ones((B, S * S)))}
    return img, f(kps), dp
