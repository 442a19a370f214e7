"""IUV-branch losses of the training step (SURVEY section 8f-2) with the reference's call surface:

    loss_U, loss_V, loss_IndexUV, loss_segAnn = body_uv_losses(u_pred, v_pred, index_pred, ann_pred, uvia_list, has_iuv)
    loss_pU, loss_pV, loss_pIndexUV           = part_iuv_losses(part_iuv_pred, part_iuv_gt, has_iuv)
    loss_Udp, loss_Vdp, loss_IndexUVdp, loss_segAnndp = dp_uvia_losses(u_pred, v_pred, index_pred, ann_pred,
                                                                       **uvia_dp_gt, has_dp=has_dp)
    loss_roi, loss_stnhm                      = stn_kps_losses(skps_hm_pred, smpl_kps_gt)
    part_iuv_gt                               = part_iuv_targets(uvia_list, thetas)

The last three are iuv_estimator.py:343-419, :137-171 and :217-230 (csrc/iuv_train.cu), forward and backward in one
pass like the first two.

`body_uv_losses` is models/danet/iuv_estimator.py:304-341; `part_iuv_losses` is the loop over the 24 part crops of
iuv_estimator.py:232-255 as one launch.  Forward and backward are ONE fused CUDA pass (csrc/losses.cu,
danet_body_uv_losses): the gradients w.r.t. the predictions are produced with the losses and handed to autograd by a
torch.autograd.Function.  No CPU path.

Deviation from the reference, stated: when no image has IUV ground truth the reference returns `torch.zeros(1)` per
loss after a host synchronisation (`torch.sum(has_iuv) > 0`); here the losses are 0-dim zeros and nothing synchronises
(the count stays on the device)."""
import torch
from torch.autograd.function import once_differentiable

from . import _lib

POINT_REGRESSION_WEIGHTS = 0.5                  # configs/danet_default.yaml:23 (cfg.DANET.POINT_REGRESSION_WEIGHTS)


def _launch(N, C, Cann, HW, pred_stride, map_stride, u, v, idx, ann, U, V, I, A, has, batch_size, point_weight, dev,
            gu, gv, gi, ga):
    """Pointers are integer device addresses (or None); returns losses [4] on `dev`."""
    with torch.cuda.device(dev):
        ws = _lib.workspace(_lib.load().danet_body_uv_losses_workspace_bytes(N, HW), dev)
        losses = torch.empty(4, device=dev)
        _lib.call("body_uv_losses", N, C, Cann, HW, pred_stride, map_stride, *map(_lib.ptr, (u, v, idx, ann, U, V, I, A, has)),
                  float(batch_size), float(point_weight), _lib.ptr(losses), *map(_lib.ptr, (gu, gv, gi, ga)), _lib.ptr(ws),
                  device=dev)
    return losses


def _f32(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def _d(t):
    """integer device address of t (None -> 0): what the launch functions take"""
    return t.data_ptr() if t is not None else 0


def _has_u8(has_iuv, dev, repeat=1):
    if has_iuv is None:
        return None
    h = (has_iuv.to(dev) != 0).to(torch.uint8)
    if repeat > 1:
        h = h.repeat_interleave(repeat)
    return h.contiguous()


class _BodyUvLosses(torch.autograd.Function):
    """losses [4] = (loss_U, loss_V, loss_IndexUV, loss_segAnn); the backward multiplies the gradients the fused pass
    already wrote by the incoming d/d losses[k]."""

    @staticmethod
    def forward(ctx, u, v, idx, ann, U, V, I, A, has, point_weight):
        dev = u.device
        B, C = u.shape[0], u.shape[1]
        HW = u.shape[2] * u.shape[3]
        u_, v_, i_ = _f32(u, dev), _f32(v, dev), _f32(idx, dev)
        U_, V_, I_ = _f32(U, dev), _f32(V, dev), _f32(I, dev)
        a_ = _f32(ann, dev) if ann is not None else None
        A_ = _f32(A, dev) if ann is not None else None
        need = [ctx.needs_input_grad[k] for k in range(4)]
        gu = torch.empty_like(u_) if need[0] else None
        gv = torch.empty_like(v_) if need[1] else None
        gi = torch.empty_like(i_) if need[2] else None
        ga = torch.empty_like(a_) if (ann is not None and need[3]) else None
        losses = _launch(B, C, a_.shape[1] if a_ is not None else 0, HW, 0, 0, _d(u_), _d(v_), _d(i_), _d(a_), _d(U_),
                         _d(V_), _d(I_), _d(A_), _d(has), float(B), point_weight, dev, _d(gu), _d(gv), _d(gi), _d(ga))
        ctx.grads = (gu, gv, gi, ga)
        ctx.dtypes = (u.dtype, v.dtype, idx.dtype, ann.dtype if ann is not None else None)
        return losses

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        out = []
        for k, t in enumerate(ctx.grads):
            out.append(None if t is None else (t * g[k]).to(ctx.dtypes[k]))
        return (*out, None, None, None, None, None, None)


def body_uv_losses(u_pred, v_pred, index_pred, ann_pred, uvia_list, has_iuv=None,
                   point_weight=POINT_REGRESSION_WEIGHTS):
    """models/danet/iuv_estimator.py:304-341.  u/v/index_pred [B,C,S,S]; ann_pred [B,Cann,S,S] or None;
    uvia_list = (Umap, Vmap, Imap, Annmap) as utils/iuvmap.py iuv_img2map returns them; has_iuv [B] or None.
    Returns (loss_U, loss_V, loss_IndexUV, loss_segAnn | None), differentiable w.r.t. the predictions."""
    _lib.require_cuda(u_pred, "u_pred")
    Umap, Vmap, Imap, Annmap = uvia_list
    if u_pred.dim() != 4 or u_pred.shape != v_pred.shape or u_pred.shape != index_pred.shape or u_pred.shape != Imap.shape:
        raise ValueError("body_uv_losses: u/v/index predictions and the target maps must share one [B,C,S,S] shape")
    if ann_pred is not None and (Annmap is None or ann_pred.shape != Annmap.shape):
        raise ValueError("body_uv_losses: ann_pred needs an Annmap of the same shape")
    if has_iuv is not None and has_iuv.shape[0] != u_pred.shape[0]:
        raise ValueError("body_uv_losses: has_iuv must have one entry per image")
    if u_pred.shape[0] == 0 or u_pred.shape[2] * u_pred.shape[3] == 0:      # nothing to sum: zeros that still carry a graph
        z = u_pred.sum() * 0 + v_pred.sum() * 0 + index_pred.sum() * 0
        return z, z, z, (ann_pred.sum() * 0 if ann_pred is not None else None)
    has = _has_u8(has_iuv, u_pred.device)
    L = _BodyUvLosses.apply(u_pred, v_pred, index_pred, ann_pred, Umap, Vmap, Imap, Annmap if ann_pred is not None else None,
                            has, point_weight)
    return L[0], L[1], L[2], (L[3] if ann_pred is not None else None)


class _PartIuvLosses(torch.autograd.Function):
    """The 24 body_uv_losses calls of iuv_estimator.py:232-255 (+ the /24 means) over part_iuv_pred [B,24,3,7,S,S]
    in place: image = (batch, part) row, u / v / index = the three 7-channel groups of a row."""

    @staticmethod
    def forward(ctx, pred, gt, has, point_weight):
        dev = pred.device
        B, P, three, C = pred.shape[:4]
        HW = pred.shape[4] * pred.shape[5]
        p_, g_ = _f32(pred, dev), _f32(gt, dev)
        grad = torch.empty_like(p_) if ctx.needs_input_grad[0] else None
        step = C * HW * 4                                         # bytes between the u, v and index groups of a row
        pb, gb, qb = p_.data_ptr(), g_.data_ptr(), _d(grad)
        q = lambda k: qb + k * step if qb else 0
        losses = _launch(B * P, C, 0, HW, three * C * HW, three * C * HW, pb, pb + step, pb + 2 * step, 0,
                         gb, gb + step, gb + 2 * step, 0, _d(has), float(B * P),
                         point_weight, dev, q(0), q(1), q(2), 0)
        ctx.grad = grad
        ctx.dtype = pred.dtype
        return losses[:3]

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        if ctx.grad is None:
            return None, None, None, None
        return (ctx.grad * g.reshape(1, 1, 3, 1, 1, 1)).to(ctx.dtype), None, None, None


def part_iuv_losses(part_iuv_pred, part_iuv_gt, has_iuv=None, point_weight=POINT_REGRESSION_WEIGHTS):
    """iuv_estimator.py:232-255: part_iuv_pred / part_iuv_gt [B,24,3,7,S,S] (u, v, index groups of the part crops).
    Returns (loss_pU, loss_pV, loss_pIndexUV) = the means over the 24 parts of body_uv_losses per part."""
    _lib.require_cuda(part_iuv_pred, "part_iuv_pred")
    if part_iuv_pred.dim() != 6 or part_iuv_pred.shape[2] != 3 or part_iuv_pred.shape != part_iuv_gt.shape:
        raise ValueError("part_iuv_losses: expected part_iuv_pred and part_iuv_gt of one shape [B,P,3,C,S,S]")
    if has_iuv is not None and has_iuv.shape[0] != part_iuv_pred.shape[0]:
        raise ValueError("part_iuv_losses: has_iuv must have one entry per image")
    if part_iuv_pred.numel() == 0:
        z = part_iuv_pred.sum() * 0
        return z, z, z
    has = _has_u8(has_iuv, part_iuv_pred.device, repeat=part_iuv_pred.shape[1])
    L = _PartIuvLosses.apply(part_iuv_pred, part_iuv_gt, has, point_weight)
    return L[0], L[1], L[2]


# ---------------------------------------------------------------------------------------------------------------------
# DensePose-point losses, STN key-point losses and part-crop IUV targets (csrc/iuv_train.cu)
# ---------------------------------------------------------------------------------------------------------------------
INDEX_WEIGHTS = 2.0                             # configs/danet_default.yaml:19 (cfg.DANET.INDEX_WEIGHTS)
PART_WEIGHTS = 0.3                              # configs/danet_default.yaml:21 (cfg.DANET.PART_WEIGHTS)
STN_KPS_WEIGHTS = 1.0                           # configs/danet_default.yaml:35 (cfg.DANET.STN_KPS_WEIGHTS)
STN_HM_WEIGHTS = 0.0                            # configs/danet_default.yaml:36 (cfg.DANET.STN_HM_WEIGHTS)
NUM_UV_CHANNELS = 25                            # cfg.DANET.NUM_PATCHES + 1


def _dp_launch(N, S, Cann, P, preds, pts, has, align, pw, part_w, index_w, dev, grads):
    """preds / pts / grads: integer device addresses (0 = NULL); returns losses [4] on `dev`."""
    with torch.cuda.device(dev):
        ws = _lib.workspace(_lib.load().danet_dp_uvia_losses_workspace_bytes(N, S * S), dev)
        losses = torch.empty(4, device=dev)
        _lib.call("dp_uvia_losses", N, S, Cann, P, *map(_lib.ptr, preds), *map(_lib.ptr, pts), _lib.ptr(has), align,
                  float(pw), float(part_w), float(index_w), _lib.ptr(losses), *map(_lib.ptr, grads), _lib.ptr(ws),
                  device=dev)
    return losses


def _stn_launch(B, J, S, hm, kps, cols, kps_weight, hm_weight, dev, groi, ghm):
    with torch.cuda.device(dev):
        ws = _lib.workspace(_lib.load().danet_stn_kps_losses_workspace_bytes(B, J), dev)
        losses = torch.empty(2, device=dev)
        _lib.call("stn_kps_losses", B, J, S, _lib.ptr(hm), _lib.ptr(kps), cols, float(kps_weight), float(hm_weight),
                  _lib.ptr(losses), _lib.ptr(groi), _lib.ptr(ghm), _lib.ptr(ws), device=dev)
    return losses


def _part_launch(B, S, C, U, V, I, theta, align, out, dev):
    with torch.cuda.device(dev):
        _lib.call("part_iuv_targets", B, S, C, *map(_lib.ptr, (U, V, I, theta)), align, _lib.ptr(out), device=dev)


def _check_labels(lab, C, sel, what):
    """int64 of a float label truncates toward zero: valid labels are (-1, C).  Only the selected images count, like
    the reference, which indexes them out before its cross_entropy."""
    bad = ~((lab > -1) & (lab < C))                              # NaN is bad too
    if sel is not None:
        bad = bad & sel.reshape(-1, *([1] * (bad.dim() - 1)))
    if bool(bad.any()):
        raise ValueError("dp_uvia_losses: %s labels outside [0, %d)" % (what, C))


class _DpUviaLosses(torch.autograd.Function):
    """losses [4] = (loss_Udp, loss_Vdp, loss_IndexUVdp, loss_segAnndp); each prediction's gradient belongs to one loss
    (u -> loss_Udp, v -> loss_Vdp, index -> loss_IndexUVdp, ann -> loss_segAnndp)."""

    @staticmethod
    def forward(ctx, u, v, idx, ann, pts, has, align, pw, part_w, index_w):
        dev = u.device
        N, S = u.shape[0], u.shape[2]
        u_, v_, i_, a_ = _f32(u, dev), _f32(v, dev), _f32(idx, dev), _f32(ann, dev)
        X, Y, I, Up, Vp, W, A = (_f32(t, dev) for t in pts)
        need = [ctx.needs_input_grad[k] for k in range(4)]
        grads = [torch.empty_like(t) if nd else None for t, nd in zip((u_, v_, i_, a_), need)]
        losses = _dp_launch(N, S, a_.shape[1], X.shape[1], [_d(t) for t in (u_, v_, i_, a_)],
                            [_d(t) for t in (X, Y, I, Up, Vp, W, A)], _d(has), 1 if align else 0, pw, part_w, index_w,
                            dev, [_d(g) for g in grads])
        ctx.grads = grads
        ctx.dtypes = (u.dtype, v.dtype, idx.dtype, ann.dtype)
        return losses

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        out = [None if t is None else (t * g[k]).to(ctx.dtypes[k]) for k, t in enumerate(ctx.grads)]
        return (*out, None, None, None, None, None, None)


def dp_uvia_losses(U_estimated, V_estimated, Index_UV, Ann_Index, body_uv_X_points, body_uv_Y_points, body_uv_I_points,
                   body_uv_Ind_points, body_uv_U_points, body_uv_V_points, body_uv_point_weights, body_uv_ann_labels,
                   body_uv_ann_weights=None, has_dp=None, align_corners=False, point_weight=POINT_REGRESSION_WEIGHTS,
                   part_weight=PART_WEIGHTS, index_weight=INDEX_WEIGHTS, check_labels=True):
    """models/danet/iuv_estimator.py:343-419 with the has_dp selection of :106-121, keyword names = the reference's
    blob names (datasets/base_dataset.py:228-232).  U/V_estimated, Index_UV [N,25,S,S]; Ann_Index [N,Cann,S,S];
    X / Y / I (/ Ind) points [N,P] (P = 196); U / V points and point weights [N,25*P] (patch-major); ann labels [N,S*S].
    `body_uv_Ind_points` and `body_uv_ann_weights` are accepted and unused, as in the reference.  align_corners=False is
    what the reference's grid_sample call means on torch >= 1.3; True reproduces torch 1.1.
    Returns (loss_Udp, loss_Vdp, loss_IndexUVdp, loss_segAnndp), differentiable w.r.t. the four predictions.
    Deviation, stated: has_dp selects images on the device (no host synchronisation, no copies of the selected
    predictions); with no image selected the losses are 0-dim zeros, not the reference's torch.zeros(1).
    check_labels=False skips the host-side label check (a host synchronisation), for callers that must stay off the
    host; a label outside the classes then contributes nothing to the losses and gradients."""
    _lib.require_cuda(U_estimated, "U_estimated")
    u, v, idx, ann = U_estimated, V_estimated, Index_UV, Ann_Index
    if u.dim() != 4 or u.shape[1] != NUM_UV_CHANNELS or u.shape[2] != u.shape[3] or v.shape != u.shape or idx.shape != u.shape:
        raise ValueError("dp_uvia_losses: U/V_estimated and Index_UV must share one [N,25,S,S] shape")
    N, S = u.shape[0], u.shape[2]
    if ann.dim() != 4 or ann.shape[0] != N or ann.shape[2:] != u.shape[2:]:
        raise ValueError("dp_uvia_losses: Ann_Index must be [N,Cann,S,S] like the U/V/index maps")
    if has_dp is not None and has_dp.shape[0] != N:
        raise ValueError("dp_uvia_losses: has_dp must have one entry per image")
    if N == 0:                                   # nothing to sum: zeros that still carry a graph
        z = u.sum() * 0 + v.sum() * 0 + idx.sum() * 0 + ann.sum() * 0
        return z, z, z, z
    X, Y, I = (t.reshape(N, -1) for t in (body_uv_X_points, body_uv_Y_points, body_uv_I_points))
    P = X.shape[1]
    if Y.shape[1] != P or I.shape[1] != P or not 1 <= P <= 256:
        raise ValueError("dp_uvia_losses: X / Y / I points must be [N,P] with 1 <= P <= 256")
    Up, Vp, W = (t.reshape(N, -1) for t in (body_uv_U_points, body_uv_V_points, body_uv_point_weights))
    if Up.shape[1] != NUM_UV_CHANNELS * P or Vp.shape[1] != NUM_UV_CHANNELS * P or W.shape[1] != NUM_UV_CHANNELS * P:
        raise ValueError("dp_uvia_losses: U / V points and point weights must be [N,25*P] (patch-major)")
    A = body_uv_ann_labels.reshape(N, -1)
    if A.shape[1] != S * S:
        raise ValueError("dp_uvia_losses: body_uv_ann_labels must hold S*S labels per image")
    sel = None if has_dp is None else (has_dp.to(u.device) == 1)           # iuv_estimator.py:108
    if check_labels:
        _check_labels(I.to(u.device), NUM_UV_CHANNELS, sel, "I_points")
        _check_labels(A.to(u.device), ann.shape[1], sel, "ann")
    has = None if sel is None else sel.to(torch.uint8).contiguous()
    L = _DpUviaLosses.apply(u, v, idx, ann, (X, Y, I, Up, Vp, W, A), has, bool(align_corners), point_weight, part_weight,
                            index_weight)
    return L[0], L[1], L[2], L[3]


class _StnKpsLosses(torch.autograd.Function):
    """losses [2] = (loss_roi, loss_stnhm); the fused pass writes d loss_roi / d hm and d loss_stnhm / d hm (one
    buffer holding their sum when only one of the losses is on)."""

    @staticmethod
    def forward(ctx, hm, kps, kps_weight, hm_weight):
        dev = hm.device
        B, J, S = hm.shape[0], hm.shape[1], hm.shape[2]
        h_, k_ = _f32(hm, dev), _f32(kps, dev)
        groi = ghm = None
        ctx.which = 0 if kps_weight != 0 else 1                 # the loss a single buffer belongs to
        if ctx.needs_input_grad[0]:
            if kps_weight != 0 and hm_weight != 0:
                groi, ghm = torch.empty_like(h_), torch.empty_like(h_)
            else:
                groi = ghm = torch.empty_like(h_)
        losses = _stn_launch(B, J, S, _d(h_), _d(k_), k_.shape[2], kps_weight, hm_weight, dev, _d(groi), _d(ghm))
        ctx.grads = (groi, ghm)
        ctx.dtype = hm.dtype
        return losses

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        groi, ghm = ctx.grads
        if groi is None:
            return None, None, None, None
        if groi is ghm:                          # one loss on: the other one is a constant zero
            out = groi * g[ctx.which]
        else:
            out = groi * g[0] + ghm * g[1]
        return out.to(ctx.dtype), None, None, None


def stn_kps_losses(skps_hm_pred, smpl_kps_gt, kps_weight=STN_KPS_WEIGHTS, hm_weight=STN_HM_WEIGHTS):
    """iuv_estimator.py:137-171: skps_hm_pred [B,24,S,S], smpl_kps_gt [B,24,2|3] (x, y in [-1, 1], weight column).
    Returns (loss_roi, loss_stnhm); each is None where the reference adds no key: its weight is not positive, or, for
    loss_roi, smpl_kps_gt has no weight column.  The centre jitter of :173-174 comes after the losses and is not part
    of them."""
    _lib.require_cuda(skps_hm_pred, "skps_hm_pred")
    hm, kps = skps_hm_pred, smpl_kps_gt
    if hm.dim() != 4 or hm.shape[2] != hm.shape[3] or hm.shape[1] == 0:
        raise ValueError("stn_kps_losses: skps_hm_pred must be [B,J,S,S]")
    if kps.dim() != 3 or kps.shape[:2] != hm.shape[:2] or kps.shape[2] not in (2, 3):
        raise ValueError("stn_kps_losses: smpl_kps_gt must be [B,J,2] or [B,J,3] with the heat maps' B and J")
    roi_on = kps_weight > 0 and kps.shape[2] == 3
    hm_on = hm_weight > 0
    if not (roi_on or hm_on):
        return None, None
    if hm.shape[0] == 0:
        z = hm.sum() * 0
        return (z if roi_on else None), (z if hm_on else None)
    kw, hw = (float(kps_weight) if roi_on else 0.0), (float(hm_weight) if hm_on else 0.0)
    L = _StnKpsLosses.apply(hm, kps.to(hm.device), kw, hw)
    return (L[0] if roi_on else None), (L[1] if hm_on else None)


def part_iuv_targets(uvia_list, thetas, align_corners=False, size=None):
    """iuv_estimator.py:217-230 with part_iuv_simp :422-445: the part-crop IUV targets part_iuv_losses takes.
    uvia_list = (Umap, Vmap, Imap[, Annmap]) [B,25,S,S] as iuv_img2map returns them (Annmap unused); thetas [B,24,2,3]
    (torch.stack of affine_para's thetas, dim 1).  `size`, when given, is the part prediction's map size: the reference
    resamples the maps by size / S with nearest interpolation, which this implements for a ratio of 1 only.
    Returns part_iuv_gt [B,24,3,7,S,S] (no gradient: the reference detaches it)."""
    Umap, Vmap, Imap = uvia_list[:3]
    _lib.require_cuda(Umap, "Umap")
    if Umap.dim() != 4 or Umap.shape[1] < NUM_UV_CHANNELS or Umap.shape[2] != Umap.shape[3] or \
            Vmap.shape != Umap.shape or Imap.shape != Umap.shape:
        raise ValueError("part_iuv_targets: U / V / I maps must share one [B,25,S,S] shape")
    B, C, S = Umap.shape[0], Umap.shape[1], Umap.shape[2]
    if size is not None and int(size) != S:
        raise ValueError("part_iuv_targets: maps of size %d for %d x %d part crops; only a ratio of 1 is supported"
                         % (S, size, size))
    if S < 2:
        raise ValueError("part_iuv_targets: maps must be at least 2 x 2")
    if tuple(thetas.shape) != (B, 24, 2, 3):
        raise ValueError("part_iuv_targets: thetas must be [B,24,2,3]")
    dev = Umap.device
    out = torch.empty(B, 24, 3, 7, S, S, device=dev)
    if B == 0:
        return out
    U_, V_, I_, t_ = (_f32(t, dev) for t in (Umap, Vmap, Imap, thetas))
    _part_launch(B, S, C, _d(U_), _d(V_), _d(I_), _d(t_), 1 if align_corners else 0, _d(out), dev)
    return out
