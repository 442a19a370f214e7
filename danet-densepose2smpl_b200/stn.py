"""The STN part crops of the IUV estimator in training mode, on the GPU (csrc/stn_train.cu):

    from danet_b200.stn import part_crops, part_thetas
    centers, thetas = part_thetas(hm, index_pred, learned_ratio, learned_offset,
                                  center_noise=torch.rand(B, 24, 2, device=dev),     # None: no jitter (eval mode)
                                  scale_noise=torch.rand(24, 2, B, device=dev))
    crops = part_crops(xd, thetas)             # [B, 24 * C, S, S], differentiable w.r.t. xd

part_thetas is iuv_estimator.py:137-140,172-191,262-301: soft-argmax centres of 10 * hm, the centre jitter, part
visibility from the index argmax and affine_para with its two scale jitters.  The noise is passed in, in the
reference's draw order (center_noise [B, 24, 2]; scale_noise [24, 2, B]: per part the draw before and the draw after the
hidden-part override), so a caller that draws it with torch.rand gets the reference's distribution.  It carries no
gradient: the reference detaches the centres and scales.

part_crops is iuv_estimator.py:193-204: 24x F.affine_grid(theta_i.detach(), xd.size()) + F.grid_sample(xd, grid),
concatenated on dim 1.  Inputs are fp32, contiguous NCHW CUDA tensors; anything else raises ValueError (there is no
fall-back to torch).  Nothing synchronises with the host and no float atomics are used: results repeat bit for bit, and
forward + backward can be captured in a CUDA graph."""
import torch
from torch.autograd.function import once_differentiable

from . import _args, _lib

NUM_PARTS = 24


class _PartCrops(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xd, thetas, align):
        dev = xd.device
        B, C, S, _ = xd.shape
        with torch.cuda.device(dev):
            crops = torch.empty(B, NUM_PARTS * C, S, S, dtype=torch.float32, device=dev)
            _lib.call("part_crops_forward", B, C, S, _lib.ptr(xd), _lib.ptr(thetas), int(align), _lib.ptr(crops),
                      device=dev)
        ctx.save_for_backward(thetas)
        ctx.shape, ctx.align = (B, C, S), align
        return crops

    @staticmethod
    @once_differentiable
    def backward(ctx, gcrops):
        if not ctx.needs_input_grad[0]:
            return None, None, None
        (thetas,) = ctx.saved_tensors
        B, C, S = ctx.shape
        dev = thetas.device
        with torch.cuda.device(dev):
            gcrops = gcrops.to(torch.float32).contiguous()
            dxd = torch.empty(B, C, S, S, dtype=torch.float32, device=dev)
            _lib.call("part_crops_backward", B, C, S, _lib.ptr(gcrops), _lib.ptr(thetas), int(ctx.align), _lib.ptr(dxd),
                      device=dev)
        return dxd, None, None


def part_crops(xd, thetas, align_corners=False):
    """The 24 part crops of xd [B, C, S, S] -> [B, 24 * C, S, S] (crop i in channels i * C .. (i + 1) * C - 1),
    bilinear with zero padding, differentiable w.r.t. xd only (theta is a constant, as in the reference).

    thetas [B, 24, 2, 3]: the torch.stack of affine_para's thetas on dim 1 (what part_thetas returns).  The sampler is
    separable: it reads theta[..., 0, 0], [0, 2], [1, 1] and [1, 2].  The off-diagonal entries must be zero and are not
    read (checking them would need a host synchronisation).  Coordinates follow F.affine_grid + F.grid_sample with the
    given align_corners, rounded step by step in fp32 without fused multiply-adds.  Each output is a 4-term fp32 sum
    (within 2^-22 sum |w x| of exact).  The backward is the exact adjoint of the forward as executed, a gather summed
    in double: within 2^-24 |dxd| + 2^-45 sum |w dcrops| of the exact adjoint."""
    where = "danet_b200.stn.part_crops"
    _args.tensor(where, "xd", xd, dim=4)
    _args.cuda(where, [("xd", xd)])
    B, C, S, S2 = xd.shape
    if S != S2 or S < 2 or B < 1 or C < 1:
        raise ValueError("%s: xd must be [B, C, S, S] with S >= 2 (got %s)" % (where, tuple(xd.shape)))
    _args.tensor(where, "thetas", thetas, dim=4)
    _args.cuda(where, [("thetas", thetas)], xd.device)
    if tuple(thetas.shape) != (B, NUM_PARTS, 2, 3):
        raise ValueError("%s: thetas must be [%d, 24, 2, 3] (got %s)" % (where, B, tuple(thetas.shape)))
    return _PartCrops.apply(xd, thetas.detach(), bool(align_corners))


def part_thetas(hm, index_pred, learned_ratio, learned_offset, *, vis_score=0.5, center_noise=None, center_jitter=0.1,
                scale_noise=None, scale_jitter=0.2, align_corners=False):
    """(stn_centers [B, 24, 2], thetas [B, 24, 2, 3]) of iuv_estimator.py:137-140,172-191,262-301, no gradient.

    hm [B, 24, Sh, Sh] (predict_hm), index_pred [B, 25, Si, Si] (predict_uv_index, raw scores), learned_ratio and
    learned_offset [24].  In order: centres = softmax_integral(10 hm) / (0.5 Sh) - 1; + center_jitter *
    (center_noise - 0.5) when center_noise [B, 24, 2] is given; visibility from the jittered centres (the bilinear
    sample of 1[argmax(index_pred) in the part's DensePose set], first maximum on ties, hidden when < vis_score; no
    check when vis_score <= 0); scale_box from the jittered centres; per part scale * relu(ratio) + relu(offset),
    * (1 + scale_jitter (r1 - 0.5)), the hidden override 0.8 scale_box (parts 1..23), * (1 + scale_jitter (r2 - 0.5))
    with (r1, r2) = scale_noise[i, :, b] when scale_noise [24, 2, B] is given.  theta = [[s, 0, cx], [0, s, cy]].
    stn_centers are the jittered centres (the reference's stn_kps_pred)."""
    where = "danet_b200.stn.part_thetas"
    _args.tensor(where, "hm", hm, dim=4)
    _args.cuda(where, [("hm", hm)])
    dev = hm.device
    B, J, Sh, Sh2 = hm.shape
    if J != NUM_PARTS or Sh != Sh2 or B < 1 or Sh < 1:
        raise ValueError("%s: hm must be [B, 24, S, S] (got %s)" % (where, tuple(hm.shape)))
    _args.tensor(where, "index_pred", index_pred, dim=4)
    _args.cuda(where, [("index_pred", index_pred)], dev)
    if index_pred.shape[0] != B or index_pred.shape[1] != 25 or index_pred.shape[2] != index_pred.shape[3] \
            or index_pred.shape[2] < 2:
        raise ValueError("%s: index_pred must be [%d, 25, S, S] with S >= 2 (got %s)"
                         % (where, B, tuple(index_pred.shape)))
    for name, t in (("learned_ratio", learned_ratio), ("learned_offset", learned_offset)):
        _args.tensor(where, name, t, dim=1)
        _args.cuda(where, [(name, t)], dev)
        if t.shape[0] != NUM_PARTS:
            raise ValueError("%s: %s must be [24] (got %s)" % (where, name, tuple(t.shape)))
    vis = _args.number(where, "vis_score", vis_score)
    cj, sj = _args.number(where, "center_jitter", center_jitter), _args.number(where, "scale_jitter", scale_jitter)
    if center_noise is not None:
        _args.tensor(where, "center_noise", center_noise, dim=3)
        _args.cuda(where, [("center_noise", center_noise)], dev)
        if tuple(center_noise.shape) != (B, NUM_PARTS, 2):
            raise ValueError("%s: center_noise must be [%d, 24, 2] (got %s)"
                             % (where, B, tuple(center_noise.shape)))
    if scale_noise is not None:
        _args.tensor(where, "scale_noise", scale_noise, dim=3)
        _args.cuda(where, [("scale_noise", scale_noise)], dev)
        if tuple(scale_noise.shape) != (NUM_PARTS, 2, B):
            raise ValueError("%s: scale_noise must be [24, 2, %d] (got %s)"
                             % (where, B, tuple(scale_noise.shape)))
    with torch.cuda.device(dev):
        centers = torch.empty(B, NUM_PARTS, 2, dtype=torch.float32, device=dev)
        thetas = torch.empty(B, NUM_PARTS, 2, 3, dtype=torch.float32, device=dev)
        _lib.call("part_thetas", B, Sh, index_pred.shape[2], _lib.ptr(hm), _lib.ptr(index_pred), _lib.ptr(learned_ratio),
                  _lib.ptr(learned_offset), vis, _lib.ptr(center_noise), cj, _lib.ptr(scale_noise), sj,
                  int(bool(align_corners)), _lib.ptr(centers), _lib.ptr(thetas), device=dev)
    return centers, thetas
