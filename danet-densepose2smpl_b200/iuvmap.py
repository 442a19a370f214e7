"""utils/iuvmap.py of the reference, CUDA-backed (csrc/glue.cu, csrc/raster.cu):
iuvmap_clean (:6-38) and iuv_img2map (:103-151, no-roi branch).  iuv_map2img (:41-100) is the
visualisation-only inverse and is composed from torch ops (off the hot path).

For training, part_drop_clean (csrc/part_drop.cu) is the differentiable join of the estimator and the regressor:
part dropout (models/danet/danet.py:193-205, 247-283) and iuvmap_clean of the global and the part maps."""
import torch
from torch.autograd.function import once_differentiable

from . import _args, _lib, constants

NUM_PARTS = 24
PARTDROP_RATE = 0.3                               # configs/danet_default.yaml:43 (cfg.DANET.PARTDROP_RATE)
_DP2SMPL = torch.tensor(constants.DP2SMPL_MAPPING, dtype=torch.int8).reshape(-1)   # host [24*6]


class _PartDropClean(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u, v, index, ann, parts, drop):
        B, S = u.shape[0], u.shape[-1]
        dev = u.device
        U, V, I, A = (t.detach().contiguous() for t in (u, v, index, ann))
        P = parts.detach()
        outs = [torch.empty_like(t) for t in (U, V, I, A)]
        oP = torch.empty(P.shape, device=dev)
        am_g = torch.empty(B, S * S, dtype=torch.uint8, device=dev)
        am_p = torch.empty(B, NUM_PARTS, S * S, dtype=torch.uint8, device=dev)
        strides = (_lib.c_i64 * 6)(*P.stride())
        with torch.cuda.device(dev):
            _lib.call("part_drop_clean_forward", B, S, A.shape[1], *map(_lib.ptr, (U, V, I, A, P)), strides,
                      _lib.ptr(drop), _lib.ptr(_DP2SMPL), *map(_lib.ptr, outs + [oP, am_g, am_p]),
                      device=dev)
        ctx.save_for_backward(am_g, am_p, drop)
        ctx.mark_non_differentiable(outs[2], outs[3])
        return (*outs, oP)

    @staticmethod
    @once_differentiable
    def backward(ctx, gu, gv, _gi, _ga, gp):
        am_g, am_p, drop = ctx.saved_tensors
        B, S = gu.shape[0], gu.shape[-1]
        dev = gu.device
        gu, gv, gp = (g.contiguous() for g in (gu, gv, gp))
        du, dv, dp = torch.empty_like(gu), torch.empty_like(gv), torch.empty_like(gp)
        with torch.cuda.device(dev):
            _lib.call("part_drop_clean_backward", B, S, _lib.ptr(drop), _lib.ptr(_DP2SMPL),
                      *map(_lib.ptr, (am_g, am_p, gu, gv, gp, du, dv, dp)), device=dev)
        return du, dv, None, None, dp, None


def part_drop_clean(u, v, index, ann, part_iuv_pred, part_drop=None):
    """Part dropout and iuvmap_clean of the IUV estimator's raw outputs, differentiable (danet.py:193-205, 247-283 with
    utils/iuvmap.py:6-38).  u / v / index [B,25,S,S], ann [B,Ca,S,S], part_iuv_pred [B,24,3,7,S,S] (any strides), fp32
    on one CUDA device.  part_drop [B,24] bool on that device (part_drop[b, d-1]: DensePose part d of image b is
    dropped) or None (no dropout, as in eval mode or with PARTDROP_RATE 0).
    Returns (u_cl, v_cl, index_cl, ann_cl, part_iuv_map [B,24,3,7,S,S]), new tensors: the inputs are not modified.
    Gradients reach u, v and the U / V maps of part_iuv_pred, bit for bit what torch autograd gives for the reference's
    expressions; index_cl and ann_cl are one-hots of argmaxes and carry no gradient.  No host synchronisation: the op
    can be captured in a CUDA graph."""
    where = "danet_b200.iuvmap.part_drop_clean"
    _args.tensor(where, "u", u, dim=4, contiguous=False)
    B, C, S = u.shape[0], u.shape[1], u.shape[-1]
    if C != 25 or u.shape[2] != S or B < 1:
        raise ValueError("%s: u must be [B,25,S,S] with B >= 1 (got %s)" % (where, tuple(u.shape)))
    _args.tensor(where, "v", v, shape=u.shape, contiguous=False)
    _args.tensor(where, "index", index, shape=u.shape, contiguous=False)
    _args.tensor(where, "ann", ann, dim=4, contiguous=False)
    if ann.shape[0] != B or tuple(ann.shape[2:]) != (S, S) or not 1 <= ann.shape[1] <= 255:
        raise ValueError("%s: ann must be [%d,Ca,%d,%d] with 1 <= Ca <= 255 (got %s)" % (where, B, S, S,
                                                                                      tuple(ann.shape)))
    _args.tensor(where, "part_iuv_pred", part_iuv_pred, shape=(B, NUM_PARTS, 3, 7, S, S), contiguous=False)
    named = [("u", u), ("v", v), ("index", index), ("ann", ann), ("part_iuv_pred", part_iuv_pred)]
    drop = None
    if part_drop is not None:
        if not isinstance(part_drop, torch.Tensor) or part_drop.dtype != torch.bool:
            raise ValueError("%s: part_drop must be a bool tensor [B,24] or None" % where)
        _args.mask(where, "part_drop", part_drop, (B, NUM_PARTS))
        named.append(("part_drop", part_drop))
        drop = part_drop.view(torch.uint8)
    _args.cuda(where, named)
    return _PartDropClean.apply(u, v, index, ann, part_iuv_pred, drop)


def draw_part_drop(B, rate=PARTDROP_RATE):
    """The reference's dropout draw (danet.py:195-197): torch.rand(24) < rate once per image, in image order, on the
    CPU generator.  Returns a bool tensor [B,24] on the CPU (part_drop_clean's part_drop once moved)."""
    rate = _args.number("danet_b200.iuvmap.draw_part_drop", "rate", rate)
    return torch.stack([torch.rand(NUM_PARTS) < rate for _ in range(B)]) if B > 0 else \
        torch.zeros(0, NUM_PARTS, dtype=torch.bool)


@torch.no_grad()
def iuvmap_clean(U_uv, V_uv, Index_UV, AnnIndex=None):
    _lib.require_cuda(Index_UV, "Index_UV")
    dev = Index_UV.device
    B, C, H, W = Index_UV.shape
    U, V, I = (t.detach().float().contiguous() for t in (U_uv, V_uv, Index_UV))
    A = AnnIndex.detach().float().contiguous() if AnnIndex is not None else None
    oU, oV, oI = torch.empty_like(U), torch.empty_like(V), torch.empty_like(I)
    oA = torch.empty_like(A) if A is not None else None
    with torch.cuda.device(dev):
        _lib.call("iuvmap_clean_nchw", B, C, A.shape[1] if A is not None else 0, H * W,
                  *map(_lib.ptr, (U, V, I, A, oU, oV, oI, oA)))
    return oU, oV, oI, oA


@torch.no_grad()
def iuv_img2map(uvimages, uv_rois=None, new_size=None):
    if uv_rois is not None:
        raise NotImplementedError("iuv_img2map: the roi branch (iuvmap.py:153-208) is unused on the DaNet path")
    _lib.require_cuda(uvimages, "uvimages")
    x = uvimages.detach().float().contiguous()
    B, _, S, S2 = x.shape
    assert S == S2
    outs = [torch.empty(B, c, S, S, device=x.device) for c in (25, 25, 25, 15)]
    with torch.cuda.device(x.device):
        _lib.call("iuv_img2map", B, S, _lib.ptr(x), *map(_lib.ptr, outs))
    return tuple(outs)


@torch.no_grad()
def iuv_map2img(U_uv, V_uv, Index_UV, AnnIndex=None, uv_rois=None, ind_mapping=None):
    """Visualisation helper (demo.py:125,136).  Pure tensor indexing, not a kernel."""
    if uv_rois is not None:
        raise NotImplementedError("iuv_map2img: roi branch unused on the DaNet path")
    K = U_uv.size(1)
    idx = torch.argmax(Index_UV, dim=1)
    if AnnIndex is not None:
        idx = idx * (torch.argmax(AnnIndex, dim=1) > 0).to(torch.int64)
    # the index channel through a K-entry table built on the host with IEEE division / multiplication: torch's CUDA
    # division by a scalar multiplies by the reciprocal, which is one ulp off the reference's CPU result for some k
    if ind_mapping is None:
        full = torch.arange(K, dtype=torch.float32) / float(K - 1)
    else:
        full = torch.arange(K, dtype=torch.float32)
        full[:len(ind_mapping)] = torch.tensor([m * (1. / 24.) for m in ind_mapping], dtype=torch.float32)
    out0 = full.to(idx.device)[idx]
    u = torch.gather(U_uv, 1, idx.unsqueeze(1)).squeeze(1) * (idx > 0)
    v = torch.gather(V_uv, 1, idx.unsqueeze(1)).squeeze(1) * (idx > 0)
    return torch.stack([out0, u, v], dim=1)
