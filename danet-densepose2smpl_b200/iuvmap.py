"""utils/iuvmap.py of the reference, CUDA-backed (csrc/glue.cu, csrc/raster.cu):
iuvmap_clean (:6-38) and iuv_img2map (:103-151, no-roi branch).  iuv_map2img (:41-100) is the
visualisation-only inverse and is composed from torch ops (off the hot path)."""
import torch

from . import _lib


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
