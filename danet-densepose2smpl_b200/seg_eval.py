"""LSP mask and part-segmentation scoring on the GPU (reference eval.py:219-266 with utils/imutils.py:11-44,89-113).

The reference renders the predicted mesh at 224 x 224 (PartRenderer), copies each map to the host, puts it back into
the original image (`uncrop`: scipy.misc.imresize to the crop size, then a paste) and compares it with the ground-truth
PNGs class by class in numpy.  Here the render stays on the device and one call (csrc/seg_eval.cu,
danet_seg_confusion) counts, per image, a 2 x 2 mask and a 9 x 7 part confusion table at the original size; every number
eval.py prints follows from the summed tables exactly (`seg_metrics`).

Host side, per image: the crop corners `ul` / `br` in float64 with the reference's own expressions (np.linalg.inv of
the crop matrix, then truncation toward zero), four integers that must equal the reference's bit for bit."""
import numpy as np
import torch

from . import _args, _lib

PART_ROWS, PART_COLS = 9, 7            # ground truth 0..6, 255, other  x  prediction 0..6
WHERE = "danet_b200.seg_eval.seg_confusion"


def crop_box(center, scale, res=224):
    """(ul, br) int arrays of uncrop (imutils.py:94-97: `transform(..., invert=1)` of the two corners, rot = 0)."""
    h = 200 * scale                                                    # get_transform, imutils.py:11-19
    t = np.zeros((3, 3))
    t[0, 0] = float(res) / h
    t[1, 1] = float(res) / h
    t[0, 2] = res * (-float(center[0]) / h + .5)
    t[1, 2] = res * (-float(center[1]) / h + .5)
    t[2, 2] = 1
    t = np.linalg.inv(t)
    corner = lambda pt: np.dot(t, np.array([pt - 1, pt - 1, 1.]).T)[:2].astype(int) + 1 - 1   # transform, :37-44
    return corner(1), corner(res + 1)


def _host_ints(where, name, a, shape):
    a = np.asarray(a)
    if a.shape != tuple(shape) or not (np.issubdtype(a.dtype, np.integer)):
        raise ValueError("%s: %s must be an integer array of shape %s (got %s %s)" % (where, name, tuple(shape), a.dtype,
                                                                                     a.shape))
    return a.astype(np.int64)


def seg_confusion(mask, parts, ul, crop_shape, orig_shape, gt_offset, mask_gt, parts_gt):
    """Per-image confusion tables of B rendered maps put back into their original images.
    mask, parts   [B,R,R] uint8 CUDA: the predicted mask (nonzero = covered, as scored) and part ids 0..6
    ul            [B,2] host ints (x, y) and crop_shape [B,2] (rows, cols) = (br - ul) swapped, as uncrop computes them
    orig_shape    [B,2] host ints (rows, cols); gt_offset [B] host ints: each image's start in the packed buffers
    mask_gt, parts_gt  1-D uint8 CUDA: the ground-truth images, row-major, packed
    -> (mask_conf [B,2,2], part_conf [B,9,7]) int64 on the maps' device: pixel counts of (gt > 0, pred > 0) and of
       (gt row: 0..6, 255, other; pred part)."""
    _args.cuda(WHERE, [("mask", mask), ("parts", parts), ("mask_gt", mask_gt), ("parts_gt", parts_gt)])
    if mask.dim() != 3 or mask.shape[1] != mask.shape[2]:
        raise ValueError("%s: mask must be [B,R,R] (got %s)" % (WHERE, tuple(mask.shape)))
    B, R = mask.shape[0], mask.shape[1]
    _args.mask(WHERE, "mask", mask, (B, R, R))
    _args.mask(WHERE, "parts", parts, (B, R, R))
    n_gt = mask_gt.numel()
    _args.mask(WHERE, "mask_gt", mask_gt, (n_gt,))
    _args.mask(WHERE, "parts_gt", parts_gt, (n_gt,))
    if mask.dtype != torch.uint8 or parts.dtype != torch.uint8 or mask_gt.dtype != torch.uint8 or \
            parts_gt.dtype != torch.uint8:
        raise ValueError("%s: mask, parts, mask_gt and parts_gt must be uint8" % WHERE)
    ul = _host_ints(WHERE, "ul", ul, (B, 2))
    crop = _host_ints(WHERE, "crop_shape", crop_shape, (B, 2))
    orig = _host_ints(WHERE, "orig_shape", orig_shape, (B, 2))
    off = _host_ints(WHERE, "gt_offset", gt_offset, (B,))
    npix = orig[:, 0] * orig[:, 1]
    if (crop < 1).any():
        raise ValueError("%s: crop_shape must be positive (got %s)" % (WHERE, crop[(crop < 1).any(1)][0]))
    if (orig < 1).any() or (npix > np.iinfo(np.int32).max).any():
        raise ValueError("%s: orig_shape must be positive with fewer than 2^31 pixels" % WHERE)
    # uncrop's numpy slices agree with "paste where the crop lies" only while the crop overlaps or touches the image;
    # past that the reference's assignment fails, so such a crop is refused here
    far = (ul[:, 0] > orig[:, 1]) | (ul[:, 0] + crop[:, 1] < 0) | (ul[:, 1] > orig[:, 0]) | (ul[:, 1] + crop[:, 0] < 0)
    if far.any():
        raise ValueError("%s: image %d's crop lies wholly outside the image" % (WHERE, int(np.nonzero(far)[0][0])))
    if (off < 0).any() or (off + npix > n_gt).any():
        raise ValueError("%s: the ground-truth images (offsets + orig sizes) exceed the packed buffers of %d bytes"
                         % (WHERE, n_gt))
    dev = mask.device
    tab = crop.sum(1)
    geom = np.stack([ul[:, 0], ul[:, 1], crop[:, 0], crop[:, 1], orig[:, 0], orig[:, 1], off,
                     np.cumsum(tab) - tab], 1).astype(np.int64)
    mask_conf = torch.empty(B, 2, 2, dtype=torch.int64, device=dev)
    part_conf = torch.empty(B, PART_ROWS, PART_COLS, dtype=torch.int64, device=dev)
    if B == 0:
        return mask_conf, part_conf
    with torch.cuda.device(dev):
        g = torch.from_numpy(geom).to(dev)
        tables = torch.empty(max(int(tab.sum()), 1), dtype=torch.int32, device=dev)
        _lib.call("seg_confusion", B, R, _lib.ptr(mask), _lib.ptr(parts), _lib.ptr(g), _lib.ptr(mask_gt),
                  _lib.ptr(parts_gt), int(npix.max()), _lib.ptr(tables), _lib.ptr(mask_conf), _lib.ptr(part_conf),
                  device=dev)
    return mask_conf, part_conf


def check_part_table(renderer):
    """The confusion has a column per part 0..6: the renderer's cube_parts table must map into them (the ids
    part_utils.py:33-35 truncates to an integer)."""
    cube = renderer.cube_parts
    if cube.numel() and not (float(cube.min()) > -1 and float(cube.max()) < PART_COLS):
        raise ValueError("danet_b200.seg_eval: PartRenderer.cube_parts holds part ids outside 0..6")


@torch.no_grad()
def score_renders(mask, parts, center, scale, orig_shape, gt_offset, mask_gt, parts_gt):
    """eval.py:219-266 for one batch after `mask, parts = renderer(vertices, camera)` (mask [B,R,R] float, parts
    [B,R,R] long on the GPU): the crop corners on the host, then seg_confusion.  center [B,2] (float32 in the
    reference's batches), scale [B] (float64), orig_shape [B,2], gt_offset [B] host arrays."""
    B, R = mask.shape[0], mask.shape[1]
    boxes = [crop_box(center[i], scale[i], R) for i in range(B)]
    ul = np.array([u for u, _ in boxes], np.int64).reshape(B, 2)
    br = np.array([b for _, b in boxes], np.int64).reshape(B, 2)
    crop_shape = np.stack([br[:, 1] - ul[:, 1], br[:, 0] - ul[:, 0]], 1)
    # uncrop resizes the float mask with scipy.misc.imresize, whose toimage bytescales it from its min..max to 0..255:
    # a mask that covers every pixel (min == max) comes out all 0, so eval.py scores it as an empty prediction
    pred_mask = (mask > 0) & ~mask.view(B, -1).all(1).view(B, 1, 1)
    return seg_confusion(pred_mask.to(torch.uint8).contiguous(), parts.to(torch.uint8).contiguous(), ul, crop_shape,
                         orig_shape, gt_offset, mask_gt, parts_gt)


def seg_metrics(mask_tables, part_tables, pixel_count):
    """eval.py's reported numbers from per-image tables (any leading shape), in its own float64 arithmetic:
    accuracy, f1 [2,1] and its mean; parts_accuracy, parts_f1 [7,1] and its mean over the 7 classes.
    pixel_count: the total pixels of the original images."""
    M = np.asarray(mask_tables, np.int64).reshape(-1, 2, 2).sum(0)
    P = np.asarray(part_tables, np.int64).reshape(-1, PART_ROWS, PART_COLS).sum(0)
    tp, fp, fn = np.zeros((2, 1)), np.zeros((2, 1)), np.zeros((2, 1))
    for c in range(2):                                 # eval.py:239-244
        tp[c] += M[c, c]
        fp[c] += M[1 - c, c]
        fn[c] += M[c, 1 - c]
    ptp, pfp, pfn = np.zeros((7, 1)), np.zeros((7, 1)), np.zeros((7, 1))
    for c in range(7):                                 # eval.py:254-260: a pixel labelled 255 is nobody's false positive
        ptp[c] += P[c, c]
        pfp[c] += P[[r for r in (0, 1, 2, 3, 4, 5, 6, 8) if r != c], c].sum()
        pfn[c] += P[c].sum() - P[c, c]
    with np.errstate(divide="ignore", invalid="ignore"):
        f1 = 2 * tp / (2 * tp + fp + fn)
        parts_f1 = 2 * ptp / (2 * ptp + pfp + pfn)
    # eval.py:262-264: 255 -> 0 on both sides, then equality (a label past 6 and not 255 matches no prediction)
    acc, pacc = 0. + (M[0, 0] + M[1, 1]), 0. + (np.trace(P) + P[7, 0])
    return {"accuracy": acc / pixel_count, "f1": f1, "f1_mean": f1.mean(), "parts_accuracy": pacc / pixel_count,
            "parts_f1": parts_f1, "parts_f1_mean": parts_f1[[0, 1, 2, 3, 4, 5, 6]].mean()}
