"""numpy restatement of the LSP mask and part-segmentation scoring (reference utils/imutils.py:11-44,89-113 `transform`
/ `uncrop`, eval.py:219-266 the metric loop).  TEST INFRASTRUCTURE.

`imresize` restates what `scipy.misc.imresize(arr, size, interp='nearest')` did in scipy <= 1.2 (scipy.misc.pilutil):
`toimage` (a 2-D float array is `bytescale`d from its min..max to 0..255, so a constant float map becomes all 0; a
uint8 array is left as it is), then Pillow's `Image.resize(..., NEAREST)`, then back to an array.  scipy.misc.pilutil
is gone from current scipy, so this is the stand-in: it runs on the installed Pillow, whose nearest-neighbour index
rule (a sequential double recurrence, `v = s/2; idx = (int)v; v += s` with s = in/out) the device tables restate."""
import numpy as np
from PIL import Image


def bytescale(data):
    """scipy.misc.pilutil.bytescale with the defaults toimage passes (cmin/cmax = data min/max, 0..255)."""
    if data.dtype == np.uint8:
        return data
    cmin, cmax = data.min(), data.max()
    cscale = cmax - cmin
    if cscale == 0:
        cscale = 1
    scale = float(255 - 0) / cscale
    bytedata = (data - cmin) * scale + 0
    return (bytedata.clip(0, 255) + 0.5).astype(np.uint8)


def imresize(arr, size, interp="nearest"):
    """scipy.misc.imresize for a 2-D array and a (rows, cols) size, nearest only (what uncrop calls)."""
    assert interp == "nearest" and np.ndim(arr) == 2
    im = Image.fromarray(np.ascontiguousarray(bytescale(np.asarray(arr))))          # 2-D uint8 -> mode 'L'
    return np.asarray(im.resize((int(size[1]), int(size[0])), resample=Image.NEAREST))


def nearest_index(n_out, n_in=224):
    """Pillow's NEAREST source index for each of n_out output pixels along one axis (the recurrence, one add after
    another)."""
    s = float(n_in) / n_out
    v = s * 0.5
    out = np.empty(n_out, np.int64)
    for i in range(n_out):
        out[i] = int(v)
        v += s
    return out


def get_transform(center, scale, res):
    """imutils.py:11-19 (rot = 0)."""
    h = 200 * scale
    t = np.zeros((3, 3))
    t[0, 0] = float(res[1]) / h
    t[1, 1] = float(res[0]) / h
    t[0, 2] = res[1] * (-float(center[0]) / h + .5)
    t[1, 2] = res[0] * (-float(center[1]) / h + .5)
    t[2, 2] = 1
    return t


def transform(pt, center, scale, res, invert=0):
    """imutils.py:37-44 (rot = 0)."""
    t = get_transform(center, scale, res)
    if invert:
        t = np.linalg.inv(t)
    new_pt = np.array([pt[0] - 1, pt[1] - 1, 1.]).T
    new_pt = np.dot(t, new_pt)
    return new_pt[:2].astype(int) + 1


def crop_box(center, scale, res=(224, 224)):
    """ul, br of uncrop (imutils.py:94-97)."""
    ul = np.array(transform([1, 1], center, scale, res, invert=1)) - 1
    br = np.array(transform([res[0] + 1, res[1] + 1], center, scale, res, invert=1)) - 1
    return ul, br


def uncrop(img, center, scale, orig_shape):
    """imutils.py:89-113 (rot = 0), with `imresize` above."""
    res = img.shape[:2]
    ul, br = crop_box(center, scale, res)
    crop_shape = [br[1] - ul[1], br[0] - ul[0]]
    new_img = np.zeros(orig_shape, dtype=np.uint8)
    new_x = max(0, -ul[0]), min(br[0], orig_shape[1]) - ul[0]
    new_y = max(0, -ul[1]), min(br[1], orig_shape[0]) - ul[1]
    old_x = max(0, ul[0]), min(orig_shape[1], br[0])
    old_y = max(0, ul[1]), min(orig_shape[0], br[1])
    img = imresize(img, crop_shape, interp="nearest")
    new_img[old_y[0]:old_y[1], old_x[0]:old_x[1]] = img[new_y[0]:new_y[1], new_x[0]:new_x[1]]
    return new_img


def confusion(pred_mask, gt_mask, pred_parts, gt_parts):
    """Per-image tables the device counts: mask [2,2] (gt > 0, pred > 0) and parts [9,7] (gt rows 0..6, then 255, then
    any other value; pred columns 0..6)."""
    m = np.zeros((2, 2), np.int64)
    np.add.at(m, ((gt_mask > 0).astype(np.int64).ravel(), (pred_mask > 0).astype(np.int64).ravel()), 1)
    g = gt_parts.astype(np.int64).ravel()
    row = np.where(g <= 6, g, np.where(g == 255, 7, 8))
    p = np.zeros((9, 7), np.int64)
    np.add.at(p, (row, pred_parts.astype(np.int64).ravel()), 1)
    return m, p


def score_image(mask224, parts224, center, scale, orig_shape, gt_mask, gt_parts):
    """One image of eval.py:219-266: (mask table, parts table, uncropped mask, uncropped parts).  mask224 is the
    renderer's float32 mask, parts224 its part ids (cast to uint8 as eval.py:250 does)."""
    pm = uncrop(np.asarray(mask224, np.float32), center, scale, orig_shape)
    pp = uncrop(np.asarray(parts224).astype(np.uint8), center, scale, orig_shape)
    m, p = confusion(pm, gt_mask, pp, gt_parts)
    return m, p, pm, pp


def metrics(mask_tables, part_tables, pixel_count):
    """eval.py's running totals from summed tables, in its own float64 arithmetic: accuracy, f1 [2,1], parts_accuracy,
    parts_f1 [7,1], and the two reported means."""
    M = np.asarray(mask_tables, np.int64).reshape(-1, 2, 2).sum(0)
    P = np.asarray(part_tables, np.int64).reshape(-1, 9, 7).sum(0)
    tp, fp, fn = np.zeros((2, 1)), np.zeros((2, 1)), np.zeros((2, 1))
    for c in range(2):
        tp[c] += M[c, c]
        fp[c] += M[1 - c, c]
        fn[c] += M[c, 1 - c]
    ptp, pfp, pfn = np.zeros((7, 1)), np.zeros((7, 1)), np.zeros((7, 1))
    for c in range(7):
        ptp[c] += P[c, c]
        pfp[c] += P[[r for r in (0, 1, 2, 3, 4, 5, 6, 8) if r != c], c].sum()
        pfn[c] += P[c].sum() - P[c, c]
    with np.errstate(divide="ignore", invalid="ignore"):
        f1 = 2 * tp / (2 * tp + fp + fn)
        parts_f1 = 2 * ptp / (2 * ptp + pfp + pfn)
    acc = 0. + (M[0, 0] + M[1, 1])
    pacc = 0. + (np.trace(P) + P[7, 0])
    return {"accuracy": acc / pixel_count, "f1": f1, "f1_mean": f1.mean(), "parts_accuracy": pacc / pixel_count,
            "parts_f1": parts_f1, "parts_f1_mean": parts_f1[[0, 1, 2, 3, 4, 5, 6]].mean()}
