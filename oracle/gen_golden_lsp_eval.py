"""Generates tests/golden/lsp_eval.npz with the REFERENCE'S OWN LSP scoring code: utils/imutils.py (`transform`,
`uncrop`) imported from the reference tree, and the loop body of eval.py:222-266 (mask and part evaluation) executed as
written, with oracle/seg_eval.py's `imresize` standing in for scipy.misc.imresize (gone from current scipy) and
`cv2.imread` answering from the in-memory ground truth.  Run in this container only:

    python -m oracle.gen_golden_lsp_eval

The cases cover crops inside the image, sticking out on every side, larger and smaller than 224, ground truth with 255
and other out-of-range values, an all-covered mask (bytescale turns it into an empty one) and an empty one."""
import importlib.util
import os
import sys
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
REF = os.environ.get("DANET_REFERENCE", "/root/reference")
R = 224

# (center x, center y, scale, orig rows, orig cols, mask kind); scale * 200 is the crop side in original pixels
CASES = [
    (150.0, 120.0, 1.0, 260, 310, "blob"),        # inside, crop 200 < 224
    (170.3, 160.7, 1.63, 360, 400, "blob"),       # inside, crop 326 > 224
    (12.0, 20.5, 0.9, 200, 240, "blob"),          # sticks out left and top
    (231.0, 190.0, 0.75, 200, 240, "blob"),       # sticks out right and bottom
    (75.0, 60.0, 1.5, 120, 150, "blob"),          # sticks out on every side
    (100.0, 100.0, 0.31, 180, 210, "blob"),       # crop 62 < 224
    (128.4, 97.2, 1.12, 210, 260, "full"),        # every pixel covered -> bytescale -> empty predicted mask
    (140.0, 110.0, 1.05, 230, 280, "empty"),      # nothing covered
    (90.25, 130.75, 1.2345, 250, 190, "blob"),
    (200.0, 112.0, 1.12, 240, 300, "blob"),       # 224 x 224: Pillow copies
]


def _load_imutils():
    sys.path.insert(0, REF)                                        # imutils imports the reference's constants
    try:
        spec = importlib.util.spec_from_file_location("ref_imutils", os.path.join(REF, "utils", "imutils.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path.remove(REF)
    from oracle import seg_eval
    mod.scipy = types.SimpleNamespace(misc=types.SimpleNamespace(imresize=seg_eval.imresize))
    return mod


def _loop_body():
    """eval.py's mask and part evaluation (from `# Mask evaluation` to `# Print intermediate results`), dedented."""
    src = open(os.path.join(REF, "eval.py")).read().split("\n")
    a = next(i for i, l in enumerate(src) if l.strip() == "# Mask evaluation (for LSP)")
    b = next(i for i, l in enumerate(src) if l.strip() == "# Print intermediate results during evaluation")
    return textwrap.dedent("\n".join(src[a:b]))


def _blob_maps(rng, kind):
    yy, xx = np.mgrid[0:R, 0:R]
    cover = np.zeros((R, R), bool)
    for _ in range(5):
        cy, cx = rng.uniform(30, 194, 2)
        ry, rx = rng.uniform(10, 60, 2)
        cover |= ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
    if kind == "full":
        cover[:] = True
    if kind == "empty":
        cover[:] = False
    parts = np.where(cover, (((yy // 17) + (xx // 23) * 3 + rng.integers(0, 7)) % 7), 0).astype(np.int64)
    return cover.astype(np.float32), parts


def _gt_maps(rng, H, W):
    yy, xx = np.mgrid[0:H, 0:W]
    m = np.zeros((H, W), np.uint8)
    p = np.zeros((H, W), np.uint8)
    for _ in range(4):
        cy, cx = rng.uniform(0, H), rng.uniform(0, W)
        ry, rx = rng.uniform(10, H / 2), rng.uniform(10, W / 2)
        inside = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1
        m[inside] = rng.choice([255, 1, 128])
        p[inside] = ((yy[inside] // 13 + xx[inside] // 19) % 7).astype(np.uint8)
    p[rng.random((H, W)) < 0.03] = 255                      # UP-3D's "ignore" label
    p[rng.random((H, W)) < 0.01] = rng.choice([7, 100, 254])  # values no class owns
    p[:3, :] = 255
    return m, p


def main():
    import torch
    sys.path.insert(0, ROOT)
    imutils = _load_imutils()
    rng = np.random.default_rng(20240611)
    masks, parts, centers, scales, shapes, gm, gp, um, up = [], [], [], [], [], [], [], [], []
    for (cx, cy, s, H, W, kind) in CASES:
        m, p = _blob_maps(rng, kind)
        g1, g2 = _gt_maps(rng, H, W)
        masks.append(m), parts.append(p), centers.append([cx, cy]), scales.append(s), shapes.append([H, W])
        gm.append(g1), gp.append(g2)
    center = np.array(centers, np.float32)
    scale = np.array(scales, np.float64)
    orig_shape = np.array(shapes, np.int64)
    names = ["%02d.png" % i for i in range(len(CASES))]
    gt = {("m" + n): a for n, a in zip(names, gm)}
    gt.update({("p" + n): a for n, a in zip(names, gp)})
    cv2 = types.SimpleNamespace(imread=lambda path, flag: gt[os.path.basename(path)].copy())
    ns = {"np": np, "os": os, "cv2": cv2, "uncrop": imutils.uncrop, "eval_masks": True, "eval_parts": True,
          "annot_path": "", "curr_batch_size": len(CASES), "mask": torch.from_numpy(np.stack(masks)),
          "parts": torch.from_numpy(np.stack(parts)),
          "batch": {"center": torch.from_numpy(center), "scale": torch.from_numpy(scale),
                    "orig_shape": torch.from_numpy(orig_shape), "maskname": ["m" + n for n in names],
                    "partname": ["p" + n for n in names]},
          "accuracy": 0., "parts_accuracy": 0., "pixel_count": 0, "parts_pixel_count": 0,
          "tp": np.zeros((2, 1)), "fp": np.zeros((2, 1)), "fn": np.zeros((2, 1)),
          "parts_tp": np.zeros((7, 1)), "parts_fp": np.zeros((7, 1)), "parts_fn": np.zeros((7, 1))}
    exec(compile(_loop_body(), "eval.py:222-266", "exec"), ns)
    for i in range(len(CASES)):                                 # the uncropped maps of the same calls
        um.append(imutils.uncrop(masks[i], center[i], scale[i], orig_shape[i]))
        up.append(imutils.uncrop(parts[i].astype(np.uint8), center[i], scale[i], orig_shape[i]))
    # ul / br of `transform` over random centres and scales (negative ul included)
    sw_center = np.concatenate([rng.uniform(-80, 700, (400, 2)), rng.uniform(0, 50, (100, 2))]).astype(np.float32)
    sw_scale = np.concatenate([rng.uniform(0.2, 6.0, 400), rng.uniform(0.5, 2.0, 100)]).astype(np.float64)
    sw_ul = np.stack([np.array(imutils.transform([1, 1], c, s, (R, R), invert=1)) - 1 for c, s in zip(sw_center, sw_scale)])
    sw_br = np.stack([np.array(imutils.transform([R + 1, R + 1], c, s, (R, R), invert=1)) - 1
                      for c, s in zip(sw_center, sw_scale)])
    assert (sw_ul < 0).any()
    flat = lambda arrs: np.concatenate([a.ravel() for a in arrs])
    out = {"mask": np.stack(masks), "parts": np.stack(parts), "center": center, "scale": scale, "orig_shape": orig_shape,
           "mask_gt": flat(gm), "parts_gt": flat(gp), "uncrop_mask": flat(um), "uncrop_parts": flat(up),
           "accuracy": np.float64(ns["accuracy"]), "pixel_count": np.int64(ns["pixel_count"]),
           "tp": ns["tp"], "fp": ns["fp"], "fn": ns["fn"], "f1": ns["f1"], "f1_mean": np.float64(ns["f1"].mean()),
           "parts_accuracy": np.float64(ns["parts_accuracy"]), "parts_pixel_count": np.int64(ns["parts_pixel_count"]),
           "parts_tp": ns["parts_tp"], "parts_fp": ns["parts_fp"], "parts_fn": ns["parts_fn"], "parts_f1": ns["parts_f1"],
           "parts_f1_mean": np.float64(ns["parts_f1"][[0, 1, 2, 3, 4, 5, 6]].mean()),
           "sweep_center": sw_center, "sweep_scale": sw_scale, "sweep_ul": sw_ul, "sweep_br": sw_br}
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "lsp_eval.npz"), **out)
    print("lsp_eval.npz written: %d images, %d pixels" % (len(CASES), out["pixel_count"]))


if __name__ == "__main__":
    main()
