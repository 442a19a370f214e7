"""LSP mask / part scoring and 3DPW ground truth on the CPU: the per-axis index tables and per-pixel uncrop mapping of
csrc/seg_eval.cu compiled for the host (DANET_SEG_HOST_CHECK) against Pillow and against the reference's own uncrop
(tests/golden/lsp_eval.npz, oracle/gen_golden_lsp_eval.py), the host crop corners against the reference's `transform`,
the oracle and the package's metric formulas against the reference loop's totals to the last bit, and the evaluation
loop's host logic (gender selection, table merging, cache validation) with the GPU pass substituted."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import seg_eval as oseg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 224


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "lsp_eval.npz"))


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("seg_host") / "libseg_host.so")
    csrc = os.path.join(ROOT, "danet-densepose2smpl_b200", "csrc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
                           "-DDANET_SEG_HOST_CHECK", "-shared", os.path.join(csrc, "seg_eval.cu"),
                           os.path.join(csrc, "api.cu"), "-o", out])
    lib = ctypes.CDLL(out)
    p = ctypes.c_void_p
    lib.danet_test_seg_table_host.argtypes = [ctypes.c_int32, ctypes.c_int32, p]
    lib.danet_test_seg_uncrop_host.argtypes = [ctypes.c_int32, p, p, p]
    return lib


def _P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def host_table(lib, n):
    out = np.zeros(n, np.int32)
    assert lib.danet_test_seg_table_host(n, R, _P(out)) == 0
    return out


def host_uncrop(lib, map224, center, scale, orig_shape):
    from danet_b200 import seg_eval
    ul, br = seg_eval.crop_box(center, scale, R)
    geom = np.array([ul[0], ul[1], br[1] - ul[1], br[0] - ul[0], orig_shape[0], orig_shape[1], 0, 0], np.int64)
    out = np.zeros(tuple(orig_shape), np.uint8)
    m = np.ascontiguousarray(map224, np.uint8)
    assert lib.danet_test_seg_uncrop_host(R, _P(m), _P(geom), _P(out)) == 0
    return out


def test_index_tables_equal_pillow_nearest_for_every_size(hostlib):
    """The device's recurrence = Pillow's resize(NEAREST) for every output size 1..2500, on both axes."""
    ramp = np.arange(R, dtype=np.uint8)
    row, col = Image.fromarray(ramp[None, :]), Image.fromarray(ramp[:, None])
    for n in range(1, 2501):
        t = host_table(hostlib, n)
        np.testing.assert_array_equal(np.asarray(row.resize((n, 1), resample=Image.NEAREST))[0], t, err_msg="cols n=%d" % n)
        np.testing.assert_array_equal(np.asarray(col.resize((1, n), resample=Image.NEAREST))[:, 0], t, err_msg="rows n=%d" % n)
    # the closed form is not the rule: it disagrees for many sizes (e.g. n = 1287, pixel 643)
    assert host_table(hostlib, 1287)[643] == 111 and int((643 + 0.5) * R / 1287) == 112


def test_crop_corners_equal_reference_transform(gold):
    """ul / br in float64 through np.linalg.inv and truncation, bit for bit with the reference's `transform`."""
    from danet_b200 import seg_eval
    assert (gold["sweep_ul"] < 0).any()
    for c, s, ul, br in zip(gold["sweep_center"], gold["sweep_scale"], gold["sweep_ul"], gold["sweep_br"]):
        u, b = seg_eval.crop_box(c, s, R)
        np.testing.assert_array_equal(u, ul)
        np.testing.assert_array_equal(b, br)


def _cases(gold):
    off = np.concatenate([[0], np.cumsum(gold["orig_shape"].prod(1))])
    for i in range(len(gold["scale"])):
        H, W = gold["orig_shape"][i]
        sl = slice(off[i], off[i + 1])
        yield (i, gold["mask"][i], gold["parts"][i], gold["center"][i], gold["scale"][i], (H, W),
               gold["mask_gt"][sl].reshape(H, W), gold["parts_gt"][sl].reshape(H, W),
               gold["uncrop_mask"][sl].reshape(H, W), gold["uncrop_parts"][sl].reshape(H, W))


def test_oracle_reproduces_reference_loop_exactly(gold):
    """oracle/seg_eval.py: the uncropped maps and every total of eval.py:222-266 (counts, accuracy, F1) to the bit."""
    from danet_b200 import seg_eval
    mt, pt = [], []
    for i, m, p, c, s, shp, gm, gp, um, up in _cases(gold):
        a, b, pm, pp = oseg.score_image(m, p, c, s, shp, gm, gp)
        np.testing.assert_array_equal(pm, um, err_msg="mask %d" % i)
        np.testing.assert_array_equal(pp, up, err_msg="parts %d" % i)
        mt.append(a), pt.append(b)
    assert int(gold["pixel_count"]) == int(gold["parts_pixel_count"]) == int(gold["orig_shape"].prod(1).sum())
    for got in (oseg.metrics(mt, pt, int(gold["pixel_count"])), seg_eval.seg_metrics(mt, pt, int(gold["pixel_count"]))):
        assert got["accuracy"] == gold["accuracy"] / gold["pixel_count"]
        assert got["parts_accuracy"] == gold["parts_accuracy"] / gold["parts_pixel_count"]
        np.testing.assert_array_equal(got["f1"], gold["f1"])
        np.testing.assert_array_equal(got["parts_f1"], gold["parts_f1"])
        assert got["f1_mean"] == gold["f1_mean"] and got["parts_f1_mean"] == gold["parts_f1_mean"]
    M, P = np.sum(mt, 0), np.sum(pt, 0)
    np.testing.assert_array_equal([M[0, 0], M[1, 1]], gold["tp"].ravel())
    np.testing.assert_array_equal(np.diag(P), gold["parts_tp"].ravel())
    assert P[7].sum() > 0 and P[8].sum() > 0                    # the golden holds 255 and other labels
    assert (gold["uncrop_mask"][_slice(gold, 6)] == 0).all()      # the all-covered render scores as empty


def _slice(gold, i):
    off = np.concatenate([[0], np.cumsum(gold["orig_shape"].prod(1))])
    return slice(off[i], off[i + 1])


def test_host_mapping_equals_reference_uncrop(gold, hostlib):
    """The kernel's per-pixel mapping (tables, ul, paste window) walked on the host = the reference's uncrop, over the
    golden's cases and random crops sticking out of ragged images on every side."""
    for i, m, p, c, s, shp, gm, gp, um, up in _cases(gold):
        np.testing.assert_array_equal(host_uncrop(hostlib, p.astype(np.uint8), c, s, shp), up, err_msg="case %d" % i)
        if not m.all():
            np.testing.assert_array_equal(host_uncrop(hostlib, (m > 0).astype(np.uint8) * 255, c, s, shp), um)
    rng = np.random.default_rng(5)
    for k in range(60):
        H, W = rng.integers(20, 500, 2)
        s = rng.uniform(0.05, 4.0)
        c = np.array([rng.uniform(-0.3, 1.3) * W, rng.uniform(-0.3, 1.3) * H], np.float32)
        ul, br = oseg.crop_box(c, s)
        if ul[0] > W or br[0] < 0 or ul[1] > H or br[1] < 0 or (br - ul < 1).any():
            continue                                              # wholly outside: the reference's paste fails
        src = rng.integers(0, 256, (R, R)).astype(np.uint8)
        np.testing.assert_array_equal(host_uncrop(hostlib, src, c, s, (H, W)), oseg.uncrop(src, c, s, (H, W)),
                                      err_msg="random %d" % k)


def test_seg_confusion_symbol_is_exported():
    from danet_b200 import _lib
    so = os.path.join(ROOT, "danet-densepose2smpl_b200", "libdanet_b200.so")
    if not os.path.exists(so):
        import __graft_entry__
        __graft_entry__.build()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "danet_b200.h")).read(), flags=re.S)
    assert re.search(r"\bdanet_seg_confusion\s*\(", hdr)
    assert "danet_seg_confusion" in _lib.SIGNATURES and hasattr(ctypes.CDLL(so), "danet_seg_confusion")


def test_seg_confusion_refuses_host_tensors():
    from danet_b200 import seg_eval
    z = torch.zeros(1, R, R, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA"):
        seg_eval.seg_confusion(z, z, [[0, 0]], [[R, R]], [[R, R]], [0], torch.zeros(R * R, dtype=torch.uint8),
                               torch.zeros(R * R, dtype=torch.uint8))


# -- the evaluation loop's host logic ---------------------------------------------------------------------------------

class _StubSmpl(object):
    """Stands in for a gendered SMPL layer: its 'H36M joints' are the pose's first 51 values times (1 + beta_0), times
    a per-model factor, so the two models' pelvis-centred joints differ."""

    def __init__(self, factor):
        self.factor = factor
        self.last = None

    def __call__(self, betas=None, body_pose=None, global_orient=None, pose2rot=True):
        assert pose2rot                                           # 3DPW's ground truth is axis-angle
        pose = torch.cat([global_orient, body_pose], 1)
        self.last = pose[:, :51].reshape(-1, 17, 3) * (1 + betas[:, :1, None]) * self.factor

    def joints_h36m(self):
        return self.last


def _pose_cache(n, seed):
    rng = np.random.default_rng(seed)
    return {"img": np.zeros((n, 3, 2, 2), np.float32), "pose": rng.normal(size=(n, 72)).astype(np.float32),
            "betas": rng.normal(size=(n, 10)).astype(np.float32), "gender": np.array(([-1, 0, 1] * n)[:n], np.int32)}


def test_3dpw_ground_truth_selects_the_female_model_where_gender_is_1():
    """-1 and 0 keep the male model's mesh, 1 takes the female model's (base_dataset.py:106-111, eval.py:196-206),
    then pelvis-centring and H36M_TO_J14; the loop hands these joints to the MPJPE pass batch by batch."""
    from danet_b200 import constants, eval_h36m
    data = _pose_cache(7, 1)
    seen = []

    def batch_fn(img, gt):
        seen.append(gt.clone())
        return {"mpjpe": gt.norm(dim=-1).mean(-1), "pred_j14": gt.clone()}
    res = eval_h36m.run_evaluation(None, "3dpw", eval_h36m.Cached3DPWDataset(data), batch_size=3, quiet=True,
                                   batch_fn=batch_fn, smpl_male=_StubSmpl(1.0), smpl_female=_StubSmpl(3.0))
    j = data["pose"][:, :51].reshape(-1, 17, 3) * (1 + data["betas"][:, :1, None])
    j = j * np.where(data["gender"] == 1, 3.0, 1.0)[:, None, None]
    want = (j - j[:, :1])[:, constants.H36M_TO_J14]
    assert [g.shape[0] for g in seen] == [3, 3, 1]
    np.testing.assert_allclose(torch.cat(seen).numpy(), want, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(res["mpjpe"], np.linalg.norm(want, axis=-1).mean(-1), rtol=1e-6)
    assert (res["recon_err"] < 1e-6).all()                     # prediction = ground truth in this stub


def test_3dpw_cache_maps_gender_strings_and_validates():
    from danet_b200 import eval_h36m
    d = _pose_cache(3, 3)
    d["gender"] = np.array(["m", "f", "x"])
    assert eval_h36m.Cached3DPWDataset(d).gender.tolist() == [0, 1, 1]
    for k, bad in (("pose", np.zeros((3, 69), np.float32)), ("betas", np.zeros((2, 10), np.float32)),
                   ("gender", np.zeros(4, np.int32))):
        e = dict(_pose_cache(3, 3), **{k: bad})
        with pytest.raises(ValueError):
            eval_h36m.Cached3DPWDataset(e)
    with pytest.raises(ValueError, match="missing"):
        eval_h36m.Cached3DPWDataset({k: v for k, v in _pose_cache(3, 3).items() if k != "betas"})
    with pytest.raises(ValueError, match="smpl_male"):
        eval_h36m.run_evaluation(None, "3dpw", eval_h36m.Cached3DPWDataset(_pose_cache(3, 3)), batch_fn=lambda *a: None)


def _seg_cache(gold):
    n = len(gold["scale"])
    return {"img": np.zeros((n, 3, 2, 2), np.float32), "center": gold["center"], "scale": gold["scale"],
            "orig_shape": gold["orig_shape"], "mask_gt": gold["mask_gt"], "parts_gt": gold["parts_gt"]}


def test_lsp_loop_merges_tables_and_reports_the_reference_numbers(gold):
    """run_evaluation('lsp') with the GPU pass replaced by the oracle: the per-image tables land in sample order across
    ragged batches, and the reported accuracy / F1 equal the reference loop's totals to the bit."""
    from danet_b200 import eval_h36m
    ds = eval_h36m.CachedSegDataset(_seg_cache(gold))
    calls = []

    def batch_fn(img, bt):
        lo = sum(calls)
        calls.append(img.shape[0])
        mt, pt = [], []
        for j in range(img.shape[0]):
            H, W = bt["orig_shape"][j]
            o = bt["gt_offset"][j]
            gm, gp = bt["mask_gt"][o:o + H * W].reshape(H, W), bt["parts_gt"][o:o + H * W].reshape(H, W)
            a, b, _, _ = oseg.score_image(gold["mask"][lo + j], gold["parts"][lo + j], bt["center"][j], bt["scale"][j],
                                          (H, W), gm, gp)
            mt.append(a), pt.append(b)
        return torch.from_numpy(np.stack(mt)), torch.from_numpy(np.stack(pt))
    res = eval_h36m.run_evaluation(None, "lsp", ds, batch_size=3, quiet=True, batch_fn=batch_fn)
    assert calls == [3, 3, 3, 1]
    assert res["mask_conf"].shape == (10, 2, 2) and res["part_conf"].shape == (10, 9, 7)
    assert res["pixel_count"] == int(gold["pixel_count"])
    assert res["accuracy"] == gold["accuracy"] / gold["pixel_count"]
    assert res["parts_accuracy"] == gold["parts_accuracy"] / gold["parts_pixel_count"]
    assert res["f1_mean"] == gold["f1_mean"] and res["parts_f1_mean"] == gold["parts_f1_mean"]
    np.testing.assert_array_equal(res["parts_f1"], gold["parts_f1"])


def test_lsp_cache_validation(gold):
    from danet_b200 import eval_h36m
    good = _seg_cache(gold)
    bads = [dict(good, mask_gt=good["mask_gt"][:-1]),                      # packed size != sum of orig sizes
            dict(good, parts_gt=np.concatenate([good["parts_gt"], [0]]).astype(np.uint8)),
            dict(good, mask_gt=good["mask_gt"].astype(np.int32)),
            dict(good, center=good["center"][:-1]),
            dict(good, scale=good["scale"][:, None]),
            dict(good, orig_shape=good["orig_shape"].astype(np.float64)),
            dict(good, orig_shape=np.where(np.arange(len(good["scale"]))[:, None] == 2, 0, good["orig_shape"])),
            {k: v for k, v in good.items() if k != "parts_gt"}]
    for i, bad in enumerate(bads):
        with pytest.raises(ValueError):
            eval_h36m.CachedSegDataset(bad)
    with pytest.raises(ValueError, match="renderer"):
        eval_h36m.run_evaluation(None, "lsp", eval_h36m.CachedSegDataset(good), quiet=True)
