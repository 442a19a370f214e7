"""CPU tests: the oracle against the reference-generated golden vectors and against the
size-independent properties of the domain; C-ABI export check (no compute without a GPU)."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import lbs, raster, synth


def test_oracle_geometry_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "geometry.npz"))
    np.testing.assert_allclose(lbs.rot6d_to_rotmat(g["x6"]), g["rot6d"], atol=2e-6)
    np.testing.assert_allclose(lbs.batch_rodrigues_quat(g["aa"]), g["rodrigues_quat"], atol=2e-6)
    p = lbs.perspective_projection(g["pts"], g["rot"], g["tr"], np.float32(5000.), g["ctr"])
    np.testing.assert_allclose(p, g["persp"], rtol=1e-5, atol=1e-2)
    # known answers: identity 6d pattern -> I ; zero axis-angle -> I
    np.testing.assert_allclose(g["rot6d"][0], np.eye(3), atol=1e-7)
    np.testing.assert_allclose(g["rodrigues_quat"][0], np.eye(3), atol=1e-6)


def test_rodrigues_variants_agree_and_are_rotations():
    rng = np.random.default_rng(0)
    aa = rng.normal(0, 0.8, (256, 3))
    a, b = lbs.batch_rodrigues_smplx(aa), lbs.batch_rodrigues_quat(aa)
    np.testing.assert_allclose(a, b, atol=1e-6)
    np.testing.assert_allclose(a @ a.transpose(0, 2, 1), np.tile(np.eye(3), (256, 1, 1)), atol=1e-7)
    np.testing.assert_allclose(np.linalg.det(a), 1.0, atol=1e-7)
    r6 = lbs.rot6d_to_rotmat(rng.normal(0, 1, (256, 6)))
    np.testing.assert_allclose(r6 @ r6.transpose(0, 2, 1), np.tile(np.eye(3), (256, 1, 1)), atol=1e-7)


def test_oracle_iuv_img2map_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "iuvmap.npz"))
    mu, mv, mi, ma = raster.iuv_img2map(g["img"])
    for a, b in ((mu, g["mu"]), (mv, g["mv"]), (mi, g["mi"]), (ma, g["ma"])):
        np.testing.assert_array_equal(a, b)


def test_lbs_rest_pose_properties(smpl_model):
    rng = np.random.default_rng(1)
    B = 3
    betas = rng.normal(0, 1, (B, 10))
    R = np.tile(np.eye(3), (B, 24, 1, 1))
    out = lbs.smpl_forward(smpl_model, betas, R[:, 1:], R[:, :1], pose2rot=False)
    v_shaped = smpl_model["v_template"][None] + np.einsum("bl,mkl->bmk", betas, smpl_model["shapedirs"].astype(np.float64))
    np.testing.assert_allclose(out["vertices"], v_shaped, atol=1e-10)
    J = np.einsum("jv,bvk->bjk", smpl_model["J_regressor"].astype(np.float64), v_shaped)
    np.testing.assert_allclose(out["smpl_joints"], J, atol=1e-10)
    assert out["joints"].shape == (B, 49, 3) and out["joints_J19"].shape == (B, 19, 3)


def test_lbs_global_rotation_commutes(smpl_model):
    rng = np.random.default_rng(2)
    betas = rng.normal(0, 1, (2, 10))
    aa = rng.normal(0, 0.3, (2, 72))
    a = lbs.smpl_forward(smpl_model, betas, aa[:, 3:], aa[:, :3], pose2rot=True)
    Rg = lbs.batch_rodrigues_smplx(np.array([[0.3, -0.2, 0.5], [1.0, 0.1, -0.4]]))
    R = a["rot_mats"].copy()
    R[:, 0] = Rg @ R[:, 0]
    b = lbs.smpl_forward(smpl_model, betas, R[:, 1:], R[:, :1], pose2rot=False)
    # rotating the root rotates everything about the (rest) root joint
    root = a["smpl_joints"][:, :1]
    # root joint position itself is unchanged by the root rotation (G_0 translation = J_0)
    np.testing.assert_allclose(b["smpl_joints"][:, 0], a["smpl_joints"][:, 0], atol=1e-7)
    expect = np.einsum("bij,bvj->bvi", Rg, a["vertices"] - root) + root
    np.testing.assert_allclose(b["vertices"], expect, atol=1e-7)


def test_lbs_fp32_close_to_fp64(smpl_model):
    rng = np.random.default_rng(3)
    betas = rng.normal(0, 1, (4, 10)).astype(np.float32)
    aa = rng.normal(0, 0.3, (4, 72)).astype(np.float32)
    a = lbs.smpl_forward(smpl_model, betas, aa[:, 3:], aa[:, :3], dtype=np.float64)
    b = lbs.smpl_forward(smpl_model, betas, aa[:, 3:], aa[:, :3], dtype=np.float32)
    assert np.abs(a["vertices"] - b["vertices"]).max() < 1e-5
    assert np.abs(a["joints"] - b["joints"]).max() < 1e-5


def test_raster_invariants(smpl_model, dp_mesh):
    rng = np.random.default_rng(4)
    betas = rng.normal(0, 1, (2, 10)).astype(np.float32)
    aa = rng.normal(0, 0.2, (2, 72)).astype(np.float32)
    verts = lbs.smpl_forward(smpl_model, betas, aa[:, 3:], aa[:, :3], dtype=np.float32)["vertices"]
    tex = synth.dp_textures(dp_mesh)
    cam = np.array([[0.9, 0.0, 0.1], [0.44, 0.0, 0.0]], np.float32)
    img, fidx, depth = raster.verts2uvimg(verts, cam, dp_mesh, tex)
    # tz = 2f/(224 s) >= far=100 for s <= 0.4464 -> empty image (SURVEY appendix B.2)
    assert (fidx[1] < 0).all() and (img[1] == 0).all()
    assert (fidx[0] >= 0).sum() > 100
    part = np.round(img[0, 0] * 24)
    vis = fidx[0] >= 0
    np.testing.assert_array_equal(part[vis], dp_mesh["FaceIndices"][fidx[0][vis]])
    assert (part[~vis] == 0).all()
    # vertical flip: mirroring the scene in y flips the rows of the coverage mask
    v2 = verts.copy(); v2[..., 1] *= -1
    cam2 = cam.copy(); cam2[:, 2] *= -1
    # (mirroring flips triangle winding -> everything back-faces; use coverage of the un-mirrored depth instead)
    assert np.isfinite(depth[0][vis]).all() and (depth[0][vis] > 0.1).all() and (depth[0][vis] < 100).all()
    # the texture_size==1 blend perturbs colours but never the recovered part id (iuvmap.py:111 round())
    img1, fidx1, _ = raster.verts2uvimg(verts, cam, dp_mesh, tex, tex_mode=1)
    np.testing.assert_array_equal(fidx1, fidx)
    np.testing.assert_array_equal(np.round(img1[:, 0] * 24), np.round(img[:, 0] * 24))
    assert np.abs(img1 - img).max() < 0.01


def test_c_abi_v5_exports_every_declared_symbol():
    """Header = SIGNATURES = exports, and the network's inference launches are not exported: their entry is the step
    record (danet_net_run_step, network programs)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(root, "danet-densepose2smpl_b200", "libdanet_b200.so")
    if not os.path.exists(so):
        import __graft_entry__
        __graft_entry__.build()
    hdr = open(os.path.join(root, "include", "danet_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(danet_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 30
    lib = ctypes.CDLL(so)
    for name in sorted(declared):
        assert hasattr(lib, name), "libdanet_b200.so does not export %s" % name
    from danet_b200 import _lib
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    for name in ("nchw_to_nhwc", "fuse_sum", "maxpool3x3s2", "iuv_clean_global", "iuv_clean_parts", "stn_params",
                 "stn_sample", "gcn_pose_head", "conv2d"):
        assert not hasattr(lib, "danet_" + name), "libdanet_b200.so still exports danet_%s" % name
    l = _lib.load()
    assert l.danet_version() == 5


def test_product_does_not_import_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "danet-densepose2smpl_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), fn


def test_get_parts_and_iuv_map2img_match_reference_golden():
    """PartRenderer.get_parts (utils/part_utils.py:27-36) and iuv_map2img (utils/iuvmap.py:41-70): host-side
    tensor code of the SURVEY 8f rows, pinned against outputs of the reference functions themselves
    (tests/golden/part_utils.npz, made by `python -m oracle.gen_golden part_utils`)."""
    import os
    import torch
    from danet_b200.part_utils import PartRenderer
    from danet_b200.iuvmap import iuv_map2img
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "part_utils.npz"))
    faces = np.array([[0, 1, 2], [1, 2, 3]])
    pr = PartRenderer(faces=faces, textures=np.zeros((2, 3), np.float32), cube_parts=g["cube"], num_smpl_verts=4)
    out = pr.get_parts(torch.from_numpy(g["parts"]), torch.from_numpy(g["mask"]))
    assert out.dtype == torch.int64
    np.testing.assert_array_equal(out.numpy(), g["out"])
    U, V, I, A = (torch.from_numpy(g[k]) for k in ("U", "V", "I", "A"))
    np.testing.assert_array_equal(iuv_map2img(U, V, I).numpy(), g["img"])
    np.testing.assert_array_equal(iuv_map2img(U, V, I, A).numpy(), g["img_a"])
