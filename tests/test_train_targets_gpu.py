"""Training targets on the GPU (csrc/targets.cu, danet_b200.targets): geometry.estimate_translation against the
reference's golden and the fp64 bound, prepare_targets stage by stage against oracle/train_targets.py and
oracle/raster.c, the rasteriser's per-image selection, no host synchronisation, CUDA-graph replay, determinism, and the
outputs feeding the existing losses."""
import os

import numpy as np
import pytest
import torch

from oracle import lbs as olbs, raster as oraster, synth, train_targets as ot

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")
T = lambda a, **kw: torch.as_tensor(np.asarray(a), device=DEV, **kw)
U2 = 2.0 ** -24


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "train_targets.npz"))


@pytest.fixture(scope="module")
def net():
    import danet_b200
    return danet_b200.build_synthetic_danet(width=32, seed=0, device=DEV)


def translation_batch(B, seed):
    """B images of 24 .. 2 weighted joints at depths 5 .. 100, some key points outside the image."""
    rng = np.random.default_rng(seed)
    S = rng.normal(0, 0.4, (B, 49, 3))
    t = np.stack([rng.uniform(-0.3, 0.3, B), rng.uniform(-0.3, 0.3, B), rng.uniform(5, 100, B)], 1)
    p = S + t[:, None]
    uv = 5000. * p[..., :2] / p[..., 2:] + 112. + rng.normal(0, 2.0, (B, 49, 2))
    uv[::5] += 250.
    conf = rng.choice([1.0, 0.3, 0.0, 0.8], (B, 49))
    k = rng.integers(2, 25, B)
    for b in range(B):
        conf[b, 25 + k[b]:] = 0.0
        conf[b, 25:25 + k[b]] = np.maximum(conf[b, 25:25 + k[b]], 0.3)
    return S.astype(np.float32), np.concatenate([uv, conf[..., None]], -1).astype(np.float32)


def test_estimate_translation_matches_reference_golden(gold):
    from danet_b200.geometry import estimate_translation
    S, j = gold["et_S"], gold["et_joints_2d"]
    got = estimate_translation(T(S), T(j)).cpu().numpy()
    ref = gold["et_trans_np"]
    assert (np.abs(got - ref) <= ot.translation_bound(S, j, ref)).all()
    assert (got == gold["et_trans"]).mean() > 0.9           # mostly the reference's fp32 bits


@pytest.mark.parametrize("B", [0, 1, 16, 4097])
def test_estimate_translation_bound_and_singular_rows(B):
    from danet_b200.geometry import estimate_translation
    S, j = translation_batch(max(B, 1), seed=B)
    S, j = S[:B], j[:B]
    got = estimate_translation(T(S), T(j))
    assert got.shape == (B, 3) and got.dtype == torch.float32 and got.device == DEV
    if B == 0:
        return
    got = got.cpu().numpy()
    ref = ot.estimate_translation(S, j)
    assert (np.abs(got - ref) <= ot.translation_bound(S, j, ref)).all()
    # zero every confidence of some images: exactly those rows are NaN, the rest keep their bits
    sing = np.arange(B) % 7 == 3
    j2 = j.copy()
    j2[sing, :, 2] = 0.0
    got2 = estimate_translation(T(S), T(j2)).cpu().numpy()
    assert np.isnan(got2[sing]).all() and np.isfinite(got2[~sing]).all()
    np.testing.assert_array_equal(got2[~sing], got[~sing])


def random_inputs(B, seed, model):
    rng = np.random.default_rng(seed)

    def pose(n):
        p = rng.normal(0, 0.25, (n, 72))
        p[:, :3] = [np.pi, 0, 0] + rng.normal(0, 0.1, (n, 3))
        return p.astype(np.float32)
    fit_pose, gt_pose = pose(B), pose(B)
    fit_betas = rng.normal(0, 1.2, (B, 10)).astype(np.float32)
    gt_betas = rng.normal(0, 1.2, (B, 10)).astype(np.float32)
    flags = {k: (rng.random(B) < 0.5).astype(np.uint8) for k in ("has_smpl", "has_dp", "iuv_annotated")}
    J = olbs.smpl_forward(model, gt_betas, gt_pose[:, 3:], gt_pose[:, :3])["joints"]
    t = np.stack([rng.uniform(-0.2, 0.2, B), rng.uniform(-0.2, 0.2, B), rng.uniform(20, 60, B)], 1)
    p = J + t[:, None]
    uv = 5000. * p[..., :2] / p[..., 2:] / 112. + rng.normal(0, 0.02, (B, 49, 2))
    conf = rng.choice([1.0, 0.3, 0.0], (B, 49), p=[0.6, 0.2, 0.2])
    conf[:, 25:30] = 1.0
    kp = np.concatenate([uv, conf[..., None]], -1).astype(np.float32)
    batch = dict(keypoints=kp, pose=gt_pose, betas=gt_betas, smpl_2dkps=rng.uniform(-1, 1, (B, 24, 3)).astype(np.float32),
                 **flags)
    return batch, fit_pose, fit_betas, (rng.random(B) < 0.5).astype(np.uint8)


def to_dev(batch):
    return {k: T(v, dtype=torch.bool) if k == "has_smpl" else T(v) for k, v in batch.items()}


@pytest.mark.parametrize("B", [1, 7, 16, 64])
def test_prepare_targets_against_oracle(net, B):
    from danet_b200 import geometry
    from danet_b200.iuvmap import iuv_img2map
    from danet_b200.targets import prepare_targets
    model, mesh = synth.make_smpl_model(0), synth.make_dp_mesh(0)
    batch, fp, fb, fv = random_inputs(B, 100 + B, model)
    use_fv = B % 2 == 1
    out = prepare_targets(net, to_dev(batch), T(fp), T(fb), fit_valid=T(fv) if use_fv else None)
    o = {k: (v.cpu().numpy() if torch.is_tensor(v) else [m.cpu().numpy() for m in v]) for k, v in out.items()}
    # merge and flags: exactly
    pose, betas, valid, has_iuv = ot.fit_merge(fp, fb, batch["pose"], batch["betas"], batch["has_smpl"],
                                               batch["iuv_annotated"], fv if use_fv else None)
    for k, v in (("opt_pose", pose), ("opt_betas", betas), ("valid_fit", valid), ("has_iuv", has_iuv)):
        np.testing.assert_array_equal(o[k], v, err_msg=k)
    # SMPL outputs within the SMPL suite's tolerances
    ref = olbs.smpl_forward(model, betas, pose[:, 3:], pose[:, :3], pose2rot=True)
    assert np.abs(o["target_verts"] - ref["vertices"]).max() < 1e-4
    assert np.abs(o["opt_joints"] - ref["joints"]).max() < 1e-4
    # the translation on the device's joints: the fp64 bound
    kpd = ot.denormalise(batch["keypoints"])
    t_ref = ot.estimate_translation(o["opt_joints"], kpd)
    assert (np.abs(o["opt_cam_t"] - t_ref) <= ot.translation_bound(o["opt_joints"], kpd, t_ref)).all()
    np.testing.assert_array_equal(o["opt_cam_t"], geometry.estimate_translation(
        out["opt_joints"], T(kpd)).cpu().numpy())
    # target_cam, target_smpl_kps, target on the device's translation and joints, fp64: a stated fp32 bound
    sj = olbs.smpl_forward(model, betas, pose[:, 3:], pose[:, :3], pose2rot=True)["smpl_joints"].astype(np.float32)
    c = ot.cam_targets(o["opt_joints"], sj, batch["keypoints"], pose, betas, has_iuv, batch["has_dp"],
                       batch["smpl_2dkps"], cam_t=o["opt_cam_t"])
    # cam: two fp32 roundings (1/t_z, the product); kps: the projection's fp32 chain on pixel magnitudes (|u| / 112 + 2)
    assert (np.abs(o["target_cam"] - c["target_cam"]) <= 4 * U2 * np.abs(c["target_cam"])).all()
    kb = 16 * U2 * (np.abs(c["target_smpl_kps"]) + 2)
    assert (np.abs(o["target_smpl_kps"] - c["target_smpl_kps"]) <= kb).all()
    np.testing.assert_array_equal(o["target"][:, 3:13], betas)
    assert np.abs(o["target"][:, 13:] - c["target"][:, 13:]).max() < 4e-6            # fp32 quaternion Rodrigues
    np.testing.assert_array_equal(o["target"][:, 13:], geometry.batch_rodrigues(
        out["opt_pose"].reshape(-1, 3), flavor="quat").reshape(B, 216).cpu().numpy())   # the one rodrigues_quat
    if B >= 7:
        assert not np.array_equal(o["target"][:, 13:], geometry.batch_rodrigues(
            out["opt_pose"].reshape(-1, 3), flavor="smplx").reshape(B, 216).cpu().numpy())
    R = o["target"][:, 13:].reshape(B, 24, 3, 3)
    tj = olbs.smpl_forward(model, o["target"][:, 3:13], R[:, 1:], R[:, :1], pose2rot=False)["smpl_joints"]
    assert np.abs(o["target_smpl_joints"] - tj).max() < 1e-4
    # the render: the face index of oracle/raster.c on selected images, background elsewhere
    sel = has_iuv.astype(bool)
    img, fidx, _ = net.iuv_renderer._render(out["target_verts"], out["target_cam"], want_face_idx=True, select=out["has_iuv"])
    fidx = fidx.cpu().numpy()
    np.testing.assert_array_equal(img.cpu().numpy(), o["uv_image_gt"])
    if sel.any():
        _, rf, _ = oraster.verts2uvimg(o["target_verts"][sel], o["target_cam"][sel], mesh, synth.dp_textures(mesh))
        np.testing.assert_array_equal(fidx[sel], rf)
    assert (fidx[~sel] == -1).all() and (o["uv_image_gt"][~sel] == 0).all()
    maps = net.iuv_renderer.verts2maps(out["target_verts"], out["target_cam"])[1]
    zero = [m.cpu().numpy() for m in iuv_img2map(torch.zeros(1, 3, 56, 56, device=DEV))]
    for k, (m, full) in enumerate(zip(o["uvia_list"], maps)):
        np.testing.assert_array_equal(m[sel], full.cpu().numpy()[sel])
        np.testing.assert_array_equal(m[~sel], np.broadcast_to(zero[k], m[~sel].shape))


def test_unselected_images_with_bad_cameras_are_background(net):
    rng = np.random.default_rng(5)
    betas, aa = rng.normal(0, 1, (4, 10)).astype(np.float32), rng.normal(0, 0.3, (4, 72)).astype(np.float32)
    smpl = net.iuv2smpl.smpl
    verts = smpl(betas=T(betas), body_pose=T(aa[:, 3:]), global_orient=T(aa[:, :3]), pose2rot=True).vertices
    cam = T([[0.9, 0.0, 0.1], [float("nan"), 0.0, 0.0], [-0.8, 0.1, 0.0], [0.8, 0.0, 0.0]], dtype=torch.float32)
    sel = T([1, 0, 0, 1], dtype=torch.uint8)
    r = net.iuv_renderer
    img, fidx, maps = r._render(verts, cam, want_maps=True, want_face_idx=True, select=sel)
    full_img, full_fidx, full_maps = r._render(verts, cam, want_maps=True, want_face_idx=True)
    for b in (0, 3):
        assert torch.equal(img[b], full_img[b]) and torch.equal(fidx[b], full_fidx[b])
    for b in (1, 2):                                              # NaN camera, t_z < 0: never rendered
        assert (img[b] == 0).all() and (fidx[b] == -1).all()


def test_select_all_is_bit_identical_to_raster_iuv(net):
    r = net.iuv_renderer
    rng = np.random.default_rng(9)
    smpl = net.iuv2smpl.smpl
    B = 6
    aa = rng.normal(0, 0.3, (B, 72)).astype(np.float32)
    verts = smpl(betas=T(rng.normal(0, 1, (B, 10)).astype(np.float32)), body_pose=T(aa[:, 3:]),
                 global_orient=T(aa[:, :3]), pose2rot=True).vertices
    cam = T(np.stack([rng.uniform(0.7, 1.0, B), rng.uniform(-0.1, 0.1, B), rng.uniform(-0.1, 0.1, B)], 1).astype(np.float32))
    a = r._render(verts, cam, want_maps=True, want_face_idx=True)
    b = r._render(verts, cam, want_maps=True, want_face_idx=True, select=torch.ones(B, dtype=torch.uint8, device=DEV))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))


def _inputs(net, B=16, seed=3):
    batch, fp, fb, fv = random_inputs(B, seed, synth.make_smpl_model(0))
    return to_dev(batch), T(fp), T(fb), T(fv)


def test_no_host_sync_graph_replay_and_determinism(net):
    from danet_b200.targets import prepare_targets
    batch, fp, fb, fv = _inputs(net)
    run = lambda: prepare_targets(net, batch, fp, fb, fit_valid=fv)
    e1, e2 = run(), run()
    torch.cuda.synchronize()
    flat = lambda o: [o[k] for k in sorted(o) if k != "uvia_list"] + list(o["uvia_list"])
    assert all(torch.equal(a, b) for a, b in zip(flat(e1), flat(e2)))
    torch.cuda.set_sync_debug_mode("error")
    try:
        run()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = run()
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(flat(cap), flat(e1)))


def test_empty_batch(net):
    from danet_b200.targets import prepare_targets
    z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=DEV)
    batch = {"keypoints": z(0, 49, 3), "pose": z(0, 72), "betas": z(0, 10), "smpl_2dkps": z(0, 24, 3),
             "has_smpl": z(0, dtype=torch.bool), "has_dp": z(0, dtype=torch.uint8), "iuv_annotated": z(0, dtype=torch.uint8)}
    out = prepare_targets(net, batch, z(0, 72), z(0, 10))
    assert out["target"].shape == (0, 229) and out["uv_image_gt"].shape == (0, 3, 56, 56)
    assert [m.shape[1] for m in out["uvia_list"]] == [25, 25, 25, 15]


def test_outputs_feed_the_losses(net):
    from danet_b200 import losses
    from danet_b200.regressor import gcn_head, gcn_head_losses
    from danet_b200.smpl import smpl_losses
    from danet_b200.targets import prepare_targets
    B = 8
    batch, fp, fb, fv = _inputs(net, B=B, seed=21)
    t = prepare_targets(net, batch, fp, fb)
    gen = torch.Generator(device=DEV).manual_seed(1)
    rot = (0.1 * torch.randn(B, 24, 128, generator=gen, device=DEV)).requires_grad_()
    gp = (0.1 * torch.randn(B, 13, generator=gen, device=DEV)).requires_grad_()
    net.train()
    try:
        out = gcn_head(net, rot, gp)
    finally:
        net.eval()
    para = out["para"]
    para.retain_grad()
    L = dict(gcn_head_losses(out, t["target"], t["target_smpl_joints"], batch["has_smpl"]))
    L.update(smpl_losses(net.iuv2smpl.smpl, para, t["target"], batch["keypoints"], torch.zeros(B, 24, 4, device=DEV),
                         t["target_verts"], torch.zeros(B, dtype=torch.uint8, device=DEV), batch["has_smpl"]))
    preds = [torch.randn(B, c, 56, 56, generator=gen, device=DEV).requires_grad_() for c in (25, 25, 25, 15)]
    uv = losses.body_uv_losses(*preds, t["uvia_list"], has_iuv=t["has_iuv"])
    hm = torch.rand(B, 24, 56, 56, generator=gen, device=DEV).requires_grad_()
    roi, stnhm = losses.stn_kps_losses(hm, t["target_smpl_kps"])
    terms = list(L.values()) + [x for x in uv if x is not None] + [x for x in (roi, stnhm) if x is not None]
    total = sum(x.sum() for x in terms)
    assert torch.isfinite(total)
    total.backward()
    assert para.grad is not None and torch.isfinite(para.grad).all() and para.grad.abs().sum() > 0
    assert rot.grad is not None and torch.isfinite(rot.grad).all()
