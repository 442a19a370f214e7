"""GPU parity: fused SMPL layer (csrc/lbs.cu via the C ABI) vs the CPU oracle.
Tolerance from BASELINE.json north_star: vertices / joints within 1e-4 abs (fp32)."""
import numpy as np
import pytest
import torch

from oracle import lbs, synth

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _inputs(B, seed):
    rng = np.random.default_rng(seed)
    betas = rng.normal(0, 1, (B, 10)).astype(np.float32)
    aa = rng.normal(0, 0.3, (B, 72)).astype(np.float32)
    x6 = rng.normal(0, 1, (B, 24, 6)).astype(np.float32)
    return betas, aa, x6


def _check(out, ref, smpl):
    assert np.abs(out.vertices.cpu().numpy() - ref["vertices"]).max() < TOL
    assert np.abs(out.joints.cpu().numpy() - ref["joints"]).max() < TOL
    assert np.abs(out.smpl_joints.cpu().numpy() - ref["smpl_joints"]).max() < TOL
    assert np.abs(out.joints_J19.cpu().numpy() - ref["joints_J19"]).max() < TOL
    assert np.abs(smpl.joints_h36m().cpu().numpy() - ref["joints_h36m"]).max() < TOL


@pytest.mark.parametrize("B", [1, 4, 7, 64])
def test_smpl_axis_angle(smpl_model, B):
    import danet_b200
    dev = torch.device("cuda:0")
    smpl = danet_b200.SMPL(smpl_model, batch_size=B).to(dev)
    betas, aa, _ = _inputs(B, B)
    out = smpl(betas=torch.from_numpy(betas).to(dev), body_pose=torch.from_numpy(aa[:, 3:]).to(dev),
               global_orient=torch.from_numpy(aa[:, :3]).to(dev), pose2rot=True)
    ref = lbs.smpl_forward(smpl_model, betas, aa[:, 3:], aa[:, :3], pose2rot=True, dtype=np.float64)
    _check(out, ref, smpl)
    assert out.vertices.shape == (B, 6890, 3) and out.joints.shape == (B, 49, 3)


@pytest.mark.parametrize("B", [517, 1100])
def test_smpl_large_batch_tensor_core_route(smpl_model, B):
    """B >= 512: the blend-shape + pose-corrective contraction runs as a split-fp16 exact-mode GEMM on the wgmma
    engine (chunks of 1024 bodies; 517 / 1100 are ragged against the 8-body rows, the 128-row tiles and the chunk),
    followed by the skinning phases.  Same 1e-4 bar; bodies_per_cta = -1 forces the fused fp32 kernel for comparison."""
    import danet_b200
    dev = torch.device("cuda:0")
    smpl = danet_b200.SMPL(smpl_model, batch_size=B).to(dev)
    betas, aa, _ = _inputs(B, B)
    args = dict(betas=torch.from_numpy(betas).to(dev), body_pose=torch.from_numpy(aa[:, 3:]).to(dev),
                global_orient=torch.from_numpy(aa[:, :3]).to(dev), pose2rot=True)
    out = smpl(**args)
    ref = lbs.smpl_forward(smpl_model, betas, aa[:, 3:], aa[:, :3], pose2rot=True, dtype=np.float64)
    _check(out, ref, smpl)
    v_gemm = out.vertices.clone()
    out2 = smpl(bodies_per_cta=-1, **args)
    d = (out2.vertices - v_gemm).abs().max().item()
    print("GEMM route vs fused fp32 kernel: max |dv| = %.3e; vs fp64 oracle: %.3e" %
          (d, np.abs(v_gemm.cpu().numpy() - ref["vertices"]).max()))
    assert d < 2e-5


@pytest.mark.parametrize("nb", [1, 2, 4, 8, 16])
def test_smpl_rotmat_all_body_blockings(smpl_model, nb):
    import danet_b200
    dev = torch.device("cuda:0")
    B = 19                                   # ragged against every blocking
    smpl = danet_b200.SMPL(smpl_model).to(dev)
    betas, aa, x6 = _inputs(B, 100 + nb)
    R = lbs.rot6d_to_rotmat(x6.reshape(-1, 6)).reshape(B, 24, 3, 3).astype(np.float32)
    out = smpl(betas=torch.from_numpy(betas).to(dev), body_pose=torch.from_numpy(R[:, 1:]).to(dev),
               global_orient=torch.from_numpy(R[:, :1]).to(dev), pose2rot=False, bodies_per_cta=nb)
    ref = lbs.smpl_forward(smpl_model, betas, R[:, 1:], R[:, :1], pose2rot=False, dtype=np.float64)
    _check(out, ref, smpl)


def test_smpl_rot6d_frontend_and_dense_weights():
    import danet_b200
    dev = torch.device("cuda:0")
    model = synth.make_smpl_model(5, dense_weights=True)     # exercises the dense skinning path
    smpl = danet_b200.SMPL(model).to(dev)
    B = 5
    betas, _, x6 = _inputs(B, 7)
    out = smpl(betas=torch.from_numpy(betas).to(dev), pose6d=torch.from_numpy(x6).to(dev))
    R = lbs.rot6d_to_rotmat(x6.reshape(-1, 6).astype(np.float64)).reshape(B, 24, 3, 3)
    ref = lbs.smpl_forward(model, betas, R[:, 1:], R[:, :1], pose2rot=False, dtype=np.float64)
    _check(out, ref, smpl)


def test_smpl_rest_pose_is_template_plus_shape(smpl_model):
    import danet_b200
    dev = torch.device("cuda:0")
    smpl = danet_b200.SMPL(smpl_model, batch_size=2).to(dev)
    out = smpl()                                               # all defaults -> zeros, like smplx
    np.testing.assert_allclose(out.vertices[0].cpu().numpy(), smpl_model["v_template"], atol=1e-6)
    betas = torch.randn(2, 10, device=dev)
    out = smpl(betas=betas, pose2rot=False)
    vs = smpl_model["v_template"][None] + np.einsum("bl,mkl->bmk", betas.cpu().numpy(), smpl_model["shapedirs"])
    np.testing.assert_allclose(out.vertices.cpu().numpy(), vs, atol=1e-5)


def test_smpl_large_batch_property(smpl_model):
    """Full-size batch: linearity property instead of the (slow) oracle -- with identity pose the
    vertices are affine in beta: v(b1)+v(b2)-v(0) == v(b1+b2)."""
    import danet_b200
    dev = torch.device("cuda:0")
    smpl = danet_b200.SMPL(smpl_model).to(dev)
    B = 4096
    g = torch.Generator(device="cpu").manual_seed(0)
    b1 = torch.randn(B, 10, generator=g).to(dev)
    b2 = torch.randn(B, 10, generator=g).to(dev)
    v = lambda b: smpl(betas=b, pose2rot=False).vertices
    lhs = v(b1) + v(b2) - v(torch.zeros_like(b1))
    assert (lhs - v(b1 + b2)).abs().max().item() < 1e-4


def test_mpjpe_kernel(smpl_model):
    import danet_b200
    from danet_b200.smpl import mpjpe_h36m
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    j17 = rng.normal(0, 0.3, (9, 17, 3)).astype(np.float32)
    gt = rng.normal(0, 0.3, (9, 14, 3)).astype(np.float32)
    got = mpjpe_h36m(torch.from_numpy(j17).to(dev), torch.from_numpy(gt).to(dev)).cpu().numpy()
    np.testing.assert_allclose(got, lbs.mpjpe_h36m(j17.astype(np.float64), gt), atol=1e-6)


def test_smpl_backward_matches_fp64_finite_differences(smpl_model):
    """LBS backward (danet_smpl_backward): dL/dbetas and dL/dR for L = <w_v, vertices> + <w_j, smpl_joints> against
    central finite differences of the fp64 oracle (oracle/lbs.py), every beta and every rotation-matrix entry."""
    import danet_b200
    dev = torch.device("cuda:0")
    B = 2
    rng = np.random.default_rng(42)
    betas = rng.normal(0, 1, (B, 10))
    x6 = rng.normal(0, 1, (B, 24, 6))
    R = lbs.rot6d_to_rotmat(x6.reshape(-1, 6)).reshape(B, 24, 3, 3).astype(np.float64)
    wv = rng.normal(0, 1, (B, 6890, 3))
    wj = rng.normal(0, 1, (B, 24, 3))

    def loss(be, Rm):
        o = lbs.smpl_forward(smpl_model, be, Rm[:, 1:], Rm[:, :1], pose2rot=False, dtype=np.float64)
        return (o["vertices"] * wv).sum() + (o["smpl_joints"] * wj).sum()
    eps = 1e-5
    gb_fd = np.zeros_like(betas)
    for i in range(B):
        for l in range(10):
            bp, bm = betas.copy(), betas.copy()
            bp[i, l] += eps; bm[i, l] -= eps
            gb_fd[i, l] = (loss(bp, R) - loss(bm, R)) / (2 * eps)
    gR_fd = np.zeros_like(R)
    for i in range(B):
        for j in range(24):
            for e in range(9):
                Rp, Rm_ = R.copy(), R.copy()
                Rp[i, j].reshape(-1)[e] += eps; Rm_[i, j].reshape(-1)[e] -= eps
                gR_fd[i, j].reshape(-1)[e] = (loss(betas, Rp) - loss(betas, Rm_)) / (2 * eps)
    smpl = danet_b200.SMPL(smpl_model, batch_size=B).to(dev)
    t = lambda a: torch.from_numpy(a.astype(np.float32)).to(dev)
    gb, gR = smpl.backward_lbs(t(betas), t(R), t(wv), t(wj))
    sb, sR = np.abs(gb_fd).max(), np.abs(gR_fd).max()
    eb = np.abs(gb.cpu().numpy() - gb_fd).max() / sb
    eR = np.abs(gR.cpu().numpy() - gR_fd).max() / sR
    print("LBS backward vs fp64 finite differences: rel err dbeta %.2e dR %.2e" % (eb, eR))
    assert eb < 2e-4 and eR < 2e-4


def _oracle_smpl_losses(model, para, target, target_kps, target_kps3d, target_verts, has_kp3d, has_smpl, w,
                        focal=5000.0, img=224, openpose_weight=0.0, gt_weight=1.0):
    """fp64 numpy restatement of smpl_regressor.py:170-215 + criteria :248-300 (test infrastructure)."""
    B = para.shape[0]
    cam, betas, rot = para[:, :3], para[:, 3:13], para[:, 13:].reshape(B, 24, 3, 3)
    o = lbs.smpl_forward(model, betas, rot[:, 1:], rot[:, :1], pose2rot=False, dtype=np.float64)
    verts, joints = o["vertices"], o["joints"]
    cam_t = np.stack([cam[:, 1], cam[:, 2], 2 * focal / (img * cam[:, 0] + 1e-9)], -1)
    pts = joints + cam_t[:, None]
    kp2d = focal * pts[..., :2] / pts[..., 2:3] / (img / 2.0)
    conf = target_kps[:, :, -1:].copy()
    conf[:, :25] *= openpose_weight
    conf[:, 25:] *= gt_weight
    total = w["keypoints_2d"] * (conf * (kp2d - target_kps[:, :, :-1]) ** 2).mean()
    s3 = has_kp3d.astype(bool)
    gt3, c3 = target_kps3d[s3, :, :3], target_kps3d[s3, :, 3:]
    pj = joints[s3][:, 25:]
    gt3 = gt3 - ((gt3[:, 2] + gt3[:, 3]) / 2)[:, None]
    pj = pj - ((pj[:, 2] + pj[:, 3]) / 2)[:, None]
    total += w["keypoints_3d"] * (c3 * (pj - gt3) ** 2).mean()
    ss = has_smpl.astype(bool)
    total += w["smpl_verts"] * np.abs(verts[ss] - target_verts[ss]).mean()
    total += w["smpl_pose"] * ((rot[ss] - target[ss, 13:].reshape(-1, 24, 3, 3)) ** 2).mean()
    total += w["smpl_betas"] * ((betas[ss] - target[ss, 3:13]) ** 2).mean()
    total += (np.exp(-cam[:, 0] * 10) ** 2).mean()
    return total


def test_differentiable_smpl_and_training_losses_match_fp64_finite_differences(smpl_model):
    """The SMPL branch of the reference's training step (smpl_regressor.py:170-215): losses on top of the differentiable
    SMPL layer (CUDA forward + danet_smpl_backward through a torch.autograd.Function, including the 49-joint selection /
    extra-regressor path); d(total loss)/d(para) against central finite differences of an fp64 restatement."""
    import danet_b200
    from danet_b200.smpl import smpl_losses
    dev = torch.device("cuda:0")
    B = 3
    rng = np.random.default_rng(7)
    x6 = rng.normal(0, 1, (B, 24, 6))
    R = lbs.rot6d_to_rotmat(x6.reshape(-1, 6)).reshape(B, 216)
    para = np.concatenate([np.stack([rng.uniform(0.6, 1.1, B), rng.normal(0, .05, B), rng.normal(0, .05, B)], 1),
                           rng.normal(0, 1, (B, 10)), R + rng.normal(0, 0.02, (B, 216))], 1)
    target = para + rng.normal(0, 0.1, para.shape)
    kps = np.concatenate([rng.uniform(-1, 1, (B, 49, 2)), rng.uniform(0, 1, (B, 49, 1))], -1)
    kps3d = np.concatenate([rng.normal(0, .3, (B, 24, 3)), rng.uniform(0, 1, (B, 24, 1))], -1)
    tverts = rng.normal(0, .5, (B, 6890, 3))
    has3 = np.array([1, 0, 1]); hass = np.array([1, 1, 0])
    w = {"keypoints_2d": 3.0, "keypoints_3d": 300.0, "smpl_pose": 60.0, "smpl_betas": 0.06, "smpl_verts": 60.0}
    smpl = danet_b200.SMPL(smpl_model, batch_size=B).to(dev)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32)).to(dev)
    p = t(para).requires_grad_(True)
    losses = smpl_losses(smpl, p, t(target), t(kps), t(kps3d), t(tverts), t(has3), t(hass), weights=w)
    total = sum(losses.values())
    total.backward()
    g = p.grad.cpu().numpy().astype(np.float64)
    f = lambda pp: _oracle_smpl_losses(smpl_model, pp, target, kps, kps3d, tverts, has3, hass, w)
    want_total = f(para)
    assert abs(total.item() - want_total) / abs(want_total) < 1e-4, (total.item(), want_total)
    idx = [(b, k) for b in range(B) for k in list(range(13)) + list(rng.choice(np.arange(13, 229), 30, replace=False))]
    eps = 1e-5
    fd = np.zeros(len(idx)); got = np.zeros(len(idx))
    for n, (b, k) in enumerate(idx):
        pp, pm = para.copy(), para.copy()
        pp[b, k] += eps; pm[b, k] -= eps
        fd[n] = (f(pp) - f(pm)) / (2 * eps)
        got[n] = g[b, k]
    rel = np.abs(got - fd).max() / np.abs(fd).max()
    print("training-loss gradient vs fp64 finite differences: max rel err %.2e over %d entries" % (rel, len(idx)))
    assert rel < 5e-4
    # plain inference calls are untouched (no autograd graph, same numbers)
    with torch.no_grad():
        o = smpl(betas=p[:, 3:13], body_pose=p[:, 13:].reshape(B, 24, 3, 3)[:, 1:], global_orient=p[:, 13:].reshape(B, 24, 3, 3)[:, :1],
                 pose2rot=False)
    assert not o.vertices.requires_grad
