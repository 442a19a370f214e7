"""GPU half of the SMPL forward sweep (tests/smpl_fwd_sweep_common.py): every case's vertices, joints, smpl_joints,
joints_J19, H36M joints and front-end rotations held element by element to the bound against the fp64 reference; the
exact relations the kernels hold by construction (blocking, route, chunk and batch independence, isolation of
non-finite bodies); the argument refusals; and danet_mpjpe_h36m against fp64."""
import ctypes
import functools

import numpy as np
import pytest
import torch

from oracle import lbs as olbs
import fp64_bound as fb
import smpl_fwd_sweep_common as sc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
_WORST = {}


@functools.lru_cache(maxsize=None)
def _smpl(name, h36m=True):
    import danet_b200
    m = sc.model(name)
    return danet_b200.SMPL(m if h36m else sc.without_h36m(m)).to(DEV)


def _smpl_of(case):
    return _smpl(case.model, case.out != "no_h36m")


def _d(t):
    return None if t is None else t.to(DEV)


def _run(smpl, front, inp, nbc):
    """{output: tensor} of one SMPL forward"""
    B = inp.betas.shape[0]
    kw = dict(betas=_d(inp.betas), transl=_d(inp.transl), bodies_per_cta=nbc)
    pose = _d(inp.pose)
    if front == "rotmat":
        kw.update(body_pose=pose[:, 1:], global_orient=pose[:, :1], pose2rot=False)
    elif front == "aa":
        kw.update(body_pose=pose[:, 1:].reshape(B, 69), global_orient=pose[:, 0], pose2rot=True)
    else:
        kw.update(pose6d=pose)
    out = smpl(**kw)
    res = {"verts": out.vertices, "joints": out.joints, "smpl_joints": out.smpl_joints, "joints_J19": out.joints_J19}
    if smpl.joints_h36m() is not None:
        res["joints_h36m"] = smpl.joints_h36m()
    if front != "rotmat":
        res["rotmats"] = smpl.last_rotmats
    return {k: v.clone() for k, v in res.items()}


@pytest.mark.parametrize("case", sc.CASES, ids=sc.case_id)
def test_case_meets_the_bound(case):
    mdl = sc.model(case.model)
    inp = sc.make_inputs(case)
    got = _run(_smpl_of(case), case.front, inp, case.nbc)
    idx = sc.bodies(case)
    ref = sc.reference(case, mdl, sc.subset(inp, idx), device=DEV, with_h36m=case.out != "no_h36m")
    assert set(got) == set(ref)
    fails = []
    for name, (r, M, slack, C) in ref.items():
        g = got[name][idx].reshape(r.shape)
        q, e = fb.worst(g, r, fb.U24 * M, fb.U24 * r.abs() + fb.TINY + slack)[0], fb.err_ratio(g, r, fb.U24 * M)
        key = (sc.skin_path(case), name)
        _WORST[key] = max(_WORST.get(key, -np.inf), q / C)
        print("%s %s: worst |err| / (2^-24 M) = %.3g, beyond the floor and slack %.3g (C = %d)"
              % (sc.case_id(case), name, e, q, C))
        if not q <= C:
            fails.append((name, q, C))
    assert not fails, fails


def test_print_worst_ratio_per_route_and_output():
    """the worst (|error| - floor - slack) / (C 2^-24 M) of the cases above, per skinning path and output"""
    for (path, name), v in sorted(_WORST.items()):
        print("route %-8s %-12s worst error / bound %.3g" % (path, name, v))


# ----------------------------------------------------------------------------------------------------------------------
# exact relations
# ----------------------------------------------------------------------------------------------------------------------
def _equal(a, b, keys=None):
    keys = a.keys() if keys is None else keys
    bad = [k for k in keys if not torch.equal(a[k], b[k])]
    assert not bad, bad


@pytest.mark.parametrize("name,B", [("packed", 1), ("packed", 19), ("dense", 33), ("nv129", 19), ("packed", 511)])
def test_fused_outputs_do_not_depend_on_the_blocking(name, B):
    c = sc.Case(name, B, "rotmat", "typical", "normal", 0, "h36m")
    inp = sc.make_inputs(c, seed=3)
    smpl = _smpl(name)
    want = _run(smpl, "rotmat", inp, 0)
    for nbc in (1, 2, 4, 8, 16, -1):
        _equal(_run(smpl, "rotmat", inp, nbc), want)


@pytest.mark.parametrize("front", ["aa", "r6d"])
def test_pose_outputs_are_identical_on_both_routes(front):
    """smpl_joints and rotmats come from k_smpl_pose on both routes"""
    c = sc.Case("packed", 600, front, "typical", "normal", 0, "h36m")
    inp = sc.make_inputs(c, seed=4)
    smpl = _smpl("packed")
    _equal(_run(smpl, front, inp, 0), _run(smpl, front, inp, -1), ("smpl_joints", "rotmats"))


@pytest.mark.parametrize("name,nbc", [("packed", 0), ("dense", 1), ("nv129", 16)])
def test_gemm_outputs_do_not_depend_on_chunk_or_batch(name, nbc):
    """body k of B = 1100 equals body k of the first 600, and body 500 + k equals body k of bodies 500..1099 (another
    chunk, another place in it, another GEMM row block)"""
    c = sc.Case(name, 1100, "r6d", "typical", "normal", nbc, "h36m")
    inp = sc.make_inputs(c, seed=5)
    smpl = _smpl(name)
    full = _run(smpl, "r6d", inp, nbc)
    for lo in (0, 500):
        part = _run(smpl, "r6d", sc.subset(inp, slice(lo, lo + 600)), nbc)
        _equal({k: v[lo:lo + 600] for k, v in full.items()}, part)


@pytest.mark.parametrize("name,B,nbc", [("packed", 37, 0), ("dense", 21, 16), ("packed", 1030, 0), ("dense", 1030, 1),
                                        ("nv129", 523, 4)])
def test_non_finite_body_leaves_the_others_bit_identical(name, B, nbc):
    """NaN betas, a NaN rotation entry and +-inf in other bodies, among them the batch's last (whose rows the
    partial CTAs repeat) and bodies in the last GEMM chunk, whose row block is padded past B; the workspace is filled
    with NaN before the poisoned run, so the padded rows of the feature planes hold NaN"""
    c = sc.Case(name, B, "rotmat", "typical", "normal", nbc, "h36m")
    inp = sc.make_inputs(c, seed=6)
    smpl = _smpl(name)
    clean = _run(smpl, "rotmat", inp, nbc)
    betas, pose = inp.betas.clone(), inp.pose.clone()
    bad = sorted({0, B // 2, B - 1, B - 3})
    betas[bad[0], 0] = float("nan")
    pose[bad[1], 5, 1, 2] = float("inf")
    betas[bad[2], -1] = -float("inf")
    pose[bad[3], 0, 0, 0] = float("nan")
    smpl._ws[(DEV.index,)].fill_(0xFF)
    got = _run(smpl, "rotmat", sc.Inputs(betas, pose, None), nbc)
    keep = [i for i in range(B) if i not in bad]
    _equal({k: v[keep] for k, v in got.items()}, {k: v[keep] for k, v in clean.items()})
    assert not torch.isfinite(got["verts"][bad]).flatten(1).all(1).any()


# ----------------------------------------------------------------------------------------------------------------------
# argument refusals: they return before anything is launched
# ----------------------------------------------------------------------------------------------------------------------
def _abi_forward(smpl, B, nbc, with_verts=True):
    from danet_b200 import _lib
    lib = _lib.load()
    h = smpl._handle(DEV)
    betas = torch.zeros(B, 10, device=DEV)
    pose = torch.zeros(B, 24, 3, device=DEV)
    nan = lambda *s: torch.full(s, float("nan"), device=DEV)
    verts, joints, sj, jh, rot = nan(B, 6890, 3), nan(B, 49, 3), nan(B, 24, 3), nan(B, 17, 3), nan(B, 24, 3, 3)
    ws = _lib.workspace(lib.danet_smpl_workspace_bytes(h, B), DEV)
    rc = lib.danet_smpl_forward(h, B, _lib.ptr(betas), _lib.ptr(pose), 1, _lib.ptr(verts if with_verts else None),
                                _lib.ptr(joints), _lib.ptr(sj), _lib.ptr(jh), _lib.ptr(rot), _lib.ptr(ws), nbc,
                                _lib.stream_ptr(DEV))
    torch.cuda.synchronize()
    msg = lib.danet_last_error()
    return rc, (msg.decode() if msg else ""), (verts, joints, sj, jh, rot)


@pytest.mark.parametrize("B", [7, 600])
@pytest.mark.parametrize("nbc", [3, 5, 32, -2, -16])
def test_bad_bodies_per_cta_is_refused_on_both_routes(B, nbc):
    rc, msg, outs = _abi_forward(_smpl("packed"), B, nbc)
    assert rc != 0 and "bodies_per_cta" in msg, (rc, msg)
    assert all(torch.isnan(o).all() for o in outs)            # nothing ran, not even the pose kernel
    rc, msg, outs = _abi_forward(_smpl("packed"), B, 0)
    assert rc == 0 and torch.isfinite(outs[0]).all()


@pytest.mark.parametrize("B", [7, 600])
def test_joint_outputs_without_verts_are_refused(B):
    rc, msg, outs = _abi_forward(_smpl("packed"), B, 0, with_verts=False)
    assert rc != 0 and "verts" in msg, (rc, msg)
    assert all(torch.isnan(o).all() for o in outs)


# ----------------------------------------------------------------------------------------------------------------------
# danet_mpjpe_h36m: per sample (1/14) sum_j |(p_j - p_0) - g_j|, against fp64 with the bound
#     |got - r| <= C_MPJPE 2^-24 M + 2^-24 |r| + 2^-149,   M = (1/14) sum_j |D_j|,  D_j = |p_j| + |p_0| + |g_j|
# the differences move each coordinate by 2 units of D (N_DIFF), the three-term sum of squares and sqrtf add 4
# (N_NORM), the 14-term sum and the division 14 (N_MEAN)
# ----------------------------------------------------------------------------------------------------------------------
N_DIFF, N_NORM, N_MEAN = 2, 4, 14
C_MPJPE = N_DIFF + N_NORM + N_MEAN


@pytest.mark.parametrize("regime", ["unit", "far_from_origin", "tiny", "exact_match"])
def test_mpjpe_meets_the_bound(regime):
    from danet_b200.smpl import mpjpe_h36m
    rng = np.random.default_rng(11)
    B = 133
    j17 = rng.normal(0, 0.3, (B, 17, 3))
    gt = rng.normal(0, 0.3, (B, 14, 3))
    if regime == "far_from_origin":                 # p_j - p_0 cancels: 100 m from the origin, 0.3 m apart
        j17 += rng.normal(0, 100, (B, 1, 3))
    elif regime == "tiny":
        j17, gt = j17 * 1e-6, gt * 1e-6
    elif regime == "exact_match":                   # zero error in fp32 arithmetic: the result is exactly 0
        j17 = j17.astype(np.float32).astype(np.float64)
        gt = (j17 - j17[:, :1])[:, olbs.H36M_TO_J14]
    j17, gt = j17.astype(np.float32), gt.astype(np.float32)
    got = mpjpe_h36m(torch.from_numpy(j17).to(DEV), torch.from_numpy(gt).to(DEV)).cpu().double().numpy()
    p, g = j17.astype(np.float64), gt.astype(np.float64)
    r = olbs.mpjpe_h36m(p, g)
    D = np.abs(p[:, olbs.H36M_TO_J14]) + np.abs(p[:, :1]) + np.abs(g)
    M = np.sqrt((D ** 2).sum(-1)).mean(-1)
    err = np.abs(got - r)
    q = (err - fb.U24 * np.abs(r) - fb.TINY) / (fb.U24 * M)
    print("mpjpe %s: worst |err| / (2^-24 M) = %.3g (C = %d)" % (regime, (err / (fb.U24 * M)).max(), C_MPJPE))
    assert (q <= C_MPJPE).all(), q.max()
    if regime == "exact_match":
        assert (got == 0).all()
