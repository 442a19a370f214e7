"""Training targets on the CPU: the fp64 oracle (oracle/train_targets.py) against the golden the reference's own code
wrote (oracle/gen_golden_train_targets.py), the per-image translation solve of csrc/targets.cu compiled for the host
(DANET_TARGETS_HOST_CHECK) against estimate_translation_np at a componentwise fp64 bound and bit for bit against a
Python restatement of its operation order, seeded defects that these checks must catch, and argument refusals."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import synth, train_targets as ot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("keypoints", "pose", "betas", "has_smpl", "has_dp", "iuv_annotated", "smpl_2dkps")


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "train_targets.npz"))


@pytest.fixture(scope="module")
def model():
    return synth.make_smpl_model(0)


@pytest.mark.parametrize("tag", ["a_", "b_"])
def test_oracle_reproduces_reference_golden(gold, model, tag):
    g = gold
    fv = g["fit_valid"] if tag == "b_" else None
    o = ot.prepare_targets(model, {k: g[k] for k in KEYS}, g["fit_pose"], g["fit_betas"], fit_valid=fv)
    for k in ("opt_pose", "opt_betas", "valid_fit", "has_iuv", "opt_joints", "opt_cam_t"):
        np.testing.assert_array_equal(np.asarray(o[k]), g[tag + k], err_msg=k)
    for k in ("target_smpl_kps", "target_cam", "target", "target_smpl_joints"):   # fp64 vs the reference's fp32
        np.testing.assert_allclose(o[k], g[tag + k], rtol=1e-6, atol=5e-7, err_msg=k)
    assert g[tag + "opt_betas"][3, 2] == np.float32(3.7)           # a ground-truth beta above 3 survives
    assert (g[tag + "opt_betas"][1] == 0).all()                   # an extreme fit is zeroed


def test_golden_translation_is_the_fp32_rounding_of_estimate_translation_np(gold):
    np.testing.assert_array_equal(gold["et_trans"], gold["et_trans_np"].astype(np.float32))
    np.testing.assert_array_equal(ot.estimate_translation(gold["et_S"], gold["et_joints_2d"]), gold["et_trans_np"])


# -- the host build of the device arithmetic -------------------------------------------------------------------------

@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("targets_host") / "libtargets_host.so")
    csrc = os.path.join(ROOT, "danet-densepose2smpl_b200", "csrc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
                           "-DDANET_TARGETS_HOST_CHECK", "-shared", os.path.join(csrc, "targets.cu"),
                           os.path.join(csrc, "api.cu"), "-o", out])
    lib = ctypes.CDLL(out)
    p = ctypes.c_void_p
    lib.danet_test_estimate_translation_host.argtypes = [ctypes.c_int32, p, p, ctypes.c_int32, ctypes.c_double,
                                                         ctypes.c_double, p, p]
    lib.danet_test_estimate_translation_host.restype = ctypes.c_int
    return lib


def host_solve(lib, S, kp, normalised=False, f=5000., img=224., fp64=False):
    """The fp32 translations, or with fp64=True their fp64 values before the final rounding."""
    S, kp = np.ascontiguousarray(S, np.float32), np.ascontiguousarray(kp, np.float32)
    out, out64 = np.zeros((S.shape[0], 3), np.float32), np.zeros((S.shape[0], 3), np.float64)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert lib.danet_test_estimate_translation_host(S.shape[0], P(S), P(kp), int(normalised), f, img, P(out), P(out64)) == 0
    np.testing.assert_array_equal(out, out64.astype(np.float32))
    return out64 if fp64 else out


def sweep_cases(seed=7):
    """24 to 2 weighted joints, depths 5 to 100, key points at and outside the image, and two images far outside it
    (|O - x| > F), where LU's partial pivoting swaps rows."""
    rng = np.random.default_rng(seed)
    depths = np.geomspace(5, 100, 6)
    S, K = [], []
    for k in (24, 17, 9, 4, 2):
        for d in depths:
            s = rng.normal(0, 0.4, (49, 3))
            t = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), d])
            p = s + t
            uv = 5000. * p[:, :2] / p[:, 2:] + 112. + rng.normal(0, 2.0, (49, 2))
            if rng.random() < 0.4:
                uv += rng.choice([-1, 1], 2) * rng.uniform(150, 400, 2)     # outside the image
            conf = rng.choice([1.0, 0.3, 0.55, 0.9], 49)
            conf[25 + k:] = 0.0
            S.append(s)
            K.append(np.concatenate([uv, conf[:, None]], 1))
    for off in ((9000., 0.), (0., -12000.)):
        s = rng.normal(0, 0.4, (49, 3))
        uv = 5000. * (s[:, :2] + [0.1, 0.1]) / (s[:, 2:] + 8) + 112. + off
        S.append(s)
        K.append(np.concatenate([uv, np.full((49, 1), 0.3)], 1))
    return np.asarray(S, np.float32), np.asarray(K, np.float32)


def emulate(S, kp, f=5000., img=224., sqrt64=False, pivot=True):
    """The operation order of csrc/targets.cu in Python floats (IEEE fp64, no FMA): per-joint terms, the 32-lane xor
    tree, LU with partial pivoting; the fp64 solution.  sqrt64 / pivot=False are seeded defects."""
    O = img / 2.
    out = np.zeros((S.shape[0], 3))
    for b in range(S.shape[0]):
        lanes = [[0.0] * 9 for _ in range(32)]
        for j in range(24):
            X, Y, Z = (float(v) for v in S[b, 25 + j])
            x, y, c = (float(v) for v in kp[b, 25 + j])
            w = math.sqrt(c) if sqrt64 else float(np.sqrt(np.float32(c)))
            q = [[w * f, w * 0.0, w * (O - x)], [w * 0.0, w * f, w * (O - y)]]
            cc = [w * ((x - O) * Z - f * X), w * ((y - O) * Z - f * Y)]
            lanes[j] = [q[0][r] * q[0][s] + q[1][r] * q[1][s] for r, s in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]
            lanes[j] += [q[0][k] * cc[0] + q[1][k] * cc[1] for k in range(3)]
        for o in (16, 8, 4, 2, 1):
            lanes = [[lanes[l][e] + lanes[l ^ o][e] for e in range(9)] for l in range(32)]
        t = lanes[0]
        a = [[t[0], t[1], t[2]], [t[1], t[3], t[4]], [t[2], t[4], t[5]]]
        r = [t[6], t[7], t[8]]
        singular = False
        for k in range(3):
            p = k
            if pivot:
                for i in range(k + 1, 3):
                    if abs(a[i][k]) > abs(a[p][k]):
                        p = i
            singular |= a[p][k] == 0.0
            a[k], a[p], r[k], r[p] = a[p], a[k], r[p], r[k]
            for i in range(k + 1, 3):
                l = a[i][k] / a[k][k] if a[k][k] != 0.0 else math.nan
                a[i] = [a[i][jj] - l * a[k][jj] if jj > k else a[i][jj] for jj in range(3)]
                r[i] = r[i] - l * r[k]
        if singular:
            out[b] = np.nan
            continue
        x2 = r[2] / a[2][2]
        x1 = (r[1] - a[1][2] * x2) / a[1][1]
        x0 = (r[0] - a[0][1] * x1 - a[0][2] * x2) / a[0][0]
        out[b] = [x0, x1, x2]
    return out


def assert_within_bound(got, S, kp, ref):
    bound = ot.translation_bound(S, kp, ref)
    err = np.abs(got.astype(np.float64) - ref)
    assert (err <= bound).all(), (err / bound).max()


def test_host_solve_on_golden_cases_within_bound_of_estimate_translation_np(gold, hostlib):
    got = host_solve(hostlib, gold["et_S"], gold["et_joints_2d"])
    assert_within_bound(got, gold["et_S"], gold["et_joints_2d"], gold["et_trans_np"])


def test_host_solve_conditioning_sweep(hostlib):
    S, kp = sweep_cases()
    got = host_solve(hostlib, S, kp)
    ref = ot.estimate_translation(S, kp)
    assert np.isfinite(ref).all()
    assert_within_bound(got, S, kp, ref)
    np.testing.assert_array_equal(host_solve(hostlib, S, kp, fp64=True), emulate(S, kp))   # the documented order


def test_host_solve_denormalises_like_the_trainer(gold, hostlib):
    g = gold
    got = host_solve(hostlib, g["a_opt_joints"], g["keypoints"], normalised=True)
    np.testing.assert_array_equal(got, host_solve(hostlib, g["a_opt_joints"], ot.denormalise(g["keypoints"])))
    assert_within_bound(got, g["a_opt_joints"], ot.denormalise(g["keypoints"]),
                        ot.estimate_translation(g["a_opt_joints"], ot.denormalise(g["keypoints"])))


def test_zero_confidence_image_is_nan_and_others_unaffected(hostlib):
    S, kp = sweep_cases()
    S, kp = S[:4].copy(), kp[:4].copy()
    base = host_solve(hostlib, S, kp)
    kp[2, :, 2] = 0.0
    got = host_solve(hostlib, S, kp)
    assert np.isnan(got[2]).all()
    np.testing.assert_array_equal(np.delete(got, 2, 0), np.delete(base, 2, 0))
    assert np.isnan(ot.estimate_translation(S[2:3], kp[2:3])).all()     # numpy: LinAlgError
    kp[1, 30, 2] = -0.5                                                  # a negative confidence: NaN weight
    assert np.isnan(host_solve(hostlib, S, kp)[1]).all()


# -- seeded defects ----------------------------------------------------------------------------------------------------

def test_seeded_fp64_sqrt_is_caught(hostlib):
    S, kp = sweep_cases()
    assert (emulate(S, kp, sqrt64=True) != host_solve(hostlib, S, kp, fp64=True)).any()


def test_seeded_no_pivoting_is_caught(hostlib):
    S, kp = sweep_cases()
    assert (emulate(S, kp, pivot=False) != host_solve(hostlib, S, kp, fp64=True)).any()


def test_seeded_clamp_after_merge_is_caught(gold):
    g = gold
    pose, betas, _, _ = ot.fit_merge(g["fit_pose"], g["fit_betas"], g["pose"], g["betas"], g["has_smpl"],
                                     g["iuv_annotated"])
    np.testing.assert_array_equal(betas, g["a_opt_betas"])
    hs = g["has_smpl"].astype(bool)
    wrong = np.where(hs[:, None], g["betas"], g["fit_betas"])           # merge first ...
    wrong[(np.abs(wrong) > 3).any(-1)] = 0.                              # ... then clamp
    assert (wrong != g["a_opt_betas"]).any()


def test_seeded_rodrigues_flavour_swap_is_caught(gold):
    """The smplx flavour differs from the quaternion route in fp32; the oracle's fp32 quaternion route reproduces the
    reference's `target` rotations more closely than the smplx route does on these poses."""
    from oracle import lbs as olbs
    g = gold
    aa = g["a_opt_pose"].reshape(-1, 3).astype(np.float32)
    ref = g["a_target"][:, 13:].reshape(-1, 3, 3)
    dq = np.abs(olbs.batch_rodrigues_quat(aa) - ref).max()
    ds = np.abs(olbs.batch_rodrigues_smplx(aa) - ref).max()
    assert dq < ds, (dq, ds)


# -- argument refusals -------------------------------------------------------------------------------------------------

ET = "danet_b200.geometry.estimate_translation: "
PT = "danet_b200.targets.prepare_targets: "
NO_CPU = "must be a CUDA tensor (there is no CPU path)"


def _t(*shape, dtype=torch.float32):
    return torch.zeros(shape, dtype=dtype)


def _et(S=None, j=None, **kw):
    from danet_b200.geometry import estimate_translation
    S = _t(2, 49, 3) if S is None else S
    j = _t(2, 49, 3) if j is None else j
    return lambda: estimate_translation(S, j, **kw)


ET_CASES = [
    ("S-type", "S must be a tensor (got list)", _et(S=[0.0])),
    ("S-dtype", "S must be float32 (got torch.float64)", _et(S=_t(2, 49, 3, dtype=torch.float64))),
    ("S-rank", "S must be 3-D (got (2, 147))", _et(S=_t(2, 147))),
    ("S-shape", "S must have shape (2, 49, 3) (got (2, 24, 3))", _et(S=_t(2, 24, 3))),
    ("S-layout", "S must be contiguous", _et(S=_t(2, 3, 49).transpose(1, 2))),
    ("joints-shape", "joints_2d must have shape (2, 49, 3) (got (3, 49, 3))", _et(j=_t(3, 49, 3))),
    ("joints-dtype", "joints_2d must be float32 (got torch.float16)", _et(j=_t(2, 49, 3, dtype=torch.float16))),
    ("focal", "focal_length must be a number (got None)", _et(focal_length=None)),
    ("img-size", "img_size must be a number (got '224')", _et(img_size="224")),
    ("cpu", "S " + NO_CPU, _et()),
]


@pytest.mark.parametrize("text,fn", [pytest.param(t, f, id=i) for i, t, f in ET_CASES])
def test_estimate_translation_refusals(text, fn):
    with pytest.raises(ValueError, match=re.escape(ET + text)):
        fn()


class _Model:
    def __init__(self):
        import danet_b200
        self.iuv2smpl = type("P", (), {})()
        self.iuv2smpl.smpl = danet_b200.SMPL(synth.make_smpl_model(0))
        self.iuv_renderer = object()


@pytest.fixture(scope="module")
def cpu_model():
    return _Model()


def _batch(B=2, **over):
    b = {"keypoints": _t(B, 49, 3), "pose": _t(B, 72), "betas": _t(B, 10), "smpl_2dkps": _t(B, 24, 3),
         "has_smpl": _t(B, dtype=torch.bool), "has_dp": _t(B, dtype=torch.uint8), "iuv_annotated": _t(B, dtype=torch.bool)}
    b.update(over)
    return {k: v for k, v in b.items() if v is not None}


PT_CASES = [
    ("batch-type", "batch must be a dict (got list)", lambda m: (m, [], _t(2, 72), _t(2, 10)), {}),
    ("batch-key", "batch must have the key 'has_dp'", lambda m: (m, _batch(has_dp=None), _t(2, 72), _t(2, 10)), {}),
    ("keypoints-rank", "batch['keypoints'] must be 3-D (got (2, 147))",
     lambda m: (m, _batch(keypoints=_t(2, 147)), _t(2, 72), _t(2, 10)), {}),
    ("pose-shape", "batch['pose'] must have shape (2, 72) (got (2, 69))",
     lambda m: (m, _batch(pose=_t(2, 69)), _t(2, 72), _t(2, 10)), {}),
    ("betas-dtype", "batch['betas'] must be float32 (got torch.float64)",
     lambda m: (m, _batch(betas=_t(2, 10, dtype=torch.float64)), _t(2, 72), _t(2, 10)), {}),
    ("flag-dtype", "batch['has_smpl'] must be bool or uint8 (got torch.int64)",
     lambda m: (m, _batch(has_smpl=_t(2, dtype=torch.int64)), _t(2, 72), _t(2, 10)), {}),
    ("flag-shape", "batch['iuv_annotated'] must have shape (2,) (got (3,))",
     lambda m: (m, _batch(iuv_annotated=_t(3, dtype=torch.bool)), _t(2, 72), _t(2, 10)), {}),
    ("opt-pose", "opt_pose must have shape (2, 72) (got (1, 72))", lambda m: (m, _batch(), _t(1, 72), _t(2, 10)), {}),
    ("opt-betas", "opt_betas must be contiguous", lambda m: (m, _batch(), _t(2, 72), _t(10, 2).t()), {}),
    ("fit-valid", "fit_valid must be bool or uint8 (got torch.float32)", lambda m: (m, _batch(), _t(2, 72), _t(2, 10)),
     {"fit_valid": _t(2)}),
    ("focal", "focal_length must be a number (got 'f')", lambda m: (m, _batch(), _t(2, 72), _t(2, 10)),
     {"focal_length": "f"}),
    ("img-res", "img_res must be a positive int (got 224.0)", lambda m: (m, _batch(), _t(2, 72), _t(2, 10)),
     {"img_res": 224.0}),
    ("model", "model must have iuv2smpl.smpl and iuv_renderer", lambda m: (object(), _batch(), _t(2, 72), _t(2, 10)), {}),
    ("cpu", "move the model to a CUDA device (there is no CPU path)", lambda m: (m, _batch(), _t(2, 72), _t(2, 10)), {}),
]


@pytest.mark.parametrize("text,args,kw", [pytest.param(t, a, k, id=i) for i, t, a, k in PT_CASES])
def test_prepare_targets_refusals(cpu_model, text, args, kw):
    from danet_b200.targets import prepare_targets
    with pytest.raises(ValueError, match=re.escape(PT + text)):
        prepare_targets(*args(cpu_model), **kw)
