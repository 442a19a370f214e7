"""CPU tests of the training STN ops and the HRNet fuse (csrc/stn_train.cu, csrc/bn_train.cu): the exported entries
and their host-side argument checks, the Python wrappers' refusals, the fp64 oracle (oracle/stn_train.py) against the
golden the reference's own code produced (oracle/gen_golden_stn_train.py), and -- compiled for the host with
DANET_STN_HOST_CHECK -- the proof that the part-crop gather visits exactly the forward's (crop pixel -> input pixel,
weight) pairs, for every degenerate theta."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import stn_train as oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "danet-densepose2smpl_b200", "libdanet_b200.so")
NEW = ["danet_hr_fuse_forward", "danet_hr_fuse_backward", "danet_part_crops_forward", "danet_part_crops_backward",
       "danet_part_thetas"]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "stn_train.npz"))


# ------------------------------------------------------------------------------------------------
# library entries and argument checks (no launch happens: every call below is refused on the host)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        pytest.skip("libdanet_b200.so not built")
    from danet_b200 import _lib
    return _lib.load()


def test_library_exports_the_new_entries(lib):
    from danet_b200 import _lib
    for name in NEW:
        assert name in _lib.SIGNATURES and hasattr(lib, name)


def test_host_checks_refuse_bad_arguments(lib):
    P = ctypes.c_void_p(16)
    null = ctypes.c_void_p(0)
    terms = (ctypes.c_void_p * 4)(16, 16, 16, 16)
    fac = lambda *f: (ctypes.c_int32 * 4)(*(list(f) + [1] * (4 - len(f))))
    fw = lib.danet_hr_fuse_forward
    assert fw(0, 4, 8, 8, 1, terms, fac(1), 1, P, null) < 0                 # N = 0
    assert fw(1, 4, 8, 8, 0, terms, fac(1), 1, P, null) < 0                 # no term
    assert fw(1, 4, 8, 8, 5, terms, fac(1), 1, P, null) < 0                 # 5 terms
    assert fw(1, 4, 8, 8, 2, terms, fac(1, 3), 1, P, null) < 0              # factor 3
    assert fw(1, 4, 8, 8, 2, terms, fac(1, 16), 1, P, null) < 0             # factor 16
    assert fw(1, 4, 6, 6, 2, terms, fac(1, 4), 1, P, null) < 0              # 4 does not divide 6
    assert fw(1, 4, 8, 8, 1, terms, fac(1), 1, null, null) < 0              # y null
    assert fw(1, 4, 8, 8, 2, (ctypes.c_void_p * 4)(16, 0, 0, 0), fac(1, 2), 1, P, null) < 0
    bw = lib.danet_hr_fuse_backward
    assert bw(1, 4, 8, 8, 3, P, P, P, null) < 0
    assert bw(1, 4, 8, 8, 0, P, P, P, null) < 0
    assert bw(1, 4, 8, 8, 2, null, P, P, null) < 0
    assert bw(1, 4, 8, 8, 2, P, P, null, null) < 0
    for f in (lib.danet_part_crops_forward, lib.danet_part_crops_backward):
        assert f(0, 4, 8, P, P, 0, P, null) < 0
        assert f(1, 0, 8, P, P, 0, P, null) < 0
        assert f(1, 4, 1, P, P, 0, P, null) < 0
        assert f(1, 4, 8, null, P, 0, P, null) < 0
        assert f(1, 4, 8, P, null, 0, P, null) < 0
        assert f(1, 4, 8, P, P, 0, null, null) < 0
        assert f(1, 4 * 65536, 2, P, P, 0, P, null) < 0      # more channel chunks than a grid dimension holds
        assert f(2731, 4, 8, P, P, 0, P, null) < 0           # B * 24 past 65535
    th = lib.danet_part_thetas
    args = lambda **k: [k.get(n, d) for n, d in (("B", 1), ("Sh", 8), ("Si", 8), ("hm", P), ("idx", P), ("r", P), ("o", P),
                                                 ("vis", 0.5), ("cn", null), ("cj", 0.1), ("sn", null), ("sj", 0.2),
                                                 ("al", 0), ("c", P), ("t", P), ("st", null))]
    assert th(*args(B=0)) < 0
    assert th(*args(Si=1)) < 0
    assert th(*args(hm=null)) < 0
    assert th(*args(idx=null)) < 0                      # visibility needs the index scores
    assert th(*args(r=null)) < 0
    assert th(*args(t=null)) < 0


def _cpu(shape, dtype=torch.float32):
    return torch.zeros(shape, dtype=dtype)


def test_wrappers_refuse_bad_input():
    from danet_b200.layers import hr_fuse
    from danet_b200.stn import part_crops, part_thetas
    t = _cpu((1, 4, 8, 8))
    bad_fuse = [([], []), ([t] * 5, [1] * 5), ([t], [3]), ([t], [True]), ([t, t], [1]),
                ([t.double()], [1]), ([_cpu((4, 8, 8))], [1]), ([_cpu((1, 4, 8, 16))[..., ::2]], [1]),
                ([t, _cpu((1, 4, 3, 4))], [1, 2]), ([t, _cpu((1, 2, 4, 4))], [1, 2]), ([t], [1])]
    for terms, factors in bad_fuse:
        with pytest.raises(ValueError):
            hr_fuse(terms, factors)
    xd, th = _cpu((2, 4, 8, 8)), _cpu((2, 24, 2, 3))
    for a, b in ((xd.double(), th), (xd, th.double()), (_cpu((2, 4, 8, 6)), th), (_cpu((2, 4, 1, 1)), th),
                 (xd, _cpu((2, 23, 2, 3))), (xd, _cpu((1, 24, 2, 3))), (_cpu((2, 4, 8, 16))[..., ::2], th),
                 (xd, th)):                                                   # the last: CPU tensors
        with pytest.raises(ValueError):
            part_crops(a, b)
    hm, idx, r = _cpu((2, 24, 8, 8)), _cpu((2, 25, 8, 8)), _cpu(24)
    for kw in (dict(hm=_cpu((2, 23, 8, 8))), dict(hm=hm.double()), dict(index_pred=_cpu((2, 24, 8, 8))),
               dict(index_pred=_cpu((1, 25, 8, 8))), dict(learned_ratio=_cpu(23)), dict(learned_offset=_cpu((24, 1))),
               dict(center_noise=_cpu((2, 24, 3))), dict(scale_noise=_cpu((2, 24, 2))), dict(vis_score="x"),
               dict(center_jitter=None), dict()):
        a = dict(hm=hm, index_pred=idx, learned_ratio=r, learned_offset=r)
        a.update(kw)
        with pytest.raises(ValueError):
            part_thetas(a.pop("hm"), a.pop("index_pred"), a.pop("learned_ratio"), a.pop("learned_offset"), **a)


# ------------------------------------------------------------------------------------------------
# fp64 oracle against the reference's golden
# ------------------------------------------------------------------------------------------------
def test_oracle_thetas_match_reference_golden(gold):
    g = gold
    vis, cj, sj = (float(x) for x in g["stn_params"])
    c, th, scores = oracle.part_thetas(g["hm"], g["index_pred"], g["learned_ratio"], g["learned_offset"], vis,
                                       g["center_noise"], cj, g["scale_noise"], sj)
    near = np.abs(scores - vis) < 1e-5                                    # visibility decisions on a near-tie
    assert not near.any(), "golden has a visibility near-tie: %s" % np.argwhere(near)
    np.testing.assert_allclose(c, g["stn_centers"], atol=1e-5)
    np.testing.assert_allclose(th, g["thetas"], atol=1e-5)
    assert (g["thetas"][..., 0, 1] == 0).all() and (g["thetas"][..., 1, 0] == 0).all()
    hidden = scores[:, 1:] < vis
    assert hidden.any() and (~hidden).any(), "the golden exercises both visibility outcomes"


def test_oracle_crops_match_reference_golden(gold):
    g = gold
    crops, _, scale, _ = oracle.part_crops(g["xd"], g["thetas"])
    # torch's affine_grid (a batched matmul) rounds the coordinates differently: agreement within the sampler's
    # Lipschitz bound of a few fp32 ulps of the coordinate
    np.testing.assert_allclose(crops, g["part_maps"], atol=2e-5)


def test_oracle_fuse_matches_reference_golden(gold):
    for i in range(4):
        terms = [gold["fuse%d_t%d" % (i, j)] for j in range(4)]
        factors = [int(f) for f in gold["fuse%d_factors" % i]]
        assert sorted(set(factors) - {1}) == sorted({2 ** (j - i) for j in range(i + 1, 4)})
        y = oracle.hr_fuse(terms, factors)
        np.testing.assert_allclose(y, gold["fuse%d_y" % i], atol=1e-5, rtol=1e-6)
        # the golden's fp32 output is the list-order fp32 sum, bit for bit
        acc = None
        for t, f in zip(terms, factors):
            u = t.repeat(f, 2).repeat(f, 3)
            acc = u if acc is None else (acc + u).astype(np.float32)
        assert np.array_equal(np.maximum(acc, np.float32(0)), gold["fuse%d_y" % i])


# ------------------------------------------------------------------------------------------------
# the gather visits exactly the forward's contributions (host build of the kernels' own functions)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("stn_host") / "libstn_host.so")
    csrc = os.path.join(ROOT, "danet-densepose2smpl_b200", "csrc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
                           "-DDANET_STN_HOST_CHECK", "-shared", os.path.join(csrc, "stn_train.cu"),
                           os.path.join(csrc, "api.cu"), "-o", out])
    lib = ctypes.CDLL(out)
    p, i32, i64, f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float
    for fn in (lib.danet_test_crop_forward_pairs, lib.danet_test_crop_gather_pairs):
        fn.argtypes, fn.restype = [i32, i32, p, p, p, i64], i64
    lib.danet_test_crop_candidates.argtypes = [i32, i32, f, f, i32, p, p]
    lib.danet_test_crop_candidates.restype = None
    lib.danet_test_crop_coord.argtypes = [i32, i32, f, f, i32]
    lib.danet_test_crop_coord.restype = f
    return lib


def _thetas(S):
    """(s, c) per axis: realistic, every degenerate form, and tiny scales placed on a pixel boundary"""
    edge = lambda S, align, q: (2.0 * q + 1.0) / S - 1.0 if not align else 2.0 * q / (S - 1) - 1.0
    out = [(0.3, 0.1), (0.55, -0.4), (1.0, 0.0), (1.7, 0.2), (3.5, -0.9),      # realistic and > 1
           (0.0, 0.0), (0.0, 0.37), (0.0, -1.0), (0.0, 5.0),                     # scale 0: one point
           (1e-7, 0.2), (3e-6, -0.5), (1e-4, 0.9), (1e-30, 0.0), (2e-3, 0.0),     # tiny
           (0.4, 1.6), (0.4, -2.5), (0.9, 40.0), (0.2, -1e4),                     # centres off the map
           (3e7, 0.1), (0.5, 3e9), (1e20, -1e20), (-0.6, 0.1),                    # huge coordinates, negative scale
           (float("nan"), 0.0), (0.3, float("inf"))]
    for q in (0, 1, S // 2):                                          # tiny scales centred exactly on a tap boundary
        for a in (0, 1):
            out += [(1e-7, edge(S, a, q) + 1.0 / S), (5e-6, edge(S, a, q) + 0.5 / S)]
    return out


def _pairs(fn, S, align, th):
    cap = 8 * S * S + 64
    rec = np.zeros((cap, 4), np.int32)
    w = np.zeros(cap, np.float32)
    n = fn(S, align, th.ctypes.data_as(ctypes.c_void_p), rec.ctypes.data_as(ctypes.c_void_p),
           w.ctypes.data_as(ctypes.c_void_p), cap)
    assert n >= 0, "record overflow"
    return rec[:n], w[:n]


@pytest.mark.parametrize("S", [2, 3, 7, 16, 56])
@pytest.mark.parametrize("align", [0, 1])
def test_gather_visits_exactly_the_forward_pairs(hostlib, S, align):
    lo, hi = ctypes.c_int32(), ctypes.c_int32()
    axes = _thetas(S)
    # the 2-D check over axis pairs (x form, y form); each axis form appears on both axes
    combos = [(axes[k], axes[(k * 7 + 3) % len(axes)]) for k in range(len(axes))]
    for (sx, cx), (sy, cy) in combos:
        th = np.array([sx, 0, cx, 0, sy, cy], np.float32)
        fwd, fw = _pairs(hostlib.danet_test_crop_forward_pairs, S, align, th)
        gat, gw = _pairs(hostlib.danet_test_crop_gather_pairs, S, align, th)
        key = lambda r: [tuple(x) for x in r]
        F = dict(zip(key(fwd), fw.view(np.uint32)))
        G = dict(zip(key(gat), gw.view(np.uint32)))
        assert len(F) == len(fwd) and len(G) == len(gat), "a pair recorded twice"
        assert F == G, "theta %s S=%d align=%d: forward %d pairs, gather %d" % (th, S, align, len(F), len(G))
        # every forward pair lies in the gather's candidate ranges of its axis
        for (py, px, yy, xx) in F:
            hostlib.danet_test_crop_candidates(S, align, float(th[0]), float(th[2]), xx, ctypes.byref(lo), ctypes.byref(hi))
            assert lo.value <= px <= hi.value
            hostlib.danet_test_crop_candidates(S, align, float(th[4]), float(th[5]), yy, ctypes.byref(lo), ctypes.byref(hi))
            assert lo.value <= py <= hi.value


@pytest.mark.parametrize("S", [2, 3, 7, 16, 56])
@pytest.mark.parametrize("align", [0, 1])
def test_numpy_coordinates_are_the_kernels(hostlib, S, align):
    """oracle.crop_coords (the GPU tests' tight oracle) restates crop_coord bit for bit"""
    for s, c in _thetas(S):
        ref = np.array([hostlib.danet_test_crop_coord(S, align, s, c, p) for p in range(S)], np.float32)
        with np.errstate(invalid="ignore", over="ignore"):
            got = oracle.crop_coords(S, s, c, align)
        assert np.array_equal(ref.view(np.uint32), got.view(np.uint32)) or \
            (np.isnan(ref) == np.isnan(got)).all() and np.array_equal(ref[~np.isnan(ref)], got[~np.isnan(got)]), (s, c)
