"""Exact mode's CTA work unit, the tile pair, read from the library on the CPU (danet_conv_tc_cta_geometry): which tiles
pair, what a pair copies into shared memory, that every convolution of the W32 / W48 plans (and the input-gradient
pieces and the SMPL blend GEMM) still fits the shared-memory plan, and the weight stream of the W48 batch-64 step."""
import ctypes
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

EXACT = 4


def _lib():
    from danet_b200 import _lib as L
    return L, L.load()


def _desc(N, H, W, Cin, Cout, k, s, G, exact=True):
    L, _ = _lib()
    return L.ConvDesc(N, H, W, Cin, Cout, k, s, k // 2, G, 1, EXACT if exact else 0)


def _geometry(*shape, exact=True):
    L, lib = _lib()
    out = (ctypes.c_int64 * 8)()
    assert lib.danet_conv_tc_geometry(ctypes.byref(_desc(*shape, exact=exact)), ctypes.cast(out, ctypes.c_void_p)) == 0
    return dict(zip(("tile_h", "tile_w", "tiles", "nstack", "products", "macs", "a_bytes", "b_bytes"), list(out)))


def _cta(*shape, exact=True):
    L, lib = _lib()
    out = (ctypes.c_int64 * 4)()
    assert lib.danet_conv_tc_cta_geometry(ctypes.byref(_desc(*shape, exact=exact)), ctypes.cast(out, ctypes.c_void_p)) == 0
    return dict(zip(("tiles_per_unit", "units", "w_bytes", "a_bytes"), list(out)))


def _check_pair(shape, units):
    g, c = _geometry(*shape), _cta(*shape)
    assert c["tiles_per_unit"] == 2
    assert c["units"] == units, (shape, c, g)
    assert c["w_bytes"] == g["b_bytes"]                 # one weight stream for both tiles
    assert c["a_bytes"] == 2 * g["a_bytes"]             # two halos
    return g, c


def test_tall_maps_pair_tile_rows():
    g, _ = _check_pair((64, 56, 56, 48, 48, 3, 1, 1), 64 * 2 * 7)        # 4 tile rows -> 2 pairs per tile column
    assert g["tiles"] == 64 * 4 * 7
    _check_pair((64, 40, 40, 64, 64, 3, 1, 1), 64 * 2 * 5)              # 3 tile rows: the last one has no partner
    _check_pair((1536, 56, 56, 64, 64, 7, 2, 1), 1536 * 1 * 4)           # the limb stem: Ho = 28, 2 tile rows
    _check_pair((1536, 56, 56, 48, 24, 3, 1, 24), 1536 * 2 * 7)          # weight sets: rows of one image, one set


def test_one_row_maps_pair_image_groups():
    _check_pair((64, 14, 14, 192, 192, 3, 1, 1), 32 * 2 * 3)            # 3 N tiles of 64 channels, 2 tile columns
    _check_pair((63, 14, 14, 192, 192, 3, 1, 1), 32 * 2 * 3)            # odd image count: the last pair is unpaired


def test_weight_sets_pair_groups_of_one_set():
    g, _ = _check_pair((1536, 2, 2, 128, 128, 3, 1, 24), 24 * 7 * 2)    # 13 groups of 5 images per set -> 7 pairs
    assert g["nstack"] == 5 and g["tiles"] == 24 * 13 * 2


def test_stacked_stride2_maps_pair_groups():
    g, _ = _check_pair((64, 7, 7, 128, 256, 3, 2, 1), 11 * 4)           # 22 groups of 3 stacked images, 4 N tiles
    assert g["nstack"] == 3
    g, _ = _check_pair((1536, 4, 4, 256, 128, 3, 2, 24), 24 * 7 * 2)
    assert g["nstack"] == 5


def test_smpl_blend_gemm_pairs_rows():
    # the SMPL blend-shape GEMM: 512 bodies as one 64 x 8 "image", 224 features -> 20672 vertex coordinates
    g, c = _check_pair((1, 64, 8, 224, 20672, 1, 1, 1), 2 * 323)
    assert c["units"] * 2 == g["tiles"]


def test_fast_mode_work_unit_is_one_tile():
    shape = (64, 56, 56, 48, 48, 3, 1, 1)
    g, c = _geometry(*shape, exact=False), _cta(*shape, exact=False)
    assert (c["tiles_per_unit"], c["units"], c["w_bytes"], c["a_bytes"]) == (1, g["tiles"], g["b_bytes"], g["a_bytes"])


def _plan_groups(width):
    import danet_b200
    from oracle.net_ops import TorchEmulOps
    net = danet_b200.build_synthetic_danet(width=width, seed=0, device="cpu", conv_algo="tc")
    plan = net.plan_for(1, "cpu", ops=TorchEmulOps())
    return [[cv["d"] for cv in s.args[0]] for s in plan.steps if s.name == "conv_group"]


def _c8(c):
    return (c + 7) // 8 * 8


@pytest.mark.parametrize("width", [32, 48])
def test_every_plan_launch_fits_the_ring_depths(width):
    L, lib = _lib()
    shapes = set()
    for group in _plan_groups(width):
        descs = (L.ConvDesc * len(group))()
        for i, d in enumerate(group):
            descs[i] = L.ConvDesc(d["N"] * 64, d["H"], d["W"], d["Cin"], d["Cout"], d["ksize"], d["stride"], d["pad"],
                                  d["wsets"], 1, EXACT)
            shapes.add((d["N"] * 64, d["H"], d["W"], d["Cin"], d["Cout"], d["ksize"], d["stride"], d["wsets"]))
        st = (ctypes.c_int32 * 2)()
        assert lib.danet_conv_tc_config(len(group), descs, ctypes.cast(st, ctypes.c_void_p)) == 0
        assert st[0] >= 2 and st[1] >= 2, list(st)
    # the input-gradient pieces of every convolution (conv.conv2d): 1x1 / 3x3 stride-1 problems on the output map with
    # input and output channels swapped
    for (N, H, W, Cin, Cout, k, s, G) in shapes:
        Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
        for kp in ((1, 3) if k > 1 else (1,)):
            d = L.ConvDesc(N, Ho, Wo, _c8(Cout), _c8(Cin), kp, 1, kp // 2, G, 0, EXACT)
            assert lib.danet_conv_tc_supported(ctypes.byref(d)) == 1, (N, Ho, Wo, Cout, Cin, kp, G)


def test_w48_b64_weight_stream_halved():
    from conv_census import census
    c = census(48, 64, "exact")
    # 75.1 GB of weight blocks per step when every 16x8 tile streamed its own
    assert c["total"]["w_bytes"] <= 0.55 * 75.1e9, c["total"]["w_bytes"]
