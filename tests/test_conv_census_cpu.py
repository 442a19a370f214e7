"""Tile geometry of the wgmma convolution engine, read from the library (danet_conv_tc_geometry) on the CPU: small-map
stacking with several weight sets and at stride 2, and the census of the HRNet-W48 plan at batch 64 (tools/conv_census.py)."""
import ctypes
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _geometry(N, H, W, Cin, Cout, k, s, G, exact=True):
    from danet_b200 import _lib as L
    out = (ctypes.c_int64 * 8)()
    d = L.ConvDesc(N, H, W, Cin, Cout, k, s, k // 2, G, 1, 4 if exact else 0)
    assert L.load().danet_conv_tc_geometry(ctypes.byref(d), ctypes.cast(out, ctypes.c_void_p)) == 0
    return dict(zip(("tile_h", "tile_w", "tiles", "nstack", "products", "macs", "a_bytes", "b_bytes"), list(out)))


@pytest.mark.parametrize("exact", [True, False])
def test_weight_sets_stack_images_of_one_set(exact):
    # 1536 = 64 batch entries x 24 parts; 2x2 maps (hs = 3 rows): five images of one part per 16-row tile
    g = _geometry(1536, 2, 2, 128, 128, 3, 1, 24, exact)
    assert g["nstack"] == 5
    ntn = 2 if exact else 1                             # N tiles: 2 x 64 channels (exact), 1 x 128 (fast)
    assert g["tiles"] == 24 * ((64 + 4) // 5) * ntn
    assert g["products"] == (3 if exact else 1)


def test_stride2_small_maps_stack():
    g = _geometry(1536, 4, 4, 256, 128, 3, 2, 24)       # Ho = 2, two parity rows of taps: 3-row boxes
    assert g["nstack"] == 5
    g = _geometry(64, 7, 7, 128, 256, 3, 2, 1)          # Ho = 4: 5-row boxes
    assert g["nstack"] == 3
    g = _geometry(64, 14, 14, 192, 384, 3, 2, 1)        # Ho = 7: 8-row boxes
    assert g["nstack"] == 2
    g = _geometry(64, 28, 28, 96, 192, 3, 2, 1)         # Ho = 14: no stacking
    assert g["nstack"] == 1


def test_large_maps_keep_their_tiles():
    g = _geometry(64, 56, 56, 48, 48, 3, 1, 1)
    assert (g["tile_h"], g["tile_w"], g["nstack"]) == (16, 8, 1)
    assert g["tiles"] == 64 * 4 * 7                     # one 48-wide N tile
    assert g["b_bytes"] == 5 * 24 * 1024                # 9 taps in blocks of 2 (hi/lo rows of 48 channels at 128 B)
    assert g["a_bytes"] == 2 * 18 * 10 * 128            # hi + lo halo planes


def test_w48_b64_census_small_maps_no_longer_one_image_per_tile():
    from conv_census import census
    c = census(48, 64, "exact")
    rows = {r["shape"]: r for r in c["shapes"]}
    # efficiency (useful / issued MACs) with one image per 128-pixel tile, as the engine tiled these shapes before
    # small-map stacking covered weight sets and stride 2
    one_image = {"1536x2x2 128->128 3x3/s1 ws24": 4 / 128., "1536x4x4 256->128 3x3/s2 ws24": 4 / 128.,
                 "64x4x4 256->512 3x3/s2 ws1": 4 / 128., "64x7x7 128->256 3x3/s2 ws1": 16 / 128.,
                 "1536x7x7 128->256 1x1/s2 ws1": 16 / 128., "1536x4x4 256->128 1x1/s2 ws24": 4 / 128.}
    for shape, eff in one_image.items():
        assert shape in rows, shape
        assert rows[shape]["img_per_tile"] > 1, rows[shape]
        assert rows[shape]["eff"] > 2.5 * eff, rows[shape]
    # every shape keeps at least its pinned efficiency, and the step issues no more MACs than pinned
    with open(os.path.join(ROOT, "tests", "golden", "conv_census_w48_b64.json")) as f:
        pinned = json.load(f)
    assert set(rows) == set(pinned["eff"])
    for shape, eff in pinned["eff"].items():
        assert rows[shape]["eff"] >= eff - 1e-6, (shape, rows[shape]["eff"], eff)
    assert c["total"]["issued_macs"] <= pinned["issued_macs"]
