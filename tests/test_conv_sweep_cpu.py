"""The convolution sweep's case table covers every coverage class (tests/conv_sweep_common.py), judged through
danet_conv_tc_dispatch, the engine's own report of what the kernel does with a shape.  No GPU."""
import ctypes

import pytest

import conv_sweep_common as S


def _geometry(case):
    from danet_b200 import _lib as L
    d = L.ConvDesc(*case[:7], case[5] // 2, case[7], 0, S.EXACT_FLAG if case[12] == "exact" else 0)
    g, c = (ctypes.c_int64 * 8)(), (ctypes.c_int64 * 4)()
    assert L.load().danet_conv_tc_geometry(ctypes.byref(d), ctypes.cast(g, ctypes.c_void_p)) == 0
    assert L.load().danet_conv_tc_cta_geometry(ctypes.byref(d), ctypes.cast(c, ctypes.c_void_p)) == 0
    return list(g), list(c)


def test_every_class_has_a_case():
    cov = S.coverage()
    missing = [name for name, cases in cov.items() if not cases]
    assert not missing, "coverage classes without a case:\n  " + "\n  ".join(missing)


def test_every_tile_body_is_listed():
    cov = S.coverage()
    for p, widths in (("exact", range(16, 65, 16)), ("fast", range(16, 257, 16))):
        for nt in widths:
            for form in ("full", "ragged"):
                assert cov["%s NT %d, %s last N tile" % (p, nt, form)], (p, nt, form)


@pytest.mark.parametrize("drop", [5, 33, 118, 141])
def test_the_classes_notice_a_missing_case(drop):
    """the table has no slack in the classes these cases alone cover: deleting one turns its class red"""
    full, less = S.coverage(), S.coverage(S.CASES[:drop] + S.CASES[drop + 1:])
    only = [name for name in full if full[name] == [drop]]
    assert only, "case %d is not the only case of any class: pick another" % drop
    assert all(not less[name] for name in only)


def test_cases_are_distinct_and_supported():
    assert len(set(S.CASES)) == len(S.CASES)
    for c in S.CASES:
        assert c[9] in ("none", "f32", "planes") and c[10] in ("f32", "planes", "both") and c[12] in ("exact", "fast"), c
        assert S.report(c)["NT"] > 0


def test_unsupported_shapes_are_refused():
    for exact in (True, False):
        assert S.dispatch(1, 20, 20, 64, 64, 7, 1, 1, exact) is None        # 49 taps in one parity plane
        assert S.dispatch(1, 20, 20, 64, 64, 5, 1, 1, exact) is None
        assert S.dispatch(1, 20, 20, 64, 64, 3, 3, 1, exact) is None
        assert S.dispatch(1, 20, 20, 60, 64, 3, 1, 1, exact) is None        # channels: multiples of 8
        assert S.dispatch(1, 20, 20, 64, 60, 3, 1, 1, exact) is None
        assert S.dispatch(1, 20, 20, 64, 64, 3, 1, 1, exact, pad=0) is None
        assert S.dispatch(1, 1 << 15, 1 << 15, 8, 8, 1, 1, 1, exact) is None   # 2^33 elements: 32-bit element offsets
        assert S.dispatch(4, 2056, 2056, 8, 64, 1, 1, 1, exact) is not None     # just past 2^30: taken


def test_report_agrees_with_the_geometry_entries():
    for c in S.CASES:
        r, (g, cta) = S.report(c), _geometry(c)
        N, H, W, Cin, Cout, k, s, G = c[:8]
        assert g[3] == r["nstack"], c
        groups = N if r["nstack"] == 1 else G * -(-(-(-N // G)) // r["nstack"])
        assert g[2] == groups * r["tiles_h"] * r["tiles_w"] * r["ntn"], c
        # issued MACs of one product per tile: 128 pixels x NT x 16 channels per K step x K steps x taps
        ksteps = (r["nchunks"] - 1) * (r["KCH"] // 16) + r["kv_last"]
        assert g[5] % (128 * r["NT"] * 16 * ksteps) == 0, c
        taps = g[5] // (128 * r["NT"] * 16 * ksteps)
        assert r["ntap"] <= taps <= k * k and (taps == k * k or s == 2), c
        assert g[7] % r["nblk"] == 0 and cta[2] == g[7], c                   # whole weight blocks
        if c[12] == "exact":
            assert cta[0] == 2 and cta[1] == r["pairs"] and 0 <= r["pairs_past"] <= r["pairs"], c
            assert 2 * r["pairs"] - r["pairs_past"] >= g[2], c                # every tile is in a pair
        else:
            assert cta[0] == 1 and cta[1] == g[2] and r["pairs"] == 0 and r["closes"] == 0, c
        assert r["last_nt"] == Cout - (r["ntn"] - 1) * r["NT"] and 0 < r["last_nt"] <= r["NT"], c
        assert Ho_tiles(c) == (r["tiles_h"], r["tiles_w"]), c


def Ho_tiles(c):
    Ho, Wo = S.out_hw(c)
    return (Ho + 15) // 16, (Wo + 7) // 8


def test_segments_follow_the_close_rule():
    """what the kernel-side constant implies: a segment closes once it holds 8 main-chain MMAs, so none but a tile's
    last holds fewer, none holds more than 7 plus one weight block, and the segments add up to the tile's MMAs"""
    longest = 0
    for Cin in range(8, 520, 8):
        for Cout in range(8, 72, 8):
            for k, s in ((1, 1), (1, 2), (3, 1), (3, 2), (7, 2)):
                r = S.dispatch(1, 20, 20, Cin, Cout, k, s, 1, True)
                ksteps = (r["nchunks"] - 1) * (r["KCH"] // 16) + r["kv_last"]
                mmas = ksteps * (k * k if s == 1 else {1: 1, 3: 9, 7: 49}[k])
                assert 1 <= r["closes"] <= mmas // 8 + 1 and r["closes"] == 1 + r["closes_plane_end"] + r["closes_mid_plane"]
                assert r["longest"] <= 7 + r["TG"] * (r["KCH"] // 16) and r["longest"] * r["closes"] >= mmas
                longest = max(longest, r["longest"])
    assert longest == S.LONGEST_SEGMENT


def test_stacked_boxes_are_tma_aligned():
    """a stacked image's halo box starts hs halo rows after the previous one's; TMA needs that offset 128-byte aligned"""
    stacked = 0
    for exact in (True, False):
        for k, s, tcols in ((1, 1, 1), (1, 2, 1), (3, 1, 3), (3, 2, 2), (7, 2, 4)):
            for H in range(1, 18):
                for Cin in (8, 16, 24, 32, 40, 64, 72):
                    r = S.dispatch(3, H, H, Cin, 16, k, s, 1, exact)
                    if r["nstack"] > 1:
                        stacked += 1
                        assert (r["hs"] * (8 + tcols - 1) * r["SWB"]) % 128 == 0, (H, Cin, k, s, r)
    assert stacked > 100
