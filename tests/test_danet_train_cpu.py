"""CPU tests of the part dropout + iuvmap_clean join (danet_b200.iuvmap.part_drop_clean, draw_part_drop): the oracle's
restatement against the reference's own DaNet._forward (tests/golden/danet_train.npz, oracle/gen_golden_danet_train.py),
the (crop, channel) table, the seeded draws, the argument refusals and the C ABI exports."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import danet_train as odt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "danet_train.npz"))


def _case(g, name):
    training, rate, seed = g["%s_meta" % name]
    B, S = int(g["B"]), int(g["S"])
    leaves = odt.make_leaves(B, S, int(g["leaf_seed"]) + int(seed))
    G1, G2 = odt.make_probes(B, S, int(g["probe_seed"]) + int(seed))
    drop = torch.as_tensor(g["%s_drop" % name]) if training else None
    return leaves, (G1, G2), drop, bool(training), float(rate), int(seed)


def run_and_grad(op, leaves, probes, drop):
    """op on fresh leaves, then the gradients of <G1, cat[u_cl, v_cl, index_cl]> + <G2, part maps>"""
    xs = [t.detach().clone().requires_grad_() for t in leaves]
    out = op(*xs, drop)
    G1, G2 = probes
    probe = (G1 * torch.cat(out[:3], 1)).sum() + (G2 * out[4]).sum()
    grads = torch.autograd.grad(probe, xs, allow_unused=True)
    return out, grads


@pytest.mark.parametrize("name", ["r03_s0", "r03_s1", "r09_s0", "r09_s1", "eval"])
def test_oracle_matches_reference_golden(name):
    g = _golden()
    leaves, probes, drop, _, _, _ = _case(g, name)
    out, grads = run_and_grad(odt.part_drop_clean, leaves, probes, drop)
    for k, t in zip(("u_cl", "v_cl", "index_cl", "ann_cl", "part_iuv_map"), out):
        assert odt.bits_equal(t, torch.as_tensor(g["%s_%s" % (name, k)])), k
    assert grads[2] is None and grads[3] is None
    for k, t in zip(("g_u", "g_v", "g_parts"), (grads[0], grads[1], grads[4])):
        assert odt.bits_equal(t, torch.as_tensor(g["%s_%s" % (name, k)])), k


def test_golden_covers_the_corner_cases():
    """a dropped part's zero wins the argmax somewhere, and NaN reaches outputs and gradients"""
    g = _golden()
    wins = 0
    for name in ("r03_s0", "r09_s0"):
        drop = g["%s_drop" % name]
        best = g["%s_index_cl" % name].argmax(1)                       # [B,S,S]
        for b in range(drop.shape[0]):
            wins += int(sum(((best[b] == d + 1) & drop[b, d]).sum() for d in range(24)))
        assert np.isnan(g["%s_u_cl" % name]).any() and np.isnan(g["%s_g_parts" % name]).any()
        neg0 = lambda a: ((a == 0) & np.signbit(a)).any()
        assert neg0(g["%s_index_cl" % name]) and not neg0(g["%s_g_u" % name])
    assert wins > 0
    assert ((g["eval_g_u"] == 0) & np.signbit(g["eval_g_u"])).any()       # no dropout: -0.0 gradients survive


def test_crop_channel_table_matches_the_reference_comprehension():
    from danet_b200 import constants, iuvmap
    table = iuvmap._DP2SMPL.reshape(24, 6)
    for part in range(1, 25):
        mine = [(i, m + 1) for i in range(24) for m in range(6) if int(table[i, m]) == part]
        assert mine == odt.crop_channels(constants.DP2SMPL_MAPPING, part), part
    pairs = [odt.crop_channels(constants.DP2SMPL_MAPPING, p) for p in range(1, 25)]
    twice = sorted({i for ch in pairs for i in {c for c, _ in ch if sum(1 for c2, _ in ch if c2 == c) == 2}})
    assert twice == [7, 8, 10, 11, 12, 15, 20, 21, 22, 23]


def test_draw_part_drop_is_the_reference_draw():
    from danet_b200.iuvmap import draw_part_drop
    g = _golden()
    for name in ("r03_s0", "r03_s1", "r09_s0", "r09_s1"):
        _, _, drop, _, rate, seed = _case(g, name)
        torch.manual_seed(seed)
        d = draw_part_drop(int(g["B"]), rate)
        assert d.dtype == torch.bool and torch.equal(d, drop), name
        assert [[k + 1 for k in range(24) if row[k]] for row in d.tolist()] == odt.zero_idxs(drop)


def _args_ok(B=2, S=4):
    return [torch.zeros(B, 25, S, S), torch.zeros(B, 25, S, S), torch.zeros(B, 25, S, S), torch.zeros(B, 15, S, S),
            torch.zeros(B, 24, 3, 7, S, S), torch.zeros(B, 24, dtype=torch.bool)]


@pytest.mark.parametrize("pos,bad,msg", [
    (0, torch.zeros(2, 24, 4, 4), "u must be"),
    (0, torch.zeros(2, 25, 4, 4, dtype=torch.float64), "u must be float32"),
    (0, torch.zeros(0, 25, 4, 4), "u must be"),
    (0, torch.zeros(2, 25, 4, 5), "u must be"),
    (1, torch.zeros(2, 25, 4, 3), "v must have shape"),
    (2, "index", "index must be a tensor"),
    (3, torch.zeros(2, 15, 3, 3), "ann must be"),
    (3, torch.zeros(2, 300, 4, 4), "ann must be"),
    (4, torch.zeros(2, 24, 3, 6, 4, 4), "part_iuv_pred must have shape"),
    (5, torch.zeros(2, 24), "part_drop must be a bool tensor"),
    (5, torch.zeros(3, 24, dtype=torch.bool), "part_drop must have shape"),
    (5, torch.zeros(24, 2, dtype=torch.bool).t(), "part_drop must be contiguous"),
    (None, None, "must be a CUDA tensor"),
])
def test_part_drop_clean_refuses_bad_arguments(pos, bad, msg):
    from danet_b200.iuvmap import part_drop_clean
    a = _args_ok()
    if pos is not None:
        a[pos] = bad
    with pytest.raises(ValueError, match="danet_b200.iuvmap.part_drop_clean: .*" + msg):
        part_drop_clean(*a)


def test_draw_part_drop_refuses_a_non_number():
    from danet_b200.iuvmap import draw_part_drop
    with pytest.raises(ValueError, match="draw_part_drop: rate must be a number"):
        draw_part_drop(2, "0.3")


def test_entries_are_exported():
    so = os.path.join(ROOT, "danet-densepose2smpl_b200", "libdanet_b200.so")
    if not os.path.exists(so):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(so)
    from danet_b200 import _lib
    for name in ("danet_part_drop_clean_forward", "danet_part_drop_clean_backward"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES


def test_danet_forward_refuses_bad_arguments():
    from danet_b200.training import danet_forward

    class NotANet(torch.nn.Module):
        pass
    with pytest.raises(ValueError, match="danet_b200.training.danet_forward: model must be a danet_b200.DaNet"):
        danet_forward(NotANet(), {"img": torch.zeros(1, 3, 224, 224)})


def test_signatures_match_the_header_argument_counts():
    """every declaration in include/danet_b200.h has as many arguments as its SIGNATURES entry"""
    import re
    from danet_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "danet_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    for m in re.finditer(r"\b(danet_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", hdr):
        name, args = m.group(1), m.group(2).strip()
        if name not in _lib.SIGNATURES:
            continue
        n = 0 if args in ("", "void") else args.count(",") + 1
        assert n == len(_lib.SIGNATURES[name][1]), (name, n, len(_lib.SIGNATURES[name][1]))


def test_oracle_leaves_the_process_as_it_found_it():
    """the reference's iuvmap_clean is loaded without leaving ref_import.load()'s shims behind"""
    import sys
    import torch.cuda.comm as comm
    before = (os.getcwd(), list(sys.path), torch.Tensor.cuda, comm.broadcast)
    leaves = odt.make_leaves(1, 4, 0)
    odt.part_drop_clean(*leaves, torch.zeros(1, 24, dtype=torch.bool))
    assert (os.getcwd(), list(sys.path), torch.Tensor.cuda, comm.broadcast) == before
    assert "neural_renderer" not in sys.modules or getattr(sys.modules["neural_renderer"], "__file__", None)
