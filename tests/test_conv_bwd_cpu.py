"""The numpy fp64 restatement of the convolution backward (oracle/conv_bwd.py) against torch CPU fp64 autograd of
torch.nn.functional.conv2d: the rotated / parity-class kernels of the input gradient with their interleave and crop,
and the weight and bias gradient sums.  No GPU needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import conv_bwd as cb

CASES = [  # (B, cin per group, cout per group, H, W, k, stride, groups)
    (2, 5, 6, 9, 8, 1, 1, 1), (2, 5, 6, 9, 8, 1, 2, 1), (2, 5, 6, 8, 9, 3, 1, 1), (2, 5, 6, 9, 9, 3, 2, 1),
    (2, 5, 6, 8, 8, 3, 2, 1), (2, 4, 3, 11, 10, 7, 1, 1), (2, 4, 3, 11, 10, 7, 2, 1), (1, 3, 4, 12, 12, 7, 2, 1),
    (2, 3, 2, 7, 7, 3, 2, 1), (2, 2, 3, 4, 4, 3, 1, 24), (2, 2, 3, 4, 5, 3, 2, 24), (1, 2, 2, 4, 4, 1, 2, 24),
    (1, 2, 2, 5, 5, 7, 2, 24),
]


def _torch_ref(x, w, b, gy, stride, groups):
    xt, wt, bt = (torch.from_numpy(a).requires_grad_() for a in (x, w, b))
    y = F.conv2d(xt, wt, bt, stride=stride, padding=w.shape[-1] // 2, groups=groups)
    y.backward(torch.from_numpy(gy))
    return y.detach().numpy(), xt.grad.numpy(), wt.grad.numpy(), bt.grad.numpy()


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d_c%d-%d_%dx%d_k%d_s%d_g%d" % c)
def test_restatement_matches_torch_autograd(case):
    B, cin, cout, H, W, k, s, G = case
    rng = np.random.default_rng(hash(case) & 0xFFFF)
    x = rng.normal(size=(B, G * cin, H, W))
    w = rng.normal(size=(G * cout, cin, k, k))
    b = rng.normal(size=(G * cout,))
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    gy = rng.normal(size=(B, G * cout, Ho, Wo))
    y_ref, dx_ref, dw_ref, db_ref = _torch_ref(x, w, b, gy, s, G)
    y = cb.conv_fwd(x, w, s, G) + b[None, :, None, None]
    dx = cb.dgrad(gy, w, H, W, s, G)
    dw, db = cb.wgrad(x, gy, k, s, G)
    for got, ref in ((y, y_ref), (dx, dx_ref), (dw, dw_ref), (db, db_ref)):
        assert got.shape == ref.shape
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-11)


@pytest.mark.parametrize("k,s,taps,npieces", [(1, 1, 1, 1), (3, 1, 9, 1), (1, 2, 1, 1), (3, 2, 28, 4), (7, 2, 81, 9)])
def test_executed_taps(k, s, taps, npieces):
    """Tap overhead of the parity decomposition: 3x3/s2 runs 1 + 9 + 9 + 9 taps for 9; 7x7/s2 nine 3x3 pieces, 81 for 49
    (every piece is a 1x1 or 3x3 stride-1 problem the engine runs)."""
    assert cb.executed_taps(k, s) == taps
    assert len(cb.dgrad_pieces(k, s)) == npieces
    assert all(p[2] in (1, 3) for p in cb.dgrad_pieces(k, s))


def test_stride1_class_is_the_rotated_filter():
    rng = np.random.default_rng(3)
    w = rng.normal(size=(6, 4, 3, 3))
    (piece,) = cb.dgrad_pieces(3, 1)
    wc = cb.dgrad_piece_weights(w, 3, 1, piece)
    np.testing.assert_array_equal(wc, w[:, :, ::-1, ::-1].transpose(1, 0, 2, 3))
