"""The ResNet training layers without a GPU: the library exports the BatchNorm / max-pool entries, their workspace size
follows the chunk formula, the host checks refuse bad sizes and null pointers before any launch, and
danet_b200.layers refuses every input it does not support with ValueError."""
import ctypes
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("danet_bn2d_workspace_bytes", "danet_bn2d_forward", "danet_bn2d_backward", "danet_maxpool3x3s2_nchw_forward",
           "danet_maxpool3x3s2_nchw_backward")


@pytest.fixture(scope="module")
def lib():
    so = os.path.join(ROOT, "danet-densepose2smpl_b200", "libdanet_b200.so")
    if not os.path.exists(so):
        import __graft_entry__
        __graft_entry__.build()
    from danet_b200 import _lib
    return _lib.load()


def test_library_exports_the_entries(lib):
    from danet_b200 import _lib
    for sym in ENTRIES:
        assert hasattr(lib, sym), sym
        assert sym in _lib.SIGNATURES, sym


@pytest.mark.parametrize("N,C,HW", [(384, 64, 3136), (384, 64, 784), (16, 64, 3136), (384, 128, 49), (16, 3072, 4),
                                    (2, 512, 4), (1, 1, 16384), (3, 5, 20000), (70000, 3, 1)])
def test_workspace_follows_the_chunk_formula(lib, N, C, HW):
    ipc = max(1, 16384 // HW)                     # images per chunk: at least 16384 elements of a channel, >= 1 image
    nchunk = (N + ipc - 1) // ipc
    part = (2 * nchunk * C * 8 + 255) // 256 * 256
    assert lib.danet_bn2d_workspace_bytes(N, C, HW) == part + C * 8 * 4


def test_workspace_of_unsupported_sizes_is_zero(lib):
    assert lib.danet_bn2d_workspace_bytes(0, 8, 8) == 0
    assert lib.danet_bn2d_workspace_bytes(8, 0, 8) == 0
    assert lib.danet_bn2d_workspace_bytes(8, 8, 0) == 0
    assert lib.danet_bn2d_workspace_bytes(1 << 20, 1 << 10, 1 << 4) == 0      # 2^34 elements


def _err(lib):
    return lib.danet_last_error().decode()


def _fake(n):
    """distinct non-null, 256-byte aligned addresses: the host checks run before anything touches them"""
    return [ctypes.c_void_p(0x100000 * (i + 1)) for i in range(n)]


def test_forward_host_checks(lib):
    x, w, b, rm, rv, y, save, ws = _fake(8)
    args = lambda **k: dict(dict(N=2, C=4, HW=9, x=x, w=w, b=b, rm=rm, rv=rv, training=1, y=y, save=save, ws=ws), **k)

    def call(a):
        return lib.danet_bn2d_forward(a["N"], a["C"], a["HW"], a["x"], a["w"], a["b"], a["rm"], a["rv"], a["training"], 0.1,
                                      1e-5, None, 1, a["y"], a["save"], None, a["ws"], None)
    for bad, msg in [(dict(N=0), "bad sizes"), (dict(C=-1), "bad sizes"), (dict(x=None), "non-null"),
                     (dict(w=None), "non-null"), (dict(rv=None), "non-null"), (dict(save=None), "non-null"),
                     (dict(ws=None), "workspace"), (dict(ws=ctypes.c_void_p(0x100004)), "workspace"),
                     (dict(N=1, HW=1), "more than one value")]:
        assert call(args(**bad)) < 0, bad
        assert msg in _err(lib), (bad, _err(lib))


def test_backward_host_checks(lib):
    x, y, dy, w, save, dx, ws = _fake(7)

    def call(N=2, C=4, HW=9, x=x, y=y, dy=dy, save=save, relu=1, training=1, ws=ws):
        return lib.danet_bn2d_backward(N, C, HW, x, y, dy, w, save, training, relu, dx, None, None, None, ws, None)
    for bad, msg in [(dict(HW=0), "bad sizes"), (dict(dy=None), "non-null"), (dict(save=None), "non-null"),
                     (dict(y=None), "relu needs"), (dict(ws=None), "workspace"), (dict(N=1, HW=1), "more than one value")]:
        assert call(**bad) < 0, bad
        assert msg in _err(lib), (bad, _err(lib))


def test_max_pool_host_checks(lib):
    x, y, slot = _fake(3)
    assert lib.danet_maxpool3x3s2_nchw_forward(2, 3, 0, 5, x, y, slot, None) < 0 and "bad sizes" in _err(lib)
    assert lib.danet_maxpool3x3s2_nchw_forward(2, 3, 5, 5, x, y, None, None) < 0 and "non-null" in _err(lib)
    assert lib.danet_maxpool3x3s2_nchw_backward(-1, 3, 5, 5, x, slot, y, None) < 0 and "bad sizes" in _err(lib)
    assert lib.danet_maxpool3x3s2_nchw_backward(2, 3, 5, 5, None, slot, y, None) < 0 and "non-null" in _err(lib)


def _bn_inputs(N=2, C=3, H=4, W=4, dtype=torch.float32):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(N, C, H, W, generator=g).to(dtype)
    return x, torch.zeros(C, dtype=dtype), torch.ones(C, dtype=dtype), torch.ones(C, dtype=dtype), torch.zeros(C, dtype=dtype)


def test_batch_norm_refuses_unsupported_inputs():
    from danet_b200.layers import batch_norm
    x, rm, rv, w, b = _bn_inputs()
    with pytest.raises(ValueError, match="CUDA tensor"):
        batch_norm(x, rm, rv, w, b, True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="float32"):
        batch_norm(*_bn_inputs(dtype=torch.float64), True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="float32"):
        batch_norm(x.half(), rm, rv, w, b, True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="float32"):
        batch_norm(x, rm, rv, w, b, True, 0.1, 1e-5, residual=x.double())
    for i, name in enumerate(("running_mean", "running_var", "weight", "bias")):
        args = [rm, rv, w, b]
        args[i] = None
        with pytest.raises(ValueError, match=name):
            batch_norm(x, *args, True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="momentum"):
        batch_norm(x, rm, rv, w, b, True, None, 1e-5)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        batch_norm(x[:1, :, :1, :1].contiguous(), rm, rv, w, b, True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="contiguous"):
        batch_norm(x.transpose(2, 3), rm, rv, w, b, True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="4-D"):
        batch_norm(x.view(2, 3, 16), rm, rv, w, b, True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="shape"):
        batch_norm(x, rm[:2], rv, w, b, True, 0.1, 1e-5)
    with pytest.raises(ValueError, match="shape"):
        batch_norm(x, rm, rv, w, b, True, 0.1, 1e-5, residual=x[:1])


def test_max_pool_refuses_unsupported_arguments():
    from danet_b200.layers import max_pool2d
    x = torch.relu(torch.randn(2, 3, 9, 9))
    for args in [(2, 2, 1), (3, 1, 1), (3, 2, 0), (3, None, 1), ((3, 2), 2, 1), (3, (2, 1), 1)]:
        with pytest.raises(ValueError, match="only kernel_size=3|equal pair"):
            max_pool2d(x, *args)
    with pytest.raises(ValueError, match="only kernel_size=3"):
        max_pool2d(x, 3, 2, 1, dilation=2)
    with pytest.raises(ValueError, match="only kernel_size=3"):
        max_pool2d(x, 3, 2, 1, ceil_mode=True)
    with pytest.raises(ValueError, match="only kernel_size=3"):
        max_pool2d(x, 3, 2, 1, return_indices=True)
    with pytest.raises(ValueError, match="CUDA tensor"):
        max_pool2d(x, 3, 2, 1)
    with pytest.raises(ValueError, match="float32"):
        max_pool2d(x.double(), 3, 2, 1)
