"""CPU tests of the dense IUV losses (SURVEY section 8f-2, models/danet/iuv_estimator.py:304-341,232-255):
the numpy oracle against the golden the reference's own function produced under torch autograd, and the kernel's
per-pixel arithmetic (csrc/losses.cu compiled with DANET_LOSSES_HOST_CHECK: the same __host__ __device__ function
walked on the host) against the same golden -- no GPU involved."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import losses as olosses

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "losses.npz"))


def _weighted(grads, w):
    return {k: (None if g is None else g * wk) for (k, g), wk in zip(grads.items(), w)}


def test_oracle_body_uv_losses_match_reference_golden(gold):
    g = gold
    w = g["grad_weights"]
    for tag, has in (("all", None), ("some", g["has_some"])):
        L, gr = olosses.body_uv_losses(g["u"], g["v"], g["i"], g["a"], [g["U"], g["V"], g["I"], g["A"]], has)
        np.testing.assert_allclose(L, g["L_" + tag], rtol=2e-6)
        for k, name in zip(("u", "v", "index", "ann"), ("gu", "gv", "gi", "ga")):
            np.testing.assert_allclose(gr[k] * w[("u", "v", "index", "ann").index(k)], g["%s_%s" % (name, tag)], atol=2e-7)
    L, gr = olosses.body_uv_losses(g["u"], g["v"], g["i"], g["a"], [g["U"], g["V"], g["I"], g["A"]], np.zeros(3))
    np.testing.assert_array_equal(L, g["L_none"])
    assert all(np.abs(x).max() == 0 for x in gr.values())


def test_oracle_part_losses_match_reference_golden(gold):
    g = gold
    L, gr = olosses.part_iuv_losses(g["part_pred"], g["part_gt"], g["part_has"])
    np.testing.assert_allclose(L, g["part_L"], rtol=2e-6)
    np.testing.assert_allclose(gr * g["grad_weights"][:3].reshape(1, 1, 3, 1, 1, 1), g["part_grad"], atol=2e-7)


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc not available")
    out = str(tmp_path_factory.mktemp("losses_host") / "liblosses_host.so")
    csrc = os.path.join(ROOT, "danet-densepose2smpl_b200", "csrc")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC",
                           "-DDANET_LOSSES_HOST_CHECK", "-shared", os.path.join(csrc, "losses.cu"), os.path.join(csrc, "api.cu"),
                           "-o", out])
    lib = ctypes.CDLL(out)
    p, i32, i64, f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float
    lib.danet_test_body_uv_losses_host.argtypes = [i32, i32, i32, i32, i64, i64] + [p] * 9 + [f, f] + [p] * 5
    lib.danet_test_body_uv_losses_host.restype = ctypes.c_int
    return lib


def _host_call(lib, N, C, Cann, HW, ps, ms, u, v, i, a, U, V, I, A, has, bs, pw, grads):
    P = lambda x: None if x is None else x.ctypes.data_as(ctypes.c_void_p)
    L = np.zeros(4, np.float32)
    assert lib.danet_test_body_uv_losses_host(N, C, Cann, HW, ps, ms, P(u), P(v), P(i), P(a), P(U), P(V), P(I), P(A), P(has),
                                              bs, pw, P(L), *[P(x) for x in grads]) == 0
    return L


def test_kernel_arithmetic_on_host_matches_reference_golden(gold, hostlib):
    g = gold
    c = lambda x: np.ascontiguousarray(x, np.float32)
    u, v, i, a, U, V, I, A = (c(g[k]) for k in ("u", "v", "i", "a", "U", "V", "I", "A"))
    B, C, S = u.shape[0], u.shape[1], u.shape[2]
    w = g["grad_weights"]
    for tag, has in (("all", None), ("some", np.ascontiguousarray(g["has_some"], np.uint8)), ("none", np.zeros(3, np.uint8))):
        gr = [np.full_like(u, 7), np.full_like(v, 7), np.full_like(i, 7), np.full_like(a, 7)]
        L = _host_call(hostlib, B, C, a.shape[1], S * S, 0, 0, u, v, i, a, U, V, I, A, has, float(B), 0.5, gr)
        np.testing.assert_allclose(L, g["L_" + tag], rtol=3e-6)
        if tag == "none":
            assert all(np.abs(x).max() == 0 for x in gr)
            continue
        for k, name in enumerate(("gu", "gv", "gi", "ga")):
            np.testing.assert_allclose(gr[k] * w[k], g["%s_%s" % (name, tag)], atol=3e-7)
    # the 24-part loop as one strided walk over part_iuv_pred [B,P,3,C,S,S]
    pp, pg = c(g["part_pred"]), c(g["part_gt"])
    Bp, Pn, _, Cp = pp.shape[:4]
    HW = S * S
    has = np.repeat(np.ascontiguousarray(g["part_has"], np.uint8), Pn)
    grad = np.full_like(pp, 7)
    flat, gflat, tflat = pp.reshape(-1), grad.reshape(-1), pg.reshape(-1)
    step = Cp * HW
    L = _host_call(hostlib, Bp * Pn, Cp, 0, HW, 3 * step, 3 * step, flat, flat[step:], flat[2 * step:], None,
                   tflat, tflat[step:], tflat[2 * step:], None, has, float(Bp * Pn), 0.5,
                   [gflat, gflat[step:], gflat[2 * step:], None])
    np.testing.assert_allclose(L[:3], g["part_L"], rtol=3e-6)
    assert L[3] == 0
    np.testing.assert_allclose(grad * w[:3].reshape(1, 1, 3, 1, 1, 1), g["part_grad"], atol=3e-7)


def test_losses_module_refuses_cpu_tensors():
    import torch
    from danet_b200 import losses
    x = torch.zeros(1, 25, 4, 4)
    with pytest.raises(RuntimeError):
        losses.body_uv_losses(x, x, x, None, [x, x, x, None])
    with pytest.raises(RuntimeError):
        losses.part_iuv_losses(torch.zeros(1, 24, 3, 7, 4, 4), torch.zeros(1, 24, 3, 7, 4, 4))


def test_autograd_layer_over_a_test_double_of_the_kernel(gold, hostlib, monkeypatch):
    """Host logic of danet_b200.losses (pointer / stride arithmetic of the part layout, which gradients are requested,
    scaling by the incoming gradient) with the kernel layer replaced by the host walk of the same per-pixel function."""
    import torch
    from danet_b200 import losses

    def fake_launch(N, C, Cann, HW, ps, ms, u, v, idx, ann, U, V, I, A, has, bs, pw, dev, gu, gv, gi, ga):
        L = torch.zeros(4)
        P = lambda x: ctypes.c_void_p(x if x else 0)
        assert hostlib.danet_test_body_uv_losses_host(N, C, Cann, HW, ps, ms, P(u), P(v), P(idx), P(ann), P(U), P(V), P(I), P(A),
                                                      P(has), bs, pw, P(L.data_ptr()), P(gu), P(gv), P(gi), P(ga)) == 0
        return L

    monkeypatch.setattr(losses, "_launch", fake_launch)
    g = gold
    t = lambda k, grad=False: torch.tensor(g[k], dtype=torch.float32).requires_grad_(grad)
    w = torch.tensor(g["grad_weights"])
    u, v, i, a = t("u", True), t("v", True), t("i", True), t("a", True)
    has = losses._has_u8(torch.tensor(g["has_some"]), torch.device("cpu"))
    L = losses._BodyUvLosses.apply(u, v, i, a, t("U"), t("V"), t("I"), t("A"), has, 0.5)
    np.testing.assert_allclose(L.detach().numpy(), g["L_some"], rtol=3e-6)
    (L * w).sum().backward()
    for x, name in ((u, "gu"), (v, "gv"), (i, "gi"), (a, "ga")):
        np.testing.assert_allclose(x.grad.numpy(), g[name + "_some"], atol=3e-7)
    # only the index logits ask for a gradient; no annotation head
    i2 = t("i", True)
    L = losses._BodyUvLosses.apply(t("u"), t("v"), i2, None, t("U"), t("V"), t("I"), None, None, 0.5)
    (3 * L[2]).backward()
    np.testing.assert_allclose(i2.grad.numpy(), g["gi_all"], atol=3e-7)
    assert float(L[3].detach()) == 0.0
    # part layout
    pp = t("part_pred", True)
    hp = losses._has_u8(torch.tensor(g["part_has"]), torch.device("cpu"), repeat=pp.shape[1])
    L = losses._PartIuvLosses.apply(pp, t("part_gt"), hp, 0.5)
    np.testing.assert_allclose(L.detach().numpy(), g["part_L"], rtol=3e-6)
    (L * w[:3]).sum().backward()
    np.testing.assert_allclose(pp.grad.numpy(), g["part_grad"], atol=3e-7)


def test_kernel_arithmetic_on_host_matches_oracle_on_random_shapes(hostlib):
    """Shapes the golden does not cover: odd pixel counts, a single channel, C = 25 / 15 heads, padded image strides,
    soft (non one-hot) target maps with exact ties (first maximum wins), |d| on both sides of the smooth-L1 knee."""
    rng = np.random.default_rng(11)
    for (N, C, Ca, H, W, pad) in ((1, 1, 0, 1, 1, 0), (2, 7, 0, 3, 5, 0), (3, 25, 15, 7, 3, 13), (5, 4, 2, 2, 2, 4), (4, 25, 15, 9, 9, 0)):
        HW = H * W
        ps, ms = C * HW + pad, C * HW + 2 * pad
        f = lambda n, stride: rng.normal(0, 1.5, (n, stride)).astype(np.float32)
        u, v, i = f(N, ps), f(N, ps), f(N, ps) * 2
        U, V = f(N, ms), f(N, ms)
        I = np.maximum(f(N, ms), 0)                                    # about half the entries are exactly 0 (masked out)
        I[:, :HW] = I[:, HW:2 * HW] if C > 1 else I[:, :HW]            # channel 0 ties channel 1: argmax must take channel 0
        a = f(N, Ca * HW) if Ca else None
        A = np.abs(f(N, Ca * HW)) if Ca else None
        has = (rng.random(N) > 0.3).astype(np.uint8)
        has[0] = 1
        view = lambda x, stride, c: x[:, :c * HW].reshape(N, c, H, W)
        Lr, gr = olosses.body_uv_losses(view(u, ps, C), view(v, ps, C), view(i, ps, C), view(a, 0, Ca) if Ca else None,
                                        [view(U, ms, C), view(V, ms, C), view(I, ms, C), view(A, 0, Ca) if Ca else None], has)
        gu, gv, gi = np.full_like(u, 7), np.full_like(v, 7), np.full_like(i, 7)
        ga = np.full_like(a, 7) if Ca else None
        L = _host_call(hostlib, N, C, Ca, HW, ps, ms, u, v, i, a, U, V, I, A, has, float(N), 0.5, [gu, gv, gi, ga])
        np.testing.assert_allclose(L, Lr, rtol=5e-6, atol=1e-7)
        for got, ref, c in ((gu, gr["u"], C), (gv, gr["v"], C), (gi, gr["index"], C)):
            np.testing.assert_allclose(got[:, :c * HW].reshape(N, c, H, W), ref, atol=2e-7)
            assert np.all(got[:, c * HW:] == 7)                         # the padding between images is never written
        if Ca:
            np.testing.assert_allclose(ga.reshape(N, Ca, H, W), gr["ann"], atol=2e-7)
