"""Helpers of the tensor-core convolution tests: run one convolution through the C ABI
(danet_conv_tc_group, split-fp16 activations) and return the result next to an fp64 torch reference."""
import ctypes

import torch
import torch.nn.functional as F

DEV = "cuda:0"


def lib():
    from danet_b200 import _lib
    return _lib


def split(x, want_lo=True):
    """fp32 [..] cuda tensor -> (hi, lo) fp16 planes through danet_act_split."""
    L = lib()
    hi = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    lo = torch.empty(x.shape, dtype=torch.float16, device=x.device) if want_lo else None
    L.check(L.load().danet_act_split(x.numel(), L.ptr(x), L.ptr(hi), L.ptr(lo), L.stream_ptr()), "act_split")
    return hi, lo


def merge(hi, lo):
    L = lib()
    y = torch.empty(hi.shape, dtype=torch.float32, device=hi.device)
    L.check(L.load().danet_act_merge(hi.numel(), L.ptr(hi), L.ptr(lo), L.ptr(y), L.stream_ptr()), "act_merge")
    return y


def desc(case, exact):
    L = lib()
    N, H, W, Cin, Cout, k, s, G, relu, _ = case
    d = L.ConvDesc()
    d.N, d.H, d.W, d.Cin, d.Cout, d.ksize, d.stride, d.pad, d.wsets, d.relu = N, H, W, Cin, Cout, k, s, k // 2, G, relu
    d.flags = 4 if exact else 0
    return d


def pack(d, w):
    L = lib()
    nbytes = int(L.load().danet_conv_tc_packed_bytes(ctypes.byref(d)))
    assert nbytes > 0, "shape not supported by the tensor-core path"
    out = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
    L.check(L.load().danet_conv_tc_pack(ctypes.byref(d), L.ptr(w), L.ptr(out), L.stream_ptr()), "conv_tc_pack")
    return out


def make_case(case, seed=None):
    """Deterministic inputs of one case: x [N,H,W,Cin], w [G,k*k*Cin,Cout], b [G,Cout], res or None (CPU fp32)."""
    N, H, W, Cin, Cout, k, s, G, relu, has_res = case
    g = torch.Generator().manual_seed((hash(case) if seed is None else seed) & 0xFFFF)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    x = torch.randn(N, H, W, Cin, generator=g)
    w = torch.randn(G, k * k * Cin, Cout, generator=g) * (1.0 / (k * k * Cin)) ** 0.5
    b = torch.randn(G, Cout, generator=g) * 0.1
    res = torch.randn(N, Ho, Wo, Cout, generator=g) if has_res else None
    return x, w, b, res


def reference(case, x, w, b, res, dtype=torch.float64):
    N, H, W, Cin, Cout, k, s, G, relu, has_res = case
    xs = x.to(dtype).permute(0, 3, 1, 2)
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    out = torch.empty(N, Cout, Ho, Wo, dtype=dtype)
    for g in range(G):
        wg = w[g].to(dtype).reshape(k, k, Cin, Cout).permute(3, 2, 0, 1)
        out[g::G] = F.conv2d(xs[g::G], wg, b[g].to(dtype), stride=s, padding=k // 2)
    out = out.permute(0, 2, 3, 1)
    if res is not None:
        out = out + res.to(dtype)
    if relu:
        out = torch.relu(out)
    return out


def problem(d, x_planes, wpk, bias, res=None, res_planes=None, y_f32=None, y_planes=None):
    L = lib()
    p = L.ConvProblem()
    p.d = d
    p.x = L.Act(None, x_planes[0].data_ptr(), x_planes[1].data_ptr() if x_planes[1] is not None else None)
    if res is not None:
        p.res = L.Act(res.data_ptr(), None, None)
    elif res_planes is not None:
        p.res = L.Act(None, res_planes[0].data_ptr(), res_planes[1].data_ptr() if res_planes[1] is not None else None)
    else:
        p.res = L.Act(None, None, None)
    p.y = L.Act(y_f32.data_ptr() if y_f32 is not None else None,
                y_planes[0].data_ptr() if y_planes is not None else None,
                y_planes[1].data_ptr() if (y_planes is not None and y_planes[1] is not None) else None)
    p.w_packed = wpk.data_ptr()
    p.bias = bias.data_ptr() if bias is not None else None
    return p


def launch(problems):
    L = lib()
    arr = (L.ConvProblem * len(problems))(*problems)
    L.check(L.load().danet_conv_tc_group(len(problems), arr, L.stream_ptr()), "conv_tc_group")


def run_case(case, exact, res_as_planes=False, seed=None):
    """Returns (y_f32 from the kernel, merged output planes, fp64 reference), all CPU."""
    N, H, W, Cin, Cout, k, s, G, relu, has_res = case
    x, w, b, res = make_case(case, seed)
    ref = reference(case, x, w, b, res)
    d = desc(case, exact)
    xc, wc, bc = x.to(DEV), w.to(DEV), b.to(DEV)
    xp = split(xc, want_lo=exact)
    wpk = pack(d, wc)
    Ho, Wo = ref.shape[1], ref.shape[2]
    y = torch.full((N, Ho, Wo, Cout), float("nan"), device=DEV)
    yh = torch.full((N, Ho, Wo, Cout), float("nan"), dtype=torch.float16, device=DEV)
    yl = torch.full((N, Ho, Wo, Cout), float("nan"), dtype=torch.float16, device=DEV) if exact else None
    rc = res.to(DEV) if has_res else None
    rp = split(rc, want_lo=exact) if (has_res and res_as_planes) else None
    p = problem(d, xp, wpk, bc, res=None if res_as_planes else rc, res_planes=rp, y_f32=y, y_planes=(yh, yl))
    launch([p])
    torch.cuda.synchronize()
    return y.cpu(), merge(yh, yl).cpu(), ref


def prepare(case, exact, x, w, b, res, res_kind="f32", out_kind="both"):
    """One problem of a launch from CPU tensors, with the residual as res_kind (none | f32 | planes; fast mode's planes
    are the hi plane alone), the outputs of out_kind (f32 | planes | both), NaN-filled, and b = None for a NULL bias.
    Returns (problem, (y_f32, y_hi, y_lo), tensors the launch needs alive)."""
    N, H, W, Cin, Cout, k, s = case[:7]
    Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    d = desc(case, exact)
    xp = split(x.to(DEV), want_lo=exact)
    wpk = pack(d, w.to(DEV))
    bc = b.to(DEV) if b is not None else None
    rc = res.to(DEV) if (res is not None and res_kind != "none") else None
    rp = split(rc, want_lo=exact) if (rc is not None and res_kind == "planes") else None
    nan = lambda dt: torch.full((N, Ho, Wo, Cout), float("nan"), dtype=dt, device=DEV)
    y = nan(torch.float32) if out_kind in ("f32", "both") else None
    yh = nan(torch.float16) if out_kind in ("planes", "both") else None
    yl = nan(torch.float16) if (yh is not None and exact) else None
    p = problem(d, xp, wpk, bc, res=rc if rp is None else None, res_planes=rp, y_f32=y,
                y_planes=(yh, yl) if yh is not None else None)
    return p, (y, yh, yl), (xp, wpk, bc, rc, rp)


def collect(outs):
    """(y_f32, y_hi, y_lo) of prepare, after the launch -> {view name: CPU tensor}: f32, hi, lo, planes (merged)"""
    y, yh, yl = outs
    r = {}
    if y is not None:
        r["f32"] = y.cpu()
    if yh is not None:
        r["hi"] = yh.cpu()
        if yl is not None:
            r["lo"] = yl.cpu()
        r["planes"] = merge(yh, yl).cpu()
    return r
