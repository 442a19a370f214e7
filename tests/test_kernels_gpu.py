"""GPU unit parity of the network-half kernels (csrc/conv_simt.cu, conv_tc.cu, glue.cu) against a
plain torch fp32 reference of the same op (oracle/net_ops.py restates each op with torch)."""
import numpy as np
import pytest
import torch

from oracle.net_ops import TorchEmulOps

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from danet_b200.plan import CudaOps
    return CudaOps(DEV)


CONV_CASES = [
    # N, H, W, Cin, Cout, k, stride, wsets, relu, residual
    (2, 56, 56, 48, 48, 3, 1, 1, 1, 1),
    (2, 28, 28, 96, 96, 3, 1, 1, 1, 1),
    (3, 14, 14, 192, 192, 3, 1, 1, 0, 0),
    (2, 7, 7, 384, 384, 3, 1, 1, 1, 1),
    (2, 56, 56, 64, 256, 1, 1, 1, 1, 1),
    (2, 56, 56, 256, 64, 1, 1, 1, 1, 0),
    (2, 56, 56, 48, 96, 3, 2, 1, 0, 0),
    (1, 224, 224, 4, 64, 3, 2, 1, 1, 0),
    (2, 56, 56, 64, 64, 7, 2, 1, 1, 0),
    (48, 56, 56, 48, 24, 3, 1, 24, 0, 0),
    (48, 4, 4, 256, 128, 3, 2, 24, 1, 0),
    (48, 4, 4, 256, 128, 1, 2, 24, 0, 0),
    (2, 56, 56, 48, 92, 3, 1, 1, 0, 0),
    (2, 56, 56, 76, 64, 1, 1, 1, 1, 0),
    (5, 13, 9, 20, 36, 3, 1, 1, 1, 1),          # ragged: nothing divides the tile sizes
    (2, 14, 14, 64, 64, 3, 1, 1, 1, 1),
    (2, 28, 28, 64, 128, 3, 2, 1, 1, 0),
    (2, 28, 28, 64, 128, 1, 2, 1, 0, 0),
]


def A(t):
    """fp32 tensor -> plan.ActBuf with only the fp32 view."""
    from danet_b200.plan import ActBuf
    return ActBuf(f32=t)


def H(x, planes=2):
    """fp32 cuda tensor -> plan.ActBuf with split-fp16 planes only (through danet_act_split)."""
    from danet_b200.plan import ActBuf
    from conv_tc_common import split
    hi, lo = split(x, want_lo=planes == 2)
    return ActBuf(h=torch.stack([hi, lo]) if planes == 2 else hi[None])


def Hempty(shape, planes=2):
    from danet_b200.plan import ActBuf
    return ActBuf(h=torch.full((planes,) + tuple(shape), float("nan"), dtype=torch.float16, device=DEV))


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_simt(case):
    N, H_, W, Cin, Cout, k, s, G, relu, has_res = case
    ops, ref = _ops(), TorchEmulOps()
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    d = dict(N=N, H=H_, W=W, Cin=Cin, Cout=Cout, ksize=k, stride=s, pad=k // 2, wsets=G, relu=relu)
    Ho, Wo = (H_ + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
    x = torch.randn(N, H_, W, Cin, generator=g)
    w = torch.randn(G, k * k * Cin, Cout, generator=g) * (1.0 / (k * k * Cin)) ** 0.5
    b = torch.randn(G, Cout, generator=g) * 0.1
    res = torch.randn(N, Ho, Wo, Cout, generator=g) if has_res else None
    y_ref = torch.empty(N, Ho, Wo, Cout)
    ref.conv2d(d, A(x), w, b, A(res) if has_res else None, A(y_ref))
    y = torch.full((N, Ho, Wo, Cout), float("nan"), device=DEV)
    ops.conv2d(d, A(x.to(DEV)), w.to(DEV), b.to(DEV), A(res.to(DEV)) if has_res else None, A(y))
    torch.cuda.synchronize()
    err = (y.cpu() - y_ref).abs().max().item()
    assert err < 2e-5, (case, err)


# the tensor-core kernel needs channel counts that are multiples of 8 (the graph pads to 8)
TC_CASES = [c for c in CONV_CASES if c[3] % 8 == 0 and c[4] % 8 == 0] + [
    (1, 224, 224, 8, 64, 3, 2, 1, 1, 0),          # the stem: 3 (padded to 8) -> 64, stride 2
    (48, 2, 2, 128, 128, 3, 1, 24, 1, 1),         # limb_reslayer: 2x2 maps, 24 weight sets
    (2, 2, 2, 512, 512, 3, 1, 1, 1, 1),           # body_net layer4: 2x2 maps
    (2, 16, 8, 16, 16, 1, 1, 1, 0, 0),            # a single tile, a single K step
    (5, 13, 9, 24, 40, 3, 1, 1, 1, 1),            # ragged: nothing divides the tile sizes
    (13, 7, 7, 64, 64, 3, 1, 1, 1, 1),            # small maps: several images share a tile (2 per tile, ragged batch)
    (7, 4, 4, 64, 64, 3, 1, 1, 1, 1),             # 3 images per tile
    (11, 2, 2, 32, 48, 3, 1, 1, 1, 1),            # 5 images per tile
    (9, 4, 4, 32, 32, 1, 1, 1, 0, 0),             # 1x1 on 4x4 maps: 4 images per tile, no zero rows
]


@pytest.mark.parametrize("case", TC_CASES)
@pytest.mark.parametrize("exact", [1, 0])
def test_conv_tc(case, exact):
    """exact: split-fp16 operands, 3 MMAs -> fp32-grade (the residual is the tensor core's truncating fp32
    accumulation, growing with K); fast: single fp16 pass (10-bit mantissa operands)."""
    from conv_tc_common import run_case
    K = case[5] * case[5] * case[3]
    y, ym, ref = run_case(case, bool(exact), res_as_planes=bool(hash(case) & 1))
    tol = (2e-5 + 1.5e-8 * K) if exact else 1.5e-2
    e1, e2 = (y.double() - ref).abs().max().item(), (ym.double() - ref).abs().max().item()
    assert not torch.isnan(y).any() and e1 < tol and e2 < tol, (case, exact, e1, e2)


def test_conv_tc_multi_problem_launch():
    """Several independent convolutions (HRNet's branches at one depth: different resolutions, channel counts,
    one with a residual, one stride-2) in ONE launch == each launched alone, bit for bit."""
    from conv_tc_common import desc, launch, make_case, merge, pack, problem, split
    cases = [(2, 56, 56, 48, 48, 3, 1, 1, 1, 1), (2, 28, 28, 96, 96, 3, 1, 1, 1, 0), (2, 14, 14, 192, 192, 3, 1, 1, 0, 1),
             (2, 7, 7, 384, 384, 3, 1, 1, 1, 1), (2, 56, 56, 48, 96, 3, 2, 1, 0, 0), (2, 14, 14, 192, 48, 1, 1, 1, 0, 0)]
    for exact in (True, False):
        probs, outs, keep = [], [], []
        for c in cases:
            N, Hh, W, Cin, Cout, k, s, G, relu, has_res = c
            x, w, b, res = make_case(c, seed=3)
            d = desc(c, exact)
            xp = split(x.to(DEV), want_lo=exact)
            wpk, bc = pack(d, w.to(DEV)), b.to(DEV)
            rp = split(res.to(DEV), want_lo=exact) if has_res else None
            Ho, Wo = (Hh + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
            mk = lambda: (torch.full((N, Ho, Wo, Cout), float("nan"), dtype=torch.float16, device=DEV),
                          torch.full((N, Ho, Wo, Cout), float("nan"), dtype=torch.float16, device=DEV) if exact else None)
            y_group, y_single = mk(), mk()
            probs.append(problem(d, xp, wpk, bc, res_planes=rp, y_planes=y_group))
            launch([problem(d, xp, wpk, bc, res_planes=rp, y_planes=y_single)])
            outs.append((y_group, y_single))
            keep.append((xp, wpk, bc, rp))
        launch(probs)
        torch.cuda.synchronize()
        for (yg, ys), c in zip(outs, cases):
            assert torch.equal(yg[0], ys[0]) and (not exact or torch.equal(yg[1], ys[1])), (c, exact)
            assert not torch.isnan(merge(*yg)).any()


def test_conv_rejects_bad_arguments():
    ops = _ops()
    d = dict(N=1, H=8, W=8, Cin=3, Cout=8, ksize=3, stride=1, pad=1, wsets=1, relu=0)
    x = torch.zeros(1, 8, 8, 3, device=DEV)
    with pytest.raises(RuntimeError):
        ops.conv2d(d, A(x), x, None, None, A(x))        # Cin % 4 != 0
    d = dict(N=1, H=8, W=8, Cin=12, Cout=8, ksize=3, stride=1, pad=1, wsets=1, relu=0)
    assert not ops.conv_tc_supported(d)                 # tensor-core path: channels must be multiples of 8
    with pytest.raises(RuntimeError):
        ops.conv_tc_pack(d, torch.zeros(1, 108, 8, device=DEV))


def test_glue_kernels_vs_torch():
    ops, ref = _ops(), TorchEmulOps()
    g = torch.Generator().manual_seed(7)
    B, S, C = 3, 56, 48
    # fuse_sum with upsampling
    t0, t1, t2 = torch.randn(B, 28, 28, C, generator=g), torch.randn(B, 14, 14, C, generator=g), torch.randn(B, 7, 7, C, generator=g)
    y_ref = torch.empty(B, 28, 28, C); ref.fuse_sum([A(t0), A(t1), A(t2)], [1, 2, 4], True, A(y_ref))
    y = torch.empty(B, 28, 28, C, device=DEV)
    ops.fuse_sum([A(t0.to(DEV)), A(t1.to(DEV)), A(t2.to(DEV))], [1, 2, 4], True, A(y), (B, 28, 28, C))
    assert torch.equal(y.cpu(), y_ref)
    # split-fp16 planes in, planes + fp32 out: the planes carry 22 bits of every value
    from danet_b200.plan import ActBuf
    yh = Hempty((B, 28, 28, C)); yh.f32 = torch.empty(B, 28, 28, C, device=DEV)
    ops.fuse_sum([H(t0.to(DEV)), H(t1.to(DEV)), H(t2.to(DEV))], [1, 2, 4], True, yh, (B, 28, 28, C))
    assert (yh.f32.cpu() - y_ref).abs().max() < 4e-6
    assert (ActBuf(h=yh.h).value().cpu() - yh.f32.cpu()).abs().max() < 2e-6
    yh1 = Hempty((B, 28, 28, C), planes=1)
    ops.fuse_sum([H(t0.to(DEV), 1), H(t1.to(DEV), 1), A(t2.to(DEV))], [1, 2, 4], True, yh1, (B, 28, 28, C))
    want = torch.relu(t0.half().float() + t1.half().float().repeat_interleave(2, 1).repeat_interleave(2, 2)
                      + t2.repeat_interleave(4, 1).repeat_interleave(4, 2)).half()
    assert (yh1.h[0].cpu().float() - want.float()).abs().max() < 4e-3
    # maxpool / avgpool / linear / nchw->nhwc
    x = torch.randn(B, 28, 28, 64, generator=g)
    y_ref = torch.empty(B, 14, 14, 64); ref.maxpool(A(x), A(y_ref))
    y = torch.empty(B, 14, 14, 64, device=DEV); ops.maxpool(A(x.to(DEV)), A(y), (B, 28, 28, 64))
    assert torch.equal(y.cpu(), y_ref)
    yh = Hempty((B, 14, 14, 64)); ops.maxpool(H(x.to(DEV)), yh, (B, 28, 28, 64))
    assert (yh.value().cpu() - y_ref).abs().max() < 2e-6
    x = torch.randn(B, 2, 2, 512, generator=g)
    y_ref = torch.empty(B, 512); ref.avgpool(A(x), y_ref)
    y = torch.empty(B, 512, device=DEV); ops.avgpool(A(x.to(DEV)), y, (B, 2, 2, 512))
    assert (y.cpu() - y_ref).abs().max() < 1e-6
    y2 = torch.empty(B, 512, device=DEV); ops.avgpool(H(x.to(DEV)), y2, (B, 2, 2, 512))
    assert (y2.cpu() - y_ref).abs().max() < 2e-6
    w, b, add = torch.randn(13, 512, generator=g), torch.randn(13, generator=g), torch.randn(13, generator=g)
    o_ref = torch.empty(B, 13); ref.linear(y_ref, w, b, add, o_ref)
    o = torch.empty(B, 13, device=DEV); ops.linear(y, w.to(DEV), b.to(DEV), add.to(DEV), o)
    assert (o.cpu() - o_ref).abs().max() < 1e-4
    img = torch.randn(B, 3, 20, 20, generator=g)
    n_ref = torch.empty(B, 20, 20, 8); ref.nchw_to_nhwc(img, A(n_ref))
    n = torch.empty(B, 20, 20, 8, device=DEV); ops.nchw_to_nhwc(img.to(DEV), A(n))
    assert torch.equal(n.cpu(), n_ref)
    nh = Hempty((B, 20, 20, 8)); ops.nchw_to_nhwc(img.to(DEV), nh)
    assert (nh.value().cpu() - n_ref).abs().max() < 2e-6 and torch.equal(nh.h[0].cpu(), n_ref.half())


def test_clean_and_stn_kernels_vs_torch():
    ops, ref = _ops(), TorchEmulOps()
    g = torch.Generator().manual_seed(8)
    B, S, C = 3, 56, 48
    heads = torch.randn(B, S, S, 96, generator=g)
    heads[0, 0, 0, 50:75] = 1.0                      # exact tie -> first index
    body_r, amax_r = torch.empty(B, S, S, 80), torch.empty(B, S, S, dtype=torch.uint8)
    vis_r = [torch.empty(B, c, S, S) for c in (25, 25, 25, 15)]
    ref.clean_global(A(heads), A(body_r), amax_r, vis_r)
    body, amax = torch.empty(B, S, S, 80, device=DEV), torch.empty(B, S, S, dtype=torch.uint8, device=DEV)
    vis = [torch.empty(B, c, S, S, device=DEV) for c in (25, 25, 25, 15)]
    bb = Hempty((B, S, S, 80)); bb.f32 = body
    ops.clean_global(A(heads.to(DEV)), bb, amax, vis, (B, S, S, 96, 80))
    assert torch.equal(amax.cpu(), amax_r) and torch.equal(body.cpu(), body_r)
    from danet_b200.plan import ActBuf
    assert (ActBuf(h=bb.h).value().cpu() - body_r).abs().max() < 2e-6          # fp32 view and planes written together
    for a, b in zip(vis, vis_r):
        assert torch.equal(a.cpu(), b)
    x = torch.randn(B * 24, S, S, 24, generator=g)
    y_r, raw_r = torch.empty(B * 24, S, S, 24), torch.empty(B * 24, 21, S, S)
    ref.clean_parts(A(x), A(y_r), raw_r)
    y, raw = torch.empty(B * 24, S, S, 24, device=DEV), torch.empty(B * 24, 21, S, S, device=DEV)
    ops.clean_parts(A(x.to(DEV)), A(y), raw, (B * 24, S, S, 24, 24))
    assert torch.equal(y.cpu(), y_r) and torch.equal(raw.cpu(), raw_r)
    y16 = Hempty((B * 24, S, S, 24))                                                            # split-fp16 planes
    ops.clean_parts(A(x.to(DEV)), y16, None, (B * 24, S, S, 24, 24))
    assert torch.equal(y16.h[0].cpu(), y_r.to(torch.float16)) and (y16.value().cpu() - y_r).abs().max() < 2e-6
    # stn params + sampling, both align_corners conventions
    hm = torch.randn(B, S, S, 24, generator=g) * 0.3
    ratio, offset = torch.rand(24, generator=g) + 0.5, torch.rand(24, generator=g) * 0.2
    xd = torch.randn(B, S, S, C, generator=g)
    for ac in (0, 1):
        c_r, th_r = torch.empty(B, 1, 24, 2), torch.empty(B, 1, 24, 3)
        ref.stn_params(A(hm), amax_r, ratio, offset, 0.5, ac, c_r, th_r)
        c, th = torch.empty(B, 1, 24, 2, device=DEV), torch.empty(B, 1, 24, 3, device=DEV)
        ops.stn_params(A(hm.to(DEV)), amax, ratio.to(DEV), offset.to(DEV), 0.5, ac, c, th)
        assert (c.cpu() - c_r).abs().max() < 2e-5 and (th.cpu() - th_r).abs().max() < 2e-5
        crops_r = torch.empty(B * 24, S, S, C); ref.stn_sample(A(xd), th_r, ac, A(crops_r))
        crops = torch.empty(B * 24, S, S, C, device=DEV)
        ops.stn_sample(A(xd.to(DEV)), th_r.to(DEV), ac, A(crops), (B, S, C))
        assert (crops.cpu() - crops_r).abs().max() < 2e-4
        crops16 = Hempty((B * 24, S, S, C))
        ops.stn_sample(A(xd.to(DEV)), th_r.to(DEV), ac, crops16, (B, S, C))
        assert torch.equal(crops16.h[0], crops.to(torch.float16))           # same values, RN-rounded
        assert (crops16.value() - crops).abs().max() < 2e-6
        crops_h = Hempty((B * 24, S, S, C))                                  # planes in, planes out
        ops.stn_sample(H(xd.to(DEV)), th_r.to(DEV), ac, crops_h, (B, S, C))
        assert (crops_h.value() - crops).abs().max() < 4e-6


def test_gcn_pose_head_vs_torch():
    from danet_b200 import netgraph as ng
    ops, ref = _ops(), TorchEmulOps()
    g = torch.Generator().manual_seed(9)
    B = 5
    gb = ng.graph_buffers()
    adj = torch.stack([torch.from_numpy(gb["r2p_A"][0]), torch.from_numpy(ng.undigraph_normalize(gb["A_mask"][0] + np.eye(24)).astype(np.float32)),
                       torch.from_numpy(gb["p2r_A"][0])]).float()
    dims = [(128, 128), (128, 256), (256, 256), (256, 128), (128, 128)]
    gp = {"adj": adj, "W": [torch.randn(i, o, generator=g) * (1.0 / i) ** 0.5 for i, o in dims],
          "b": [torch.randn(o, generator=g) * 0.1 for _, o in dims],
          "bn_scale": [torch.rand(24, generator=g) + 0.5 for _ in dims], "bn_shift": [torch.randn(24, generator=g) * 0.1 for _ in dims],
          "head_w": torch.randn(144, 128, generator=g) * 0.1, "head_b": torch.randn(144, generator=g) * 0.1,
          "mean_pose": torch.tensor([1., 0, 0, 1, 0, 0] * 24)}
    rot = torch.randn(B * 24, 1, 1, 128, generator=g)
    gpara = torch.randn(B, 1, 1, 13, generator=g)
    p_ref = torch.empty(B, 1, 1, 229); ref.gcn_head(gp, rot, gpara, p_ref)
    gpc = {k: ([t.to(DEV) for t in v] if isinstance(v, list) else v.to(DEV)) for k, v in gp.items()}
    p = torch.empty(B, 1, 1, 229, device=DEV); ops.gcn_head(gpc, rot.to(DEV), gpara.to(DEV), p)
    assert (p.cpu() - p_ref).abs().max() < 5e-5
