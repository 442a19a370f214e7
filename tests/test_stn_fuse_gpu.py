"""GPU tests of danet_b200.layers.hr_fuse and danet_b200.stn (part_crops, part_thetas): the fuse bit-identical to
torch fp32 at every HRNet fuse site of W48 and W32 and its backward within its stated bound of fp64; the crops against
a tight fp64 oracle over the kernel's own fp32 coordinates (forward and backward) and loosely against torch's
affine_grid + grid_sample; the thetas against the reference's golden; repeatability, CUDA-graph replay, gradient
subsets, batch independence and refused arguments."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import stn_train as oracle

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _fuse_sites(width):
    """(stage, output i, [(C, h, factor)] per term) of the 23 fuse outputs of HRNet-W<width> at 224 x 224 input:
    2 in stage 2, 4 modules x 3 in stage 3, 4 + 4 + 1 in stage 4 (the last module keeps only output 0)"""
    C = [width * 2 ** k for k in range(4)]
    H = [56, 28, 14, 7]
    sites = []
    for stage, nb, outs in ((2, 2, [2]), (3, 3, [3, 3, 3, 3]), (4, 4, [4, 4, 1])):
        for nout in outs:
            for i in range(nout):
                sites.append((stage, i, [(C[i], H[max(i, j)], 2 ** (j - i) if j > i else 1) for j in range(nb)]))
    assert len(sites) == 23
    return sites


def _terms(site, B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(B, c, h, h, generator=g, device=DEV) for (c, h, f) in site[2]], [f for (_, _, f) in site[2]]


def _torch_fuse(terms, factors):
    y = None
    for t, f in zip(terms, factors):
        u = F.interpolate(t, scale_factor=f, mode="nearest") if f > 1 else t
        y = u if y is None else y + u
    return torch.relu(y)


@pytest.mark.parametrize("B", [2, 16])
@pytest.mark.parametrize("width", [48, 32])
def test_fuse_forward_bit_identical_at_every_site(width, B):
    from danet_b200.layers import hr_fuse
    for k, site in enumerate(_fuse_sites(width)):
        terms, factors = _terms(site, B, k)
        assert torch.equal(hr_fuse(terms, factors), _torch_fuse(terms, factors)), site


@pytest.mark.parametrize("width", [48, 32])
def test_fuse_backward_within_bound_of_fp64(width):
    from danet_b200.layers import hr_fuse
    worst = 0.0
    for k, site in enumerate(_fuse_sites(width)):
        terms, factors = _terms(site, 2, 100 + k)
        leaves = [t.clone().requires_grad_() for t in terms]
        y = hr_fuse(leaves, factors)
        gy = torch.randn(y.shape, generator=torch.Generator(device=DEV).manual_seed(k), device=DEV)
        y.backward(gy)
        d = [t.double().requires_grad_() for t in terms]
        yr = _torch_fuse(d, factors)
        yr.backward(gy.double())
        for t, r, f in zip(leaves, d, factors):
            N, C, h, w = t.shape
            absdy = (gy.double().abs() * (yr > 0)).reshape(N, C, h, f, w, f).sum((3, 5))
            bound = (f * f - 1) * 2.0 ** -24 * absdy             # f = 1: exact
            err = (t.grad.double() - r.grad).abs()
            assert (err <= bound).all(), (site, f)
            if f > 1:
                worst = max(worst, float((err / bound.clamp_min(1e-300)).max()))
    print("fuse backward: worst error / ((f^2 - 1) 2^-24 sum|dy|) = %.3f" % worst)


def test_fuse_exact_zero_sums_get_no_gradient():
    from danet_b200.layers import hr_fuse
    g = torch.Generator(device=DEV).manual_seed(7)
    a = torch.randn(2, 8, 4, 4, generator=g, device=DEV)
    b = -F.interpolate(a, scale_factor=2, mode="nearest")                  # a + b == +0 exactly everywhere
    b[:, :, :2] = b[:, :, :2] + 1.0                                        # except the top rows
    la, lb = a.clone().requires_grad_(), b.clone().requires_grad_()
    y = hr_fuse([lb, la], [1, 2])
    gy = torch.ones_like(y)
    y.backward(gy)
    ta, tb = a.clone().requires_grad_(), b.clone().requires_grad_()
    yt = torch.relu(tb + F.interpolate(ta, scale_factor=2, mode="nearest"))
    yt.backward(gy)
    assert torch.equal(y, yt) and (y[:, :, 2:] == 0).all()
    assert torch.equal(lb.grad, tb.grad) and torch.equal(la.grad, ta.grad)
    assert (lb.grad[:, :, 2:] == 0).all()


def test_fuse_without_relu_and_unaligned_terms():
    from danet_b200.layers import hr_fuse
    g = torch.Generator(device=DEV).manual_seed(8)
    big = torch.randn(2 * 3 * 12 * 12 + 1, generator=g, device=DEV)
    t0 = big[1:].reshape(2, 3, 12, 12)                                     # 4-byte offset: the scalar paths
    t1 = torch.randn(2, 3, 6, 6, generator=g, device=DEV)
    t2 = torch.randn(2, 3, 3, 3, generator=g, device=DEV)
    l = [t.clone().requires_grad_() for t in (t1, t2)]
    y = hr_fuse([t0, l[0], l[1]], [1, 2, 4], relu=False)
    yr = t0 + F.interpolate(t1, scale_factor=2) + F.interpolate(t2, scale_factor=4)
    assert torch.equal(y, yr)
    gy = torch.randn(y.shape, generator=g, device=DEV)
    y.backward(gy)
    assert torch.allclose(l[0].grad, gy.reshape(2, 3, 6, 2, 6, 2).sum((3, 5)), atol=1e-5)
    assert torch.allclose(l[1].grad, gy.reshape(2, 3, 3, 4, 3, 4).sum((3, 5)), atol=1e-5)


# ------------------------------------------------------------------------------------------------
# part crops
# ------------------------------------------------------------------------------------------------
def _realistic_thetas(B, seed):
    from danet_b200.stn import part_thetas
    g = torch.Generator(device=DEV).manual_seed(seed)
    S = 56
    yy, xx = torch.meshgrid(torch.arange(S, device=DEV), torch.arange(S, device=DEV), indexing="ij")
    c = torch.rand(B, 24, 2, generator=g, device=DEV) * (S - 12) + 6
    hm = torch.exp(-((xx - c[..., 0, None, None]) ** 2 + (yy - c[..., 1, None, None]) ** 2) / 8.0)
    idx = torch.randn(B, 25, S // 8, S // 8, generator=g, device=DEV).repeat_interleave(8, 2).repeat_interleave(8, 3)
    ratio = torch.rand(24, generator=g, device=DEV) + 0.5
    off = torch.rand(24, generator=g, device=DEV) * 0.1
    return part_thetas(hm.contiguous(), idx.contiguous(), ratio, off,
                       center_noise=torch.rand(B, 24, 2, generator=g, device=DEV),
                       scale_noise=torch.rand(24, 2, B, generator=g, device=DEV))[1]


DEGENERATE = [(0.0, 0.0, 0.0, 0.3), (0.0, 0.5, 0.0, -0.2), (1e-7, 0.1, 1e-6, -0.3), (3e-4, 0.0, 2e-3, 0.7),
              (1.7, 0.2, 2.5, -0.1), (0.4, 1.6, 0.4, -1.8), (0.3, 30.0, 0.3, 0.0), (3e7, 0.1, 0.5, 3e9),
              (-0.5, 0.2, 0.6, 0.1), (1.0, 0.0, 1.0, 0.0)]


def _degenerate_thetas(B):
    th = torch.zeros(B, 24, 2, 3, device=DEV)
    for k in range(24):
        sx, cx, sy, cy = DEGENERATE[k % len(DEGENERATE)]
        th[:, k, 0, 0], th[:, k, 0, 2], th[:, k, 1, 1], th[:, k, 1, 2] = sx, cx, sy, cy
    return th


def _crop_case(kind, B, C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    xd = torch.randn(B, C, 56, 56, generator=g, device=DEV)
    th = _realistic_thetas(B, seed) if kind == "realistic" else _degenerate_thetas(B)
    return xd, th


@pytest.mark.parametrize("align", [False, True], ids=["align0", "align1"])
@pytest.mark.parametrize("kind", ["realistic", "degenerate"])
@pytest.mark.parametrize("B,C", [(1, 32), (16, 48)])
def test_part_crops_against_fp64_oracle(kind, align, B, C):
    from danet_b200.stn import part_crops
    xd, th = _crop_case(kind, B, C, 11)
    leaf = xd.clone().requires_grad_()
    y = part_crops(leaf, th, align_corners=align)
    gy = torch.randn(y.shape, generator=torch.Generator(device=DEV).manual_seed(5), device=DEV)
    y.backward(gy)
    imgs = [0] if B == 1 else [0, B - 1]                 # the others: test_part_crops_batch_independent
    sel = lambda t: t[imgs].cpu().numpy()
    ref, dref, scale, dscale = oracle.part_crops(sel(xd), sel(th), align, dcrops=sel(gy))
    err = np.abs(sel(y.detach()) - ref)
    assert (err <= 2.0 ** -22 * scale + 1e-30).all(), err.max()
    derr = np.abs(sel(leaf.grad) - dref)
    dbound = 2.0 ** -24 * np.abs(dref) + 2.0 ** -45 * dscale
    assert (derr <= dbound + 1e-38).all(), (derr / np.maximum(dbound, 1e-38)).max()
    # torch, loosely: its affine_grid rounds the coordinates differently (a batched matmul)
    if kind == "realistic":
        tl = []
        for i in range(24):
            grid = F.affine_grid(th[:, i], list(xd.shape), align_corners=align)
            tl.append(F.grid_sample(xd, grid, align_corners=align))
        assert torch.allclose(y.detach(), torch.cat(tl, 1), atol=1e-4)


def test_part_crops_backward_against_torch_autograd():
    from danet_b200.stn import part_crops
    xd, th = _crop_case("realistic", 2, 32, 3)
    gy = torch.randn(2, 24 * 32, 56, 56, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
    a = xd.clone().requires_grad_()
    part_crops(a, th).backward(gy)
    b = xd.double().requires_grad_()
    torch.cat([F.grid_sample(b, F.affine_grid(th[:, i].double(), list(b.shape), align_corners=False), align_corners=False)
               for i in range(24)], 1).backward(gy.double())
    assert torch.allclose(a.grad.double(), b.grad, atol=2e-3, rtol=1e-4)


def test_part_crops_batch_independent_and_repeatable():
    from danet_b200.stn import part_crops
    xd, th = _crop_case("realistic", 16, 32, 21)
    th[5] = _degenerate_thetas(1)[0]
    gy = torch.randn(16, 24 * 32, 56, 56, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
    runs = []
    for _ in range(2):
        a = xd.clone().requires_grad_()
        y = part_crops(a, th)
        y.backward(gy)
        runs.append((y.detach(), a.grad))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    for b in (0, 5, 15):
        a = xd[b:b + 1].clone().requires_grad_()
        y = part_crops(a, th[b:b + 1].contiguous())
        y.backward(gy[b:b + 1])
        assert torch.equal(y.detach(), runs[0][0][b:b + 1]) and torch.equal(a.grad, runs[0][1][b:b + 1])


# ------------------------------------------------------------------------------------------------
# thetas
# ------------------------------------------------------------------------------------------------
def _golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stn_train.npz"))


def test_part_thetas_match_golden_and_oracle():
    from danet_b200.stn import part_thetas
    g = _golden()
    vis, cj, sj = (float(x) for x in g["stn_params"])
    T = lambda k: torch.tensor(g[k], device=DEV)
    c, th = part_thetas(T("hm"), T("index_pred"), T("learned_ratio"), T("learned_offset"), vis_score=vis,
                        center_noise=T("center_noise"), center_jitter=cj, scale_noise=T("scale_noise"), scale_jitter=sj)
    oc, oth, scores = oracle.part_thetas(g["hm"], g["index_pred"], g["learned_ratio"], g["learned_offset"], vis,
                                         g["center_noise"], cj, g["scale_noise"], sj)
    near = np.abs(scores - vis) < 1e-5
    print("part_thetas: %d visibility decisions within 1e-5 of vis_score" % near.sum())
    keep = ~near.any(1)                                                     # images without a near-tie
    for got, want in ((c, g["stn_centers"]), (c, oc), (th, g["thetas"]), (th, oth)):
        np.testing.assert_allclose(got.cpu().numpy()[keep], np.asarray(want)[keep], atol=1e-5)
    # eval form: no noise
    c0, th0 = part_thetas(T("hm"), T("index_pred"), T("learned_ratio"), T("learned_offset"))
    oc0, oth0, _ = oracle.part_thetas(g["hm"], g["index_pred"], g["learned_ratio"], g["learned_offset"])
    np.testing.assert_allclose(c0.cpu().numpy(), oc0, atol=1e-5)
    np.testing.assert_allclose(th0.cpu().numpy(), oth0, atol=1e-5)


def test_part_thetas_repeatable_and_batch_independent():
    from danet_b200.stn import part_thetas
    g = _golden()
    T = lambda k: torch.tensor(g[k], device=DEV)
    args = (T("hm"), T("index_pred"), T("learned_ratio"), T("learned_offset"))
    cn, sn = T("center_noise"), T("scale_noise")
    r1 = part_thetas(*args, center_noise=cn, scale_noise=sn)
    r2 = part_thetas(*args, center_noise=cn, scale_noise=sn)
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[1], r2[1])
    b = 1
    one = part_thetas(args[0][b:b + 1].contiguous(), args[1][b:b + 1].contiguous(), args[2], args[3],
                      center_noise=cn[b:b + 1].contiguous(), scale_noise=sn[:, :, b:b + 1].contiguous())
    assert torch.equal(one[1][0], r1[1][b]) and torch.equal(one[0][0], r1[0][b])


# ------------------------------------------------------------------------------------------------
# graphs, subsets, errors
# ------------------------------------------------------------------------------------------------
def test_cuda_graph_replays_eager_bits():
    from danet_b200.layers import hr_fuse
    from danet_b200.stn import part_crops
    terms, factors = _terms(_fuse_sites(32)[-1], 2, 3)
    xd, th = _crop_case("realistic", 2, 32, 4)
    leaves = [t.clone().requires_grad_() for t in terms] + [xd.clone().requires_grad_()]

    def step():
        for l in leaves:
            l.grad = None
        y = hr_fuse(leaves[:4], factors)
        c = part_crops(leaves[4], th)
        (y.square().sum() + c.square().sum()).backward()
        return y.detach().clone(), c.detach().clone(), [l.grad.clone() for l in leaves]

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
    assert all(torch.equal(a, b) for a, b in zip(out[2], eager[2]))


def test_needs_input_grad_subsets():
    from danet_b200.layers import hr_fuse
    terms, factors = _terms(_fuse_sites(32)[-1], 2, 5)
    full = [t.clone().requires_grad_() for t in terms]
    hr_fuse(full, factors).sum().backward()
    for keep in ([0], [1, 3], [2]):
        ls = [t.clone().requires_grad_(k in keep) for k, t in enumerate(terms)]
        hr_fuse(ls, factors).sum().backward()
        for k, l in enumerate(ls):
            assert (l.grad is None) == (k not in keep)
            if k in keep:
                assert torch.equal(l.grad, full[k].grad)


def test_argument_errors_on_the_device():
    """every refused argument, on CUDA tensors so that each check is reached on its own"""
    from danet_b200.layers import hr_fuse
    from danet_b200.stn import part_crops, part_thetas
    z = lambda *shape, **kw: torch.zeros(*shape, device=DEV, **kw)
    t = z(1, 4, 8, 8)
    bad_fuse = [([], []), ([t] * 5, [1] * 5), (t, [1]), ([t], 1), ([t, t], [1]), ([t], [3]), ([t], [16]), ([t], [True]),
                ([t], [1.0]), ([t.double()], [1]), ([z(4, 8, 8)], [1]), ([z(1, 4, 0, 8)], [1]), ([t.transpose(2, 3)], [1]),
                ([t, z(1, 4, 4, 4)], [1, 4]), ([t, z(1, 2, 4, 4)], [1, 2]), ([t, z(2, 4, 4, 4)], [1, 2]),
                ([z(1, 4, 6, 6), z(1, 4, 3, 3)], [1, 4]), ([t, t.cpu()], [1, 1]),
                (["x"], [1])]
    for terms, factors in bad_fuse:
        with pytest.raises(ValueError):
            hr_fuse(terms, factors)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            hr_fuse([t, t.to("cuda:1")], [1, 1])
    xd, th = z(2, 4, 8, 8), z(2, 24, 2, 3)
    bad_crops = [(xd.double(), th), (xd.half(), th), (z(4, 8, 8), th), (z(2, 4, 8, 6), th), (z(2, 4, 1, 1), th),
                 (z(0, 4, 8, 8), z(0, 24, 2, 3)), (z(2, 0, 8, 8), th), (xd.transpose(2, 3), th), (xd.cpu(), th),
                 (xd, th.double()), (xd, z(2, 24, 6)), (xd, z(2, 23, 2, 3)), (xd, z(1, 24, 2, 3)), (xd, z(2, 24, 3, 2)),
                 (xd, z(2, 24, 3, 2).transpose(2, 3)), (xd, th.cpu()), ("x", th)]
    for a, b in bad_crops:
        with pytest.raises(ValueError):
            part_crops(a, b)
    hm, idx, r = z(2, 24, 8, 8), z(2, 25, 8, 8), z(24)
    bad_thetas = [dict(hm=z(2, 23, 8, 8)), dict(hm=z(2, 24, 8, 6)), dict(hm=z(24, 8, 8)), dict(hm=hm.double()),
                  dict(hm=hm.transpose(2, 3)), dict(hm=hm.cpu()), dict(index_pred=z(2, 24, 8, 8)),
                  dict(index_pred=z(1, 25, 8, 8)), dict(index_pred=z(2, 25, 8, 6)), dict(index_pred=z(2, 25, 1, 1)),
                  dict(index_pred=idx.double()), dict(index_pred=idx.cpu()), dict(learned_ratio=z(23)),
                  dict(learned_ratio=z(24, 1)), dict(learned_ratio=r.double()), dict(learned_offset=z(25)),
                  dict(learned_offset=r.cpu()), dict(vis_score="x"), dict(vis_score=True), dict(center_jitter=None),
                  dict(scale_jitter="0.2"), dict(center_noise=z(2, 24, 3)), dict(center_noise=z(24, 2, 2)),
                  dict(center_noise=z(2, 24, 2, dtype=torch.float64)), dict(center_noise=z(2, 24, 2).cpu()),
                  dict(scale_noise=z(2, 24, 2)), dict(scale_noise=z(24, 2, 3)), dict(scale_noise=z(24, 2, 2).cpu()),
                  dict(scale_noise=z(2, 2, 24).transpose(0, 2))]
    for kw in bad_thetas:
        a = dict(hm=hm, index_pred=idx, learned_ratio=r, learned_offset=r)
        a.update(kw)
        with pytest.raises(ValueError):
            part_thetas(a.pop("hm"), a.pop("index_pred"), a.pop("learned_ratio"), a.pop("learned_offset"), **a)
    part_thetas(hm, idx, r, r)                                            # the base case itself is accepted
    part_crops(xd, th)
    hr_fuse([t, z(1, 4, 2, 2)], [1, 4])


# ------------------------------------------------------------------------------------------------
# composites against the reference's own modules in fp64
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    """the reference's modules (oracle.ref_import); the process-wide shims load() installs are undone afterwards"""
    import torch.cuda.comm as comm
    import warnings
    import yaml
    from oracle import ref_import
    saved = (os.getcwd(), torch.Tensor.cuda, comm.broadcast, yaml.load)
    try:
        with warnings.catch_warnings():
            ns = ref_import.load(32)
    finally:
        os.chdir(saved[0])
        torch.Tensor.cuda, comm.broadcast, yaml.load = saved[1:]
    return ns


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def _stage4_module(seed):
    """one stage-4 HighResolutionModule of HRNet-W32 (4 branches of 4 BasicBlocks, x2/x4/x8 upsample terms, 1-3-conv
    down chains), with non-trivial BatchNorm affine parameters and running statistics"""
    from models.module.hr_module import HighResolutionModule
    from models.module.res_module import BasicBlock
    torch.manual_seed(seed)
    C = [32, 64, 128, 256]
    m = HighResolutionModule(4, BasicBlock, [4, 4, 4, 4], list(C), list(C), "SUM", True)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.weight.data.uniform_(0.5, 1.5)
            mod.bias.data.uniform_(-0.3, 0.3)
            mod.running_mean.normal_(0, 0.1)
            mod.running_var.uniform_(0.8, 1.2)
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(2, c, 16 >> k, 16 >> k, generator=g) for k, c in enumerate(C)]
    return m.to(DEV).train(), [x.to(DEV) for x in xs]


def _stage4_fp64(m, xs, gys=None):
    import copy
    m64 = copy.deepcopy(m).double()
    pre = []
    for mod in m64.modules():
        if isinstance(mod, torch.nn.ReLU):
            mod.register_forward_pre_hook(lambda mod, inp: pre.append(inp[0].detach().clone()))
    x64 = [x.double().requires_grad_() for x in xs]
    ys = m64(list(x64))
    if gys is not None:
        sum((y * gy.double()).sum() for y, gy in zip(ys, gys)).backward()
    return [y.detach() for y in ys], x64, m64, pre


def _stage4_ours(m, xs, gys):
    from danet_b200.conv import conv2d
    from danet_b200.layers import batch_norm, hr_fuse
    P = {n: p.detach().clone().requires_grad_() for n, p in m.named_parameters()}
    R = {n: b.detach().clone() for n, b in m.named_buffers() if "running" in n}

    def conv(x, name, mod):
        return conv2d(x, P[name + ".weight"], None, mod.stride[0], mod.padding[0])

    def bn(x, name, mod, residual=None, relu=False):
        return batch_norm(x, R[name + ".running_mean"], R[name + ".running_var"], P[name + ".weight"], P[name + ".bias"],
                          True, mod.momentum, mod.eps, residual=residual, relu=relu)

    x = [t.clone().requires_grad_() for t in xs]
    br = []
    for i in range(4):
        h = x[i]
        for k, blk in enumerate(m.branches[i]):                        # res_module.py BasicBlock.forward
            n = "branches.%d.%d" % (i, k)
            o = bn(conv(h, n + ".conv1", blk.conv1), n + ".bn1", blk.bn1, relu=True)
            h = bn(conv(o, n + ".conv2", blk.conv2), n + ".bn2", blk.bn2, residual=h, relu=True)
        br.append(h)
    ys = []
    for i in range(4):                                                  # hr_module.py:161-179
        terms, factors = [], []
        for j in range(4):
            n = "fuse_layers.%d.%d" % (i, j)
            if j == i:
                terms.append(br[j])
                factors.append(1)
            elif j > i:
                seq = m.fuse_layers[i][j]
                terms.append(bn(conv(br[j], n + ".0", seq[0]), n + ".1", seq[1]))
                factors.append(2 ** (j - i))
            else:
                h = br[j]
                for k, sub in enumerate(m.fuse_layers[i][j]):
                    h = bn(conv(h, n + ".%d.0" % k, sub[0]), n + ".%d.1" % k, sub[1], relu=len(sub) == 3)
                terms.append(h)
                factors.append(1)
        ys.append(hr_fuse(terms, factors))
    sum((y * gy).sum() for y, gy in zip(ys, gys)).backward()
    return [y.detach() for y in ys], x, P, R


def test_composite_stage4_module_against_reference_fp64(ref):
    # the first seed whose fp64 ReLU inputs (about 2.8e5 of them) all keep 3e-6 RMS away from zero: a mask flip cannot
    # hide in the tolerance (the fp32 error of a pre-activation stays far below that)
    for seed in range(40):
        m, xs = _stage4_module(seed)
        pre = _stage4_fp64(m, xs)[3]
        if all(bool((z.abs() >= 3e-6 * z.pow(2).mean().sqrt()).all()) for z in pre):
            break
    else:
        pytest.fail("no seed keeps the ReLU inputs away from zero")
    g = torch.Generator(device=DEV).manual_seed(seed)
    gys = [torch.randn(x.shape, generator=g, device=DEV) for x in xs]
    y, x, P, R = _stage4_ours(m, xs, gys)
    yr, xr, m64, _ = _stage4_fp64(m, xs, gys)
    errs = {"y%d" % i: rel(a, b) for i, (a, b) in enumerate(zip(y, yr))}
    errs.update({"dx%d" % i: rel(a.grad, b.grad) for i, (a, b) in enumerate(zip(x, xr))})
    p64, b64 = dict(m64.named_parameters()), dict(m64.named_buffers())
    errs.update({"d" + n: rel(P[n].grad, p64[n].grad) for n in P})
    errs.update({n: rel(R[n], b64[n]) for n in R})
    worst = max(errs, key=errs.get)
    print("stage-4 W32 composite, seed %d: %d quantities, worst %s %.2e" % (seed, len(errs), worst, errs[worst]))
    assert len([n for n in errs if n.startswith("d") and n[1:] in P]) == len(list(m.parameters()))
    assert max(errs.values()) <= 1e-4, {k: v for k, v in errs.items() if v > 1e-4}


def test_composite_crops_grouped_conv_part_losses_against_reference_fp64(ref):
    """xd -> part_crops -> predict_partial_iuv (conv2d, groups = 24) -> part_iuv_losses(part_iuv_targets(...)),
    backward to xd and the conv's weight and bias, against iuv_estimator.py:193-255 on the reference's own layer and
    body_uv_losses in fp64"""
    from danet_b200 import losses
    from danet_b200.conv import conv2d
    from danet_b200.stn import part_crops
    from models.module.res_module import IUV_predict_layer
    B, C, S = 2, 32, 56
    torch.manual_seed(3)
    layer = IUV_predict_layer(feat_dim=C, part_out_dim=7).predict_partial_iuv.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(4)
    xd = torch.randn(B, C, S, S, generator=g, device=DEV)
    th = _realistic_thetas(B, 9)
    part = torch.randint(0, 25, (B, S, S), generator=g, device=DEV)
    I = F.one_hot(part, 25).permute(0, 3, 1, 2).float()
    U = torch.rand(B, 25, S, S, generator=g, device=DEV) * I
    V = torch.rand(B, 25, S, S, generator=g, device=DEV) * I
    gt = losses.part_iuv_targets([U, V, I], th)                        # a constant of both sides
    has = torch.tensor([True, True], device=DEV)
    coef = (0.7, 1.3, 0.9)

    x = xd.clone().requires_grad_()
    w, b = layer.weight.detach().clone().requires_grad_(), layer.bias.detach().clone().requires_grad_()
    pred = conv2d(part_crops(x, th), w, b, 1, 1, groups=24).view(B, 24, 3, 7, S, S)
    L = losses.part_iuv_losses(pred, gt, has)
    sum(c * l for c, l in zip(coef, L)).backward()

    x64 = xd.double().requires_grad_()
    l64 = layer.double()
    crops = torch.cat([F.grid_sample(x64, F.affine_grid(th[:, i].double(), list(x64.shape), align_corners=False),
                                     align_corners=False) for i in range(24)], 1)
    p64 = l64(crops).view(B, 24, 3, 7, S, S)
    gt64 = gt.double()
    Lr = [0.0, 0.0, 0.0]
    for i in range(24):                                                 # iuv_estimator.py:232-255
        li = ref.IUV_Estimator.body_uv_losses(None, p64[:, i, 0], p64[:, i, 1], p64[:, i, 2], None,
                                              [gt64[:, i, k] for k in range(3)] + [None], has)
        Lr = [a + l for a, l in zip(Lr, li[:3])]
    Lr = [l / 24.0 for l in Lr]
    sum(c * l for c, l in zip(coef, Lr)).backward()
    errs = {"loss_pU": rel(L[0], Lr[0]), "loss_pV": rel(L[1], Lr[1]), "loss_pIndexUV": rel(L[2], Lr[2]),
            "dxd": rel(x.grad, x64.grad), "dweight": rel(w.grad, l64.weight.grad), "dbias": rel(b.grad, l64.bias.grad)}
    print("crops -> grouped conv -> part losses: " + " ".join("%s %.2e" % kv for kv in errs.items()))
    assert max(errs.values()) <= 1e-4, errs
