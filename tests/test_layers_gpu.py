"""GPU tests of the ResNet training layers (danet_b200.layers): batch_norm at every BatchNorm2d site of body_net,
limb_net and limb_reslayer in its (residual, relu) form, training and eval mode, against torch fp64 autograd; inputs
with |mean| >> std and gradients far from 1; max_pool2d against torch's CUDA max_pool2d on inputs full of exact ties;
a BasicBlock with a downsample and the limb_net stem built from conv2d + batch_norm + max_pool2d against an fp64
restatement; then repeatability, CUDA-graph replay, needs_input_grad subsets, batch independence in eval mode and the
running statistics' versions."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MOM, EPS = 0.1, 1e-5
TOL_Y, TOL_G = 1e-6, 1e-5


def _resnet_sites(prefix, H, layers):
    """(name, C, H, residual, relu) of the BatchNorm2d sites of Sequential(conv1x1, BN, ReLU, SmplResNet) on H x H input
    (smpl_regressor.py:432-436,494-499; res_module.py:27-61,393-448): the stem BN, bn1 after the 7x7/s2 conv, then per
    layer two BasicBlocks (bn1 + relu, bn2 + residual + relu; the first block of layers 2-4 has a downsample BN)."""
    sites = [(prefix + ".0.bn", 64, H, False, True), (prefix + ".bn1", 64, H // 2, False, True)]
    h, C = H // 4, 64
    for li in range(1, layers + 1):
        if li > 1:
            h, C = (h + 1) // 2, C * 2
        for blk in range(2):
            sites.append(("%s.layer%d.%d.bn1" % (prefix, li, blk), C, h, False, True))
            sites.append(("%s.layer%d.%d.bn2" % (prefix, li, blk), C, h, True, True))
            if li > 1 and blk == 0:
                sites.append(("%s.layer%d.0.downsample" % (prefix, li), C, h, False, False))
    return sites


# (name, images per batch entry, C, H, residual, relu)
SITES = [(n, 24, C, H, r, a) for n, C, H, r, a in _resnet_sites("limb_net", 56, 3)] + \
        [(n, 1, C, H, r, a) for n, C, H, r, a in _resnet_sites("body_net", 56, 4)] + \
        [("limb_reslayer.layer4.0.bn1", 1, 3072, 2, False, True), ("limb_reslayer.layer4.0.bn2", 1, 3072, 2, True, True),
         ("limb_reslayer.layer4.0.downsample", 1, 3072, 2, False, False),
         ("limb_reslayer.layer4.1.bn1", 1, 3072, 2, False, True), ("limb_reslayer.layer4.1.bn2", 1, 3072, 2, True, True)]
assert len(SITES) == 42


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def make(N, C, H, residual, seed, shift=None, scale=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, device=DEV)
    u = lambda *s: torch.rand(*s, generator=g, device=DEV)
    mu = r(C) * 0.5 if shift is None else shift * torch.sign(r(C))
    sd = 0.5 + 1.5 * u(C) if scale is None else torch.full((C,), scale, device=DEV)
    x = (r(N, C, H, H) * sd.view(1, C, 1, 1) + mu.view(1, C, 1, 1)).contiguous()
    p = {"x": x, "w": 1 + 0.2 * r(C), "b": 0.2 * r(C), "rm": mu + 0.1 * r(C), "rv": sd * sd * (0.8 + 0.4 * u(C)),
         "res": r(N, C, H, H) if residual else None, "gy": r(N, C, H, H)}
    return p


def run(p, training, relu, need=(True, True, True, True)):
    from danet_b200.layers import batch_norm
    x = p["x"].clone().requires_grad_(need[0])
    w = p["w"].clone().requires_grad_(need[1])
    b = p["b"].clone().requires_grad_(need[2])
    res = p["res"].clone().requires_grad_(need[3]) if p["res"] is not None else None
    rm, rv = p["rm"].clone(), p["rv"].clone()
    y = batch_norm(x, rm, rv, w, b, training, MOM, EPS, residual=res, relu=relu)
    y.backward(p["gy"])
    return {"y": y.detach(), "rm": rm, "rv": rv, "dx": x.grad, "dw": w.grad, "db": b.grad,
            "dr": res.grad if res is not None else None}


def reference(p, training, relu, mask):
    """fp64 autograd of relu(F.batch_norm(...) + r), the ReLU mask taken from the op under test; also the fp64
    pre-activation"""
    x, w, b = (p[k].double().requires_grad_() for k in ("x", "w", "b"))
    res = p["res"].double().requires_grad_() if p["res"] is not None else None
    rm, rv = p["rm"].double(), p["rv"].double()
    z = F.batch_norm(x, rm, rv, w, b, training, MOM, EPS)
    if res is not None:
        z = z + res
    y = z * mask.double() if relu else z
    y.backward(p["gy"].double())
    return {"y": y.detach(), "rm": rm, "rv": rv, "dx": x.grad, "dw": w.grad, "db": b.grad,
            "dr": res.grad if res is not None else None}, z.detach()


def check(p, training, relu):
    got = run(p, training, relu)
    mask = got["y"] > 0
    ref, z = reference(p, training, relu, mask)
    if relu:
        flips = mask != (z > 0)
        rms = float(z.pow(2).mean().sqrt())
        assert bool((z[flips].abs() < 1e-5 * rms).all()), "ReLU mask disagrees away from zero"
    errs = {}
    for k in ("y", "rm", "rv", "dx", "dw", "db", "dr"):
        if ref[k] is None:
            assert got[k] is None
            continue
        assert got[k].dtype == torch.float32 and got[k].shape == ref[k].shape, k
        errs[k] = rel(got[k], ref[k])
        assert errs[k] <= (TOL_Y if k in ("y", "rm", "rv") else TOL_G), (k, errs)
    if not training:
        assert torch.equal(got["rm"], p["rm"]) and torch.equal(got["rv"], p["rv"])
    return errs


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("B", [2, 16])
@pytest.mark.parametrize("site", SITES, ids=[s[0] for s in SITES])
def test_sites_against_fp64_autograd(site, B, training):
    name, per, C, H, residual, relu = site
    p = make(B * per, C, H, residual, seed=1000 * B + C + H)
    errs = check(p, training, relu)
    print("%s B=%d %s %s" % (name, B, "train" if training else "eval", " ".join("%s %.1e" % kv for kv in errs.items())))


HARD = [SITES[1], SITES[21], SITES[24], SITES[38]]


@pytest.mark.parametrize("gscale", [1.0, 1e-8, 1e3])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("site", HARD, ids=[s[0] for s in HARD])
def test_hard_inputs(site, training, gscale):
    """|mean| / std = 1e3 per channel, and dy scaled far from 1: the same bounds."""
    name, per, C, H, residual, relu = site
    p = make(2 * per, C, H, residual, seed=77 + C, shift=1e3, scale=1.0)
    p["rm"] = p["x"].mean((0, 2, 3)) + 0.1                        # eval mode: running statistics near the data's
    p["rv"] = p["x"].var((0, 2, 3)) * 1.1
    p["gy"] = p["gy"] * gscale
    errs = check(p, training, relu)
    print("%s hard gy*%g %s" % (name, gscale, " ".join("%s %.1e" % kv for kv in errs.items())))


# ------------------------------------------------------------------------------------------------
# max pool
# ------------------------------------------------------------------------------------------------
def _slot_to_index(slot, H, W):
    N, C, Ho, Wo = slot.shape
    s = slot.long()
    oh = torch.arange(Ho, device=DEV).view(1, 1, Ho, 1)
    ow = torch.arange(Wo, device=DEV).view(1, 1, 1, Wo)
    return (2 * oh - 1 + s // 3) * W + (2 * ow - 1 + s % 3)


POOLS = [("limb_net_pool_B16", 384, 64, 28, 28), ("body_net_pool_B16", 16, 64, 28, 28), ("odd_7x9", 3, 5, 7, 9),
         ("2x3", 2, 3, 2, 3), ("1x1", 2, 4, 1, 1), ("5x4", 1, 7, 5, 4)]


@pytest.mark.parametrize("kind", ["relu", "quantised"])
@pytest.mark.parametrize("shape", POOLS, ids=[s[0] for s in POOLS])
def test_max_pool_against_torch(shape, kind):
    from danet_b200.layers import max_pool2d, max_pool_forward
    _, N, C, H, W = shape
    g = torch.Generator(device=DEV).manual_seed(N * C + H)
    x = torch.randn(N, C, H, W, generator=g, device=DEV)
    x = F.relu(x) if kind == "relu" else torch.randint(-2, 3, (N, C, H, W), generator=g, device=DEV).float().clamp_min(0)
    assert float((x == 0).float().mean()) > 0.3
    y_t, idx_t = F.max_pool2d(x, 3, 2, 1, return_indices=True)
    y, slot = max_pool_forward(x)
    assert torch.equal(y, y_t)
    assert torch.equal(_slot_to_index(slot, H, W), idx_t)
    xg = x.clone().requires_grad_()
    yo = max_pool2d(xg, 3, 2, 1)
    assert torch.equal(yo.detach(), y_t)
    gy = torch.randn(y.shape, generator=g, device=DEV)
    yo.backward(gy)
    ref = torch.zeros(N * C, H * W, dtype=torch.float64, device=DEV).scatter_add_(
        1, idx_t.view(N * C, -1), gy.double().view(N * C, -1)).view(N, C, H, W)
    count = torch.zeros(N * C, H * W, device=DEV).scatter_add_(
        1, idx_t.view(N * C, -1), torch.ones_like(gy).view(N * C, -1)).view(N, C, H, W)
    assert rel(xg.grad, ref) <= 1e-7
    one = count <= 1
    assert torch.equal(xg.grad[one], ref[one].float())


def test_max_pool_nan_picks_torchs_slot():
    from danet_b200.layers import max_pool_forward
    g = torch.Generator(device=DEV).manual_seed(5)
    x = F.relu(torch.randn(2, 3, 9, 9, generator=g, device=DEV))
    x[0, 0, 1, 1] = float("nan")
    x[0, 1, 2, 2] = float("nan")
    x[0, 1, 3, 3] = float("nan")
    x[1, 2, 0, :] = float("-inf")
    x[1, 2, 1, :2] = float("-inf")
    y_t, idx_t = F.max_pool2d(x, 3, 2, 1, return_indices=True)
    y, slot = max_pool_forward(x)
    assert torch.equal(y.view(torch.int32), y_t.view(torch.int32))
    assert torch.equal(_slot_to_index(slot, 9, 9), idx_t)


# ------------------------------------------------------------------------------------------------
# composition: BasicBlock with a downsample, and the limb_net stem
# ------------------------------------------------------------------------------------------------
def _bn_params(C, g):
    return {"w": 1 + 0.2 * torch.randn(C, generator=g, device=DEV), "b": 0.3 * torch.randn(C, generator=g, device=DEV),
            "rm": 0.1 * torch.randn(C, generator=g, device=DEV), "rv": 1 + 0.2 * torch.rand(C, generator=g, device=DEV)}


def _conv_w(co, ci, k, g):
    return torch.randn(co, ci, k, k, generator=g, device=DEV) * (2.0 / (ci * k * k)) ** 0.5


def _block_params(seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = {"conv1": _conv_w(128, 64, 3, g), "conv2": _conv_w(128, 128, 3, g), "down": _conv_w(128, 64, 1, g)}
    bns = {k: _bn_params(128, g) for k in ("bn1", "bn2", "dbn")}
    x = torch.randn(1, 64, 14, 14, generator=g, device=DEV)
    return x, P, bns


def _stem_params(seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = {"conv0": _conv_w(64, 21, 1, g), "conv1": _conv_w(64, 64, 7, g)}
    bns = {k: _bn_params(64, g) for k in ("bn0", "bn1")}
    x = torch.randn(1, 21, 16, 16, generator=g, device=DEV)
    return x, P, bns


def _block_forward(x, P, S, conv, bn, pool, pre):
    """res_module.py:40-56 (BasicBlock with a stride-2 downsample); pre collects the ReLU inputs"""
    out = bn(conv(x, P["conv1"], 2), S["bn1"], None, True, pre)
    out = conv(out, P["conv2"], 1)
    res = bn(conv(x, P["down"], 2), S["dbn"], None, False, pre)
    return bn(out, S["bn2"], res, True, pre)


def _stem_forward(x, P, S, conv, bn, pool, pre):
    """smpl_regressor.py:494-498 + res_module.py:445-448: 1x1 conv, BN, ReLU, 7x7/s2 conv, BN, ReLU, max pool"""
    out = bn(conv(x, P["conv0"], 1), S["bn0"], None, True, pre)
    out = bn(conv(out, P["conv1"], 2), S["bn1"], None, True, pre)
    return pool(out)


def _ours(fwd, x, P, S, gy):
    from danet_b200.conv import conv2d
    from danet_b200.layers import batch_norm, max_pool2d
    x = x.clone().requires_grad_()
    P = {k: v.clone().requires_grad_() for k, v in P.items()}
    S = {k: {n: (t.clone().requires_grad_() if n in ("w", "b") else t.clone()) for n, t in v.items()} for k, v in S.items()}
    conv = lambda t, w, s: conv2d(t, w, None, s, w.shape[-1] // 2)
    bn = lambda t, s, r, relu, pre: batch_norm(t, s["rm"], s["rv"], s["w"], s["b"], True, MOM, EPS, residual=r, relu=relu)
    y = fwd(x, P, S, conv, bn, lambda t: max_pool2d(t, 3, 2, 1), [])
    y.backward(gy)
    return y.detach(), x, P, S


def _fp64(fwd, x, P, S, gy=None):
    x = x.double().requires_grad_()
    P = {k: v.double().requires_grad_() for k, v in P.items()}
    S = {k: {n: (t.double().requires_grad_() if n in ("w", "b") else t.double()) for n, t in v.items()} for k, v in S.items()}
    conv = lambda t, w, s: F.conv2d(t, w, None, s, w.shape[-1] // 2)

    def bn(t, s, r, relu, pre):
        z = F.batch_norm(t, s["rm"], s["rv"], s["w"], s["b"], True, MOM, EPS)
        if r is not None:
            z = z + r
        if relu:
            pre.append(z.detach())
            z = F.relu(z)
        return z

    pre = []
    y = fwd(x, P, S, conv, bn, lambda t: F.max_pool2d(t, 3, 2, 1), pre)
    if gy is not None:
        y.backward(gy.double())
    return y.detach(), x, P, S, pre


def _clear_of_zero(pre):
    return all(bool((z.abs() >= 1e-4 * z.pow(2).mean().sqrt()).all()) for z in pre)


@pytest.mark.parametrize("which", ["basic_block_down", "limb_net_stem"])
def test_composition_against_fp64(which):
    fwd, make_p = (_block_forward, _block_params) if which == "basic_block_down" else (_stem_forward, _stem_params)
    # the first seed whose fp64 ReLU inputs all keep 1e-4 RMS away from zero: a mask flip cannot hide in the tolerance
    for seed in range(100):
        x, P, S = make_p(seed)
        if _clear_of_zero(_fp64(fwd, x, P, S)[4]):
            break
    else:
        pytest.fail("no seed keeps the ReLU inputs away from zero")
    y0 = _fp64(fwd, x, P, S)[0]
    gy = torch.randn(y0.shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)
    y, xo, Po, So = _ours(fwd, x, P, S, gy)
    yr, xr, Pr, Sr, _ = _fp64(fwd, x, P, S, gy)
    errs = {"y": rel(y, yr), "dx": rel(xo.grad, xr.grad)}
    for k in P:
        errs["d" + k] = rel(Po[k].grad, Pr[k].grad)
    for k in S:
        for n in ("w", "b"):
            errs["d%s.%s" % (k, n)] = rel(So[k][n].grad, Sr[k][n].grad)
        for n in ("rm", "rv"):
            errs["%s.%s" % (k, n)] = rel(So[k][n], Sr[k][n])
    print(which, "seed", seed, " ".join("%s %.1e" % kv for kv in errs.items()))
    assert max(errs.values()) <= 1e-4, errs


# ------------------------------------------------------------------------------------------------
# determinism, graphs, subsets, batch independence, versions
# ------------------------------------------------------------------------------------------------
REP = [SITES[0], SITES[21], SITES[38]]


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("site", REP, ids=[s[0] for s in REP])
def test_bit_repeatable(site, training):
    name, per, C, H, residual, relu = site
    p = make(2 * per, C, H, residual, seed=3)
    r1, r2 = run(p, training, relu), run(p, training, relu)
    for k in r1:
        assert (r1[k] is None and r2[k] is None) or torch.equal(r1[k], r2[k]), k


def test_max_pool_bit_repeatable():
    from danet_b200.layers import max_pool2d
    x = F.relu(torch.randn(48, 64, 28, 28, device=DEV))
    gy = torch.randn(48, 64, 14, 14, device=DEV)
    outs = []
    for _ in range(2):
        xg = x.clone().requires_grad_()
        y = max_pool2d(xg, 3, 2, 1)
        y.backward(gy)
        outs.append((y.detach(), xg.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_cuda_graph_replays_eager_bits():
    from danet_b200.layers import batch_norm, max_pool2d
    p = make(4, 64, 14, True, seed=11)
    rm0, rv0 = p["rm"].clone(), p["rv"].clone()

    def step(x, w, b, res, rm, rv):
        y = batch_norm(x, rm, rv, w, b, True, MOM, EPS, residual=res, relu=True)
        z = max_pool2d(y, 3, 2, 1)
        z.backward(gz)
        return z

    gz = torch.randn(4, 64, 7, 7, device=DEV)
    leaves = [p[k].clone().requires_grad_() for k in ("x", "w", "b", "res")]
    rm, rv = rm0.clone(), rv0.clone()
    eager = step(*leaves, rm, rv).detach()
    eager_g = [t.grad.clone() for t in leaves]
    eager_rs = (rm.clone(), rv.clone())
    for t in leaves:
        t.grad = None
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step(*leaves, rm, rv)
            for t in leaves:
                t.grad = None
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        z = step(*leaves, rm, rv)
    rm.copy_(rm0)
    rv.copy_(rv0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(z.detach(), eager)
    for t, e in zip(leaves, eager_g):
        assert torch.equal(t.grad, e)
    assert torch.equal(rm, eager_rs[0]) and torch.equal(rv, eager_rs[1])


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_needs_input_grad_subsets(training):
    site = SITES[21]
    p = make(4, site[2], site[3], True, seed=21)
    full = run(p, training, True)
    for need in [(True, False, False, False), (False, True, False, False), (False, False, True, False),
                 (False, False, False, True), (False, True, True, False), (True, False, False, True)]:
        got = run(p, training, True, need)
        assert torch.equal(got["y"], full["y"])
        for i, k in enumerate(("dx", "dw", "db", "dr")):
            if need[i]:
                assert torch.equal(got[k], full[k]), (need, k)
            else:
                assert got[k] is None, (need, k)


@pytest.mark.parametrize("site", [SITES[1], SITES[6], SITES[38]], ids=["HW784", "HW49", "HW4_C3072"])
def test_eval_output_does_not_depend_on_the_batch(site):
    from danet_b200.layers import batch_norm
    name, per, C, H, residual, relu = site
    p = make(5, C, H, residual, seed=9)
    r = p["res"]
    full = batch_norm(p["x"], p["rm"], p["rv"], p["w"], p["b"], False, MOM, EPS, residual=r, relu=relu)
    for i in (0, 3, 4):
        one = batch_norm(p["x"][i:i + 1], p["rm"], p["rv"], p["w"], p["b"], False, MOM, EPS,
                         residual=r[i:i + 1] if r is not None else None, relu=relu)
        assert torch.equal(one, full[i:i + 1])


def test_running_statistics_versions():
    from danet_b200.layers import batch_norm
    p = make(2, 64, 7, False, seed=4)
    rm, rv = p["rm"].clone(), p["rv"].clone()
    v0, w0 = rm._version, rv._version
    batch_norm(p["x"], rm, rv, p["w"], p["b"], False, MOM, EPS)
    assert rm._version == v0 and rv._version == w0
    batch_norm(p["x"], rm, rv, p["w"], p["b"], True, MOM, EPS)
    assert rm._version > v0 and rv._version > w0


def _fixed_order_channel_sums(a):
    """numpy replica, add for add, of the per-channel sums' order: per (channel, chunk of ipc images) 256 threads each
    add their pixels q = t, t + 256, ... image after image in double, a halving tree adds the threads, then the chunks
    are added in order and the sum rounded to fp32"""
    import numpy as np
    N, C, HW = a.shape
    ipc = max(1, 16384 // HW)
    tot = np.zeros(C)
    for j in range(-(-N // ipc)):
        acc = np.zeros((C, 256))
        for n in range(j * ipc, min(N, (j + 1) * ipc)):
            for q0 in range(0, HW, 256):
                blk = a[n, :, q0:q0 + 256].astype(np.float64)
                acc[:, :blk.shape[1]] += blk
        o = 128
        while o > 0:
            acc[:, :o] += acc[:, o:2 * o]
            o //= 2
        tot += acc[:, 0]
    return tot.astype(np.float32)


@pytest.mark.parametrize("N,C,HW", [(16, 64, 784), (40, 8, 3136), (3, 5, 20000), (384, 16, 49), (16, 96, 4)])
def test_bias_grad_keeps_its_summation_order(N, C, HW):
    """danet_conv_bias_grad runs on the per-channel sum kernel BatchNorm shares: its db is the fixed-order sum, bit for
    bit, as before that kernel learned a second sum"""
    from danet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(N + C + HW)
    dy = torch.randn(N, C, HW, generator=g, device=DEV) * torch.exp(2 * torch.randn(N, C, 1, generator=g, device=DEV))
    ws = torch.empty(int(lib.danet_conv_bias_grad_workspace_bytes(N, C, HW)), dtype=torch.uint8, device=DEV)
    db = torch.empty(C, device=DEV)
    _lib.check(lib.danet_conv_bias_grad(N, C, HW, _lib.ptr(dy), _lib.ptr(db), _lib.ptr(ws), _lib.stream_ptr(DEV)))
    want = torch.from_numpy(_fixed_order_channel_sums(dy.cpu().numpy()))
    assert torch.equal(db.cpu(), want)


def test_argument_errors_on_the_device():
    from danet_b200.layers import batch_norm, max_pool2d
    p = make(2, 8, 5, False, seed=1)
    with pytest.raises(ValueError):
        batch_norm(p["x"].transpose(2, 3), p["rm"], p["rv"], p["w"], p["b"], True, MOM, EPS)
    with pytest.raises(ValueError):
        batch_norm(p["x"], p["rm"].cpu(), p["rv"], p["w"], p["b"], True, MOM, EPS)
    with pytest.raises(ValueError):
        batch_norm(p["x"][:1, :, :1, :1].contiguous(), p["rm"], p["rv"], p["w"], p["b"], True, MOM, EPS)
    with pytest.raises(ValueError):
        max_pool2d(p["x"], 3, 1, 1)
    with pytest.raises(ValueError):
        max_pool2d(p["x"].double(), 3, 2, 1)
