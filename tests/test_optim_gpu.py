"""GPU tests of danet_b200.optim.Adam (csrc/optim.cu): each rounding of k_adam against the torch._foreach_* op it
restates, 30 steps bit-identical to torch.optim.Adam (torch's CUDA default, the foreach implementation) over sizes,
alignments, launch splits, param groups, lr changes, late and missing gradients and gradients from 2^-60 to 2^60 with
±0, subnormals, NaN and ±inf; state dicts in both directions; no host synchronisation; version counters, and infer_net
seeing the weights after training."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LARGEST = 7077888                                    # DaNet W48's largest parameter tensor (limb_reslayer.layer4.0.conv1)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _wide(n, gen, lo=-60, hi=60):
    """fp32 values sign * 2^U(lo, hi) * mantissa, with ±0, subnormals, NaN and ±inf sprinkled in"""
    e = torch.randint(lo, hi + 1, (n,), generator=gen).float()
    x = (torch.rand(n, generator=gen) + 1) * torch.exp2(e) * (torch.randint(0, 2, (n,), generator=gen) * 2 - 1)
    if n >= 16:
        k = torch.randperm(n, generator=gen)[:max(8, n // 200)]
        special = torch.tensor([0.0, -0.0, 1e-40, -3e-42, float("nan"), float("inf"), -float("inf"), 1.4e-45])
        x[k] = special[torch.arange(len(k)) % len(special)]
    return x.to(DEV)


def _fma(a, b, c):
    """fp32 fma through fp64 (the product of two fp32 values is exact in fp64)"""
    return (a.double() * b.double() + c.double()).float()


def test_each_rounding_is_the_foreach_ops():
    """the per-element forms k_adam writes down, each against the torch._foreach_* op of _multi_tensor_adam"""
    gen = torch.Generator().manual_seed(0)
    n = 1 << 20
    m = torch.randn(n, generator=gen).to(DEV)
    g = (torch.randn(n, generator=gen) * 3).to(DEV)
    v = torch.rand(n, generator=gen).to(DEV)
    f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=DEV)
    report = {}
    for w in (0.1, 0.5, 0.7):                                     # Lerp.h: both branches, contracted
        out = [m.clone()]
        torch._foreach_lerp_(out, [g], w)
        want = _fma(f32(w).expand(n), g - m, m) if w < 0.5 else _fma(-(g - m), (1 - f32(w)).expand(n), g)
        plain = m + f32(w) * (g - m) if w < 0.5 else g - (g - m) * (1 - f32(w))
        report["lerp %g" % w] = int((out[0] != plain).sum())
        assert _bits_equal(out[0], want), "lerp w=%g" % w
    c2 = 1 - 0.999
    out = [v.clone()]
    torch._foreach_addcmul_(out, [g], [g], c2)                    # fma(value, g * g, v)
    assert _bits_equal(out[0], _fma(f32(c2).expand(n), g * g, v)), "addcmul"
    report["addcmul"] = int((out[0] != v + f32(c2) * g * g).sum())
    bc2 = (1 - 0.999 ** 7) ** 0.5
    out = [v.sqrt()]
    torch._foreach_div_(out, [bc2])                               # a true division by the fp32 scalar
    assert _bits_equal(out[0], v.sqrt() / f32(bc2)), "div"
    report["div"] = int((out[0] != v.sqrt() * f32(1 / bc2)).sum())
    s = (1e-3 / (1 - 0.9 ** 7)) * -1
    d = v.sqrt() + 1e-8
    out = [g.clone()]
    torch._foreach_addcdiv_(out, [m], [d], [s])                   # fma(value, m / d, p)
    assert _bits_equal(out[0], _fma(f32(s).expand(n), m / d, g)), "addcdiv"
    report["addcdiv"] = int((out[0] != g + f32(s) * (m / d)).sum())
    print("\nelements where the other form (unfused / reciprocal) differs: %s" % report)


def _param_set(gen):
    """(name, tensor factory) of every kind of parameter the bit-identity test covers"""
    sizes = [0, 1, 3, 4, 5, 1023, 4097, (1 << 20) + 7, LARGEST]
    out = [("n%d" % n, torch.randn(n, generator=gen)) for n in sizes]
    out += [("small%d" % i, torch.randn(1 + i % 37, generator=gen)) for i in range(2100)]   # > 2 launches' tables
    return out


def _make(values, offset_view):
    ps = [torch.nn.Parameter(v.to(DEV).clone()) for v in values]
    base = torch.empty(1001, device=DEV)
    base[1:] = offset_view.to(DEV)
    ps.append(torch.nn.Parameter(base[1:]))                      # storage offset 1: the unaligned path
    assert ps[-1].data_ptr() % 16 != 0
    return ps


def _groups(ps):
    return [{"params": ps[:-400]},
            {"params": ps[-400:], "lr": 3e-2, "betas": (0.5, 0.9), "eps": 1e-6}]   # |w| >= 0.5: Lerp.h's other branch


def _assign_grads(ps, step, gen_seed):
    g = torch.Generator().manual_seed(gen_seed + step)
    grads = []
    for i, p in enumerate(ps):
        if (i == 3 and step < 5) or (i == 5 and step % 3 == 0):   # first gradient at step 5; None on some steps
            grads.append(None)
        else:
            grads.append(_wide(p.numel(), g).view_as(p) if p.numel() >= 16 else torch.randn(p.shape, generator=g).to(DEV))
    return grads


def _compare(ours, twin, a, b):
    for i, (p, q) in enumerate(zip(a, b)):
        assert _bits_equal(p.detach(), q.detach()), ("param", i)
        assert (p in ours.state) == (q in twin.state), ("state", i)
        if p in ours.state:
            s, t = ours.state[p], twin.state[q]
            assert s["step"].dtype == t["step"].dtype and float(s["step"]) == float(t["step"]), ("step", i)
            assert _bits_equal(s["exp_avg"], t["exp_avg"]), ("exp_avg", i)
            assert _bits_equal(s["exp_avg_sq"], t["exp_avg_sq"]), ("exp_avg_sq", i)


def test_thirty_steps_bit_identical_to_torch_adam():
    from danet_b200.optim import Adam
    gen = torch.Generator().manual_seed(1)
    params = _param_set(gen)
    view = torch.randn(1000, generator=gen)
    a, b = _make([v for _, v in params], view), _make([v for _, v in params], view)
    ours, twin = Adam(_groups(a), lr=1e-3), torch.optim.Adam(_groups(b), lr=1e-3)
    assert len(a) > 2000
    for step in range(1, 31):
        if step in (10, 20):
            for opt in (ours, twin):
                opt.param_groups[0]["lr"] *= 0.1                 # in place, as the reference's decay does
        grads = _assign_grads(a, step, 1000)
        for p, q, g in zip(a, b, grads):
            p.grad = None if g is None else g.clone()
            q.grad = None if g is None else g.clone()
        ours.step()
        twin.step()
        if step in (1, 4, 5, 6, 15, 30):
            _compare(ours, twin, a, b)
    assert float(ours.state[a[3]]["step"]) == 26 and float(ours.state[a[5]]["step"]) == 20
    nan = [bool(torch.isnan(p).any()) for p in a]
    print("\n30 steps over %d tensors (%d elements): bit-identical; %d tensors hold NaN"
          % (len(a), sum(p.numel() for p in a), sum(nan)))


@pytest.mark.parametrize("direction", ["torch_to_ours", "ours_to_torch"])
def test_state_dicts_continue_bit_identically(direction):
    from danet_b200.optim import Adam
    gen = torch.Generator().manual_seed(2)
    vals = [torch.randn(n, generator=gen) for n in (5, 4097, 1023, 70000)]
    view = torch.randn(1000, generator=gen)
    a, b = _make(vals, view), _make(vals, view)
    first = (torch.optim.Adam if direction == "torch_to_ours" else Adam)(a, lr=2e-3)
    for step in range(1, 4):
        for p, g in zip(a, _assign_grads(a, step, 50)):
            p.grad = g
        first.step()
    with torch.no_grad():
        for p, q in zip(a, b):
            q.copy_(p)
    second = (Adam if direction == "torch_to_ours" else torch.optim.Adam)(b, lr=1.0)
    second.load_state_dict(copy.deepcopy(first.state_dict()))    # a state dict shares the optimizer's tensors
    for step in range(4, 9):
        grads = _assign_grads(a, step, 50)
        for p, q, g in zip(a, b, grads):
            p.grad = None if g is None else g.clone()
            q.grad = None if g is None else g.clone()
        first.step()
        second.step()
    ours, twin = (second, first) if direction == "torch_to_ours" else (first, second)
    oa, ob = (b, a) if direction == "torch_to_ours" else (a, b)
    _compare(ours, twin, oa, ob)


def test_step_never_synchronises_and_bumps_versions():
    from danet_b200.optim import Adam
    ps = [torch.nn.Parameter(torch.randn(n, device=DEV)) for n in (7, 4096, 100000)]
    opt = Adam(ps, lr=1e-3)
    for p in ps:
        p.grad = torch.randn_like(p)
    torch.cuda.synchronize()
    versions = [p._version for p in ps]
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.step()                                                # creates the state
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert all(p._version > v for p, v in zip(ps, versions))
    # autograd refuses a saved parameter the kernel has rewritten, as after torch's in-place ops
    x = torch.randn(7, device=DEV, requires_grad=True)
    y = (ps[0] * x).sum()
    opt.step()
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.backward()


def test_infer_net_sees_the_trained_weights():
    """two train_steps, then eval-mode infer_net against a freshly built model loaded with the trained state_dict"""
    from danet_b200 import build_synthetic_danet
    from danet_b200.optim import Adam
    from danet_b200.training import LRDecay, train_step
    from test_train_step_gpu import make_batch
    net = build_synthetic_danet(width=32, seed=0, device=DEV)
    B = 2
    batch, opt_pose, opt_betas, fit_valid, noise, drops = make_batch(B, 5, steps=2)
    net.eval()
    before = net.infer_net(batch["img"])["para"].clone()          # caches a plan of the untrained weights
    opt = Adam(net.parameters(), lr=1e-3)
    sched = LRDecay()
    for step in (1, 2):
        train_step(net, opt, batch, opt_pose, opt_betas, step, schedule=sched, pretr_step=0, fit_valid=fit_valid,
                   part_drop=drops[step - 1], center_noise=noise[step - 1][0], scale_noise=noise[step - 1][1])
    net.eval()
    para = net.infer_net(batch["img"])["para"]
    fresh = build_synthetic_danet(width=32, seed=1, device=DEV)
    fresh.load_state_dict(net.state_dict())
    fresh.eval()
    want = fresh.infer_net(batch["img"])["para"]
    print("\ninfer_net after two steps: max |para - untrained para| = %.3g" % float((para - before).abs().max()))
    assert not torch.equal(para, before)
    assert _bits_equal(para, want)
