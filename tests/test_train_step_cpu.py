"""CPU tests of the training step's host logic: training.LRDecay against a restatement of train/trainer.py:119-128,
danet_b200.optim.Adam's bookkeeping through a test double of its kernel layer (lazy state, skipped parameters, grouping
by step count, lr read on every call, torch.optim.Adam's state-dict format), every refusal, train_step's argument
checks and parallel.broadcast_buffers over two gloo ranks."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS, GAMMA = [0, 30000, 60000], 0.1                       # configs/danet_default.yaml SOLVER


def _reference_decay(optimizer, step_count, ind):
    """train/trainer.py:119-128 as written; returns the new decay_steps_ind"""
    if ind < len(STEPS) and step_count == STEPS[ind]:
        lr = optimizer.param_groups[0]['lr']
        lr_new = lr * GAMMA
        for param_group in optimizer.param_groups:
            param_group['lr'] = lr_new
        ind += 1
    return ind


def _sgd():
    p = torch.zeros(1, requires_grad=True)
    return torch.optim.SGD([{"params": [p]}, {"params": [torch.zeros(1, requires_grad=True)], "lr": 5.0}], lr=1e-4)


def test_lr_decay_is_the_reference_rule_with_a_resume():
    from danet_b200.training import LRDecay
    ours, ref = _sgd(), _sgd()
    sched, ind = LRDecay(), 1
    seen = []
    for step in range(1, 70001):
        if step == 40001:                                   # resume: a new trainer, decay_steps_ind back at 1
            sched, ind = LRDecay(), 1
        sched(ours, step)
        ind = _reference_decay(ref, step, ind)
        assert [g["lr"] for g in ours.param_groups] == [g["lr"] for g in ref.param_groups], step
        assert sched.decay_steps_ind == ind
        seen.append(ours.param_groups[0]["lr"])
    assert seen[29998] == 1e-4 and seen[29999] == 1e-4 * 0.1 and seen[-1] == 1e-4 * 0.1   # no decay after the resume
    assert ours.param_groups[1]["lr"] == ours.param_groups[0]["lr"]


def test_lr_decay_without_a_resume_decays_twice():
    from danet_b200.training import LRDecay
    opt, sched = _sgd(), LRDecay()
    fired = [s for s in range(1, 70001) if sched(opt, s)]
    assert fired == [30000, 60000] and opt.param_groups[0]["lr"] == 1e-4 * 0.1 * 0.1


# ---------------------------------------------------------------------------------------------------------------------
class KernelDouble:
    """danet_b200.optim's kernel layer on the CPU: records every call and applies Adam with torch's CPU ops"""

    def __init__(self):
        self.calls = []

    def check_device(self, where, name, t):
        pass

    def launch(self, device, ps, gs, ms, vs, w1, beta2, c2, bc2_sqrt, eps, step_size):
        self.calls.append(dict(n=len(ps), ids=[id(p) for p in ps], w1=w1, beta2=beta2, c2=c2, bc2=bc2_sqrt, eps=eps,
                               s=step_size))
        for p, g, m, v in zip(ps, gs, ms, vs):
            m.lerp_(g, w1)
            v.mul_(beta2).addcmul_(g, g, value=c2)
            p.addcdiv_(m, v.sqrt() / bc2_sqrt + eps, value=step_size)


@pytest.fixture
def kernel(monkeypatch):
    from danet_b200 import optim
    k = KernelDouble()
    monkeypatch.setattr(optim, "_check_device", k.check_device)
    monkeypatch.setattr(optim, "_launch", k.launch)
    return k


def _params(seed, sizes=(3, 5, 7, 2)):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(n, generator=g)) for n in sizes]


def _grads(params, step, skip=()):
    g = torch.Generator().manual_seed(100 + step)
    for i, p in enumerate(params):
        p.grad = None if i in skip else torch.randn(p.shape, generator=g)


def test_bookkeeping_matches_torch_adam(kernel):
    from danet_b200.optim import Adam
    a, b = _params(0), _params(0)
    ours = Adam([{"params": a[:3]}, {"params": a[3:], "lr": 3e-2, "betas": (0.5, 0.9), "eps": 1e-6}], lr=1e-3)
    twin = torch.optim.Adam([{"params": b[:3]}, {"params": b[3:], "lr": 3e-2, "betas": (0.5, 0.9), "eps": 1e-6}],
                            lr=1e-3, foreach=False)
    for step in range(1, 9):
        skip = {2} if step < 5 else ({1} if step % 2 else set())   # a[2] first gets a gradient at step 5
        if step == 6:
            for opt in (ours, twin):
                opt.param_groups[0]["lr"] = 5e-4                   # read again on the next call
        _grads(a, step, skip)
        _grads(b, step, skip)
        kernel.calls.clear()
        ours.step()
        twin.step()
        for p, q in zip(a, b):
            assert torch.allclose(p, q, rtol=1e-6, atol=1e-7)
            assert (p in ours.state) == (q in twin.state)
            if p in ours.state:
                s, t = ours.state[p], twin.state[q]
                assert s["step"].dtype == t["step"].dtype == torch.float32 and s["step"].device.type == "cpu"
                assert s["step"].dim() == 0 and float(s["step"]) == float(t["step"])
                assert torch.allclose(s["exp_avg"], t["exp_avg"]) and torch.allclose(s["exp_avg_sq"], t["exp_avg_sq"])
        assert 2 not in [i for i, p in enumerate(a) if p in ours.state] or step >= 5
        # one call per (group, step count); a[2]'s count lags the others of group 0 from step 5 on
        groups = {}
        for gi, group in enumerate(ours.param_groups):
            for p in group["params"]:
                if p.grad is not None:
                    groups.setdefault((gi, float(ours.state[p]["step"])), []).append(id(p))
        assert sorted(sorted(c["ids"]) for c in kernel.calls) == sorted(sorted(v) for v in groups.values())
        for c in kernel.calls:
            (gi, t), = [k for k, v in groups.items() if sorted(v) == sorted(c["ids"])]
            lr, (b1, b2), eps = (ours.param_groups[gi][k] for k in ("lr", "betas", "eps"))
            assert c["s"] == (lr / (1 - b1 ** t)) * -1 and c["bc2"] == (1 - b2 ** t) ** 0.5
            assert (c["w1"], c["beta2"], c["c2"], c["eps"]) == (1 - b1, b2, 1 - b2, eps)
    assert len(kernel.calls) == 4                                  # step 8: counts 8, 6 and 4 in group 0; group 1


def test_skipped_parameters_keep_their_state(kernel):
    from danet_b200.optim import Adam
    a = _params(1)
    opt = Adam(a, lr=1e-2)
    _grads(a, 1)
    opt.step()
    before = {i: {k: v.clone() for k, v in opt.state[p].items()} for i, p in enumerate(a)}
    vals = [p.detach().clone() for p in a]
    _grads(a, 2, skip={0, 3})
    opt.step()
    for i in (0, 3):
        assert torch.equal(a[i], vals[i]) and float(opt.state[a[i]]["step"]) == 1
        assert all(torch.equal(opt.state[a[i]][k], before[i][k]) for k in before[i])
    assert float(opt.state[a[1]]["step"]) == 2


def test_state_dicts_move_both_ways(kernel):
    from danet_b200.optim import Adam
    a, b = _params(2), _params(2)
    twin = torch.optim.Adam(b, lr=1e-3)
    ours = Adam(a, lr=1e-3)
    assert ours.state_dict()["param_groups"][0].keys() == twin.state_dict()["param_groups"][0].keys()
    for step in (1, 2):
        _grads(a, step)
        _grads(b, step)
        ours.step()
        twin.step()
    so, st = ours.state_dict(), twin.state_dict()
    assert so["param_groups"] == st["param_groups"]
    assert so["state"].keys() == st["state"].keys()
    for k in so["state"]:
        assert so["state"][k].keys() == st["state"][k].keys()
        assert so["state"][k]["step"].dtype == st["state"][k]["step"].dtype
    c, d = _params(3), _params(3)
    again = Adam(c, lr=1.0)
    again.load_state_dict(st)
    back = torch.optim.Adam(d, lr=1.0)
    back.load_state_dict(so)
    assert again.param_groups[0]["lr"] == back.param_groups[0]["lr"] == 1e-3
    _grads(c, 3)
    again.step()
    assert float(again.state[c[0]]["step"]) == 3


def test_closure_and_version(kernel):
    from danet_b200.optim import Adam
    a = _params(4)
    opt = Adam(a)
    _grads(a, 1)
    v0 = [p._version for p in a]
    assert opt.step(lambda: 7.0) == 7.0
    assert all(p._version > v for p, v in zip(a, v0))


@pytest.mark.parametrize("kw,msg", [
    (dict(weight_decay=1e-4), "weight_decay must be 0"),
    (dict(amsgrad=True), "amsgrad=True is not provided"),
    (dict(maximize=True), "maximize=True is not provided"),
    (dict(capturable=True), "capturable=True is not provided"),
    (dict(differentiable=True), "differentiable=True is not provided"),
    (dict(foreach=True), "foreach must be None"),
    (dict(foreach=False), "foreach must be None"),
    (dict(fused=True), "fused must be None"),
    (dict(lr=torch.tensor(1e-3)), "lr must be a number, not a Tensor"),
    (dict(betas=(torch.tensor(0.9), 0.999)), r"betas\[0\] must be a number"),
    (dict(lr=-1.0), "need lr >= 0"),
    (dict(betas=(1.0, 0.999)), "need lr >= 0, eps >= 0 and 0 <= betas < 1"),
])
def test_adam_refuses_options(kernel, kw, msg):
    from danet_b200.optim import Adam
    with pytest.raises(ValueError, match="danet_b200.optim.Adam: " + msg):
        Adam(_params(0), **kw)


def test_adam_refuses_options_set_after_construction(kernel):
    from danet_b200.optim import Adam
    a = _params(0)
    opt = Adam(a)
    _grads(a, 1)
    opt.param_groups[0]["lr"] = torch.tensor(1e-3)
    with pytest.raises(ValueError, match="Adam.step: lr must be a number, not a Tensor"):
        opt.step()
    opt.param_groups[0]["lr"] = 1e-3
    opt.param_groups[0]["amsgrad"] = True                         # e.g. from a loaded state dict
    with pytest.raises(ValueError, match="Adam.step: amsgrad=True is not provided"):
        opt.step()
    assert not opt.state                                          # a refused step changes nothing


def test_adam_refuses_parameters(kernel):
    from danet_b200.optim import Adam
    with pytest.raises(ValueError, match=r"\['params'\]\[0\] must be float32"):
        Adam([torch.nn.Parameter(torch.zeros(3, dtype=torch.float64))])
    with pytest.raises(ValueError, match=r"\['params'\]\[0\] must be contiguous"):
        Adam([torch.nn.Parameter(torch.zeros(4, 3).t())])
    a = _params(0)
    opt = Adam(a)
    a[1].grad = torch.sparse_coo_tensor([[0]], [1.0], (5,))
    with pytest.raises(ValueError, match="has a sparse gradient"):
        opt.step()
    a[1].grad = torch.zeros(10)[::2]
    with pytest.raises(ValueError, match=r"\.grad must be contiguous"):
        opt.step()
    m = torch.nn.Parameter(torch.zeros(2, device="meta"))
    two = Adam(_params(0)[:1] + [m])
    for p in two.param_groups[0]["params"]:
        p.grad = torch.zeros_like(p)
    with pytest.raises(ValueError, match="parameters on more than one device"):
        two.step()
    assert not two.state


def test_adam_refuses_cpu_parameters():
    from danet_b200.optim import Adam
    with pytest.raises(ValueError, match=r"danet_b200.optim.Adam: .* must be a CUDA tensor \(there is no CPU path\)"):
        Adam(_params(0))


def test_adam_entry_is_bound():
    from danet_b200 import _lib
    assert "danet_adam_step" in _lib.SIGNATURES


def test_train_step_refuses_bad_arguments():
    from danet_b200.training import LRDecay, train_step
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=1.0)
    net = torch.nn.Linear(1, 1)
    batch = {"img": torch.zeros(1, 3, 224, 224)}
    cases = [((net, object(), batch, None, None, 1), dict(schedule=LRDecay()), "optimizer must be a torch.optim"),
             ((net, opt, batch, None, None, 1), dict(schedule=None), "schedule must be callable"),
             ((net, opt, [], None, None, 1), dict(schedule=LRDecay()), "batch must be a dict with 'img'"),
             ((net, opt, batch, None, None, 1.0), dict(schedule=LRDecay()), "step_count must be an int"),
             ((net, opt, batch, None, None, 1), dict(schedule=LRDecay(), pretr_step=True), "pretr_step must be an int")]
    for args, kw, msg in cases:
        with pytest.raises(ValueError, match="danet_b200.training.train_step: " + msg):
            train_step(*args, **kw)
    assert opt.param_groups[0]["lr"] == 1.0


# ---------------------------------------------------------------------------------------------------------------------
def _broadcast_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from danet_b200.parallel import broadcast_buffers
    bufs = []
    for k in range(5):                              # BatchNorm's interleaving: fp32, fp32, int64
        bufs += [torch.full((3 + k,), 10.0 * rank + k), torch.full((3 + k,), -1.0 - rank), torch.tensor(rank + 7 * k)]
    n = broadcast_buffers(bufs, bucket_bytes=48)
    torch.save((n, bufs), tmp + str(rank))
    dist.barrier()
    dist.destroy_process_group()


def test_broadcast_buffers_two_gloo_ranks(tmp_path):
    out = str(tmp_path / "bufs")
    mp.spawn(_broadcast_worker, args=(2, 29553, out), nprocs=2, join=True)
    (n0, b0), (n1, b1) = torch.load(out + "0"), torch.load(out + "1")
    assert n0 == n1 and 2 < n0 < 15                  # one int64 bucket and several byte-limited fp32 buckets
    for x, y in zip(b0, b1):
        assert x.dtype == y.dtype and torch.equal(x, y)
    assert float(b1[0][0]) == 0.0 and int(b1[2]) == 0 and int(b1[5]) == 7


def test_broadcast_buffers_without_a_group_is_a_no_op():
    from danet_b200.parallel import broadcast_buffers
    t = torch.ones(3)
    assert broadcast_buffers([t]) == 0 and torch.equal(t, torch.ones(3))
