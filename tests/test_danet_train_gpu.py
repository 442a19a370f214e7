"""GPU tests of DaNet's training join: danet_b200.iuvmap.part_drop_clean bit for bit against the reference's own
expressions run by torch on the same CUDA tensors (oracle/danet_train.py) and against the reference's DaNet._forward
(tests/golden/danet_train.npz); repeatability, no host synchronisation, CUDA-graph capture; and
danet_b200.training.danet_forward: against the same runner with the reference's dropout and clean in its op table,
the regressor's gradient reaching the estimator, the seeded draws in the reference's order and eval mode against
infer_net."""
import numpy as np
import pytest
import torch

from oracle import danet_train as odt
from estimator_train_common import Recorder, decision_flips
from oracle import estimator_train as oet
from oracle import regressor_train as ort
from test_danet_train_cpu import _case, _golden, run_and_grad

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
PARA_TOL = 1e-4                                    # bench.py's para tolerance
FLIP_BOUND = 5e-2                                  # test_estimator_train_gpu.py's bound where decisions differ
# loss_stnhm on: without it the heat-map head's bias gradient is zero up to rounding (the soft-argmax is shift-invariant)
HM_WEIGHT = 1.0


def _masks(kind, B, seed):
    if kind == "none":
        return None
    if kind == "all":
        return torch.ones(B, 24, dtype=torch.bool, device=DEV)
    if kind == "nothing":
        return torch.zeros(B, 24, dtype=torch.bool, device=DEV)
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, 24, generator=g) < 0.3).to(DEV)


def _same_all(a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        assert (x is None) == (y is None), (what, k)
        if x is not None:
            assert odt.bits_equal(x, y), (what, k)


@pytest.mark.parametrize("B,S", [(1, 56), (3, 40), (16, 56), (3, 7), (16, 7)])
@pytest.mark.parametrize("drop", ["none", "nothing", "rate0.3", "all"])
def test_op_is_bit_identical_to_the_reference_expressions(B, S, drop):
    from danet_b200.iuvmap import part_drop_clean
    leaves = [t.to(DEV) for t in odt.make_leaves(B, S, 7 * B + S)]
    probes = tuple(t.to(DEV) for t in odt.make_probes(B, S, 3 * B + S))
    mask = _masks(drop, B, B + S)
    out, grads = run_and_grad(part_drop_clean, leaves, probes, mask)
    r_out, r_grads = run_and_grad(odt.part_drop_clean, leaves, probes, mask)
    _same_all(out, r_out, "out")
    _same_all(grads, r_grads, "grad")


def test_op_reads_a_strided_part_view():
    from danet_b200.iuvmap import part_drop_clean
    B, S = 3, 12
    u, v, i, a, p = (t.to(DEV) for t in odt.make_leaves(B, S, 5))
    big = torch.randn(B, 24, 3, 9, S + 2, S, device=DEV)
    view = big[:, :, :, 1:8, 1:S + 1, :]                        # not contiguous in the channel and row strides
    view.copy_(p)
    assert not view.is_contiguous()
    probes = tuple(t.to(DEV) for t in odt.make_probes(B, S, 6))
    mask = _masks("rate0.3", B, 1)
    out, grads = run_and_grad(part_drop_clean, [u, v, i, a, view], probes, mask)
    r_out, r_grads = run_and_grad(odt.part_drop_clean, [u, v, i, a, p], probes, mask)
    _same_all(out, r_out, "out")
    _same_all(grads, r_grads, "grad")


@pytest.mark.parametrize("name", ["r03_s0", "r03_s1", "r09_s0", "r09_s1", "eval"])
def test_op_matches_reference_golden(name):
    from danet_b200.iuvmap import part_drop_clean
    g = _golden()
    leaves, probes, drop, _, _, _ = _case(g, name)
    out, grads = run_and_grad(part_drop_clean, [t.to(DEV) for t in leaves], tuple(t.to(DEV) for t in probes),
                              drop.to(DEV) if drop is not None else None)
    for k, t in zip(("u_cl", "v_cl", "index_cl", "ann_cl", "part_iuv_map"), out):
        assert odt.bits_equal(t, torch.as_tensor(g["%s_%s" % (name, k)])), k
    assert grads[2] is None and grads[3] is None
    for k, t in zip(("g_u", "g_v", "g_parts"), (grads[0], grads[1], grads[4])):
        assert odt.bits_equal(t, torch.as_tensor(g["%s_%s" % (name, k)])), k


def test_op_repeatable_no_sync_and_graph_capture_replays_eager():
    from danet_b200.iuvmap import part_drop_clean
    B, S = 4, 56
    src = [t.to(DEV) for t in odt.make_leaves(B, S, 11)]
    G1, G2 = (t.to(DEV) for t in odt.make_probes(B, S, 12))
    mask = _masks("rate0.3", B, 13)
    xs = [t.clone().requires_grad_() for t in src]

    def step():
        for x in xs:
            x.grad = None
        out = part_drop_clean(*xs, mask)
        ((G1[:, :50] * torch.cat(out[:2], 1)).sum() + (G2 * out[4]).sum()).backward()
        return [t.detach().clone() for t in out] + [xs[k].grad.clone() for k in (0, 1, 4)]
    eager = step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _same_all(eager, again, "repeat")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = part_drop_clean(*xs, mask)
        ((G1[:, :50] * torch.cat(out[:2], 1)).sum() + (G2 * out[4]).sum()).backward()
    for x in xs:
        if x.grad is not None:
            x.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    replay = [t.detach() for t in out] + [xs[k].grad for k in (0, 1, 4)]
    _same_all(eager, replay, "graph")


# ---------------------------------------------------------------------------------------------------------------------
_NETS = {}


def _net(width):
    if width not in _NETS:
        from danet_b200 import build_synthetic_danet
        net = build_synthetic_danet(width=width, seed=0, device=DEV)
        _NETS[width] = (net, {k: v.clone() for k, v in net.state_dict().items()})
    return _NETS[width]


def _restore(net, snap):
    with torch.no_grad():
        for k, v in net.state_dict().items():
            v.copy_(snap[k])


def _in_dict(net, B, seed):
    """a data batch after prepare_targets (synthetic fits and annotations) with the image and DensePose points"""
    from danet_b200.targets import prepare_targets
    rng = np.random.default_rng(seed)
    T = lambda a, dt=torch.float32: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=DEV)

    def pose(n):
        p = rng.normal(0, 0.25, (n, 72))
        p[:, :3] = [np.pi, 0, 0] + rng.normal(0, 0.1, (n, 3))
        return p
    kp = np.concatenate([rng.uniform(-0.8, 0.8, (B, 49, 2)), rng.choice([1.0, 0.3, 0.0], (B, 49, 1))], -1)
    kp[:, 25:30, 2] = 1.0
    flag = lambda: T(rng.random(B) < 0.6, torch.uint8)
    batch = dict(keypoints=T(kp), pose=T(pose(B)), betas=T(rng.normal(0, 1, (B, 10))), has_smpl=flag(),
                 has_dp=flag(), iuv_annotated=flag(), smpl_2dkps=T(rng.uniform(-1, 1, (B, 24, 3))))
    d = dict(batch)
    d.update(prepare_targets(net, batch, T(pose(B)), T(rng.normal(0, 1, (B, 10))), fit_valid=flag()))
    _, _, dp = oet.make_targets(B, seed)
    d.update(img=oet.make_image(B, seed).to(DEV), dp_dict={k: T(v) for k, v in dp.items()},
             pose_3d=T(np.concatenate([rng.normal(0, 0.3, (B, 24, 3)), rng.random((B, 24, 1)) < 0.8], -1)),
             has_pose_3d=flag(), pretrain_mode=False, vis_on=False)
    return d


def _noise(B, seed):
    from danet_b200.estimator import draw_noise
    torch.manual_seed(seed)
    return tuple(t.to(DEV) for t in draw_noise(B))


def _step(net, in_dict, training, part_drop=None, noise=(None, None), regressor_losses=True, hm_weight=None):
    """danet_forward, then the gradients of the sum of its losses w.r.t. the image and every parameter"""
    from danet_b200 import training as tr
    net.train(training)
    try:
        x = in_dict["img"].clone().requires_grad_()
        d = dict(in_dict, img=x)
        ret = tr.danet_forward(net, d, part_drop=part_drop, center_noise=noise[0], scale_noise=noise[1],
                               stn_hm_weight=hm_weight)
    finally:
        net.eval()
    L = {k: v for k, v in ret["losses"].items() if regressor_losses or k.startswith("loss_")}
    params = {k: p for k, p in net.named_parameters() if p.requires_grad and not k.startswith("iuv2smpl.smpl.")}
    grads = {}
    if training:
        g = torch.autograd.grad(sum(v.sum() for v in L.values()), [x] + list(params.values()), allow_unused=True)
        grads = dict(zip(["image"] + list(params), g))
    return ret, grads


def _bits(ret, grads):
    out = [ret["losses"][k] for k in sorted(ret["losses"])] + [ret["prediction"][k] for k in sorted(ret["prediction"])]
    out += list(ret["visualization"]["iuv_pred"]) + [ret["visualization"]["part_iuv_pred"]]
    return out + [grads[k] for k in sorted(grads)]


def _cast(d, dtype):
    c = lambda t: t.to(dtype) if torch.is_tensor(t) and t.is_floating_point() else t
    return {k: ({a: c(b) for a, b in v.items()} if isinstance(v, dict) else c(v)) for k, v in d.items()}


def _table_run(net, snap, d, training, drop, noise, dtype, record=True):
    """run_danet on the snapshot's state through oracle.danet_train.torch_table in `dtype` (cuDNN and TF32 off), and
    the gradients of the sum of the losses w.r.t. the image and every parameter"""
    from danet_b200 import synthetic
    from danet_b200.training import run_danet
    state = {k: (v.to(DEV, dtype).clone() if v.is_floating_point() else v.clone().to(DEV)) for k, v in snap.items()
             if not k.startswith("iuv2smpl.smpl.")}
    keys = [k for k, _ in net.named_parameters() if k in state]
    for k in keys:
        state[k].requires_grad_(training)
    dd = _cast(d, dtype)
    x = dd["img"].clone().requires_grad_(training)
    dd["img"] = x
    ops = Recorder(odt.torch_table(state, synthetic.make_smpl_model(0), training))
    flags = torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = False, False, False
    try:
        ret = run_danet(net.graph, state, dd, training, ops, drop, tuple(_cast({"n": n}, dtype)["n"] for n in noise),
                        0.3, HM_WEIGHT)
        grads = {}
        if training:
            g = torch.autograd.grad(sum(v.sum() for v in ret["losses"].values()), [x] + [state[k] for k in keys],
                                    allow_unused=True)
            grads = dict(zip(["image"] + keys, g))
    finally:
        torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags
    return ret, grads, state, ops


def _flat(ret):
    out = {"L_" + k: v for k, v in ret["losses"].items()}
    out.update({"p_" + k: v for k, v in ret["prediction"].items()})
    out["part_iuv_pred"] = ret["visualization"].get("part_iuv_pred")
    for k, t in zip(("u_cl", "v_cl", "index_cl", "ann_cl"), ret["visualization"]["iuv_pred"]):
        out[k] = t
    return {k: v for k, v in out.items() if v is not None}


def _clean_flips(a, b):
    """pixels whose cleaned Index argmax differs between two runs (global and part maps)"""
    va, vb = a["visualization"], b["visualization"]
    n = int((va["iuv_pred"][2].argmax(1) != vb["iuv_pred"][2].to(DEV).argmax(1)).sum())
    if "part_iuv_pred" in va:
        n += int((va["part_iuv_pred"][:, :, 2].argmax(2) != vb["part_iuv_pred"][:, :, 2].to(DEV).argmax(2)).sum())
    return n


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("width", [32, 48])
@pytest.mark.parametrize("training", [True, False])
def test_join_matches_fp64_table(B, width, training):
    """danet_forward against run_danet driven by the fp64 torch table (the estimator's and the branches' layers, the
    reference's dropout and clean, the GCN head, its losses and smpl_losses over the torch SMPL layer): losses,
    predictions, cleaned maps, parameter gradients and running statistics within 1e-5 or 4x fp32 torch's error on the
    same problem; 5 % where a ReLU, STN argmax or clean argmax decision differs from fp64's"""
    from danet_b200.regressor import _attr
    from danet_b200.training import cuda_ops, run_danet
    net, snap = _net(width)
    d = _in_dict(net, B, 30 + B)
    noise = _noise(B, B) if training else (None, None)
    drop = _masks("rate0.3", B, B) if training else None
    r64, g64, s64, rec64 = _table_run(net, snap, d, training, drop, noise, torch.float64)
    r32, g32, s32, _ = _table_run(net, snap, d, training, drop, noise, torch.float32)
    # the CUDA walk once more through a recording op table, for the decisions
    _restore(net, snap)
    net.train(training)
    try:
        rec = Recorder(cuda_ops(net))
        with torch.no_grad():
            state = {k: _attr(net, k) for k in s64 if not k.startswith("iuv2smpl.smpl.")}
            run_danet(net.graph, state, d, training, rec, drop, noise, 0.3, 0.0)
    finally:
        net.eval()
    relu_flips, amax_flips = decision_flips(rec, rec64)
    _restore(net, snap)
    ret, grads = _step(net, d, training, part_drop=drop, noise=noise, hm_weight=HM_WEIGHT)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    _restore(net, snap)
    clean_flips = _clean_flips(ret, r64)
    stats = [k for k in s64 if k.endswith(("running_mean", "running_var"))]

    def errors(o, g, st):
        f, f64 = _flat(o), _flat(r64)
        assert set(f) == set(f64), set(f) ^ set(f64)
        err = {k: ort.rel_norm(f[k].double(), f64[k]) for k in f}
        for k, t in g.items():
            assert (t is None) == (g64[k] is None), k
            if t is not None:
                err["g_" + k] = ort.rel_norm(t.double(), g64[k])
        for k in stats:
            err["st_" + k] = ort.rel_norm(st[k].double(), s64[k])
        return err
    e32 = errors(r32, g32, s32)
    err = errors(ret, grads, sd)
    downstream = amax_flips or clean_flips
    bound = {k: (FLIP_BOUND if (downstream or (relu_flips and k.startswith("g_"))) else max(1e-5, 4 * e32[k]))
             for k in err}
    k, e = max(err.items(), key=lambda kv: kv[1])
    kr, r = max(((k2, e2 / bound[k2]) for k2, e2 in err.items()), key=lambda kv: kv[1])
    print("\nW%d B=%d training=%d: worst relative error %.3g (%s, fp32 torch %.3g); decisions unlike fp64: %d ReLU, "
          "%d STN argmax, %d clean argmax; worst error / bound %.3g (%s)"
          % (width, B, training, e, k, e32[k], relu_flips, amax_flips, clean_flips, r, kr))
    assert r <= 1.0, (kr, err[kr], bound[kr])
    assert len(ret["losses"]) == (22 if training else 0) and all(v.dim() == 1 for v in ret["losses"].values())
    assert ("loss_stnhm" in ret["losses"]) == training                 # 13 estimator losses with it, 9 regressor
    assert set(ret["prediction"]) == ({"cam", "shape", "pose", "vertices", "cam_t"} if training else
                                      {"cam", "shape", "pose"})
    assert ret["metrics"] == {}


def test_regressor_gradient_reaches_the_estimator_heads():
    net, snap = _net(32)
    B = 3
    d = _in_dict(net, B, 50)
    noise, drop = _noise(B, 1), _masks("rate0.3", B, 2)
    _restore(net, snap)
    _, full = _step(net, d, True, part_drop=drop, noise=noise)
    _restore(net, snap)
    _, est_only = _step(net, d, True, part_drop=drop, noise=noise, regressor_losses=False)
    _restore(net, snap)
    heads = [k for k in full if k.startswith("img2iuv.iuv_est.") and full[k] is not None]
    assert heads
    moved = [k for k in heads if not torch.equal(full[k], est_only[k])]
    diff = max(float((full[k] - est_only[k]).abs().max()) for k in heads)
    print("\nregressor losses change %d of %d img2iuv.iuv_est gradients (max |d| %.3g)" % (len(moved), len(heads), diff))
    assert len(moved) > 0 and all(torch.isfinite(full[k]).all() for k in heads)


def test_default_draws_follow_the_reference_order():
    """no noise and no part_drop given: the STN draws, then the dropout draw, on the CPU generator"""
    from danet_b200.iuvmap import draw_part_drop
    from danet_b200.estimator import draw_noise
    net, snap = _net(32)
    B = 3
    d = _in_dict(net, B, 60)
    _restore(net, snap)
    torch.manual_seed(77)
    a = _bits(*_step(net, d, True))
    _restore(net, snap)
    torch.manual_seed(77)
    cn, sn = draw_noise(B)
    drop = draw_part_drop(B).to(DEV)
    b = _bits(*_step(net, d, True, part_drop=drop, noise=(cn.to(DEV), sn.to(DEV))))
    _restore(net, snap)
    _same_all(a, b, "seeded")


def test_eval_mode_agrees_with_infer_net():
    net, snap = _net(48)
    _restore(net, snap)
    B = 4
    d = _in_dict(net, B, 70)
    ret, _ = _step(net, d, False)
    inf = net.infer_net(d["img"])
    para = torch.cat([ret["prediction"]["cam"], ret["prediction"]["shape"], ret["prediction"]["pose"].reshape(B, -1)], 1)
    same = [bool(torch.equal(ret["visualization"]["iuv_pred"][2].argmax(1), inf["visualization"]["iuv_pred"][2].argmax(1)))]
    pi = inf["visualization"]["part_iuv_pred"][:, :, 2].argmax(2)
    same.append(bool(torch.equal(ret["visualization"]["part_iuv_pred"][:, :, 2].argmax(2), pi)))
    err = float((para.detach() - inf["para"]).abs().max())
    print("\neval danet_forward vs infer_net (W48 B=%d): argmax maps equal %s; worst |d para| %.3g" % (B, same, err))
    assert all(same), same                         # this seed's maps equal the plan's, so the bound applies
    assert err <= PARA_TOL, err
