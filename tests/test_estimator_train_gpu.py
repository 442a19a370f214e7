"""GPU tests of the IUV estimator's training path (danet_b200.estimator.iuv_estimator): against the reference's own
IUV_Estimator (tests/golden/estimator_train.npz), against the fp64 test double driven through the same walk at other
batch sizes and widths, repeatability, CUDA-graph capture, no host synchronisation, eval mode against infer_net and
gradient subsets."""
import numpy as np
import pytest
import torch

from estimator_train_common import (EP, OUTPUTS, Recorder, bn_names, decision_flips, golden, golden_image, golden_noise,
                                    golden_targets, projections, step)
from oracle import estimator_train as oet
from oracle import regressor_train as ort

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD_TOL, STATS_TOL = 5e-6, 1e-6
FLIP_BOUND = 5e-2


def _bound(e32):
    """relative error allowed: 1e-5, or 4x what fp32 torch reaches on the same problem"""
    return max(1e-5, 4 * e32)


_NETS = {}


def _net(width):
    """Synthetic DaNet with the keyed weights of seed 0 (the golden's), and a snapshot of its state."""
    if width not in _NETS:
        from danet_b200 import build_synthetic_danet
        net = build_synthetic_danet(width=width, seed=0, device=DEV)
        _NETS[width] = (net, {k: v.clone() for k, v in net.state_dict().items()})
    return _NETS[width]


def _restore(net, snap):
    with torch.no_grad():
        for k, v in net.state_dict().items():
            v.copy_(snap[k])


def _params(net):
    return {k: p for k, p in net.named_parameters() if k.startswith(EP + "iuv_est.")}


def _targets(B, seed):
    img, kps, dp = oet.make_targets(B, seed)
    f = lambda a: torch.as_tensor(a, device=DEV)
    has_iuv = torch.tensor([i % 2 == 0 for i in range(B)], device=DEV)
    has_dp = torch.tensor([float(i % 3 != 1) for i in range(B)], device=DEV)
    return dict(iuv_image_gt=f(img), smpl_kps_gt=f(kps), uvia_dp_gt={k: f(v) for k, v in dp.items()}, has_iuv=has_iuv,
                has_dp=has_dp)


def _run(net, image, training, targets=None, noise=(None, None), proj=None, scale=1.0, hm_weight=1.0, leaves=None,
         want_input_grad=True):
    """iuv_estimator, then the gradients of scale * (sum of the losses + sum_k <proj_k, out_k>).  Returns (outputs,
    losses, {name: grad})."""
    from danet_b200 import iuv_estimator
    net.train(training)
    try:
        x = image.clone().requires_grad_(want_input_grad)
        out = iuv_estimator(net, x, **(targets or {}), center_noise=noise[0], scale_noise=noise[1],
                            stn_hm_weight=hm_weight)
    finally:
        net.eval()
    u, v, idx, ann = out["uvia_pred"]
    o = dict(u=u, v=v, index=idx, ann=ann, hm=out["skps_hm_pred"], part_pred=out["part_iuv_pred"],
             centers=out["stn_kps_pred"], part_iuv_gt=out.get("part_iuv_gt"))
    total = sum(v.sum() for v in out["losses"].values()) if out["losses"] else 0
    if proj is not None:
        total = total + sum((o[k] * proj[k]).sum() for k in proj)
    leaves = {k: p for k, p in (leaves if leaves is not None else _params(net)).items() if p.requires_grad}
    if want_input_grad:
        leaves["image"] = x
    # the hm branch is reached only through the STN losses (skps_hm_pred is detached): no gradient without them
    grads = dict(zip(leaves, torch.autograd.grad(total * scale, list(leaves.values()), allow_unused=True)))
    return {k: (t.detach() if t is not None else None) for k, t in o.items()}, \
        {k: t.detach() for k, t in out["losses"].items()}, grads


# ---------------------------------------------------------------------------------------------------------------------
def test_training_step_matches_reference_golden():
    gold = golden()
    net, snap = _net(32)
    _restore(net, snap)
    img = golden_image(gold).to(DEV)
    out, L, grads = _run(net, img, True, golden_targets(gold, torch.float32, DEV), golden_noise(gold, torch.float32, DEV),
                         hm_weight=float(gold["hm_weight"]))
    err = {}
    for k, v in L.items():
        err["L_" + k] = abs(float(v.sum()) - float(gold["L_" + k])) / max(1.0, abs(float(gold["L_" + k])))
    for k in OUTPUTS + ("part_iuv_gt",):
        err[k] = ort.sketch_error(ort.sketch("out_" + k, out[k]), gold["out_" + k], out[k].numel())
    err["stn_kps_pred"] = float(np.abs(out["centers"].cpu().numpy() - gold["stn_kps_pred"]).max())
    err["g_image"] = ort.sketch_error(ort.sketch("image", grads["image"]), gold["sk_image"], grads["image"].numel())
    sd = net.state_dict()
    stats = {}
    for n in bn_names(snap):
        if not n.startswith(EP):
            continue
        for s, key in (("rm1_", ".running_mean"), ("rv1_", ".running_var")):
            stats[s + n] = ort.sketch_error(ort.sketch(s + n, sd[n + key]), gold[s + n], sd[n + key].numel())
        assert int(sd[n + ".num_batches_tracked"]) == int(gold["nbt_" + n]), n
    pg = max((ort.sketch_error(ort.sketch(k, g), gold["sk_" + k], g.numel()), k) for k, g in grads.items() if k != "image")
    _restore(net, snap)
    k, e = max(err.items(), key=lambda kv: kv[1])
    ks, es = max(stats.items(), key=lambda kv: kv[1])
    print("\ngolden W32 B=2: worst %.3g (%s); running statistics %.3g (%s); parameter gradients %.3g (%s)"
          % (e, k, es, ks, pg[0], pg[1]))
    assert e <= GOLD_TOL, (k, e)
    assert es <= STATS_TOL, (ks, es)


# ---------------------------------------------------------------------------------------------------------------------
def _state64(snap, dtype):
    return {k: (v.to(DEV, dtype).clone() if v.is_floating_point() else v.clone().to(DEV)) for k, v in snap.items()
            if k.startswith(EP)}


def _torch_step(snap, graph, img, training, targets, noise, proj, dtype):
    """the walk through the torch test double in `dtype` on the GPU (cuDNN and TF32 off), from the snapshot's state"""
    state = _state64(snap, dtype)
    cast = lambda t: t.to(dtype) if torch.is_tensor(t) and t.is_floating_point() else t
    tg = None if targets is None else {k: ({a: cast(b) for a, b in v.items()} if isinstance(v, dict) else cast(v))
                                       for k, v in targets.items()}
    nz = tuple(cast(t) for t in noise)
    pj = {k: cast(t) for k, t in proj.items()}
    rec = Recorder(oet.TorchEstimatorOps())
    flags = torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = False, False, False
    try:
        out, L, grads, gx = step(state, graph, cast(img), training, rec, tg, nz, 1.0, pj)
    finally:
        torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags
    grads["image"] = gx
    return out, L, grads, state, rec


def _errors(out, L, grads, stats, ref, scale):
    r_out, r_L, r_grads, r_state = ref[:4]
    err = {}
    for k in OUTPUTS + ("centers",):
        err[k] = ort.rel_norm(out[k], r_out[k])
    for k, v in L.items():
        err["L_" + k] = ort.rel_norm(v.reshape(-1), r_L[k].reshape(-1))
    for k, g in grads.items():
        assert (g is None) == (r_grads[k] is None), k
        if g is not None:
            err["g_" + k] = ort.rel_norm(g.double() / scale, r_grads[k])
    for n, t in stats.items():
        err["st_" + n] = ort.rel_norm(t, r_state[n])
    return err


@pytest.mark.parametrize("B", [1, 3, 16])
@pytest.mark.parametrize("width", [32, 48])
@pytest.mark.parametrize("training", [True, False])
def test_matches_fp64_double(B, width, training):
    from danet_b200.estimator import _cuda_ops, draw_noise, lower_estimator, run_estimator
    from danet_b200.regressor import _attr
    net, snap = _net(width)
    img = oet.make_image(B, 40 + B).to(DEV)
    S = net.graph.outputs["hm"].H
    proj = projections(B, S, 5, torch.float32, DEV)
    targets, noise = (None, (None, None))
    if training:
        targets = _targets(B, 60 + B)
        torch.manual_seed(B)
        noise = tuple(t.to(DEV) for t in draw_noise(B))
    ref = _torch_step(snap, net.graph, img, training, targets, noise, proj, torch.float64)
    r32 = _torch_step(snap, net.graph, img, training, targets, noise, proj, torch.float32)
    stat_keys = [k for k in ref[3] if k.endswith(("running_mean", "running_var"))]
    e32 = _errors(r32[0], r32[1], r32[2], {k: r32[3][k] for k in stat_keys}, ref, 1.0)
    # the GPU walk once more through a recording op table: ReLU and index-argmax decisions against fp64's
    _restore(net, snap)
    net.train(training)
    try:
        rec = Recorder(_cuda_ops())
        low = lower_estimator(net.graph)
        with torch.no_grad():
            state = {k: _attr(net, k) for op in low["ops"] for k in op["keys"]}
            run_estimator(low, state, img, training, rec, noise)
    finally:
        net.eval()
    relu_flips, amax_flips = decision_flips(rec, ref[4])
    worst = []
    for scale in (1e-8, 1e3):
        _restore(net, snap)
        out, L, grads = _run(net, img, training, targets, noise, proj, scale)
        sd = net.state_dict()
        err = _errors(out, L, grads, {k: sd[k] for k in stat_keys}, ref, scale)
        for n in bn_names(snap):
            if n.startswith(EP):
                assert int(sd[n + ".num_batches_tracked"]) == int(snap[n + ".num_batches_tracked"]) + int(training), n
        flips = relu_flips + amax_flips
        bound = {k: (FLIP_BOUND if flips and (k.startswith("g_") or (amax_flips and k in ("part_pred", "L_loss_pU",
                                                                                          "L_loss_pV", "L_loss_pIndexUV")))
                     else _bound(e32.get(k, 0.0))) for k in err}
        k, e = max(err.items(), key=lambda kv: kv[1])
        kr, r = max(((k2, e2 / bound[k2]) for k2, e2 in err.items()), key=lambda kv: kv[1])
        print("\nW%d B=%d training=%d scale=%g: worst relative error %.3g (%s, fp32 torch %.3g); decisions unlike fp64: "
              "%d ReLU, %d index argmax; worst error / bound %.3g (%s)"
              % (width, B, training, scale, e, k, e32.get(k, 0.0), relu_flips, amax_flips, r, kr))
        worst.append((r, kr, err[kr], bound[kr]))
    _restore(net, snap)
    r, kr, e, b = max(worst)
    assert r <= 1.0, (kr, e, b)


# ---------------------------------------------------------------------------------------------------------------------
def _step_bits(net, img, targets, noise, proj):
    out, L, grads = _run(net, img, True, targets, noise, proj)
    return [out[k] for k in OUTPUTS + ("centers", "part_iuv_gt")] + [L[k] for k in sorted(L)] + \
        [grads[k] for k in sorted(grads) if grads[k] is not None]


def test_repeatable_no_sync_and_graph_capture_replays_eager():
    net, snap = _net(32)
    B = 2
    img = oet.make_image(B, 11).to(DEV)
    targets = _targets(B, 12)
    torch.manual_seed(3)
    from danet_b200.estimator import draw_noise
    noise = tuple(t.to(DEV) for t in draw_noise(B))
    proj = projections(B, 56, 6, torch.float32, DEV)
    stat_keys = [k for k in snap if k.startswith(EP) and ("running_" in k or "num_batches" in k)]
    runs = []
    for i in range(2):
        _restore(net, snap)
        torch.cuda.synchronize()
        if i == 1:
            torch.cuda.set_sync_debug_mode("error")
        try:
            res = [t.clone() for t in _step_bits(net, img, targets, noise, proj)]
        finally:
            torch.cuda.set_sync_debug_mode("default")
        runs.append((res, {k: net.state_dict()[k].clone() for k in stat_keys}))
    (r1, s1), (r2, s2) = runs
    assert all(torch.equal(a, b) for a, b in zip(r1, r2))
    assert all(torch.equal(s1[k], s2[k]) for k in stat_keys)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _restore(net, snap)
        _step_bits(net, img, targets, noise, proj)                     # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = _step_bits(net, img, targets, noise, proj)
    _restore(net, snap)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(static, r1))
    sd = net.state_dict()
    assert all(torch.equal(sd[k], s1[k]) for k in stat_keys)
    assert int(sd[EP + "iuv_est.bn1.num_batches_tracked"]) == 1
    _restore(net, snap)


def test_default_noise_is_the_seeded_draw():
    from danet_b200.estimator import draw_noise
    net, snap = _net(32)
    B = 2
    img = oet.make_image(B, 13).to(DEV)
    targets = _targets(B, 14)
    _restore(net, snap)
    torch.manual_seed(5)
    a = _step_bits(net, img, targets, (None, None), None)
    torch.manual_seed(5)
    noise = tuple(t.to(DEV) for t in draw_noise(B))
    _restore(net, snap)
    b = _step_bits(net, img, targets, noise, None)
    _restore(net, snap)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------------------
def test_eval_mode_matches_inference():
    from danet_b200 import iuv_estimator
    from danet_b200.plan import Plan
    net, snap = _net(48)
    _restore(net, snap)
    net.eval()
    B = 3
    img = oet.make_image(B, 21).to(DEV)
    with torch.no_grad():
        out = iuv_estimator(net, img)
    assert out["losses"] == {} and "part_iuv_gt" not in out
    inf = net.infer_net(img)
    sd = {k: v for k, v in net.state_dict().items() if not k.startswith("iuv2smpl.smpl.")}
    plan = Plan(net.graph, sd, B, DEV, conv_algo="tc", precision="exact", keep_all=True)
    plan.run(img)
    torch.cuda.synchronize()
    S = net.graph.outputs["hm"].H

    def nchw(name, C):
        v = plan.out(name)
        return v.reshape(B, S, S, -1)[..., :C].permute(0, 3, 1, 2)
    heads = torch.cat(out["uvia_pred"], 1)
    err = {"heads": ort.rel_norm(heads, nchw("heads", 90)), "hm": ort.rel_norm(out["skps_hm_pred"], nchw("hm", 24)),
           "part_iuv_pred": ort.rel_norm(out["part_iuv_pred"], inf["visualization"]["part_iuv_pred"])}
    kps = float((out["stn_kps_pred"] - inf["stn_kps_pred"]).abs().max())
    print("\neval estimator vs inference (W48 B=3): relative errors %s; stn_kps_pred max |d| %.3g"
          % ({k: "%.3g" % v for k, v in err.items()}, kps))
    assert max(err.values()) < 1e-5, err
    assert kps < 1e-5, kps


# ---------------------------------------------------------------------------------------------------------------------
def test_gradient_subsets_keep_their_bits(monkeypatch):
    from danet_b200 import conv
    net, snap = _net(32)
    B = 2
    img = oet.make_image(B, 31).to(DEV)
    targets = _targets(B, 32)
    torch.manual_seed(9)
    from danet_b200.estimator import draw_noise
    noise = tuple(t.to(DEV) for t in draw_noise(B))
    P = _params(net)
    _restore(net, snap)
    _, _, full = _run(net, img, True, targets, noise)
    # no image gradient: the stem convolution is asked for no input gradient
    seen = []
    bwd = conv._Conv2d.backward

    def spy(ctx, gy):
        seen.append((ctx.geom[1], ctx.needs_input_grad[0]))
        return bwd(ctx, gy)
    monkeypatch.setattr(conv._Conv2d, "backward", staticmethod(spy))
    _restore(net, snap)
    _, _, nog = _run(net, img, True, targets, noise, want_input_grad=False)
    monkeypatch.undo()
    assert (3, False) in seen and all(need for c, need in seen if c != 3)
    assert all(torch.equal(nog[k], full[k]) for k in P)
    assert all(full[k] is not None for k in full)
    frozen = {EP + "iuv_est.conv1.weight", EP + "iuv_est.bn2.weight", EP + "iuv_est.final_pred.predict_u.weight",
              EP + "iuv_est.final_pred.predict_partial_iuv.bias", EP + "iuv_est.stage4.2.fuse_layers.0.3.0.weight"}
    assert frozen <= set(P)
    _restore(net, snap)
    try:
        for k in frozen:
            P[k].requires_grad_(False)
        _, _, sub = _run(net, img, True, targets, noise)
    finally:
        for k in frozen:
            P[k].requires_grad_(True)
    assert set(sub) == set(full) - frozen
    assert all(torch.equal(sub[k], full[k]) for k in sub)
    _restore(net, snap)
