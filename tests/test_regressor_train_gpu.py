"""GPU tests of the regressor's training path (danet_b200.regressor.body_branch / limb_branch / predictor): against the
reference's own DecomposedPredictor (tests/golden/regressor_train.npz), against the fp64 test double on full tensors
at other batch and map sizes, eval mode against infer_net, repeatability, CUDA-graph capture, batch independence,
gradient subsets and argument checks."""
import numpy as np
import pytest
import torch

from oracle import regressor_train as ort
from regressor_train_common import (RP, Recorder, branch_param_keys, bn2d_names, double_step, golden, golden_inputs,
                                    relu_flips)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    return golden()


@pytest.fixture(scope="module")
def net():
    """Synthetic DaNet with the keyed weights of seed 0 (the golden's)."""
    from danet_b200 import build_synthetic_danet
    return build_synthetic_danet(width=32, seed=0, device=DEV)


@pytest.fixture(scope="module")
def snapshot(net):
    return {k: v.clone() for k, v in net.state_dict().items()}


def _restore(net, snap):
    with torch.no_grad():
        for k, v in net.state_dict().items():
            v.copy_(snap[k])


def _state(net):
    return dict(net.named_parameters())


def _branch_params(net):
    P = _state(net)
    return {k: P[k] for k in P if k.startswith(RP) and k in set(branch_param_keys(net.state_dict()))}


def _trained(net):
    """the 157 tensors the predictor trains: the branches' 128 and the head's 29 (rot2pos / pos2rot are unused)"""
    from danet_b200.regressor import PARAM_NAMES
    P = _state(net)
    return {**_branch_params(net), **{RP + n: P[RP + n] for n in PARAM_NAMES}}


def _fp32_branch_grads(snapshot, body, part, training, g_gp, g_rf, dev):
    """(global_para, rot_feats, {key: grad}) of the test double in fp32 on `dev` (on the GPU with cuDNN and TF32 off)
    from the snapshot's state: a yardstick of what fp32 arithmetic reaches on a problem."""
    state = {k: v.clone().to(dev) for k, v in snapshot.items() if k.startswith(RP)}
    from danet_b200 import netgraph
    flags = torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = False, False, False
    try:
        return double_step(state, netgraph.danet_graph(32), body.to(dev), part.to(dev), training,
                           torch.as_tensor(np.asarray(g_gp), dtype=torch.float32, device=dev),
                           torch.as_tensor(np.asarray(g_rf), dtype=torch.float32, device=dev))
    finally:
        torch.backends.cudnn.enabled, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags


def _fp32_errors(snapshot, body, part, training, g_gp, g_rf, err_of):
    """{key: error} of fp32 torch, the larger of its CPU and GPU runs.  A ReLU or max-pool decision whose margin is
    below fp32 rounding can go the other way than in fp64 and move a whole pixel's gradient: on the 2x2 maps of the
    last blocks that is percents of a parameter gradient.  Which fp32 implementation meets such a margin depends on
    its rounding, so the bound takes the worse of two independent ones."""
    out = {}
    for dev in (torch.device("cpu"), DEV):
        for k, e in err_of(*_fp32_branch_grads(snapshot, body, part, training, g_gp, g_rf, dev)).items():
            out[k] = max(out.get(k, 0.0), e)
    return out


FLIP_BOUND = 5e-2
GRAD_BOUND = 2e-3


def _bound(e32):
    """relative error allowed: 1e-5, or 4x what fp32 torch reaches on the same problem"""
    return max(1e-5, 4 * e32)


def _zero_grads(net):
    for p in net.parameters():
        p.grad = None


def test_training_step_matches_reference_golden(gold, net, snapshot):
    from danet_b200.regressor import body_branch, gcn_head, gcn_head_losses, limb_branch, PARAM_NAMES
    _restore(net, snapshot)
    _zero_grads(net)
    net.train()
    try:
        body, part = (t.to(DEV).requires_grad_() for t in golden_inputs(gold))
        gp = body_branch(net, body)
        rf = limb_branch(net, part)
        gp.retain_grad()
        rf.retain_grad()
        out = gcn_head(net, rf, gp)
        L = gcn_head_losses(out, torch.tensor(gold["target"], dtype=torch.float32, device=DEV),
                            torch.tensor(gold["gt_joints"], dtype=torch.float32, device=DEV),
                            torch.tensor(gold["has_smpl"], device=DEV))
        (L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"] +
         (out["para"] * torch.tensor(gold["G"], dtype=torch.float32, device=DEV)).sum()).backward()
    finally:
        net.eval()
    got = {"para": out["para"], "pose0": out["joint_rotation"][0], "coord0": out["joint_position"][0],
           "coord1": out["joint_position"][1], "global_para": gp, "rot_feats": rf, "g_global_para": gp.grad,
           "g_rot_feats": rf.grad}
    worst = {}
    for k, v in got.items():
        worst[k] = ort.rel_norm(v, gold[k])
    for k in ("joint_rotation0", "joint_position0", "joint_position1"):
        worst["L_" + k] = abs(L[k].item() - float(gold["L_" + k])) / abs(float(gold["L_" + k]))
    for k, v in worst.items():
        assert v < 1e-5, (k, v)
    P = _state(net)
    # branch gradients to GRAD_BOUND or 4x the fp32 torch yardstick.  The widest are BatchNorm sums over a dy that the
    # next training-mode BatchNorm centred: limb_net.3.layer1.0.bn1.bias (fp32 torch is as far off) and body_net.1.bias,
    # where the path lands near 1e-3 and fp32 torch near 1e-6 (DESIGN section 8, f2)
    body32, part32 = golden_inputs(gold)
    e32s = _fp32_errors(snapshot, body32, part32, True, gold["g_global_para"], gold["g_rot_feats"],
                        lambda gp, rf, g: {k: ort.sketch_error(ort.sketch(k, v), gold["sk_" + k], v.numel())
                                           for k, v in g.items()})
    sk = {}
    for k, t in list(_branch_params(net).items()) + [("body_iuv", body), ("part_iuv", part)]:
        assert t.grad is not None, k
        e = ort.sketch_error(ort.sketch(k, t.grad), gold["sk_" + k], t.numel())
        e32 = e32s[k]
        sk[k] = (e, e32)
    worst_sk = sorted(((e, k, e32) for k, (e, e32) in sk.items()), reverse=True)[:8]
    print("\ngolden: widest branch gradient sketches: " + "; ".join("%s %.3g (fp32 torch %.3g)" % (k[len(RP):] if
                                                                     k.startswith(RP) else k, e, e32)
                                                                     for e, k, e32 in worst_sk))
    for k, (e, e32) in sk.items():
        assert e <= max(GRAD_BOUND, 4 * e32), (k, e, e32)
    for n in PARAM_NAMES:
        t = P[RP + n]
        assert t.grad is not None, n
        sk[RP + n] = (ort.sketch_error(ort.sketch(RP + n, t.grad), gold["sk_" + RP + n], t.numel()), 0.0)
        assert sk[RP + n][0] < 1e-4, (n, sk[RP + n])
    assert len(sk) == 159
    stats = {}
    sd = net.state_dict()
    for n in [k[4:] for k in gold.files if k.startswith("nbt_")]:
        for a, b in (("rm1_", ".running_mean"), ("rv1_", ".running_var")):
            ref = gold[a + n]
            stats[a + n] = float(np.abs(sd[n + b].cpu().numpy() - ref).max() / max(1.0, np.abs(ref).max()))
        assert int(sd[n + ".num_batches_tracked"]) == int(gold["nbt_" + n]) == 1, n
    k1, e1 = max(worst.items(), key=lambda kv: kv[1])
    k2, e2 = max(stats.items(), key=lambda kv: kv[1])
    k3, (e3, e3_32) = max(sk.items(), key=lambda kv: kv[1][0])
    print("\ngolden: outputs and losses %.3g (%s); running statistics %.3g (%s); gradient sketches %.3g (%s, fp32 torch "
          "%.3g)" % (e1, k1, e2, k2, e3, k3, e3_32))
    assert e2 < 1e-6, (k2, e2)


_REF = {}


def _reference(snapshot, B, S, training):
    """fp64 test double for one (B, S, mode): outputs, gradients for upstream (G_gp, G_rf), running statistics"""
    key = (B, S, training)
    if key not in _REF:
        state = {k: v.detach().cpu().double() if v.is_floating_point() else v.cpu().clone()
                 for k, v in snapshot.items() if k.startswith(RP)}
        from danet_b200 import netgraph
        body, part = ort.make_inputs(B, S, 100 + B * S + int(training))
        rng = np.random.default_rng(B * S)
        G_gp, G_rf = rng.normal(0, 1, (B, 13)), rng.normal(0, 1, (B, 24, 128))
        rec = Recorder(ort.TorchTrainOps())
        gp, rf, grads = double_step(state, netgraph.danet_graph(32), body, part, training, G_gp, G_rf, ops=rec)
        stats = {n: (state[n + ".running_mean"].clone(), state[n + ".running_var"].clone()) for n in bn2d_names(state)}
        e32 = _fp32_errors(snapshot, body, part, training, G_gp, G_rf,
                           lambda gp32, rf32, g32: {"global_para": ort.rel_norm(gp32, gp), "rot_feats": ort.rel_norm(rf32, rf),
                                                    **{"g_" + k: ort.rel_norm(v, grads[k]) for k, v in g32.items()}})
        _REF[key] = (body, part, G_gp, G_rf, gp, rf, grads, stats, e32, rec.bn)
    return _REF[key]


@pytest.mark.parametrize("B", [1, 3, 16])
@pytest.mark.parametrize("S", [56, 40])
@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("scale", [1e-8, 1e3])
def test_branches_match_fp64_double(net, snapshot, B, S, training, scale):
    from danet_b200.regressor import body_branch, limb_branch
    body, part, G_gp, G_rf, gp_ref, rf_ref, g_ref, stats_ref, e32, bn_ref = _reference(snapshot, B, S, training)
    _restore(net, snapshot)
    _zero_grads(net)
    net.train(training)
    try:
        b, p = body.to(DEV).requires_grad_(), part.to(DEV).requires_grad_()
        gp, rf = body_branch(net, b), limb_branch(net, p)
        torch.autograd.backward([gp, rf], [torch.tensor(G_gp * scale, dtype=torch.float32, device=DEV),
                                           torch.tensor(G_rf * scale, dtype=torch.float32, device=DEV)])
    finally:
        net.eval()
    err = {"global_para": ort.rel_norm(gp, gp_ref), "rot_feats": ort.rel_norm(rf, rf_ref),
           "g_body_iuv": ort.rel_norm(b.grad.double() / scale, g_ref["body_iuv"]),
           "g_part_iuv": ort.rel_norm(p.grad.double() / scale, g_ref["part_iuv"])}
    for k, t in _branch_params(net).items():
        assert t.grad is not None, k
        err["g_" + k] = ort.rel_norm(t.grad.double() / scale, g_ref[k])
    sd = net.state_dict()
    for n, (rm, rv) in stats_ref.items():
        err["rm_" + n], err["rv_" + n] = ort.rel_norm(sd[n + ".running_mean"], rm), ort.rel_norm(sd[n + ".running_var"], rv)
        assert int(sd[n + ".num_batches_tracked"]) == int(training), n
    # the same walk once more from the same state, recording every BatchNorm output: a ReLU decision that differs from
    # fp64 (a pre-activation within fp32 rounding of 0) moves that pixel's whole gradient, percents of a parameter
    # gradient on 2x2 maps.  Where that happens the gradients are held to FLIP_BOUND instead of the fp32 yardstick.
    from danet_b200 import regressor as R
    _restore(net, snapshot)
    net.train(training)
    try:
        rec = Recorder(R._cuda_ops())
        low = R.lower_branches(net.graph)
        with torch.no_grad():
            state = {k: R._attr(net, k) for name in ("body", "limb") for op in low[name]["ops"] for k in op["keys"]}
            R.run_branch(low["body"], state, body.to(DEV), training, rec)
            R.run_branch(low["limb"], state, part.to(DEV).reshape(B * 24, 21, S, S), training, rec)
    finally:
        net.eval()
        _restore(net, snapshot)
    flips = relu_flips(rec.bn, bn_ref)
    bound = {k: (FLIP_BOUND if flips and k.startswith("g_") else _bound(e32.get(k, 0.0))) for k in err}
    k, e = max(err.items(), key=lambda kv: kv[1])
    kr, r = max(((k2, e2 / bound[k2]) for k2, e2 in err.items()), key=lambda kv: kv[1])
    print("\nB=%d S=%d training=%d scale=%g: worst relative Frobenius error %.3g (%s, fp32 torch %.3g); ReLU decisions "
          "unlike fp64: %d; worst error / bound %.3g (%s)" % (B, S, training, scale, e, k, e32.get(k, 0.0), flips, r, kr))
    assert r <= 1.0, (kr, err[kr], bound[kr])


def _clean_inputs(net, images):
    from danet_b200.iuvmap import iuvmap_clean
    out = net.infer_net(images)
    vis = out["visualization"]
    body = torch.cat(vis["iuv_pred"][:3], 1).contiguous()
    pp = vis["part_iuv_pred"]
    parts = [torch.stack(iuvmap_clean(pp[:, i, 0], pp[:, i, 1], pp[:, i, 2])[:3], 1) for i in range(24)]
    return out["para"].clone(), body.clone(), torch.stack(parts, 1).contiguous()


def _images(B, seed):
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(seed)
    low = torch.randn(B, 3, 7, 7, generator=g)
    return (F.interpolate(low, size=224, mode="bilinear", align_corners=False) * 2 +
            0.3 * torch.randn(B, 3, 224, 224, generator=g)).to(DEV)


def test_eval_mode_matches_inference_and_plans_refold(net, snapshot):
    from danet_b200.regressor import predictor
    _restore(net, snapshot)
    net.eval()
    para, body, part = _clean_inputs(net, _images(3, 7))
    got = predictor(net, body, part)
    assert got["joint_rotation"] == [] and got["joint_position"] == []
    e = (got["para"] - para).abs().max().item()
    print("\neval predictor vs infer_net: max |d para| = %.3g" % e)
    assert e < 2e-5, e
    plan0 = net.plan_for(3, DEV)
    net.train()
    try:
        predictor(net, body, part)
    finally:
        net.eval()
    assert net.plan_for(3, DEV) is not plan0
    _restore(net, snapshot)


def _train_step(net, body, part, G, want_input_grad=True, params=None):
    from danet_b200.regressor import gcn_head_losses, predictor
    b = body.clone().requires_grad_(want_input_grad)
    p = part.clone().requires_grad_(want_input_grad)
    out = predictor(net, b, p)
    B = body.shape[0]
    tgt, gt = torch.zeros(B, 229, device=DEV), torch.zeros(B, 24, 3, device=DEV)
    L = gcn_head_losses(out, tgt, gt, torch.ones(B, device=DEV))
    total = L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"] + (out["para"] * G).sum()
    leaves = list(params) if params is not None else [t for t in net.parameters() if t.requires_grad]
    leaves += [b, p] if want_input_grad else []
    grads = torch.autograd.grad(total, leaves)
    return [out["para"].detach(), total.detach()] + list(grads)


def test_repeatable_and_graph_capture_replays_eager(net, snapshot):
    _restore(net, snapshot)
    body, part = (t.to(DEV) for t in ort.make_inputs(4, 56, 9))
    G = torch.randn(4, 229, generator=torch.Generator().manual_seed(1)).to(DEV)
    params = list(_trained(net).values())
    stat_keys = [k for k in net.state_dict() if k.startswith(RP) and ("running_" in k or "num_batches" in k)]
    net.train()
    try:
        runs = []
        for _ in range(2):
            _restore(net, snapshot)
            res = [t.clone() for t in _train_step(net, body, part, G, params=params)]
            runs.append((res, {k: net.state_dict()[k].clone() for k in stat_keys}))
        (r1, s1), (r2, s2) = runs
        assert all(torch.equal(a, b) for a, b in zip(r1, r2))
        assert all(torch.equal(s1[k], s2[k]) for k in stat_keys)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _train_step(net, body, part, G, params=params)           # warm-up on the side stream
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = _train_step(net, body, part, G, params=params)
        _restore(net, snapshot)
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(static, r1))
        sd = net.state_dict()
        assert all(torch.equal(sd[k], s1[k]) for k in stat_keys)
        assert int(sd[RP + "limb_reslayer.layer4.1.bn2.num_batches_tracked"]) == 1
    finally:
        net.eval()
        _restore(net, snapshot)


def test_eval_image_independent_of_its_batch(net, snapshot):
    from danet_b200.regressor import predictor
    _restore(net, snapshot)
    net.eval()
    body, part = (t.to(DEV) for t in ort.make_inputs(3, 56, 21))
    G = torch.randn(3, 229, generator=torch.Generator().manual_seed(2)).to(DEV)

    def run(lo, hi):
        b, p = body[lo:hi].clone().requires_grad_(), part[lo:hi].clone().requires_grad_()
        para = predictor(net, b, p)["para"]
        gb, gp = torch.autograd.grad((para * G[lo:hi]).sum(), [b, p])
        return para.detach(), gb, gp
    full = run(0, 3)
    for i in range(3):
        one = run(i, i + 1)
        assert torch.equal(one[0], full[0][i:i + 1]), i
        # the input gradients agree to rounding: the first convolutions' input gradient splits dy * 2^s into fp16
        # hi + lo with 2^s from the batch's max |dy|, so the smallest entries round at a batch-dependent position
        e = max(ort.rel_norm(one[1], full[1][i:i + 1]), ort.rel_norm(one[2], full[2][i:i + 1]))
        print("\nimage %d alone vs in its batch: input gradients %.3g" % (i, e))
        assert e < 1e-6, (i, e)


def test_gradient_subsets_keep_their_bits(net, snapshot):
    body, part = (t.to(DEV) for t in ort.make_inputs(2, 40, 4))
    G = torch.randn(2, 229, generator=torch.Generator().manual_seed(3)).to(DEV)
    P = _trained(net)
    names = list(P)
    frozen = {RP + "body_net.0.weight", RP + "limb_net.1.weight", RP + "limb_reslayer.layer4.0.conv1.weight",
              RP + "body_net.3.final_layer.bias"}
    net.train()
    try:
        _restore(net, snapshot)
        full = dict(zip(names + ["body_iuv", "part_iuv"], _train_step(net, body, part, G, params=[P[k] for k in names])[2:]))
        _restore(net, snapshot)
        _zero_grads(net)
        for k in frozen:
            P[k].requires_grad_(False)
        b, p = body.clone(), part.clone()
        from danet_b200.regressor import gcn_head_losses, predictor
        out = predictor(net, b, p)
        L = gcn_head_losses(out, torch.zeros(2, 229, device=DEV), torch.zeros(2, 24, 3, device=DEV),
                            torch.ones(2, device=DEV))
        (L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"] + (out["para"] * G).sum()).backward()
        assert b.grad is None and p.grad is None
        for k in names:
            if k in frozen:
                assert P[k].grad is None, k
            else:
                assert P[k].grad is not None and torch.equal(P[k].grad, full[k]), k
    finally:
        for k in frozen:
            P[k].requires_grad_(True)
        _zero_grads(net)
        net.eval()
        _restore(net, snapshot)


def test_refuses_bad_arguments(net):
    from danet_b200.regressor import body_branch, limb_branch, predictor
    body, part = (t.to(DEV) for t in ort.make_inputs(2, 24, 0))
    for bad in (body[:, :74], body[0], body.double(), body.cpu(), body[:, :, :, :23], body[:0]):
        with pytest.raises(ValueError):
            body_branch(net, bad.contiguous() if bad.is_cuda else bad)
    for bad in (part[:, :23], part.reshape(2, 24, 21, 24, 24), part.half(), part.cpu(), part[..., :20]):
        with pytest.raises(ValueError):
            limb_branch(net, bad)
    with pytest.raises(ValueError):
        predictor(net, body, part[:1])
    with pytest.raises(ValueError):
        body_branch(object(), body)
