"""GPU tests of the regressor head's training path (danet_b200.regressor, csrc/gcn_train.cu): against the reference's
own autograd (tests/golden/gcn_head.npz), against the fp64 restatement at other batch sizes and selections, eval mode
against the inference kernel, repeatability, CUDA-graph capture and argument checks."""
import numpy as np
import pytest
import torch

from gcn_head_common import RP, golden, golden_params, random_problem, rel_norm
from oracle import gcn_head as og

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    return golden()


@pytest.fixture(scope="module")
def net(gold):
    """Synthetic DaNet (keyed weights, seed 0: the golden's) with the golden's edge_importance."""
    from danet_b200 import build_synthetic_danet
    m = build_synthetic_danet(width=32, seed=0, device=DEV)
    with torch.no_grad():
        m.iuv2smpl.smpl_para_Outs.edge_importance.copy_(torch.from_numpy(gold["edge_importance"]))
    return m


def _set_bn(net, bn):
    mod = net.iuv2smpl.smpl_para_Outs
    with torch.no_grad():
        for n, (rm, rv) in bn.items():
            m = mod.get_submodule(n)
            m.running_mean.copy_(torch.as_tensor(np.asarray(rm, np.float32)))
            m.running_var.copy_(torch.as_tensor(np.asarray(rv, np.float32)))
            m.num_batches_tracked.zero_()


def _params(net):
    from danet_b200.regressor import PARAM_NAMES
    mod = net.iuv2smpl.smpl_para_Outs
    return {n: mod.get_parameter(n) for n in PARAM_NAMES}


def _step(net, rot, gp, target, gt, has, G):
    """forward + head losses + <G, para>, backward; returns (out, losses, {name: grad})."""
    from danet_b200.regressor import TRAINING_ONLY, gcn_head, gcn_head_losses
    P = _params(net)
    rot = torch.as_tensor(rot, device=DEV).requires_grad_()
    gp = torch.as_tensor(gp, device=DEV).requires_grad_()
    out = gcn_head(net, rot, gp)
    total = (out["para"] * torch.as_tensor(G, device=DEV)).sum()
    L = None
    if net.training:
        L = gcn_head_losses(out, torch.as_tensor(target, device=DEV), torch.as_tensor(gt, device=DEV),
                            torch.as_tensor(has, device=DEV))
        total = total + L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"]
    names = [n for n in P if net.training or n not in TRAINING_ONLY]
    gr = torch.autograd.grad(total, [P[n] for n in names] + [rot, gp])
    grads = dict(zip(names + ["rot_feats", "global_para"], gr))
    return out, L, grads


def test_training_step_matches_reference_golden(gold, net):
    g = gold
    _, _, bn = golden_params(g)
    _set_bn(net, bn)
    net.train()
    from danet_b200.regressor import gcn_head, gcn_head_losses
    rot = torch.tensor(g["rot_feats"], device=DEV, requires_grad=True)
    gp = torch.tensor(g["global_para"], device=DEV, requires_grad=True)
    out = gcn_head(net, rot, gp)
    L = gcn_head_losses(out, torch.tensor(g["target"], device=DEV), torch.tensor(g["gt_joints"], device=DEV),
                        torch.tensor(g["has_smpl"], device=DEV))
    for p in _params(net).values():
        p.grad = None
    (L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"] +
     (out["para"] * torch.tensor(g["G"], device=DEV)).sum()).backward()
    net.eval()
    got = {"para": out["para"], "pose0": out["joint_rotation"][0], "coord0": out["joint_position"][0],
           "coord1": out["joint_position"][1]}
    for k, v in got.items():
        assert np.abs(v.detach().cpu().numpy() - g[k]).max() < 1e-5, k
    for k in ("joint_rotation0", "joint_position0", "joint_position1"):
        assert abs(L[k].item() - float(g["L_" + k])) <= 1e-5 * abs(float(g["L_" + k])), k
    P = _params(net)
    mod = net.iuv2smpl.smpl_para_Outs
    for n in og.PARAM_NAMES:
        assert P[n].grad is not None, n
        e = rel_norm(P[n].grad.cpu().numpy(), g["g_" + n])
        assert e < 1e-4, (n, e)
    assert mod.get_buffer("mean_pose").grad is None
    assert rel_norm(rot.grad.cpu().numpy(), g["g_rot_feats"]) < 1e-4
    assert rel_norm(gp.grad.cpu().numpy(), g["g_global_para"]) < 1e-4
    for n in og.BN_NAMES:
        m = mod.get_submodule(n)
        assert np.abs(m.running_mean.cpu().numpy() - g["rm1_" + n]).max() < 1e-6, n
        assert np.abs(m.running_var.cpu().numpy() - g["rv1_" + n]).max() < 1e-6, n
        assert int(m.num_batches_tracked.item()) == int(g["nbt_" + n]) == 1


@pytest.mark.parametrize("B", [1, 16, 64])
@pytest.mark.parametrize("has", ["all", "some", "none"])
def test_training_step_matches_fp64_restatement(gold, net, B, has):
    P, buf, bn = golden_params(gold)
    _set_bn(net, bn)
    rot, gpara, target, gt, h, G = random_problem(B, has, seed=B * 10 + len(has))
    net.train()
    out, L, grads = _step(net, rot, gpara, target, gt, h, G)
    net.eval()
    ref, sv = og.forward(P, buf, bn, rot, gpara, training=True)
    Lr, (gp0, gc0, gc1) = og.losses(ref["pose0"], ref["coord0"], ref["coord1"], target, gt, h)
    Gr = og.backward(P, sv, {"para": G, "pose0": gp0, "coord0": gc0, "coord1": gc1}, training=True)
    # fp32 against fp64: rot6d's Gram-Schmidt amplifies rounding where a 6d pair is nearly parallel (up to ~5e-5 on a
    # few of the 13 824 rotation entries at B = 64); the gradients below are held to 1e-4 in norm
    np.testing.assert_allclose(out["para"].detach().cpu().numpy(), ref["para"], atol=1e-4)
    np.testing.assert_allclose(out["joint_rotation"][0].detach().cpu().numpy(), ref["pose0"], atol=1e-4)
    for k in range(2):
        np.testing.assert_allclose(out["joint_position"][k].detach().cpu().numpy(), ref["coord%d" % k], atol=2e-5, rtol=1e-5)
    got_L = np.array([L[k].item() for k in ("joint_rotation0", "joint_position0", "joint_position1")])
    if has == "none":
        assert (got_L == 0).all()
        gz = torch.autograd.grad(sum(L.values()), [out["joint_rotation"][0]] + out["joint_position"])
        assert all((t == 0).all() for t in gz)
    else:
        np.testing.assert_allclose(got_L, Lr, rtol=1e-5)
    # gradients: 1e-4 in norm, or within 4x of what fp32 autograd over the torch restatement reaches on this device
    # (dW = (A X)^T dY sums 24 B rows whose BatchNorm-centred dY cancel: fp32 loses digits there whatever the order)
    t = lambda x, rg=False: torch.tensor(np.asarray(x, np.float32), device=DEV, requires_grad=rg)
    Pt = {k: t(v, True) for k, v in P.items()}
    rt, gt32 = t(rot, True), t(gpara, True)
    p32 = og.torch_head(Pt, {k: t(v) for k, v in buf.items()}, {k: (t(a), t(b)) for k, (a, b) in bn.items()}, rt, gt32)
    tot = sum((a * t(b)).sum() for a, b in zip(p32, (G, gp0, gc0, gc1)))
    g32 = dict(zip(list(grads), torch.autograd.grad(tot, [Pt[n] for n in list(grads)[:-2]] + [rt, gt32])))
    for n, gv in grads.items():
        e, e32 = rel_norm(gv.cpu().numpy(), Gr[n]), rel_norm(g32[n].cpu().numpy(), Gr[n])
        assert e < max(1e-4, 4 * e32), (n, e, e32)
    for n in og.BN_NAMES:
        m = net.iuv2smpl.smpl_para_Outs.get_submodule(n)
        assert np.abs(m.running_mean.cpu().numpy() - ref["bn"][n][0]).max() < 1e-6
        assert np.abs(m.running_var.cpu().numpy() - ref["bn"][n][1]).max() < 1e-6


def test_eval_mode_matches_inference_kernel_and_plan_sees_new_statistics(gold, net):
    from danet_b200.plan import CudaOps
    from danet_b200.regressor import gcn_head
    _, _, bn = golden_params(gold)
    _set_bn(net, bn)
    net.eval()
    B = 4
    rot, gpara, target, gt, h, G = random_problem(B, "some", seed=7)
    rot_t, gp_t = torch.tensor(rot, device=DEV), torch.tensor(gpara, device=DEV)

    def infer(plan):
        p = torch.empty(B, 1, 1, 229, device=DEV)
        CudaOps(DEV).gcn_head(plan.gcn, rot_t.reshape(B * 24, 1, 1, 128), gp_t.reshape(B, 1, 1, 13), p)
        return p.reshape(B, 229)

    plan0 = net.plan_for(B, DEV)
    para = gcn_head(net, rot_t, gp_t)["para"]
    assert (para - infer(plan0)).abs().max().item() < 1e-6
    # eval mode is differentiable (frozen BatchNorm) and leaves the running statistics alone
    rot_g = rot_t.clone().requires_grad_()
    out = gcn_head(net, rot_g, gp_t)
    assert out["joint_rotation"] == [] and out["joint_position"] == []
    out["para"].sum().backward()
    assert rot_g.grad is not None and rot_g.grad.abs().sum() > 0
    # a training-mode call moves the running statistics: the plan cache rebuilds, and eval mode follows them
    net.train()
    gcn_head(net, torch.tensor(rot * 1.3, device=DEV), gp_t)
    net.eval()
    plan1 = net.plan_for(B, DEV)
    assert plan1 is not plan0
    para1 = gcn_head(net, rot_t, gp_t)["para"]
    assert (para1 - para).abs().max().item() > 1e-4
    assert (para1 - infer(plan1)).abs().max().item() < 1e-6


def test_repeatable_bit_for_bit(gold, net):
    _, _, bn = golden_params(gold)
    rot, gpara, target, gt, h, G = random_problem(16, "some", seed=3)
    res = []
    for _ in range(2):
        _set_bn(net, bn)
        net.train()
        out, L, grads = _step(net, rot, gpara, target, gt, h, G)
        net.eval()
        res.append((out, L, grads))
    (o1, L1, g1), (o2, L2, g2) = res
    assert torch.equal(o1["para"], o2["para"]) and torch.equal(o1["joint_rotation"][0], o2["joint_rotation"][0])
    assert all(torch.equal(a, b) for a, b in zip(o1["joint_position"], o2["joint_position"]))
    assert all(torch.equal(L1[k], L2[k]) for k in L1)
    assert all(torch.equal(g1[k], g2[k]) for k in g1)


def test_cuda_graph_replay_equals_eager(gold, net):
    from danet_b200.regressor import PARAM_NAMES, gcn_head, gcn_head_losses
    _, _, bn = golden_params(gold)
    rot, gpara, target, gt, h, G = random_problem(16, "some", seed=11)
    rot_t, gp_t = torch.tensor(rot, device=DEV, requires_grad=True), torch.tensor(gpara, device=DEV, requires_grad=True)
    tgt, gtj, hs, Gt = (torch.tensor(x, device=DEV) for x in (target, gt, h, G))
    P = _params(net)
    leaves = [P[n] for n in PARAM_NAMES] + [rot_t, gp_t]

    def step():
        out = gcn_head(net, rot_t, gp_t)
        L = gcn_head_losses(out, tgt, gtj, hs)
        total = L["joint_rotation0"] + L["joint_position0"] + L["joint_position1"] + (out["para"] * Gt).sum()
        grads = list(torch.autograd.grad(total, leaves))
        return [out["para"].detach(), total.detach()] + grads     # keep no graph alive across the capture

    net.train()
    _set_bn(net, bn)
    eager = [t.clone() for t in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                           # warm-up on the side stream (library load, allocator)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    _set_bn(net, bn)
    graph.replay()
    torch.cuda.synchronize()
    net.eval()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


def test_refuses_bad_arguments(net):
    from danet_b200.regressor import gcn_head, gcn_head_losses
    net.train()
    try:
        with pytest.raises(RuntimeError):
            gcn_head(net, torch.zeros(2, 24, 128), torch.zeros(2, 13, device=DEV))
        with pytest.raises(RuntimeError):
            gcn_head(net, torch.zeros(2, 24, 128, device=DEV), torch.zeros(2, 13))
        for r, g in (((2, 24, 127), (2, 13)), ((2, 23, 128), (2, 13)), ((2, 24, 128), (3, 13)), ((2, 24, 128), (2, 12)),
                     ((0, 24, 128), (0, 13)), ((48, 128), (2, 13))):
            with pytest.raises(ValueError):
                gcn_head(net, torch.zeros(*r, device=DEV), torch.zeros(*g, device=DEV))
        out = gcn_head(net, torch.rand(2, 24, 128, device=DEV), torch.zeros(2, 13, device=DEV))
        tgt, gt = torch.zeros(2, 229, device=DEV), torch.zeros(2, 24, 3, device=DEV)
        gcn_head_losses(out, tgt, gt, torch.ones(2, device=DEV))
        with pytest.raises(ValueError):
            gcn_head_losses(out, tgt, gt, torch.ones(3, device=DEV))
        with pytest.raises(ValueError):
            gcn_head_losses(out, tgt[:, :228], gt, torch.ones(2, device=DEV))
        with pytest.raises(ValueError):
            gcn_head_losses(out, tgt, gt[:, :23], torch.ones(2, device=DEV))
        cpu = {"joint_rotation": [t.cpu() for t in out["joint_rotation"]],
               "joint_position": [t.cpu() for t in out["joint_position"]]}
        with pytest.raises(RuntimeError):
            gcn_head_losses(cpu, tgt.cpu(), gt.cpu(), torch.ones(2))
        net.eval()
        with pytest.raises(ValueError):                   # eval mode has no intermediate outputs
            gcn_head_losses(gcn_head(net, torch.rand(2, 24, 128, device=DEV), torch.zeros(2, 13, device=DEV)), tgt, gt,
                            torch.ones(2, device=DEV))
    finally:
        net.eval()
