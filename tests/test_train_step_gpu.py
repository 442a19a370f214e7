"""GPU tests of danet_b200.training.train_step: bit-identical to the reference's train_step loop written out on the same
CUDA ops with torch.optim.Adam (through a pretraining step and a learning-rate decay), repeatable, the total loss falling
over 20 steps, and two ranks over NCCL (skipped below two GPUs)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_batch(B, seed, steps, device=DEV):
    """a data batch (prepare_targets' keys, the image, DensePose points, 3-D joints), the fits, and per step the STN
    noise and part-dropout masks, all drawn once"""
    from danet_b200.estimator import draw_noise
    from danet_b200.iuvmap import draw_part_drop
    from oracle import estimator_train as oet
    rng = np.random.default_rng(seed)
    T = lambda a, dt=torch.float32: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=device)

    def pose(n):
        p = rng.normal(0, 0.25, (n, 72))
        p[:, :3] = [np.pi, 0, 0] + rng.normal(0, 0.1, (n, 3))
        return p
    kp = np.concatenate([rng.uniform(-0.8, 0.8, (B, 49, 2)), rng.choice([1.0, 0.3, 0.0], (B, 49, 1))], -1)
    kp[:, 25:30, 2] = 1.0
    flag = lambda: T(rng.random(B) < 0.6, torch.uint8)
    _, _, dp = oet.make_targets(B, seed)
    batch = dict(keypoints=T(kp), pose=T(pose(B)), betas=T(rng.normal(0, 1, (B, 10))), has_smpl=flag(),
                 has_dp=flag(), iuv_annotated=flag(), smpl_2dkps=T(rng.uniform(-1, 1, (B, 24, 3))),
                 img=oet.make_image(B, seed).to(device), dp_dict={k: T(v) for k, v in dp.items()},
                 pose_3d=T(np.concatenate([rng.normal(0, 0.3, (B, 24, 3)), rng.random((B, 24, 1)) < 0.8], -1)),
                 has_pose_3d=flag())
    torch.manual_seed(seed)
    noise, drops = [], []
    for _ in range(steps):
        cn, sn = draw_noise(B)
        noise.append((cn.to(device), sn.to(device)))
        drops.append(draw_part_drop(B).to(device))
    return batch, T(pose(B)), T(rng.normal(0, 1, (B, 10))), flag(), noise, drops


def _bits_equal(a, b):
    if a.dtype == torch.float32:
        return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))
    return torch.equal(a, b)


def _reference_loop(net, opt, batch, opt_pose, opt_betas, fit_valid, noise, drops, steps, lr_steps, pretr_step):
    """train/trainer.py:117-244 and base_trainer.py:70-74 written out on the same CUDA ops, with the caller's optimizer"""
    from danet_b200.targets import prepare_targets
    from danet_b200.training import danet_forward
    decay_steps_ind, all_losses = 1, []
    for step_count in range(1, steps + 1):
        if decay_steps_ind < len(lr_steps) and step_count == lr_steps[decay_steps_ind]:
            lr_new = opt.param_groups[0]['lr'] * 0.1
            for param_group in opt.param_groups:
                param_group['lr'] = lr_new
            decay_steps_ind += 1
        net.train()
        input_batch = dict(batch)
        input_batch['pretrain_mode'] = False if step_count > pretr_step else True
        input_batch.update(prepare_targets(net, batch, opt_pose, opt_betas, fit_valid=fit_valid))
        ret = danet_forward(net, input_batch, part_drop=drops[step_count - 1], center_noise=noise[step_count - 1][0],
                            scale_noise=noise[step_count - 1][1])
        loss_tatal = 0
        losses_dict = {}
        for loss_key in ret['losses']:
            loss_tatal += ret['losses'][loss_key]
            losses_dict['loss_{}'.format(loss_key)] = ret['losses'][loss_key].detach()
        opt.zero_grad()
        loss_tatal.backward()
        opt.step()
        losses_dict['loss_tatal'] = loss_tatal.detach()
        all_losses.append(losses_dict)
    return all_losses


def _ours(net, opt, batch, opt_pose, opt_betas, fit_valid, noise, drops, steps, lr_steps, pretr_step):
    from danet_b200.training import LRDecay, train_step
    sched, outs = LRDecay(steps=lr_steps), []
    for step in range(1, steps + 1):
        outs.append(train_step(net, opt, batch, opt_pose, opt_betas, step, schedule=sched, pretr_step=pretr_step,
                               fit_valid=fit_valid, part_drop=drops[step - 1], center_noise=noise[step - 1][0],
                               scale_noise=noise[step - 1][1]))
    return outs


def _nets(width=32):
    from danet_b200 import build_synthetic_danet
    a = build_synthetic_danet(width=width, seed=0, device=DEV)
    b = build_synthetic_danet(width=width, seed=0, device=DEV)
    b.load_state_dict(a.state_dict())
    return a, b


def _same_model(na, nb, oa, ob):
    for (k, p), (_, q) in zip(na.named_parameters(), nb.named_parameters()):
        assert _bits_equal(p.detach(), q.detach()), k
        assert (p in oa.state) == (q in ob.state), k
        if p in oa.state:
            assert float(oa.state[p]["step"]) == float(ob.state[q]["step"]), k
            for s in ("exp_avg", "exp_avg_sq"):
                assert _bits_equal(oa.state[p][s], ob.state[q][s]), (k, s)
    for (k, x), (_, y) in zip(na.named_buffers(), nb.named_buffers()):
        assert _bits_equal(x, y), k


def test_train_step_is_the_reference_loop_bit_for_bit():
    """W32, B = 2, three steps: step 1 in pretraining (pretr_step=1), a decay at step 3 (steps=(0, 3))"""
    from danet_b200.optim import Adam
    B, steps, lr_steps = 2, 3, (0, 3)
    batch, opt_pose, opt_betas, fit_valid, noise, drops = make_batch(B, 11, steps)
    na, nb = _nets()
    oa = Adam(na.parameters(), lr=1e-4)
    ob = torch.optim.Adam(nb.parameters(), lr=1e-4)
    outs = _ours(na, oa, batch, opt_pose, opt_betas, fit_valid, noise, drops, steps, lr_steps, 1)
    ref = _reference_loop(nb, ob, batch, opt_pose, opt_betas, fit_valid, noise, drops, steps, lr_steps, 1)
    for step, ((output, losses), want) in enumerate(zip(outs, ref), 1):
        assert list(losses) == list(want), step
        for k in losses:
            assert losses[k].device.type == "cuda" and not losses[k].requires_grad
            assert _bits_equal(losses[k], want[k]), (step, k)
        assert (output["pred_vertices"] is None) == (step == 1) and (output["pred_cam_t"] is None) == (step == 1)
        assert set(output) == {"pred_vertices", "opt_vertices", "pred_cam_t", "opt_cam_t", "visualization"}
    _same_model(na, nb, oa, ob)
    assert oa.param_groups[0]["lr"] == ob.param_groups[0]["lr"] == 1e-4 * 0.1
    reg = [p for k, p in na.named_parameters() if k.startswith("iuv2smpl.") and p in oa.state]
    est = [p for k, p in na.named_parameters() if k.startswith("img2iuv.") and p in oa.state]
    assert reg and est
    assert {float(oa.state[p]["step"]) for p in reg} == {2.0} and {float(oa.state[p]["step"]) for p in est} == {3.0}
    print("\n%d losses per step; loss_tatal %s" % (len(outs[-1][1]), [float(o[1]["loss_tatal"]) for o in outs]))


def test_train_step_is_repeatable():
    from danet_b200.optim import Adam
    batch, opt_pose, opt_betas, fit_valid, noise, drops = make_batch(2, 12, 2)
    runs = []
    for _ in range(2):
        na, _ = _nets()
        opt = Adam(na.parameters(), lr=1e-4)
        outs = _ours(na, opt, batch, opt_pose, opt_betas, fit_valid, noise, drops, 2, (0, 30000), 0)
        runs.append((na, opt, outs))
    (na, oa, outs_a), (nb, ob, outs_b) = runs
    _same_model(na, nb, oa, ob)
    for (_, la), (_, lb) in zip(outs_a, outs_b):
        assert all(_bits_equal(la[k], lb[k]) for k in la)


def test_it_trains():
    """a fixed batch with fixed noise and masks: the total loss after 20 steps at lr 1e-4 is below the first step's"""
    from danet_b200.optim import Adam
    B, steps = 4, 20
    batch, opt_pose, opt_betas, fit_valid, noise, drops = make_batch(B, 13, 1)
    na, _ = _nets()
    opt = Adam(na.parameters(), lr=1e-4)
    outs = _ours(na, opt, batch, opt_pose, opt_betas, fit_valid, noise * steps, drops * steps, steps, (0, 30000), 0)
    tot = [float(o[1]["loss_tatal"]) for o in outs]
    print("\nloss_tatal over %d steps: %s" % (steps, " ".join("%.4g" % t for t in tot)))
    assert all(np.isfinite(tot)) and tot[-1] < tot[0]


# ---------------------------------------------------------------------------------------------------------------------
def _nccl_worker(rank, world, port, tmp):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from danet_b200 import build_synthetic_danet
    from danet_b200.optim import Adam
    from danet_b200.training import LRDecay, train_step
    net = build_synthetic_danet(width=32, seed=0, device=dev)
    opt = Adam(net.parameters(), lr=1e-4)
    sched = LRDecay()
    after_one = None
    for step in (1, 2):
        # each rank its own shard: a different seed per rank
        batch, opt_pose, opt_betas, fit_valid, noise, drops = make_batch(2, 100 + 10 * rank + step, 1, device=dev)
        train_step(net, opt, batch, opt_pose, opt_betas, step, schedule=sched, pretr_step=0, fit_valid=fit_valid,
                   part_drop=drops[0], center_noise=noise[0][0], scale_noise=noise[0][1])
        if step == 1:
            after_one = {k: p.detach().cpu().clone() for k, p in net.named_parameters()}
    state = {"params": {k: p.detach().cpu() for k, p in net.named_parameters()},
             "buffers": {k: b.cpu() for k, b in net.named_buffers()},
             "opt": {k: {s: (v.cpu() if torch.is_tensor(v) else v) for s, v in opt.state[p].items()}
                     for k, p in net.named_parameters() if p in opt.state},
             "after_one": after_one}
    torch.save(state, tmp + str(rank))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_over_nccl(tmp_path):
    from danet_b200 import build_synthetic_danet
    from danet_b200.optim import Adam
    from danet_b200.targets import prepare_targets
    from danet_b200.training import danet_forward
    out = str(tmp_path / "rank")
    mp.spawn(_nccl_worker, args=(2, 29561, out), nprocs=2, join=True)
    r0, r1 = torch.load(out + "0"), torch.load(out + "1")
    for part in ("params", "buffers"):
        for k in r0[part]:
            assert _bits_equal(r0[part][k], r1[part][k]), (part, k)
    for k in r0["opt"]:
        for s in ("exp_avg", "exp_avg_sq", "step"):
            assert _bits_equal(r0["opt"][k][s], r1["opt"][k][s]), (k, s)
    # step 1 on one GPU: both shards' gradients, averaged as (g0 + g1) / 2 in fp32, then the optimizer step
    net = build_synthetic_danet(width=32, seed=0, device=DEV)
    grads = []
    for rank in (0, 1):
        ref = build_synthetic_danet(width=32, seed=0, device=DEV)
        ref.load_state_dict(net.state_dict())
        ref.train()
        batch, opt_pose, opt_betas, fit_valid, noise, drops = make_batch(2, 100 + 10 * rank + 1, 1)
        d = dict(batch, pretrain_mode=False)
        d.update(prepare_targets(ref, batch, opt_pose, opt_betas, fit_valid=fit_valid))
        ret = danet_forward(ref, d, part_drop=drops[0], center_noise=noise[0][0], scale_noise=noise[0][1])
        total = 0
        for v in ret["losses"].values():
            total += v
        total.backward()
        grads.append({k: p.grad for k, p in ref.named_parameters()})
    for k, p in net.named_parameters():
        g0, g1 = grads[0][k], grads[1][k]
        p.grad = None if g0 is None else (g0 + g1) / 2
    Adam(net.parameters(), lr=1e-4).step()
    for k, p in net.named_parameters():
        assert _bits_equal(p.detach().cpu(), r0["after_one"][k]), k
