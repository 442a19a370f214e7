"""Generates tests/golden/gcn_head.npz by driving the REFERENCE'S OWN DecomposedPredictor.forward
(models/danet/smpl_regressor.py:676-928, 'gcn' branch :844-895) in training mode on the CPU:

    python -m oracle.gen_golden_gcn_head

Weights are the keyed ones (danet_b200.synthetic.keyed_state_dict, seed 0), except `edge_importance`, which is set
around 1 with some negative entries so that relu'(E) = 0 is exercised.  body_net, limb_net and limb_reslayer are stubs:
body_net returns a fixed leaf (the head sees it + mean_cam_shape, :696) and limb_reslayer returns a fixed leaf
`rot_feats`, so every operation between those leaves and `para` is the reference's code.  The loss is the three head
losses of SMPL_Regressor.forward (:147-166, with the reference's own l1_losses and nn.MSELoss) plus <G, para> for a
fixed random G, which stands in for d(smpl_losses)/d(para).  Recorded: the inputs, para, pose0, coord0, coord1, each
loss, the gradient of every head parameter and of rot_feats / global_para, the running statistics before and after the
step and the graph buffers."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
B, SEED = 4, 0
HAS_SMPL = [1, 0, 1, 1]
RP = "iuv2smpl.smpl_para_Outs."


def gen(ns):
    torch = ns.torch
    nn = torch.nn
    from danet_b200 import synthetic
    from oracle import gcn_head as og
    from models.danet.smpl_regressor import SMPL_Regressor
    rng = np.random.default_rng(2718)
    mp = synthetic.make_mean_params(SEED)
    pred = ns.DecomposedPredictor(None, (torch.tensor(mp["cam"]).reshape(1, 3), torch.tensor(mp["shape"]).reshape(1, 10),
                                         torch.tensor(mp["pose"]).reshape(1, 144)), pretrained=False)
    rsd = {RP + k: v for k, v in pred.state_dict().items()}
    ksd = synthetic.keyed_state_dict(rsd, SEED)
    E = (1.0 + 0.3 * rng.standard_normal((1, 24, 24))).astype(np.float32)
    mask = ksd[RP + "A_mask"].numpy()[0] > 0
    on = np.argwhere(mask)
    for r, c in on[rng.choice(len(on), 12, replace=False)]:
        E[0, r, c] = -abs(E[0, r, c]) - 0.05                                   # relu'(E) = 0 on 12 live edges
    ksd[RP + "edge_importance"] = torch.tensor(E)
    pred.load_state_dict({k[len(RP):]: v for k, v in ksd.items()}, strict=True)
    bn_before = {n: (pred.state_dict()[n + ".running_mean"].numpy().copy(), pred.state_dict()[n + ".running_var"].numpy().copy())
                 for n in og.BN_NAMES}

    rot_feats = torch.tensor(rng.uniform(0, 1.5, (B, 24, 128)).astype(np.float32), requires_grad=True)
    body_out = torch.tensor(rng.normal(0, 0.2, (B, 13)).astype(np.float32), requires_grad=True)

    class Body(nn.Module):
        def forward(self, x):
            return body_out * 1.0, None                     # a non-leaf: :696 adds mean_cam_shape in place

    class Limb(nn.Module):
        def forward(self, x):
            return None, {"x4": torch.zeros(B * 24, 1, 1, 1)}

    class LimbRes(nn.Module):
        def forward(self, x):
            return rot_feats.view(B, 24 * 128, 1, 1)

    pred.body_net, pred.limb_net, pred.limb_reslayer = Body(), Limb(), LimbRes()
    pred.train()
    out = pred(torch.zeros(B, 75, 1, 1), torch.zeros(B, 24 * 3, 1, 1))
    para = out["para"]
    assert len(out["joint_rotation"]) == 1 and len(out["joint_position"]) == 2

    target = np.concatenate([rng.normal(0, 0.3, (B, 13)), rng.normal(0, 0.5, (B, 216))], 1).astype(np.float32)
    gt_joints = rng.normal(0, 0.3, (B, 24, 3)).astype(np.float32)
    has = torch.tensor(HAS_SMPL, dtype=torch.uint8)
    tgt = torch.tensor(target)
    losses = {}
    loss_rot = nn.MSELoss()(out["joint_rotation"][0][has == 1], tgt[:, 13:][has == 1]) * og.SMPL_POSE_WEIGHTS
    losses["joint_rotation0"] = loss_rot
    for i, c in enumerate(out["joint_position"]):
        losses["joint_position%d" % i] = SMPL_Regressor.l1_losses(None, c, torch.tensor(gt_joints), has) * og.JOINT_POSITION_WEIGHTS
    G = rng.normal(0, 1, (B, 229)).astype(np.float32)
    total = sum(losses.values()) + (para * torch.tensor(G)).sum()
    params = dict(pred.named_parameters())
    names = og.PARAM_NAMES
    leaves = [params[n] for n in names] + [rot_feats, body_out]
    grads = torch.autograd.grad(total, leaves)
    rec = {"rot_feats": rot_feats.detach().numpy(), "global_para": (body_out + pred.mean_cam_shape).detach().numpy(),
           "target": target, "gt_joints": gt_joints, "has_smpl": np.array(HAS_SMPL, np.uint8), "G": G,
           "edge_importance": E, "para": para.detach().numpy(), "pose0": out["joint_rotation"][0].detach().numpy(),
           "coord0": out["joint_position"][0].detach().numpy(), "coord1": out["joint_position"][1].detach().numpy()}
    for k, v in losses.items():
        rec["L_" + k] = np.float32(v.detach().reshape(()).item())
    for n, g in zip(names + ["rot_feats", "global_para"], grads):
        rec["g_" + n] = g.numpy()
    sd = pred.state_dict()
    for n in og.BN_NAMES:
        rec["rm0_" + n], rec["rv0_" + n] = bn_before[n]
        rec["rm1_" + n], rec["rv1_" + n] = sd[n + ".running_mean"].numpy(), sd[n + ".running_var"].numpy()
        rec["nbt_" + n] = np.int64(sd[n + ".num_batches_tracked"].item())
    for k in og.BUFFER_NAMES:
        rec["buf_" + k] = sd[k].numpy()
    np.savez_compressed(os.path.join(GOLD, "gcn_head.npz"), **rec)
    print("gcn_head.npz written:", {k: float(v) for k, v in rec.items() if k.startswith("L_")})


def main():
    sys.path.insert(0, ROOT)
    from oracle import ref_import
    ns = ref_import.load(48)
    os.makedirs(GOLD, exist_ok=True)
    gen(ns)


if __name__ == "__main__":
    main()
