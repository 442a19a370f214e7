"""tests/golden/danet_train.npz: the reference's own DaNet._forward (models/danet/danet.py:140-366, INPUT_MODE 'iuv',
DECOMPOSED) run unbound on a stand-in `self`, for the part dropout and iuvmap_clean between the IUV estimator and the
regressor.

    python -m oracle.gen_golden_danet_train

The stand-in's img2iuv returns clones of seeded raw maps (oracle.danet_train.make_leaves: negative-only pixels, 0.0 /
-0.0 ties, NaN and +-inf) that are leaves requiring grad; its iuv2smpl returns the probe loss <G1, iuv_map> +
<G2, part_iuv_map> (oracle.danet_train.make_probes); opt_pose is zero and has_iuv false, so no renderer or SMPL runs
(opt_pose only makes the reference define uv_image_gt, which the stand-in ignores).  Each case
records the drop masks the reference drew (its own torch.rand calls after torch.manual_seed(seed)), the cleaned maps
and the gradients of the leaves.  Inputs are regenerated from their seeds by the tests."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
B, S = 3, 8
CASES = [("r03_s0", True, 0.3, 0), ("r03_s1", True, 0.3, 1), ("r09_s0", True, 0.9, 0), ("r09_s1", True, 0.9, 1),
         ("eval", False, 0.3, 2)]
LEAF_SEED, PROBE_SEED = 100, 200


class _Stub(object):
    pass


def run_case(ns, training, rate, seed):
    from models.danet import danet as ref_danet
    from danet_b200 import constants
    from oracle import danet_train as odt
    ns.cfg.DANET.INPUT_MODE, ns.cfg.DANET.DECOMPOSED, ns.cfg.DANET.PARTDROP_RATE = "iuv", True, rate
    leaves = [t.requires_grad_() for t in odt.make_leaves(B, S, LEAF_SEED + seed)]
    G1, G2 = odt.make_probes(B, S, PROBE_SEED + seed)
    me = _Stub()
    me.training = training
    me.img2iuv = lambda *a, **k: {"uvia_pred": [t.clone() for t in leaves[:4]], "part_iuv_pred": leaves[4].clone()}
    me.img2iuv.dp2smpl_mapping = constants.DP2SMPL_MAPPING
    seen = {}

    def iuv2smpl(d):
        seen["part_iuv_map"] = d["part_iuv_map"]
        probe = (G1 * d["iuv_map"]).sum() + (G2 * d["part_iuv_map"]).sum()
        return {"losses": {"probe": probe}, "metrics": {}, "visualization": {}, "prediction": {}}
    me.iuv2smpl = iuv2smpl
    draws, rand = [], torch.rand

    def recording_rand(*a, **k):
        r = rand(*a, **k)
        draws.append(r.clone())
        return r
    torch.manual_seed(seed)
    torch.rand = recording_rand
    try:
        ret = ref_danet.DaNet._forward(me, {"img": torch.zeros(B, 3, 4, 4), "pretrain_mode": False, "vis_on": False,
                                            "opt_pose": torch.zeros(B, 72), "opt_betas": torch.zeros(B, 10),
                                            "target_cam": torch.zeros(B, 3), "has_iuv": torch.zeros(B)})
    finally:
        torch.rand = rand
    assert len(draws) == (B if training else 0)
    drop = torch.stack([d < rate for d in draws]).numpy() if training else np.zeros((B, 24), bool)
    grads = torch.autograd.grad(ret["losses"]["probe"].sum(), leaves, allow_unused=True)
    assert grads[2] is None and grads[3] is None       # Index and Ann reach the loss only through argmaxes
    out = dict(drop=drop)
    for k, t in zip(("u_cl", "v_cl", "index_cl", "ann_cl"), ret["visualization"]["iuv_pred"]):
        out[k] = t.detach().numpy()
    out["part_iuv_map"] = ret["visualization"]["part_iuv_pred"].detach().numpy()
    for k, g in zip(("g_u", "g_v", "g_parts"), (grads[0], grads[1], grads[4])):
        out[k] = g.numpy()
    return out


def main():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_import
    cwd = os.getcwd()
    ns = ref_import.load()
    rec = dict(B=np.int64(B), S=np.int64(S), leaf_seed=np.int64(LEAF_SEED), probe_seed=np.int64(PROBE_SEED),
               cases=np.array([c[0] for c in CASES]))
    for name, training, rate, seed in CASES:
        rec["%s_meta" % name] = np.array([float(training), rate, seed])
        for k, v in run_case(ns, training, rate, seed).items():
            rec["%s_%s" % (name, k)] = v
    os.chdir(cwd)
    np.savez_compressed(os.path.join(GOLD, "danet_train.npz"), **rec)
    print("wrote", os.path.join(GOLD, "danet_train.npz"))


if __name__ == "__main__":
    main()
