"""Generates tests/golden/stn_train.npz with the REFERENCE'S OWN code on the CPU:

    python -m oracle.gen_golden_stn_train

Thetas: IUV_Estimator.forward in training mode (models/danet/iuv_estimator.py:125-204) with the backbone replaced by a
stub that returns fixed predict_hm / predict_uv_index / xd, centre and scale jitter on (the configured 0.1 and 0.2),
and torch.rand patched to record its draws.  Recorded: the soft-argmax + jitter centres (stn_kps_pred), affine_para's
thetas, part_maps (the 24 crops of xd) and the draws, as center_noise [B,24,2] and scale_noise [24,2,B].
Fuse: the HighResolutionModule of models/module/hr_module.py with 4 branches of a few channels on small maps: per
output i, the terms entering the fuse sum (the branch itself or the fuse conv + BN, before the nearest upsample),
their factors and the module's output."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

B, S, CX = 3, 16, 4
FUSE_C, FUSE_H = [2, 4, 6, 8], 16


def gen_thetas(ns, out):
    torch = ns.torch
    cfg = ns.cfg
    cfg.DANET.HEATMAP_SIZE = S
    cfg.DANET.STN_CENTER_JITTER = 0.1
    cfg.DANET.STN_SCALE_JITTER = 0.2
    cfg.DANET.STN_HM_WEIGHTS = 0.0
    torch.Tensor.get_device = lambda self: -1 if not self.is_cuda else self.device.index
    rng = np.random.default_rng(2718)
    # peaked heat maps (realistic centres) and index scores whose argmax forms blobs
    hm = rng.normal(0, 0.05, (B, 24, S, S)).astype(np.float32)
    yy, xx = np.mgrid[0:S, 0:S]
    for b in range(B):
        for j in range(24):
            cx, cy = rng.uniform(2, S - 3, 2)
            hm[b, j] += np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / 4.0).astype(np.float32)
    index = rng.normal(0, 1, (B, 25, S // 4, S // 4)).repeat(4, 2).repeat(4, 3).astype(np.float32)
    index += rng.normal(0, 0.3, index.shape).astype(np.float32)
    xd = rng.normal(0, 1, (B, CX, S, S)).astype(np.float32)
    kps = np.concatenate([rng.uniform(-0.9, 0.9, (B, 24, 2)), np.ones((B, 24, 1))], 2).astype(np.float32)

    class FinalPred(torch.nn.Module):
        def predict_partial_iuv(self, part_maps):
            out["part_maps"] = part_maps.detach().numpy()
            return torch.zeros(B, 24 * 21, S, S)

    class Stub(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.final_pred = FinalPred()

        def forward(self, data):
            z = torch.zeros(B, 25, S, S)
            return {"predict_u": z, "predict_v": z, "predict_uv_index": torch.tensor(index),
                    "predict_ann_index": torch.zeros(B, 15, S, S), "predict_hm": torch.tensor(hm), "xd": torch.tensor(xd)}

    est = ns.IUV_Estimator(pretrained=False)
    est.iuv_est = Stub()
    est.train()
    with torch.no_grad():
        est.learned_ratio.copy_(torch.tensor(rng.uniform(-0.2, 1.5, 24).astype(np.float32)))
        est.learned_offset.copy_(torch.tensor(rng.uniform(-0.1, 0.2, 24).astype(np.float32)))
    thetas_rec = []
    orig_affine = est.affine_para

    def affine_rec(*a, **k):
        th, sc = orig_affine(*a, **k)
        thetas_rec.append(torch.stack([t.detach() for t in th], 1))
        return th, sc
    est.affine_para = affine_rec
    draws = []
    orig_rand = torch.rand
    gen = torch.Generator().manual_seed(99)

    def rand_rec(*size, **kw):
        r = orig_rand(*size, generator=gen)
        draws.append(r.clone())
        return r
    torch.rand = rand_rec
    try:
        ret = est(torch.zeros(B, 3, 4 * S, 4 * S), None, torch.tensor(kps))
    finally:
        torch.rand = orig_rand
    assert len(draws) == 1 + 48 and tuple(draws[0].shape) == (B, 24, 2), [tuple(d.shape) for d in draws]
    out.update(hm=hm, index_pred=index, xd=xd, learned_ratio=est.learned_ratio.detach().numpy(),
               learned_offset=est.learned_offset.detach().numpy(), center_noise=draws[0].numpy(),
               scale_noise=torch.stack(draws[1:]).reshape(24, 2, B).numpy(),
               stn_centers=ret["stn_kps_pred"].numpy(), thetas=thetas_rec[-1].numpy(),
               stn_params=np.array([0.5, 0.1, 0.2], np.float32))         # STN_PART_VIS_SCORE, CENTER / SCALE_JITTER


def gen_fuse(ns, out):
    torch = ns.torch
    from models.module.hr_module import HighResolutionModule
    from models.module.res_module import BasicBlock
    torch.manual_seed(5)
    m = HighResolutionModule(4, BasicBlock, [1, 1, 1, 1], list(FUSE_C), list(FUSE_C), "SUM").train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.weight.data.uniform_(0.5, 1.5)
            mod.bias.data.uniform_(-0.3, 0.3)
    xs = [torch.randn(2, c, FUSE_H >> k, FUSE_H >> k) for k, c in enumerate(FUSE_C)]
    with torch.no_grad():
        ys = m([x.clone() for x in xs])
        br = [m.branches[k](x) for k, x in enumerate(xs)]
        for i in range(4):
            terms, factors = [], []
            for j in range(4):
                if j == i:
                    t, f = br[j], 1
                elif j > i:
                    t, f = m.fuse_layers[i][j][1](m.fuse_layers[i][j][0](br[j])), 2 ** (j - i)
                else:
                    t, f = m.fuse_layers[i][j](br[j]), 1
                terms.append(t.numpy())
                factors.append(f)
            for j, t in enumerate(terms):
                out["fuse%d_t%d" % (i, j)] = t
            out["fuse%d_factors" % i] = np.array(factors, np.int32)
            out["fuse%d_y" % i] = ys[i].numpy()


def main():
    sys.path.insert(0, ROOT)
    from oracle import ref_import
    ns = ref_import.load(48)
    out = {}
    gen_thetas(ns, out)
    gen_fuse(ns, out)
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "stn_train.npz"), **out)
    print("stn_train.npz written:", sorted(out))


if __name__ == "__main__":
    main()
