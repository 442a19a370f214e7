"""Generates tests/golden/estimator_train.npz by driving the REFERENCE'S OWN IUV_Estimator.forward
(models/danet/iuv_estimator.py:58-260, INPUT_MODE='iuv', DECOMPOSED=True) in float64 and training mode on the CPU, with
the real HRNet backbone:

    python -m oracle.gen_golden_estimator

HRNet W32 (NUM_CHANNELS), pretrained=False, keyed weights (danet_b200.synthetic.keyed_state_dict, seed 0), B = 2,
224 x 224 images (oracle.estimator_train.make_image(B, seed), the first seed from IMAGE_SEED on whose index
head keeps the margin below).  STN_HM_WEIGHTS is set to 1 so that loss_stnhm
exists.  torch.rand is wrapped so that each draw is the fp32 draw a float32 run makes (then widened) and is recorded:
the centre jitter [B,24,2], then per part the two scale jitters [B].  The batch mixes has_iuv (image 0) and has_dp
(image 1).  The index head keeps a top-2 margin of at least 1e-3 at the four pixels around every part centre, so
part visibility is not a near-tie.

Recorded: every loss; sketches (oracle.regressor_train.sketch) of the four raw heads, hm, part_iuv_pred, part_iuv_gt,
xd; the thetas and stn_kps_pred in full; running-statistics sketches and num_batches_tracked of every BatchNorm2d;
and a gradient sketch of every iuv_est parameter and of the image, for the loss sum(losses)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
B, WIDTH, SEED, IMAGE_SEED, NOISE_SEED, TARGET_SEED = 2, 32, 0, 100, 7, 31415
HM_WEIGHT = 1.0
HAS_IUV = [1, 0]
HAS_DP = [0, 1]
EP = "img2iuv."


def centre_margin(index, centers):
    """smallest top-2 margin of the index scores at the four pixels around each part centre (parts 1..23)"""
    top = np.sort(index, axis=1)
    marg = top[:, -1] - top[:, -2]                                   # [B,S,S]
    Si = index.shape[-1]
    worst = np.inf
    for b in range(index.shape[0]):
        for i in range(1, 24):
            ix = ((centers[b, i, 0] + 1) * Si - 1) / 2
            iy = ((centers[b, i, 1] + 1) * Si - 1) / 2
            for yy in (int(np.floor(iy)), int(np.floor(iy)) + 1):
                for xx in (int(np.floor(ix)), int(np.floor(ix)) + 1):
                    if 0 <= xx < Si and 0 <= yy < Si:
                        worst = min(worst, marg[b, yy, xx])
    return worst


def gen(ns):
    torch = ns.torch
    nn = torch.nn
    from danet_b200 import synthetic
    from oracle import ref_import
    from oracle import estimator_train as oet
    from oracle import regressor_train as ort
    ref_import._set_width(ns.cfg, WIDTH)
    ns.cfg.DANET.STN_HM_WEIGHTS = HM_WEIGHT
    torch.Tensor.get_device = lambda self: -1 if not self.is_cuda else self.device.index
    # iuvmap_clean returns its one-hot index maps as .float() (utils/iuvmap.py:8): exact values, widened for the
    # visibility sample of iuv_estimator.py:180
    grid_sample = torch.nn.functional.grid_sample
    torch.nn.functional.grid_sample = lambda x, g, *a, **k: grid_sample(x.to(g.dtype), g, *a, **k)
    est = ns.IUV_Estimator(pretrained=False)
    rsd = {EP + k: v for k, v in est.state_dict().items()}
    ksd = synthetic.keyed_state_dict(rsd, SEED)
    est.load_state_dict({k[len(EP):]: v for k, v in ksd.items()}, strict=True)
    est.double().train()
    # float64 from here on (affine_para builds its thetas in the default dtype); the keyed weights above are drawn in
    # float32, as the product's build_synthetic_danet draws them
    torch.set_default_dtype(torch.float64)
    sd0 = {k: v.clone() for k, v in est.state_dict().items()}
    bns = [n for n, m in est.named_modules() if isinstance(m, nn.BatchNorm2d)]

    iuv, kps, dp = oet.make_targets(B, TARGET_SEED)
    draws, thetas_rec = [], []
    rand = torch.rand
    affine = est.affine_para

    def affine_rec(*a, **k):
        th, sc = affine(*a, **k)
        thetas_rec.append(torch.stack([t.detach() for t in th], 1))
        return th, sc
    est.affine_para = affine_rec

    def rec_rand(*size, **kw):
        r = rand(*size, dtype=torch.float32)                         # what a float32 run draws
        draws.append(r.clone())
        return r.double()
    for image_seed in range(IMAGE_SEED, IMAGE_SEED + 64):            # the first image without a near-tie visibility
        est.load_state_dict(sd0)
        del draws[:], thetas_rec[:]
        img32 = oet.make_image(B, image_seed)
        image = img32.double().requires_grad_()
        torch.manual_seed(NOISE_SEED)
        torch.rand = rec_rand
        try:
            ret = est(image, torch.tensor(iuv).double(), torch.tensor(kps).double(),
                      uvia_dp_gt={k: torch.tensor(v).double() for k, v in dp.items()},
                      has_iuv=torch.tensor(HAS_IUV, dtype=torch.bool), has_dp=torch.tensor(HAS_DP, dtype=torch.float64))
        finally:
            torch.rand = rand
        margin = centre_margin(ret["uvia_pred"][2].detach().numpy(), ret["stn_kps_pred"].numpy())
        print("image seed %d: centre margin %.3g" % (image_seed, margin))
        if margin >= 1e-3:
            break
    assert margin >= 1e-3, margin
    assert len(draws) == 1 + 48 and tuple(draws[0].shape) == (B, 24, 2), [tuple(d.shape) for d in draws]
    center_noise = draws[0].numpy()
    scale_noise = torch.stack([torch.stack(draws[1 + 2 * i:3 + 2 * i]) for i in range(24)]).numpy()
    losses = ret["losses"]
    names = sorted(losses)
    assert len(names) == 13, names
    u, v, idx, ann = ret["uvia_pred"]
    total = sum(losses[k].sum() for k in names)
    params = dict(est.named_parameters())
    pnames = [n for n in params if n.startswith("iuv_est.")]
    grads = torch.autograd.grad(total, [params[n] for n in pnames] + [image], allow_unused=True)
    assert all(g is not None for g in grads), [n for n, g in zip(pnames, grads) if g is None]

    rec = {"B": np.int64(B), "width": np.int64(WIDTH), "image_seed": np.int64(image_seed),
           "noise_seed": np.int64(NOISE_SEED), "hm_weight": np.float64(HM_WEIGHT),
           "checksum_image": ort.input_checksum(img32), "iuv_image_gt": iuv, "smpl_kps_gt": kps,
           "has_iuv": np.array(HAS_IUV, np.uint8), "has_dp": np.array(HAS_DP, np.float32),
           "center_noise": center_noise, "scale_noise": scale_noise, "centre_margin": np.float64(margin),
           "thetas": thetas_rec[-1].numpy()}
    for k, val in dp.items():
        rec["dp_" + k] = val
    for k in names:
        rec["L_" + k] = np.float64(losses[k].detach().sum().item())
    outs = {"u": u, "v": v, "index": idx, "ann": ann, "hm": ret["skps_hm_pred"], "part_pred": ret["part_iuv_pred"],
            "part_iuv_gt": ret["part_iuv_gt"]}
    for k, t in outs.items():
        rec["out_" + k] = ort.sketch("out_" + k, t.detach())
    rec["stn_kps_pred"] = ret["stn_kps_pred"].numpy()
    for n, g in zip(pnames + ["image"], grads):
        key = EP + n if n in params else n
        rec["sk_" + key] = ort.sketch(key, g)
    sd = est.state_dict()
    for n in bns:
        key = EP + n
        rec["rm1_" + key] = ort.sketch("rm1_" + key, sd[n + ".running_mean"])
        rec["rv1_" + key] = ort.sketch("rv1_" + key, sd[n + ".running_var"])
        rec["nbt_" + key] = np.int64(sd[n + ".num_batches_tracked"].item())
        assert torch.equal(sd0[n + ".running_mean"], ksd[key + ".running_mean"].double())
    np.savez_compressed(os.path.join(GOLD, "estimator_train.npz"), **rec)
    print("estimator_train.npz written (%d BatchNorm2d, %d parameters, centre margin %.3g):" % (len(bns), len(pnames), margin),
          {k: float(v) for k, v in rec.items() if k.startswith("L_")})


def main():
    sys.path.insert(0, ROOT)
    from oracle import ref_import
    ns = ref_import.load(WIDTH)
    os.makedirs(GOLD, exist_ok=True)
    gen(ns)


if __name__ == "__main__":
    main()
