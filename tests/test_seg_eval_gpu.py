"""LSP scoring and 3DPW evaluation on the GPU: danet_seg_confusion (csrc/seg_eval.cu) against the oracle's per-image
tables over the reference-generated golden cases and a ragged random sweep in one launch, run-to-run identity, the
whole LSP loop (synthetic network, SMPL and PartRenderer) against the oracle chain to the last bit, the 3DPW loop with
mixed genders against oracle/lbs.py per gender, and two GPUs against one."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from net_common import build
from oracle import seg_eval as oseg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = 224


def _pack(cases):
    """cases: (mask224 float, parts224 int, center, scale, (H, W), gt mask, gt parts) -> inputs of score_renders."""
    dev = torch.device("cuda:0")
    mask = torch.from_numpy(np.stack([c[0] for c in cases]).astype(np.float32)).to(dev)
    parts = torch.from_numpy(np.stack([c[1] for c in cases]).astype(np.int64)).to(dev)
    center = np.array([c[2] for c in cases], np.float32)
    scale = np.array([c[3] for c in cases], np.float64)
    shapes = np.array([c[4] for c in cases], np.int64)
    off = np.concatenate([[0], np.cumsum(shapes.prod(1))])[:-1]
    mgt = torch.from_numpy(np.concatenate([c[5].ravel() for c in cases])).to(dev)
    pgt = torch.from_numpy(np.concatenate([c[6].ravel() for c in cases])).to(dev)
    return mask, parts, center, scale, shapes, off, mgt, pgt


def _golden_cases():
    g = np.load(os.path.join(ROOT, "tests", "golden", "lsp_eval.npz"))
    off = np.concatenate([[0], np.cumsum(g["orig_shape"].prod(1))])
    out = []
    for i in range(len(g["scale"])):
        H, W = g["orig_shape"][i]
        sl = slice(off[i], off[i + 1])
        out.append((g["mask"][i], g["parts"][i], g["center"][i], g["scale"][i], (H, W), g["mask_gt"][sl].reshape(H, W),
                    g["parts_gt"][sl].reshape(H, W)))
    return out


def _random_cases(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        H, W = (int(v) for v in rng.integers(30, 700, 2))
        s = float(rng.uniform(0.1, 4.0))
        c = np.array([rng.uniform(-0.3, 1.3) * W, rng.uniform(-0.3, 1.3) * H], np.float32)
        ul, br = oseg.crop_box(c, s)
        if ul[0] > W or br[0] < 0 or ul[1] > H or br[1] < 0 or (br - ul < 1).any():
            continue
        cover = rng.random((R, R)) < rng.uniform(0, 1) if len(out) % 5 else np.ones((R, R), bool)
        parts = np.where(cover, rng.integers(0, 7, (R, R)), 0)
        gm = ((rng.random((H, W)) < 0.5) * rng.integers(1, 256)).astype(np.uint8)
        gp = rng.choice(np.array([0, 1, 2, 3, 4, 5, 6, 255, 7, 200], np.uint8), (H, W),
                        p=[.3, .1, .1, .1, .1, .1, .1, .05, .03, .02])
        out.append((cover.astype(np.float32), parts, c, s, (H, W), gm, gp))
    return out


def _oracle_tables(cases):
    res = [oseg.score_image(*c) for c in cases]
    return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])


@pytest.mark.parametrize("which", ["golden", "random"])
def test_confusion_equals_oracle_in_one_launch(which):
    from danet_b200 import seg_eval
    cases = _golden_cases() if which == "golden" else _random_cases(40, 11)
    mc, pc = seg_eval.score_renders(*_pack(cases))
    wm, wp = _oracle_tables(cases)
    np.testing.assert_array_equal(mc.cpu().numpy(), wm)
    np.testing.assert_array_equal(pc.cpu().numpy(), wp)
    assert (mc.sum((1, 2)).cpu().numpy() == np.array([c[4][0] * c[4][1] for c in cases])).all()
    if which == "golden":
        g = np.load(os.path.join(ROOT, "tests", "golden", "lsp_eval.npz"))
        m = seg_eval.seg_metrics(mc.cpu().numpy(), pc.cpu().numpy(), int(g["pixel_count"]))
        assert m["f1_mean"] == g["f1_mean"] and m["parts_f1_mean"] == g["parts_f1_mean"]
        assert m["accuracy"] == g["accuracy"] / g["pixel_count"]
        assert m["parts_accuracy"] == g["parts_accuracy"] / g["parts_pixel_count"]


def test_confusion_is_repeatable():
    from danet_b200 import seg_eval
    args = _pack(_random_cases(24, 12))
    a = [t.clone() for t in seg_eval.score_renders(*args)]
    b = seg_eval.score_renders(*args)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_confusion_refuses_a_crop_outside_the_image():
    from danet_b200 import seg_eval
    z = torch.zeros(1, R, R, dtype=torch.uint8, device="cuda:0")
    gt = torch.zeros(100, dtype=torch.uint8, device="cuda:0")
    with pytest.raises(ValueError, match="outside"):
        seg_eval.seg_confusion(z, z, [[20, 0]], [[10, 10]], [[10, 10]], [0], gt, gt)
    with pytest.raises(ValueError, match="exceed"):
        seg_eval.seg_confusion(z, z, [[0, 0]], [[10, 10]], [[10, 11]], [0], gt, gt)


class _InView(torch.nn.Module):
    """The synthetic network with its predicted camera replaced by one that puts the body in view: random weights
    predict cameras whose render covers nothing, which would leave the mask and part counts untested."""

    def __init__(self, net):
        super().__init__()
        self.net, self.iuv2smpl = net, net.iuv2smpl

    def infer_net(self, x):
        para = self.net.infer_net(x)["para"].clone()
        para[:, :3] = torch.tensor([0.9, 0.0, 0.1], device=para.device)
        return {"para": para}


def _renderer(net):
    from danet_b200 import synthetic
    from danet_b200.part_utils import PartRenderer
    return PartRenderer(faces=net.iuv2smpl.smpl.faces, **synthetic.make_part_assets(0))


def _lsp_cache(n):
    from danet_b200 import synthetic
    return synthetic.make_eval_cache("lsp", n, seed=3)


def test_lsp_loop_equals_oracle_chain():
    """run_evaluation('lsp'): network -> SMPL -> PartRenderer -> uncrop + counts on the GPU; the oracle chain takes the
    same renders to the host and scores them with the numpy restatement of eval.py:219-266."""
    from danet_b200 import eval_h36m
    net = _InView(build(32, "cuda:0", conv_algo="auto"))
    rend = _renderer(net)
    data = _lsp_cache(40)
    ds = eval_h36m.CachedSegDataset(data)
    res = eval_h36m.run_evaluation(net, "lsp", ds, batch_size=16, quiet=True, renderer=rend)
    smpl = net.iuv2smpl.smpl
    mt, pt, covered = [], [], 0
    for lo in range(0, 40, 16):
        img, bt = ds.batch(lo, min(40, lo + 16))
        para = net.infer_net(img.cuda())["para"]
        rot = para[:, 13:].reshape(-1, 24, 3, 3)
        v = smpl(betas=para[:, 3:13].contiguous(), body_pose=rot[:, 1:], global_orient=rot[:, :1], pose2rot=False).vertices
        mask, parts = rend(v, para[:, :3].contiguous())
        covered += int(mask.sum())
        for j in range(img.shape[0]):
            H, W = bt["orig_shape"][j]
            o = bt["gt_offset"][j]
            a, b, _, _ = oseg.score_image(mask[j].cpu().numpy(), parts[j].cpu().numpy(), bt["center"][j], bt["scale"][j],
                                          (H, W), bt["mask_gt"][o:o + H * W].reshape(H, W),
                                          bt["parts_gt"][o:o + H * W].reshape(H, W))
            mt.append(a), pt.append(b)
    assert covered > 16 * 1000
    np.testing.assert_array_equal(res["mask_conf"], np.stack(mt))
    np.testing.assert_array_equal(res["part_conf"], np.stack(pt))
    want = oseg.metrics(mt, pt, int((data["orig_shape"][:, 0] * data["orig_shape"][:, 1]).sum()))
    for k in ("accuracy", "f1_mean", "parts_accuracy", "parts_f1_mean"):
        assert res[k] == want[k] or (np.isnan(res[k]) and np.isnan(want[k])), k


def test_3dpw_loop_matches_oracle_chain_with_mixed_genders():
    from danet_b200 import constants, eval_h36m, synthetic
    from oracle import lbs
    net = build(32, "cuda:0", conv_algo="auto")
    data = synthetic.make_eval_cache("3dpw", 48, seed=5)
    assert set(data["gender"].tolist()) == {-1, 0, 1}
    models = synthetic.make_gendered_smpl_models(0)
    male, female = eval_h36m.gendered_smpl(models, device=torch.device("cuda:0"))
    res = eval_h36m.run_evaluation(net, "3dpw", eval_h36m.Cached3DPWDataset(data), batch_size=16, quiet=True,
                                   smpl_male=male, smpl_female=female)
    ds = eval_h36m.Cached3DPWDataset(data)
    para = np.concatenate([net.infer_net(ds.batch(lo, lo + 16)[0].cuda())["para"].cpu().numpy() for lo in range(0, 48, 16)])
    R_ = para[:, 13:].reshape(-1, 24, 3, 3)
    pred = lbs.smpl_forward(synthetic.make_smpl_model(0), para[:, 3:13], R_[:, 1:], R_[:, :1], pose2rot=False,
                            dtype=np.float64)["joints_h36m"]
    gts = {g: lbs.smpl_forward(models[g], data["betas"], data["pose"][:, 3:], data["pose"][:, :3], pose2rot=True,
                               dtype=np.float64)["joints_h36m"] for g in ("male", "female")}
    gt = np.where((data["gender"] == 1)[:, None, None], gts["female"], gts["male"])
    gt = (gt - gt[:, :1])[:, constants.H36M_TO_J14]
    want = lbs.mpjpe_h36m(pred, gt)
    np.testing.assert_allclose(res["mpjpe"], want, atol=1e-5)
    # the gender matters: scoring every image against the male model moves the female images' errors
    gm = (gts["male"] - gts["male"][:, :1])[:, constants.H36M_TO_J14]
    f = data["gender"] == 1
    assert np.abs(lbs.mpjpe_h36m(pred, gm)[f] - want[f]).max() > 1e-3


def _worker(rank, world, port, out):
    import torch.distributed as dist
    from danet_b200 import eval_h36m
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    net = _InView(build(32, "cuda:%d" % rank, conv_algo="auto"))
    res = eval_h36m.run_evaluation(net, "lsp", eval_h36m.CachedSegDataset(_lsp_cache(36)), batch_size=8, quiet=True,
                                   renderer=_renderer(net))
    if rank == 0:
        torch.save({k: res[k] for k in ("mask_conf", "part_conf", "f1_mean", "parts_f1_mean")}, out)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_lsp_loop_two_gpus_equals_one(tmp_path):
    from danet_b200 import eval_h36m
    out = str(tmp_path / "lsp2.pt")
    mp.spawn(_worker, args=(2, 29563, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    net = _InView(build(32, "cuda:0", conv_algo="auto"))
    want = eval_h36m.run_evaluation(net, "lsp", eval_h36m.CachedSegDataset(_lsp_cache(36)), batch_size=8, quiet=True,
                                    renderer=_renderer(net))
    np.testing.assert_array_equal(got["mask_conf"], want["mask_conf"])
    np.testing.assert_array_equal(got["part_conf"], want["part_conf"])
