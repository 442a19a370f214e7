"""Evaluation loop of the reference's eval.py (run_evaluation, eval.py:57-299) for all five of its datasets --
h36m-p1 / h36m-p2 / 3dpw / mpi-inf-3dhp (3D pose) and lsp (silhouette and part segmentation) -- over CACHED network
inputs, image-sharded across ranks.

    python -m danet_b200.eval_h36m --checkpoint data/pretrained_model/danet_model_h36m_itw.pt \
           --cache data/dataset_extras/h36m_valid_protocol2_cached.npz --batch_size 32
    python -m danet_b200.eval_h36m --checkpoint ... --dataset lsp --cache lsp_test_cached.npz
    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 -m danet_b200.eval_h36m ...    (r::world batches)

The cache is what the reference's BaseDataset hands to the model and the metric (eval.py:142-147,196-200): the
cropped / normalised image tensor `img` [N,3,224,224] float32 (or uint8 RGB crops [N,224,224,3], which are normalised
here like datasets/base_dataset.py does), plus per dataset:
    h36m-p1 / h36m-p2 / mpi-inf-3dhp   `pose_3d` [N,24,4], optionally `imgname` [N]
    3dpw    `pose` [N,72] (axis-angle), `betas` [N,10], `gender` [N] (-1 none, 0 male, 1 female; or 'm' / 'f')
    lsp     `center` [N,2], `scale` [N], `orig_shape` [N,2] (rows, cols), and `mask_gt` / `parts_gt`: the ground-truth
            mask and part PNGs (read as cv2.imread(..., 0) does) packed row-major, image after image, into flat uint8
            arrays
Caches are validated (lengths, and the packed sizes against orig_shape); a bad cache raises ValueError.  Cropping from
raw frames (cv2, BaseDataset) is a data-loader concern and stays with the reference.

What runs where:
    model.infer_net -> SMPL -> J_regressor_h36m joints -> MPJPE      GPU (evaluate.evaluate_batch: one fused pass)
    3dpw ground truth: male and female SMPL (gendered_smpl) with the same regressor, selected per image where
        gender == 1 (gt_joints_3dpw)                                   GPU
    reconstruction error (Procrustes / PA-MPJPE, utils/pose_utils.py:10-76)   host numpy SVD, as in the reference
    lsp: PartRenderer -> uncrop to the original size -> 2x2 mask and 9x7 part confusion tables per image
        (seg_eval.score_renders, csrc/seg_eval.cu)                    GPU; the crop corners on the host in float64
    per-sample results: one all-reduce at the end (the lsp tables are integers, so the merge is exact)
Results are printed like the reference prints them (eval.py:269-299) and returned as a dict.
"""
import argparse
import os

import numpy as np
import torch

from . import constants
from .evaluate import evaluate_batch

IMG_NORM_MEAN = np.array([0.485, 0.456, 0.406], dtype=np.float32)       # constants.py:10-11 of the reference
IMG_NORM_STD = np.array([0.229, 0.224, 0.225], dtype=np.float32)


def compute_similarity_transform(S1, S2):
    """Similarity transform (s, R, t) taking S1 [N,3] closest to S2 [N,3] (orthogonal Procrustes, det R = +1);
    returns the transformed S1.  utils/pose_utils.py:10-57."""
    X1 = S1.T.astype(np.float64)
    X2 = S2.T.astype(np.float64)
    mu1, mu2 = X1.mean(axis=1, keepdims=True), X2.mean(axis=1, keepdims=True)
    X1c, X2c = X1 - mu1, X2 - mu2
    var1 = np.sum(X1c ** 2)
    K = X1c.dot(X2c.T)
    U, _s, Vh = np.linalg.svd(K)
    V = Vh.T
    Z = np.eye(U.shape[0])
    Z[-1, -1] *= np.sign(np.linalg.det(U.dot(V.T)))
    R = V.dot(Z.dot(U.T))
    scale = np.trace(R.dot(K)) / var1
    t = mu2 - scale * R.dot(mu1)
    return (scale * R.dot(X1) + t).T


def reconstruction_error(S1, S2):
    """Per-sample PA-MPJPE of S1 [B,J,3] against S2 [B,J,3] (utils/pose_utils.py:66-76, reduction=None)."""
    out = np.zeros(S1.shape[0])
    for i in range(S1.shape[0]):
        hat = compute_similarity_transform(S1[i], S2[i])
        out[i] = np.sqrt(((hat - S2[i]) ** 2).sum(axis=-1)).mean()
    return out


class CachedPoseDataset(object):
    """Cached inputs of a 3D-pose evaluation set (see module docstring)."""

    def __init__(self, path_or_dict):
        z = np.load(path_or_dict, allow_pickle=True) if isinstance(path_or_dict, str) else path_or_dict
        self.img = z["img"]
        self.pose_3d = np.asarray(z["pose_3d"], dtype=np.float32)
        self.imgname = [str(s) for s in z["imgname"]] if "imgname" in z else None
        if self.img.shape[0] != self.pose_3d.shape[0]:
            raise ValueError("cache: img and pose_3d disagree on the number of samples")

    def __len__(self):
        return self.img.shape[0]

    def batch(self, lo, hi):
        return _images(self.img[lo:hi]), self.pose_3d[lo:hi]


def _images(img):
    """Cached network inputs -> float32 NCHW: RGB crops [n,224,224,3] uint8 are normalised (base_dataset.py:170-173)."""
    if img.dtype == np.uint8:
        x = img.astype(np.float32) / 255.0
        x = (x - IMG_NORM_MEAN) / IMG_NORM_STD
        img = np.ascontiguousarray(x.transpose(0, 3, 1, 2))
    return torch.from_numpy(np.ascontiguousarray(img, dtype=np.float32))


def _load(path_or_dict):
    return np.load(path_or_dict, allow_pickle=True) if isinstance(path_or_dict, str) else path_or_dict


def _need(z, keys, what):
    missing = [k for k in keys if k not in z]
    if missing:
        raise ValueError("%s cache: missing %s" % (what, ", ".join(missing)))


class Cached3DPWDataset(object):
    """Cached 3DPW inputs: `img`, SMPL ground truth `pose` [N,72] (axis-angle) and `betas` [N,10], `gender` [N]
    (-1 / 0 / 1, or the dataset's 'm' / 'f' strings, mapped like base_dataset.py:106-111: 0 for 'm', 1 otherwise)."""

    def __init__(self, path_or_dict):
        z = _load(path_or_dict)
        _need(z, ("img", "pose", "betas", "gender"), "3dpw")
        self.img = z["img"]
        self.pose = np.asarray(z["pose"], dtype=np.float32)
        self.betas = np.asarray(z["betas"], dtype=np.float32)
        g = np.asarray(z["gender"])
        self.gender = np.array([0 if str(v) == "m" else 1 for v in g], np.int32) if g.dtype.kind in "USO" else \
            g.astype(np.int32)
        n = self.img.shape[0]
        if self.pose.shape != (n, 72) or self.betas.shape != (n, 10) or self.gender.shape != (n,):
            raise ValueError("3dpw cache: img %s, pose %s, betas %s and gender %s disagree (want [N,72], [N,10], [N])"
                             % (self.img.shape, self.pose.shape, self.betas.shape, self.gender.shape))

    def __len__(self):
        return self.img.shape[0]

    def batch(self, lo, hi):
        return _images(self.img[lo:hi]), self.pose[lo:hi], self.betas[lo:hi], self.gender[lo:hi]


class CachedSegDataset(object):
    """Cached LSP inputs: `img`, the crop `center` [N,2] and `scale` [N], the original image size `orig_shape` [N,2]
    (rows, cols), and the ground-truth mask and part images (cv2.imread(..., 0) of eval.py:235,252) packed row-major,
    image after image, into the flat uint8 arrays `mask_gt` and `parts_gt`."""

    def __init__(self, path_or_dict):
        z = _load(path_or_dict)
        _need(z, ("img", "center", "scale", "orig_shape", "mask_gt", "parts_gt"), "lsp")
        self.img = z["img"]
        self.center = np.asarray(z["center"]).astype(np.float32)        # base_dataset.py: center.astype(np.float32)
        self.scale = np.asarray(z["scale"]).astype(np.float64)          # float(sc * scale)
        self.orig_shape = np.asarray(z["orig_shape"])
        self.mask_gt, self.parts_gt = np.asarray(z["mask_gt"]), np.asarray(z["parts_gt"])
        n = self.img.shape[0]
        if self.center.shape != (n, 2) or self.scale.shape != (n,) or self.orig_shape.shape != (n, 2):
            raise ValueError("lsp cache: img %s, center %s, scale %s and orig_shape %s disagree (want [N,2], [N], [N,2])"
                             % (self.img.shape, self.center.shape, self.scale.shape, self.orig_shape.shape))
        if self.orig_shape.dtype.kind not in "iu" or (self.orig_shape < 1).any():
            raise ValueError("lsp cache: orig_shape must hold positive integers")
        for k in ("mask_gt", "parts_gt"):
            a = getattr(self, k)
            if a.dtype != np.uint8 or a.ndim != 1:
                raise ValueError("lsp cache: %s must be a flat uint8 array (got %s %s)" % (k, a.dtype, a.shape))
        self.orig_shape = self.orig_shape.astype(np.int64)
        npix = self.orig_shape[:, 0] * self.orig_shape[:, 1]
        self.offset = np.concatenate([[0], np.cumsum(npix)]).astype(np.int64)
        if self.mask_gt.size != self.offset[-1] or self.parts_gt.size != self.offset[-1]:
            raise ValueError("lsp cache: mask_gt (%d) and parts_gt (%d) must hold the %d pixels orig_shape gives"
                             % (self.mask_gt.size, self.parts_gt.size, self.offset[-1]))

    def __len__(self):
        return self.img.shape[0]

    def batch(self, lo, hi):
        a, b = self.offset[lo], self.offset[hi]
        return _images(self.img[lo:hi]), {"center": self.center[lo:hi], "scale": self.scale[lo:hi],
                                          "orig_shape": self.orig_shape[lo:hi], "gt_offset": self.offset[lo:hi] - a,
                                          "mask_gt": self.mask_gt[a:b], "parts_gt": self.parts_gt[a:b]}


def gendered_smpl(model_path="data/smpl", J_regressor_h36m=None, device=None):
    """The male and female SMPL layers of eval.py:72-77, each with the H36M regressor (eval.py:80; by default
    data/J_regressor_h36m.npy).  model_path: the SMPL directory, or a dict {'male': model, 'female': model}."""
    from .smpl import SMPL
    out = []
    for g in ("male", "female"):
        m = model_path[g] if isinstance(model_path, dict) else model_path
        s = SMPL(m, gender=g, J_regressor_h36m=J_regressor_h36m)
        out.append(s.to(device) if device is not None else s)
    return tuple(out)


@torch.no_grad()
def gt_joints_3dpw(smpl_male, smpl_female, pose, betas, gender):
    """eval.py:196-206: the ground-truth mesh of smpl_male, replaced by smpl_female's where gender == 1 (-1 and 0 keep
    the male model), through the H36M regressor, centred on H36M joint 0 and mapped with H36M_TO_J14 -> [n,14,3].
    Selecting the regressed joints per image equals regressing the selected meshes: each image's joints depend on its
    own mesh only."""
    pose = torch.as_tensor(pose, dtype=torch.float32)
    betas = torch.as_tensor(betas, dtype=torch.float32)
    joints = []
    for smpl in (smpl_male, smpl_female):
        smpl(betas=betas, body_pose=pose[:, 3:], global_orient=pose[:, :3], pose2rot=True)
        j = smpl.joints_h36m()
        if j is None:
            raise ValueError("3dpw: the gendered SMPL layers need J_regressor_h36m (eval.py:80)")
        joints.append(j)
    female = torch.as_tensor(np.asarray(gender) == 1, device=joints[0].device).view(-1, 1, 1)
    j17 = torch.where(female, joints[1], joints[0])
    return (j17 - j17[:, :1])[:, constants.H36M_TO_J14]


def run_evaluation(model, dataset_name, dataset, result_file=None, batch_size=32, log_freq=50, group=None, quiet=False,
                   batch_fn=None, smpl_male=None, smpl_female=None, renderer=None):
    """eval.py:57-299.  Every rank holds the dataset; batch b is evaluated by rank b % world (image-sharded, SURVEY
    section 8e) and the per-sample results are all-reduced once at the end.
    Pose datasets (h36m-p1 / h36m-p2 / 3dpw / mpi-inf-3dhp) return dict(mpjpe [N] m, recon_err [N] m, mpjpe_mm,
    recon_err_mm, per_action); batch_fn(images, gt_j14) -> dict(mpjpe, pred_j14) replaces the GPU pass (host-logic
    tests).  3dpw takes its ground truth from smpl_male / smpl_female (`gendered_smpl`, `gt_joints_3dpw`).
    lsp needs `renderer` (a PartRenderer) and returns what `run_segmentation` returns."""
    if dataset_name == "lsp":
        return run_segmentation(model, dataset, renderer, result_file, batch_size, log_freq, group, quiet, batch_fn)
    if dataset_name == "3dpw" and (smpl_male is None or smpl_female is None):
        raise ValueError("3dpw: pass smpl_male and smpl_female (eval.py:72-77; see gendered_smpl)")
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank(group) if world > 1 else 0
    j17 = dataset_name == "mpi-inf-3dhp"                    # eval.py:139-140: 17 joints there, the 14 LSP joints otherwise
    if batch_fn is None:
        dev = next(model.parameters()).device
        smpl = model.iuv2smpl.smpl
        batch_fn = lambda im, gt: evaluate_batch(model, smpl, im.to(dev), gt.to(dev), shard=False, joints17=j17)
    else:
        dev = torch.device("cpu")
    nj = 17 if j17 else 14
    n = len(dataset)
    nb = (n + batch_size - 1) // batch_size
    mpjpe = np.zeros(n)
    recon = np.zeros(n)
    done = np.zeros(n, dtype=bool)
    pred_joints = np.zeros((n, nj, 3), dtype=np.float32)
    for b in range(rank, nb, world):
        lo, hi = b * batch_size, min(n, (b + 1) * batch_size)
        if dataset_name == "3dpw":
            img, pose, betas, gender = dataset.batch(lo, hi)
            gt = gt_joints_3dpw(smpl_male, smpl_female, pose, betas, gender).cpu()
        else:
            img, pose_3d = dataset.batch(lo, hi)
            gt = torch.from_numpy(pose_3d[:, constants.J24_TO_J17 if j17 else constants.J24_TO_J14, :3].copy())     # eval.py:189-190
        out = batch_fn(img, gt)                              # this rank's batch only (the loop deals the batches)
        e = out["mpjpe"].cpu().numpy()
        pj = out["pred_j14"].cpu().numpy()
        mpjpe[lo:hi] = e
        recon[lo:hi] = reconstruction_error(pj, gt.numpy())                        # host SVD, as the reference does
        pred_joints[lo:hi] = pj
        done[lo:hi] = True
        if not quiet and rank == 0 and (b // world) % log_freq == log_freq - 1:
            print("MPJPE: " + str(1000 * mpjpe[done].mean()))
            print("Reconstruction Error: " + str(1000 * recon[done].mean()))
            print()
    if world > 1:
        buf = torch.from_numpy(np.stack([mpjpe, recon, done.astype(np.float64)])).to(dev if dist.get_backend(group) == "nccl" else "cpu")
        pred_joints = pred_joints.astype(np.float32)
        dist.all_reduce(buf, group=group)                                             # disjoint supports: sum = merge
        pj = torch.from_numpy(pred_joints).to(buf.device)
        dist.all_reduce(pj, group=group)
        mpjpe, recon, cnt = buf[0].cpu().numpy(), buf[1].cpu().numpy(), buf[2].cpu().numpy()
        pred_joints = pj.cpu().numpy()
        assert (cnt == 1).all()
    res = {"mpjpe": mpjpe, "recon_err": recon, "mpjpe_mm": 1000 * mpjpe.mean(), "recon_err_mm": 1000 * recon.mean(),
           "pred_joints": pred_joints, "per_action": {}}
    if dataset_name == "h36m-p2" and dataset.imgname is not None:
        acts = {}
        for i, name in enumerate(dataset.imgname):
            a = name.split("/")[-1].split(".")[0].split("_")[1]                       # eval.py:150-157
            acts.setdefault(a, []).append(i)
        for a, idx in acts.items():
            res["per_action"][a] = (1000 * mpjpe[idx].mean(), 1000 * recon[idx].mean())
    if result_file is not None and rank == 0:
        np.savez(result_file, pred_joints=pred_joints, mpjpe=mpjpe, recon_err=recon)
    if not quiet and rank == 0:
        print("*** Final Results ***")
        print("MPJPE: " + str(res["mpjpe_mm"]))
        print("Reconstruction Error: " + str(res["recon_err_mm"]))
        print()
        if res["per_action"]:
            print(["action err"] + [str(v[1]) for v in res["per_action"].values()] + list(res["per_action"].keys()))
    return res


def _print_segmentation(m):
    print("Accuracy: ", m["accuracy"])                                  # eval.py:276-282
    print("F1: ", m["f1_mean"])
    print()
    print("Parts Accuracy: ", m["parts_accuracy"])
    print("Parts F1 (BG): ", m["parts_f1_mean"])
    print()


def run_segmentation(model, dataset, renderer, result_file=None, batch_size=32, log_freq=50, group=None, quiet=False,
                     batch_fn=None):
    """eval.py:57-299 for lsp: the predicted mesh rendered by `renderer` (PartRenderer), put back into each original
    image and scored against the ground-truth mask and parts on the GPU (seg_eval.score_renders).  Batch b is evaluated
    by rank b % world; the per-image integer tables are all-reduced once at the end (exact).  Returns dict(mask_conf
    [N,2,2], part_conf [N,9,7] int64, pixel_count, accuracy, f1 [2,1], f1_mean, parts_accuracy, parts_f1 [7,1],
    parts_f1_mean).  batch_fn(images, batch) -> (mask_conf, part_conf) of the batch replaces the GPU pass (host-logic
    tests); `batch` is CachedSegDataset.batch's dict."""
    import torch.distributed as dist
    from . import seg_eval
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank(group) if world > 1 else 0
    if batch_fn is None:
        if renderer is None:
            raise ValueError("lsp: pass renderer, a PartRenderer (eval.py:131-132)")
        seg_eval.check_part_table(renderer)
        dev = next(model.parameters()).device
        smpl = model.iuv2smpl.smpl

        def batch_fn(im, bt):
            para = model.infer_net(im.to(dev))["para"]                                    # eval.py:164-173
            rot = para[:, 13:].reshape(-1, 24, 3, 3)
            verts = smpl(betas=para[:, 3:13].contiguous(), body_pose=rot[:, 1:], global_orient=rot[:, :1],
                         pose2rot=False).vertices
            mask, parts = renderer(verts, para[:, :3].contiguous())                      # eval.py:219-220
            return seg_eval.score_renders(mask, parts, bt["center"], bt["scale"], bt["orig_shape"], bt["gt_offset"],
                                          torch.from_numpy(bt["mask_gt"]).to(dev), torch.from_numpy(bt["parts_gt"]).to(dev))
    else:
        dev = torch.device("cpu")
    n = len(dataset)
    nb = (n + batch_size - 1) // batch_size
    npix = dataset.orig_shape[:, 0] * dataset.orig_shape[:, 1]
    tables = np.zeros((n, 4 + seg_eval.PART_ROWS * seg_eval.PART_COLS + 1), np.int64)   # mask | parts | done
    for b in range(rank, nb, world):
        lo, hi = b * batch_size, min(n, (b + 1) * batch_size)
        img, bt = dataset.batch(lo, hi)
        mc, pc = batch_fn(img, bt)
        tables[lo:hi, :4] = mc.cpu().numpy().reshape(hi - lo, 4)
        tables[lo:hi, 4:-1] = pc.cpu().numpy().reshape(hi - lo, -1)
        tables[lo:hi, -1] = 1
        if not quiet and rank == 0 and (b // world) % log_freq == log_freq - 1:
            d = tables[:, -1] == 1
            _print_segmentation(seg_eval.seg_metrics(tables[d, :4], tables[d, 4:-1], npix[d].sum()))
    if world > 1:
        buf = torch.from_numpy(tables).to(dev if dist.get_backend(group) == "nccl" else "cpu")
        dist.all_reduce(buf, group=group)                                             # disjoint supports: sum = merge
        tables = buf.cpu().numpy()
        assert (tables[:, -1] == 1).all()
    mask_conf = tables[:, :4].reshape(n, 2, 2)
    part_conf = tables[:, 4:-1].reshape(n, seg_eval.PART_ROWS, seg_eval.PART_COLS)
    res = {"mask_conf": mask_conf, "part_conf": part_conf, "pixel_count": int(npix.sum())}
    res.update(seg_eval.seg_metrics(mask_conf, part_conf, res["pixel_count"]))
    if result_file is not None and rank == 0:
        np.savez(result_file, mask_conf=mask_conf, part_conf=part_conf)
    if not quiet and rank == 0:
        print("*** Final Results ***")
        _print_segmentation(res)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--checkpoint", default=None, help="path to the network checkpoint (the reference's .pt with a 'model' entry)")
    ap.add_argument("--dataset", default="h36m-p2", choices=["h36m-p1", "h36m-p2", "lsp", "3dpw", "mpi-inf-3dhp"])
    ap.add_argument("--cache", required=True, help="npz of the dataset's cached inputs (see module docstring)")
    ap.add_argument("--batch_size", default=32, type=int)
    ap.add_argument("--log_freq", default=50, type=int)
    ap.add_argument("--result_file", default=None)
    ap.add_argument("--smpl_mean_params", default="data/smpl_mean_params.npz")
    ap.add_argument("--legacy_align_corners", action="store_true",
                    help="torch<=1.2 affine_grid/grid_sample semantics (the released checkpoint was trained under torch 1.1)")
    ap.add_argument("--precision", default="exact", choices=["exact", "fast"])
    ap.add_argument("--synthetic", action="store_true",
                    help="random weights and synthetic SMPL / PartRenderer assets (no licensed files)")
    ap.add_argument("--smpl_model_dir", default="data/smpl", help="SMPL_{MALE,FEMALE}.pkl for 3dpw (path_config.py)")
    args = ap.parse_args(argv)
    import torch.distributed as dist
    from . import synthetic
    from .danet import DaNet, build_synthetic_danet
    from .part_utils import PartRenderer
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        dist.init_process_group("nccl", device_id=dev)
    if args.synthetic:
        model = build_synthetic_danet(width=48, device=dev, precision=args.precision, legacy_align_corners=args.legacy_align_corners)
    else:
        model = DaNet(args, args.smpl_mean_params, pretrained=False, precision=args.precision,
                      legacy_align_corners=args.legacy_align_corners)
        ck = torch.load(args.checkpoint, map_location="cpu")
        model.load_state_dict(ck["model"], strict=False)                               # eval.py:333-334
        model = model.to(dev).eval()
    extra = {}
    if args.dataset == "3dpw":
        dataset = Cached3DPWDataset(args.cache)
        h36m = model.iuv2smpl.smpl.J_regressor_h36m                        # eval.py:80: one regressor for every model
        models = synthetic.make_gendered_smpl_models(0) if args.synthetic else args.smpl_model_dir
        extra["smpl_male"], extra["smpl_female"] = gendered_smpl(models, None if h36m is None else h36m.cpu().numpy(), dev)
    elif args.dataset == "lsp":
        dataset = CachedSegDataset(args.cache)
        if args.synthetic:
            extra["renderer"] = PartRenderer(faces=model.iuv2smpl.smpl.faces, **synthetic.make_part_assets(0))
        else:
            extra["renderer"] = PartRenderer()                                # part_utils.py's data files
    else:
        dataset = CachedPoseDataset(args.cache)
    res = run_evaluation(model, args.dataset, dataset, args.result_file, args.batch_size, args.log_freq, **extra)
    if dist.is_initialized():
        dist.destroy_process_group()
    return res


if __name__ == "__main__":
    main()
