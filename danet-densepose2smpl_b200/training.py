"""DaNet's training forward (models/danet/danet.py:140-366, INPUT_MODE='iuv', DECOMPOSED=True) on the GPU, as one
differentiable call:

    from danet_b200.targets import prepare_targets
    from danet_b200.training import danet_forward
    batch.update(prepare_targets(model, batch, opt_pose, opt_betas, fit_valid=...))
    ret = danet_forward(model, batch)
    sum(v.sum() for v in ret['losses'].values()).backward()

It is composition, in the reference's order, over the graph walks the estimator and the regressor already lower:
    1. the IUV estimator and its 12 losses (13 with loss_stnhm), as danet_b200.estimator.iuv_estimator
    2. in training mode with partdrop_rate > 0, the part dropout draw (after the estimator's STN draws, so a seeded run
       draws the reference's masks) unless part_drop is given; then danet_b200.iuvmap.part_drop_clean (eval mode:
       clean only)
    3. body_net, limb_net + limb_reslayer and the GCN head on cat[u_cl, v_cl, index_cl] and the cleaned part maps, as
       danet_b200.regressor.predictor
    4. in training mode, danet_b200.regressor.gcn_head_losses and danet_b200.smpl.smpl_losses
so the estimator's U and V heads receive the gradient of the regressor's losses.

in_dict is the reference's input_batch after input_batch.update(prepare_targets(...)): 'img' [B,3,224,224], and in
training mode 'keypoints' [B,49,3], 'pose_3d' [B,24,4], 'has_pose_3d', 'target' [B,229], 'target_smpl_joints',
'target_verts', 'valid_fit' (the regressor's has_smpl, danet.py:322); optional 'uv_image_gt', 'target_smpl_kps',
'dp_dict', 'has_iuv', 'has_dp' (the estimator's losses, danet_b200.estimator) and 'pretrain_mode' (skips steps 3-4,
danet.py:245).  'vis_on' visualisations (TensorBoard only) are not provided.

Returns the reference's four dicts: 'losses' (0-dim losses unsqueezed to [1], danet.py:358-364), 'metrics' (empty),
'visualization' ('iuv_pred': the cleaned maps, detached; 'part_iuv_pred': the cleaned part maps) and 'prediction'
('cam', 'shape', 'pose', and in training mode 'vertices' and 'cam_t').

`train_step` is the reference's whole training step around danet_forward: the learning-rate decay (`LRDecay`), the
pretraining phase, prepare_targets, the loss sum, the backward, the gradient average over ranks and the optimizer step.

`run_danet` walks the lowered estimator and regressor ops of the network graph (danet_b200.estimator.run_estimator,
danet_b200.regressor.run_branch) on a state dictionary through an op table: `cuda_ops(model)` here, an fp64 torch table
in the tests.  `danet_forward` checks the arguments, draws the noise and passes the model's state and the CUDA ops."""
import functools
import types

import torch
import torch.distributed as dist

from . import _args
from .iuvmap import NUM_PARTS, PARTDROP_RATE

FOCAL_LENGTH, IMG_RES = 5000.0, 224                # constants.FOCAL_LENGTH, cfg.DANET.INIMG_SIZE
TRAIN_KEYS = ("keypoints", "pose_3d", "has_pose_3d", "target", "target_smpl_joints", "target_verts", "valid_fit")


def cuda_ops(model):
    """The op table of danet_forward: the estimator's and the branches' layers, part_drop_clean, the GCN head of
    `model` (gcn_head(rot_feats, global_para)), its losses and smpl_losses on model.iuv2smpl.smpl."""
    from . import estimator, iuvmap, regressor, smpl
    ops = vars(estimator._cuda_ops()).copy()
    ops.update(vars(regressor._cuda_ops()))
    ops.update(draw_part_drop=iuvmap.draw_part_drop, part_drop_clean=iuvmap.part_drop_clean,
               gcn_head=functools.partial(regressor.gcn_head, model), gcn_head_losses=regressor.gcn_head_losses,
               smpl_losses=functools.partial(smpl.smpl_losses, model.iuv2smpl.smpl))
    return types.SimpleNamespace(**ops)


def run_danet(graph, state, in_dict, training, ops, part_drop=None, noise=(None, None), partdrop_rate=PARTDROP_RATE,
              stn_hm_weight=0.0):
    """Steps 1-4 of the module docstring on `state` (state_dict keys -> tensors; BatchNorm statistics are updated in
    place in training mode) through `ops`."""
    from .estimator import estimator_losses, lower_estimator, run_estimator
    from .regressor import lower_branches, run_branch
    image = in_dict["img"]
    B = image.shape[0]
    pred = run_estimator(lower_estimator(graph), state, image.contiguous(), training, ops, noise)
    losses = {}
    if training:
        losses, _ = estimator_losses(pred, ops, in_dict.get("uv_image_gt"), in_dict.get("target_smpl_kps"),
                                     in_dict.get("dp_dict"), in_dict.get("has_iuv"), in_dict.get("has_dp"),
                                     stn_hm_weight)
    drop = None
    if training and partdrop_rate > 0:
        drop = part_drop if part_drop is not None else ops.draw_part_drop(B, partdrop_rate).to(image.device)
    u_cl, v_cl, index_cl, ann_cl, part_iuv_map = ops.part_drop_clean(pred["u"], pred["v"], pred["index"],
                                                                     pred["ann"], pred["part_pred"], drop)
    ret = {"losses": losses, "metrics": {}, "prediction": {},
           "visualization": {"iuv_pred": [t.detach() for t in (u_cl, v_cl, index_cl, ann_cl)]}}
    if not in_dict.get("pretrain_mode", False):
        ret["visualization"]["part_iuv_pred"] = part_iuv_map
        br = lower_branches(graph)
        S = part_iuv_map.shape[-1]
        global_para = run_branch(br["body"], state, torch.cat([u_cl, v_cl, index_cl], 1), training, ops)
        rot_feats = run_branch(br["limb"], state, part_iuv_map.reshape(B * NUM_PARTS, 21, S, S), training, ops)
        out = ops.gcn_head(rot_feats.reshape(B, NUM_PARTS, -1), global_para)
        para = out["para"]
        ret["prediction"].update(cam=para[:, :3], shape=para[:, 3:13], pose=para[:, 13:].reshape(-1, 24, 3, 3))
        if training:
            has_smpl = in_dict["valid_fit"]
            losses.update(ops.gcn_head_losses(out, in_dict["target"], in_dict["target_smpl_joints"], has_smpl))
            losses.update(ops.smpl_losses(para, in_dict["target"], in_dict["keypoints"], in_dict["pose_3d"],
                                          in_dict["target_verts"], in_dict["has_pose_3d"], has_smpl,
                                          focal_length=FOCAL_LENGTH, img_size=IMG_RES, outputs=ret["prediction"]))
    ret["losses"] = {k: (v.unsqueeze(0) if v.dim() == 0 else v) for k, v in losses.items()}
    return ret


def danet_forward(model, in_dict, *, part_drop=None, center_noise=None, scale_noise=None,
                  partdrop_rate=PARTDROP_RATE, stn_hm_weight=None):
    """DaNet._forward for INPUT_MODE='iuv', DECOMPOSED=True in model.training's mode; see the module docstring.
    part_drop: bool [B,24] on the model's device (part_drop[b, d-1]: DensePose part d of image b is dropped), training
    mode with partdrop_rate > 0 only; drawn like the reference (danet_b200.iuvmap.draw_part_drop) when not given.
    center_noise / scale_noise / stn_hm_weight: as in danet_b200.estimator.iuv_estimator.
    partdrop_rate: cfg.DANET.PARTDROP_RATE."""
    from .estimator import prepare_estimator
    from .regressor import _model_state
    where = "danet_b200.training.danet_forward"
    if getattr(model, "graph", None) is None or getattr(model, "iuv2smpl", None) is None:
        raise ValueError("%s: model must be a danet_b200.DaNet (it has no network graph)" % where)
    if not isinstance(in_dict, dict) or "img" not in in_dict:
        raise ValueError("%s: in_dict must be a dict with 'img'" % where)
    if in_dict.get("vis_on", False):
        raise ValueError("%s: vis_on visualisations (TensorBoard only) are not provided" % where)
    rate = _args.number(where, "partdrop_rate", partdrop_rate)
    if rate < 0:
        raise ValueError("%s: partdrop_rate must be >= 0 (got %g)" % (where, rate))
    image = in_dict["img"]
    _args.tensor(where, "img", image, dim=4, contiguous=False)
    B = image.shape[0]
    training = bool(model.training)
    if part_drop is not None:
        if not training or rate == 0:
            raise ValueError("%s: part_drop is training-mode dropout with partdrop_rate > 0" % where)
        if not isinstance(part_drop, torch.Tensor) or part_drop.dtype != torch.bool:
            raise ValueError("%s: part_drop must be a bool tensor [B,24]" % where)
        _args.mask(where, "part_drop", part_drop, (B, NUM_PARTS))
        _args.cuda(where, [("img", image), ("part_drop", part_drop)])
    if training and not in_dict.get("pretrain_mode", False):
        missing = [k for k in TRAIN_KEYS if in_dict.get(k) is None]
        if missing:
            raise ValueError("%s: training mode needs in_dict[%s] (prepare_targets and the data batch)"
                             % (where, ", ".join(repr(k) for k in missing)))
    _, state, training, hm_w, noise = prepare_estimator(
        where, model, image, in_dict.get("uv_image_gt"), in_dict.get("target_smpl_kps"), in_dict.get("dp_dict"),
        in_dict.get("has_iuv"), in_dict.get("has_dp"), center_noise, scale_noise, stn_hm_weight)
    for branch in ("body", "limb"):
        state.update(_model_state(model, branch)[1])
    return run_danet(model.graph, state, in_dict, training, cuda_ops(model), part_drop, noise, rate, hm_w)


BN_BUFFERS = ("running_mean", "running_var", "num_batches_tracked")


class LRDecay:
    """The reference's learning-rate decay (train/trainer.py:119-128, configs/danet_default.yaml SOLVER) as it is
    written: decay_steps_ind starts at 1, and when step_count == steps[decay_steps_ind] every param group's lr becomes
    param_groups[0]['lr'] * gamma and the index moves on.  A trainer that resumes builds a new one, so the index restarts
    at 1 there too, as in the reference (where a resume past steps[1] therefore never decays again)."""

    def __init__(self, steps=(0, 30000, 60000), gamma=0.1):
        self.steps = tuple(int(s) for s in steps)
        self.gamma = _args.number("danet_b200.training.LRDecay", "gamma", gamma)
        self.decay_steps_ind = 1

    def __call__(self, optimizer, step_count):
        """Apply the rule for `step_count`; returns True when it decayed the learning rate."""
        if self.decay_steps_ind < len(self.steps) and step_count == self.steps[self.decay_steps_ind]:
            lr_new = optimizer.param_groups[0]["lr"] * self.gamma
            for param_group in optimizer.param_groups:
                param_group["lr"] = lr_new
            self.decay_steps_ind += 1
            return True
        return False


def train_step(model, optimizer, batch, opt_pose, opt_betas, step_count, *, schedule, pretr_step=5000, fit_valid=None,
               part_drop=None, center_noise=None, scale_noise=None, partdrop_rate=PARTDROP_RATE, stn_hm_weight=None,
               group=None):
    """Trainer.train_step (train/trainer.py:117-244) on the GPU, in the reference's order:
        1. schedule(optimizer, step_count) (the learning-rate decay, LRDecay); 2. model.train();
        3. pretrain_mode = step_count <= pretr_step (train/base_trainer.py:70-74);
        4. danet_b200.targets.prepare_targets(model, batch, opt_pose, opt_betas, fit_valid=) merged into the batch;
        5. danet_forward; 6. loss_tatal, the sum of the losses from 0 in dict order; 7. optimizer.zero_grad();
        8. loss_tatal.backward(); 9. with a process group of more than one rank, the gradient average
           (parallel.all_reduce_gradients); 10. optimizer.step();
        11. with more than one rank, rank 0's BatchNorm statistics and counters on every rank (parallel.broadcast_buffers),
            so every rank ends the step with the same model, as DistributedDataParallel's broadcast_buffers gives.
    batch: the data batch (prepare_targets' keys, 'img', 'pose_3d', 'has_pose_3d' and the estimator's optional
    annotations; see danet_forward).  opt_pose / opt_betas / fit_valid: the fits the caller looked up (FitsDict).
    part_drop / center_noise / scale_noise / partdrop_rate / stn_hm_weight: as in danet_forward.  optimizer: any
    torch.optim optimizer (danet_b200.optim.Adam is the reference's Adam in one pass).

    Returns the reference's (output, losses): output 'pred_vertices', 'opt_vertices', 'pred_cam_t', 'opt_cam_t'
    (the prediction entries None in pretraining mode) and 'visualization'; losses 'loss_<key>' and 'loss_tatal' as
    detached device tensors, so that the step never waits for the GPU (call .item() where the values are logged)."""
    from .parallel import all_reduce_gradients, broadcast_buffers
    from .targets import prepare_targets
    where = "danet_b200.training.train_step"
    if not isinstance(optimizer, torch.optim.Optimizer):
        raise ValueError("%s: optimizer must be a torch.optim.Optimizer (got %s)" % (where, type(optimizer).__name__))
    if not callable(schedule):
        raise ValueError("%s: schedule must be callable as schedule(optimizer, step_count) (e.g. LRDecay())" % where)
    if not isinstance(batch, dict) or "img" not in batch:
        raise ValueError("%s: batch must be a dict with 'img'" % where)
    for name, v in (("step_count", step_count), ("pretr_step", pretr_step)):
        if isinstance(v, bool) or not isinstance(v, int):
            raise ValueError("%s: %s must be an int (got %r)" % (where, name, v))
    schedule(optimizer, step_count)
    model.train()
    in_dict = dict(batch)
    in_dict["pretrain_mode"] = step_count <= pretr_step
    targets = prepare_targets(model, batch, opt_pose, opt_betas, fit_valid=fit_valid)
    in_dict.update(targets)
    ret = danet_forward(model, in_dict, part_drop=part_drop, center_noise=center_noise, scale_noise=scale_noise,
                        partdrop_rate=partdrop_rate, stn_hm_weight=stn_hm_weight)
    loss_tatal = 0
    losses = {}
    for k, v in ret["losses"].items():
        loss_tatal += v
        losses["loss_%s" % k] = v.detach()
    optimizer.zero_grad()
    loss_tatal.backward()
    ranks = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    if ranks > 1:
        all_reduce_gradients(model.parameters(), group)
    optimizer.step()
    if ranks > 1:
        broadcast_buffers([b for n, b in model.named_buffers() if n.endswith(BN_BUFFERS)], group)
    pretrain = in_dict["pretrain_mode"]
    output = {"pred_vertices": None if pretrain else ret["prediction"]["vertices"].detach(),
              "opt_vertices": targets["target_verts"],
              "pred_cam_t": None if pretrain else ret["prediction"]["cam_t"].detach(),
              "opt_cam_t": targets["opt_cam_t"],
              "visualization": ret["visualization"]}
    losses["loss_tatal"] = loss_tatal.detach()
    return output, losses
