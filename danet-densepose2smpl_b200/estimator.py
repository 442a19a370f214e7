"""Training path of the IUV estimator (iuv_estimator.py:58-260, INPUT_MODE='iuv', DECOMPOSED=True) on the GPU:

    from danet_b200.estimator import iuv_estimator
    out = iuv_estimator(model, image, iuv_image_gt, smpl_kps_gt, uvia_dp_gt, has_iuv, has_dp)
    sum(out['losses'].values()).backward()

image [B,3,224,224] fp32 on the model's CUDA device.  `model.training` selects the mode, as in danet_b200.regressor.
Training mode normalises with batch statistics and updates every running_mean / running_var (momentum 0.1, unbiased
variance, copied in place so DaNet.plan_for refolds) and num_batches_tracked; eval mode uses the running statistics.

The targets come from danet_b200.targets.prepare_targets(...) and the data batch without reshaping:
    iuv_image_gt = targets['uv_image_gt']        [B,3,S,S] (S = 56, the heads' map size)
    smpl_kps_gt  = targets['target_smpl_kps']    [B,24,3]  (x, y in [-1, 1], weight)
    has_iuv      = targets['has_iuv']            [B]
    uvia_dp_gt   = the batch's DensePose blobs   {'body_uv_X_points': ..., ...} (danet_b200.losses.dp_uvia_losses)
    has_dp       = batch['has_dp']               [B]
Each target is optional; a loss is computed only where the reference computes it (training mode, its targets given).

Returns a dict:
    'losses'         loss_U, loss_V, loss_IndexUV, loss_segAnn (iuv_image_gt); loss_Udp, loss_Vdp, loss_IndexUVdp,
                     loss_segAnndp (uvia_dp_gt); loss_roi, and loss_stnhm when stn_hm_weight > 0 (smpl_kps_gt);
                     loss_pU, loss_pV, loss_pIndexUV (iuv_image_gt).  Empty in eval mode.
    'uvia_pred'      [U, V, Index, Ann] raw heads [B,25|25|25|15,S,S]
    'part_iuv_pred'  [B,24,3,7,S,S]
    'stn_kps_pred'   [B,24,2] (detached), 'skps_hm_pred' [B,24,S,S] (detached)
    'part_iuv_gt'    [B,24,3,7,S,S], training mode with iuv_image_gt
The result is differentiable w.r.t. image and every img2iuv.iuv_est.* parameter.  learned_ratio and learned_offset get
no gradient: the reference detaches the thetas.

STN noise.  In training mode the reference draws torch.rand on the host: the centre jitter (iuv_estimator.py:174, only
with smpl_kps_gt) and then, per part, the two scale jitters of affine_para (:285, :291).  When center_noise [B,24,2]
and scale_noise [24,2,B] are not given, they are drawn in that order on the CPU generator and moved to the device, so
after the same torch.manual_seed the draws are the reference's.  When both are given, nothing touches the host: no
synchronisation and no `torch.sum(has_dp) > 0` test (dp_uvia_losses selects on the device, and the DensePose labels are
not range-checked on the host; a label outside the classes contributes nothing), so forward, losses and backward can be
captured in a CUDA graph.  Eval mode takes no noise and no jitter, as the reference.

The network is not restated here: `lower_estimator` walks the ops of the network graph (model.graph) from `image` to
xd, the four heads and hm, on through the STN to the grouped predict_partial_iuv, and lowers each op once per graph:
    conv (one part)    conv2d, then batch_norm(residual=, relu=) when the op has BatchNorm (regressor._lower_op)
    conv (four parts)  one conv2d over the out-channel concatenation of the U | V | Index | Ann weights and biases,
                       split into the four maps
    fuse               hr_fuse(terms, factors, relu)
    stn_params         part_thetas(hm, raw index head, learned_ratio, learned_offset, noise)
    stn_sample         part_crops(xd, thetas)
    grouped conv       conv2d(groups=24) on the crops [B, 24 C, S, S]
The cleaning ops (clean_global, clean_parts) end the walk: cleaning, part dropout and the regressor are not part of
the estimator.  `run_estimator` runs the lowered ops through an op table (the CUDA one here; the tests substitute an
fp64 torch one)."""
import functools
import types
import weakref

import torch

from . import _args
from .regressor import BN_EPS, BN_MOMENTUM, _attr, _lower_op

EP = "img2iuv."
VIS_SCORE = 0.5                                   # configs/danet_default.yaml:41 (cfg.DANET.STN_PART_VIS_SCORE)
CENTER_JITTER = 0.1                               # configs/danet_default.yaml:38 (cfg.DANET.STN_CENTER_JITTER)
SCALE_JITTER = 0.2                                # configs/danet_default.yaml:39 (cfg.DANET.STN_SCALE_JITTER)
HEADS = ("u", "v", "index", "ann")                # the parts of the heads convolution, in channel order
STOPS = ("clean_global", "clean_parts")           # graph ops that end the walk
NUM_PARTS = 24
_LOWERED = weakref.WeakKeyDictionary()
WHERE = "lower_estimator"


def _inputs(op, heads):
    """the tensor names an op reads; the first is the one that puts the op on the walk"""
    kind = op["op"]
    if kind == "conv":
        return [op["x"].name] + ([op["res"].name] if op["res"] is not None else [])
    if kind == "fuse":
        return [t.name for t, _ in op["terms"]]
    if kind == "stn_params":                      # training reads the raw index head, not the cleaned argmax map
        return [op["hm"].name, heads]
    if kind == "stn_sample":
        return [op["x"].name, op["theta"].name]
    x = op.get("x")
    return [x.name] if x is not None else []


def _lower(op, heads):
    kind = op["op"]
    if kind == "conv" and len(op["parts"]) > 1:
        parts = op["parts"]
        if op["bn"] or op["relu"] or op["res"] is not None or op["groups"] != 1:
            raise ValueError("%s: a multi-part convolution with BatchNorm, ReLU, residual or groups has no training "
                             "lowering" % WHERE)
        w = tuple(k + ".weight" for k, _, _ in parts)
        b = tuple(k + ".bias" for k, _, has in parts if has)
        if b and len(b) != len(parts):
            raise ValueError("%s: the parts of %s must all have a bias or none" % (WHERE, parts[0][0]))
        y = op["y"].name
        return [dict(op="conv2d", x=op["x"].name, y=y, weight=w, bias=b or None, stride=op["stride"],
                     padding=op["pad"], groups=1, split=tuple(c for _, c, _ in parts),
                     ys=tuple("%s:%s" % (y, h) for h in HEADS[:len(parts)]), keys=w + b)]
    if kind == "conv":
        return _lower_op(op, WHERE)
    if kind == "fuse":
        return [dict(op="hr_fuse", terms=[t.name for t, _ in op["terms"]], factors=[f for _, f in op["terms"]],
                     y=op["y"].name, relu=op["relu"], keys=())]
    if kind == "stn_params":
        return [dict(op="part_thetas", hm=op["hm"].name, index=heads + ":index", y=op["theta"].name,
                     centers=op["centers"].name, keys=(EP + "learned_ratio", EP + "learned_offset"))]
    if kind == "stn_sample":
        return [dict(op="part_crops", x=op["x"].name, theta=op["theta"].name, y=op["y"].name, keys=())]
    raise ValueError("%s: graph op %r has no training lowering" % (WHERE, kind))


def _walk(graph):
    heads, dst = graph.outputs["heads"].name, graph.outputs["part_pred"].name
    live, out = {"image"}, []
    for i, op in enumerate(graph.ops):
        ins = _inputs(op, heads)
        if not ins or ins[0] not in live:
            continue
        if op["op"] in STOPS:
            continue
        missing = [n for n in ins if n not in live]
        if missing:
            raise ValueError("%s: input %s of graph op %d (%s) is not on the estimator's path" % (WHERE, missing[0], i,
                                                                                                 op["op"]))
        for t in _lower(op, heads):
            t["gop"] = i
            out.append(t)
            live.update(t["ys"] if "ys" in t else [t["y"]])
            if t["op"] == "part_thetas":
                live.add(t["centers"])
        if op.get("y") is not None:
            live.add(op["y"].name)
            if op["y"].name == dst:
                return out
    raise ValueError("%s: the graph has no path from image to %s" % (WHERE, dst))


def lower_estimator(graph):
    """{'ops': the lowered ops from image to the part prediction, 'out': names of xd, the heads, hm, thetas, centres and
    the part prediction}, once per graph (a weak dictionary keyed by the graph)."""
    low = _LOWERED.get(graph)
    if low is None:
        ops = _walk(graph)
        h = graph.outputs["heads"].name
        th = next(op for op in ops if op["op"] == "part_thetas")
        low = dict(ops=ops, out=dict(xd=graph.outputs["xd"].name, heads=["%s:%s" % (h, k) for k in HEADS],
                                     hm=graph.outputs["hm"].name, thetas=th["y"], centers=th["centers"],
                                     part_pred=graph.outputs["part_pred"].name))
        _LOWERED[graph] = low
    return low


def run_estimator(low, state, image, training, ops, noise=(None, None)):
    """Runs the lowered ops (lower_estimator(graph)) on image [B,3,H,W].  `state` maps state_dict keys to tensors;
    `ops` provides conv2d, batch_norm, hr_fuse, part_thetas and part_crops with the signatures of danet_b200.conv,
    danet_b200.layers and danet_b200.stn.  noise = (center_noise [B,24,2] or None, scale_noise [24,2,B] or None): a
    jitter is applied where its noise is given.  Training mode adds 1 to every num_batches_tracked.
    Returns {'u', 'v', 'index', 'ann', 'hm', 'xd', 'centers', 'thetas', 'part_pred' [B,24,3,7,S,S]}."""
    center_noise, scale_noise = noise
    env = {"image": image}
    for op in low["ops"]:
        kind = op["op"]
        if kind == "conv2d":
            w, b = op["weight"], op["bias"]
            if isinstance(w, tuple):              # the heads: one convolution over the concatenated parts
                w = torch.cat([state[k] for k in w], 0)
                b = torch.cat([state[k] for k in b], 0) if b else None
            else:
                w, b = state[w], (state[b] if b else None)
            y = ops.conv2d(env[op["x"]], w, b, op["stride"], op["padding"], 1, op["groups"])
            if "split" in op:
                for name, t in zip(op["ys"], torch.split(y, op["split"], 1)):
                    env[name] = t.contiguous()
                continue
        elif kind == "batch_norm":
            p = lambda k: state["%s.%s" % (op["bn"], k)]
            y = ops.batch_norm(env[op["x"]], p("running_mean"), p("running_var"), p("weight"), p("bias"), training,
                               BN_MOMENTUM, BN_EPS, residual=env[op["res"]] if op["res"] else None, relu=op["relu"])
        elif kind == "hr_fuse":
            y = ops.hr_fuse([env[n] for n in op["terms"]], op["factors"], op["relu"])
        elif kind == "part_thetas":
            env[op["centers"]], y = ops.part_thetas(
                env[op["hm"]], env[op["index"]], state[op["keys"][0]], state[op["keys"][1]], vis_score=VIS_SCORE,
                center_noise=center_noise, center_jitter=CENTER_JITTER if center_noise is not None else 0.0,
                scale_noise=scale_noise, scale_jitter=SCALE_JITTER if scale_noise is not None else 0.0)
        else:
            y = ops.part_crops(env[op["x"]], env[op["theta"]])
        env[op["y"]] = y
    if training:
        with torch.no_grad():
            for op in low["ops"]:
                if op["op"] == "batch_norm":
                    state[op["bn"] + ".num_batches_tracked"].add_(1)
    o = low["out"]
    pp = env[o["part_pred"]]
    out = {k: env[n] for k, n in zip(HEADS, o["heads"])}
    out.update(hm=env[o["hm"]], xd=env[o["xd"]], centers=env[o["centers"]], thetas=env[o["thetas"]],
               part_pred=pp.view(pp.shape[0], NUM_PARTS, 3, -1, pp.shape[2], pp.shape[3]))
    return out


def estimator_losses(pred, ops, iuv_image_gt=None, smpl_kps_gt=None, uvia_dp_gt=None, has_iuv=None, has_dp=None,
                     stn_hm_weight=0.0):
    """The training losses of iuv_estimator.py:97-121,142-171,217-256 on run_estimator's output, through the op table's
    iuv_img2map, body_uv_losses, dp_uvia_losses, stn_kps_losses, part_iuv_targets and part_iuv_losses.
    Returns (losses dict with the reference's keys, part_iuv_gt or None)."""
    L, part_gt = {}, None
    u, v, idx, ann = (pred[k] for k in HEADS)
    if iuv_image_gt is not None:
        uvia = ops.iuv_img2map(iuv_image_gt)
        L["loss_U"], L["loss_V"], L["loss_IndexUV"], L["loss_segAnn"] = ops.body_uv_losses(u, v, idx, ann, uvia, has_iuv)
    if uvia_dp_gt is not None:
        L["loss_Udp"], L["loss_Vdp"], L["loss_IndexUVdp"], L["loss_segAnndp"] = ops.dp_uvia_losses(
            u, v, idx, ann, has_dp=has_dp, **uvia_dp_gt)
    if smpl_kps_gt is not None:
        roi, stnhm = ops.stn_kps_losses(pred["hm"], smpl_kps_gt, hm_weight=stn_hm_weight)
        if stnhm is not None:
            L["loss_stnhm"] = stnhm
        if roi is not None:
            L["loss_roi"] = roi
    if iuv_image_gt is not None:
        part_gt = ops.part_iuv_targets(uvia, pred["thetas"])
        L["loss_pU"], L["loss_pV"], L["loss_pIndexUV"] = ops.part_iuv_losses(pred["part_pred"], part_gt, has_iuv)
    return L, part_gt


def _cuda_ops():
    from . import conv, iuvmap, layers, losses, stn
    return types.SimpleNamespace(conv2d=conv.conv2d, batch_norm=layers.batch_norm, hr_fuse=layers.hr_fuse,
                                 part_thetas=stn.part_thetas, part_crops=stn.part_crops, iuv_img2map=iuvmap.iuv_img2map,
                                 body_uv_losses=losses.body_uv_losses,
                                 dp_uvia_losses=functools.partial(losses.dp_uvia_losses, check_labels=False),
                                 stn_kps_losses=losses.stn_kps_losses, part_iuv_targets=losses.part_iuv_targets,
                                 part_iuv_losses=losses.part_iuv_losses)


def draw_noise(B, center=True):
    """The reference's STN draws, in its order, on the CPU generator: (center_noise [B,24,2] or None, scale_noise
    [24,2,B])."""
    cn = torch.rand(B, NUM_PARTS, 2) if center else None
    sn = torch.stack([torch.stack([torch.rand(B), torch.rand(B)]) for _ in range(NUM_PARTS)])
    return cn, sn


def iuv_estimator(model, image, iuv_image_gt=None, smpl_kps_gt=None, uvia_dp_gt=None, has_iuv=None, has_dp=None, *,
                  center_noise=None, scale_noise=None, stn_hm_weight=None):
    """IUV_Estimator.forward (iuv_estimator.py:58-260) for INPUT_MODE='iuv', DECOMPOSED=True in model.training's mode.
    See the module docstring.  stn_hm_weight: cfg.DANET.STN_HM_WEIGHTS (default danet_b200.losses.STN_HM_WEIGHTS)."""
    low, state, training, hm_w, noise = prepare_estimator("danet_b200.estimator.iuv_estimator", model, image,
                                                          iuv_image_gt, smpl_kps_gt, uvia_dp_gt, has_iuv, has_dp,
                                                          center_noise, scale_noise, stn_hm_weight)
    ops = _cuda_ops()
    pred = run_estimator(low, state, image.contiguous(), training, ops, noise)
    ret = {"losses": {}, "uvia_pred": [pred[k] for k in HEADS], "part_iuv_pred": pred["part_pred"],
           "stn_kps_pred": pred["centers"].detach(), "skps_hm_pred": pred["hm"].detach()}
    if training:
        ret["losses"], part_gt = estimator_losses(pred, ops, iuv_image_gt, smpl_kps_gt, uvia_dp_gt, has_iuv, has_dp,
                                                  hm_w)
        if part_gt is not None:
            ret["part_iuv_gt"] = part_gt
    return ret


def prepare_estimator(where, model, image, iuv_image_gt, smpl_kps_gt, uvia_dp_gt, has_iuv, has_dp, center_noise,
                      scale_noise, stn_hm_weight):
    """iuv_estimator's argument checks and STN draws: (lowered ops, state, training, stn_hm_weight, noise)."""
    from . import losses
    graph = getattr(model, "graph", None)
    if graph is None:
        raise ValueError("%s: model must be a danet_b200.DaNet (it has no network graph)" % where)
    low = lower_estimator(graph)
    state = {k: _attr(model, k) for op in low["ops"] for k in op["keys"]}
    dev = state[low["ops"][0]["weight"]].device
    # shapes and combinations first, then devices
    _args.tensor(where, "image", image, dim=4, contiguous=False)
    size = graph.tensors["image"].H
    if tuple(image.shape[1:]) != (3, size, size) or image.shape[0] < 1:
        raise ValueError("%s: image must be [B,3,%d,%d] with B >= 1 (got %s)" % (where, size, size, tuple(image.shape)))
    B, S = image.shape[0], graph.outputs["hm"].H
    training = bool(model.training)
    hm_w = losses.STN_HM_WEIGHTS if stn_hm_weight is None else _args.number(where, "stn_hm_weight", stn_hm_weight)
    if not training and (center_noise is not None or scale_noise is not None):
        raise ValueError("%s: center_noise / scale_noise are training-mode jitter (eval mode has none)" % where)
    if center_noise is not None and smpl_kps_gt is None:
        raise ValueError("%s: center_noise needs smpl_kps_gt (the reference jitters the centres only with key points)"
                         % where)
    noise = (("center_noise", center_noise, (B, NUM_PARTS, 2)), ("scale_noise", scale_noise, (NUM_PARTS, 2, B)))
    for name, n, shape in noise:
        if n is not None:
            _args.tensor(where, name, n, shape=shape)
    named = [(name, n) for name, n, _ in noise if n is not None]
    if training:
        if iuv_image_gt is not None:
            _args.tensor(where, "iuv_image_gt", iuv_image_gt, shape=(B, 3, S, S), contiguous=False)
            named.append(("iuv_image_gt", iuv_image_gt))
        if smpl_kps_gt is not None:
            _args.tensor(where, "smpl_kps_gt", smpl_kps_gt, dim=3, contiguous=False)
            if tuple(smpl_kps_gt.shape[:2]) != (B, NUM_PARTS) or smpl_kps_gt.shape[2] not in (2, 3):
                raise ValueError("%s: smpl_kps_gt must be [%d,24,2|3] (got %s)" % (where, B, tuple(smpl_kps_gt.shape)))
            named.append(("smpl_kps_gt", smpl_kps_gt))
        if uvia_dp_gt is not None:
            if not isinstance(uvia_dp_gt, dict):
                raise ValueError("%s: uvia_dp_gt must be a dict of the DensePose blobs" % where)
            named += [(k, v) for k, v in uvia_dp_gt.items() if v is not None]
        for name, f in (("has_iuv", has_iuv), ("has_dp", has_dp)):
            if f is not None:
                if not isinstance(f, torch.Tensor) or f.dim() != 1 or f.shape[0] != B:
                    raise ValueError("%s: %s must be a tensor with one entry per image (%d)" % (where, name, B))
                named.append((name, f))
    if dev.type != "cuda":
        raise ValueError("%s: move the model to a CUDA device (there is no CPU path)" % where)
    _args.cuda(where, [("image", image)] + named, dev)
    if training:
        if scale_noise is None:
            cn, sn = draw_noise(B, center_noise is None and smpl_kps_gt is not None)
            center_noise = center_noise if center_noise is not None else (cn.to(dev) if cn is not None else None)
            scale_noise = sn.to(dev)
        elif center_noise is None and smpl_kps_gt is not None:
            center_noise = torch.rand(B, NUM_PARTS, 2).to(dev)
    return low, state, training, hm_w, (center_noise, scale_noise)
