"""Training path of the decomposed regressor's head (smpl_regressor.py:844-895, GCN.py:29-92), forward and backward on
the GPU (csrc/gcn_train.cu):

    from danet_b200.regressor import gcn_head, gcn_head_losses
    out = gcn_head(model, rot_feats, global_para)      # {'para', 'joint_rotation', 'joint_position'}
    losses = gcn_head_losses(out, target, gt_smpl_joints, has_smpl)

`rot_feats` [B,24,128] is limb_reslayer's output as the head sees it (smpl_regressor.py:725,860); `global_para` [B,13]
is body_net's output + mean_cam_shape (:696).  `para` [B,229] feeds danet_b200.smpl.smpl_losses unchanged.

`model.training` selects BatchNorm's mode, as in the reference.  Training mode normalises with batch statistics, updates
running_mean / running_var (momentum 0.1, unbiased variance) and num_batches_tracked with in-place tensor ops (so
DaNet.plan_for sees the new version and refolds the inference weights), and returns the intermediate supervision
outputs: 'joint_rotation' = [pose0 [B,216]], 'joint_position' = [coord0, coord1] [B,24,3].  Eval mode normalises with
the running statistics (frozen BatchNorm, still differentiable) and both lists are empty.

One torch.autograd.Function takes the head's 29 parameters as inputs: after backward every one of them has .grad
(pose_regressors.0 and coord_regressors only in training mode, where they are used), and so do rot_feats and
global_para.  Nothing synchronises with the host, and forward + backward + losses can be captured in a CUDA graph.

Deviation from the reference, stated: with no image selected by has_smpl the head losses are 0-dim zeros with a zero
gradient; the reference raises NameError there (`pred` is undefined at smpl_regressor.py:153).

The three ResNet branches in front of the head (smpl_regressor.py:688-725) train through the same module:

    from danet_b200.regressor import body_branch, limb_branch, predictor
    global_para = body_branch(model, body_iuv)          # [B,13] = body_net(body_iuv) + mean_cam_shape
    rot_feats   = limb_branch(model, part_iuv)          # [B,24,128]: limb_net -> limb_reslayer -> average pool
    out         = predictor(model, body_iuv, part_iuv)  # gcn_head(model, rot_feats, global_para)

body_iuv [B,75,S,S] is cat[U,V,I] of the cleaned maps, part_iuv [B,24,3,7,S,S] the cleaned per-part maps, both fp32 on
the model's CUDA device, any S.  The branches are not restated here: `lower_branches` walks the regressor ops of the
network graph (model.graph, the description parameter registration and the inference plan consume) from `body_iuv` to
`global_para` and from `part_iuv_clean` to `rot_feats`, and lowers each op once per graph into differentiable ops:
conv2d (danet_b200.conv), batch_norm fused with residual and ReLU, max_pool2d, adaptive_avg_pool2d and linear
(danet_b200.layers).  A limb tensor is NCHW [24B, C, H, W], the same memory as [B, 24C, H, W]: the grouped convolutions
of limb_reslayer and their BatchNorm2d(24 * 128) take the second view (statistics over the batch), limb_net's
BatchNorm2d(64) the first (statistics pooled over the parts).  model.training selects BatchNorm's mode as in gcn_head;
training mode also adds 1 to every num_batches_tracked.  Inputs that do not require grad get no input gradient (the
first convolution then skips its input gradient)."""
import ctypes
import types
import weakref

import torch
from torch.autograd.function import once_differentiable

from . import _args, _lib

LAYERS = [("r2p_gcn", 0), ("refine_gcn", 0), ("refine_gcn", 1), ("refine_gcn", 2), ("p2r_gcn", 0)]
DIMS = [(128, 128), (128, 256), (256, 256), (256, 128), (128, 128)]
PARAM_NAMES = []
for _n, _i in LAYERS:
    PARAM_NAMES += ["%s.gc.%d.weight" % (_n, _i), "%s.gc.%d.bias" % (_n, _i),
                    "%s.act.%d.0.weight" % (_n, _i), "%s.act.%d.0.bias" % (_n, _i)]
PARAM_NAMES += ["edge_importance"]
for _h in ("pose_regressors", "coord_regressors"):
    for _i in range(2):
        PARAM_NAMES += ["%s.%d.1.weight" % (_h, _i), "%s.%d.1.bias" % (_h, _i)]
BN_NAMES = ["%s.act.%d.0" % (n, i) for n, i in LAYERS]
# parameters only the intermediate supervision heads of training mode use
TRAINING_ONLY = {"pose_regressors.0.1.weight", "pose_regressors.0.1.bias", "coord_regressors.0.1.weight",
                 "coord_regressors.0.1.bias", "coord_regressors.1.1.weight", "coord_regressors.1.1.bias"}
SMPL_POSE_WEIGHTS = 60.0                          # configs/danet_default.yaml:25 (cfg.DANET.SMPL_POSE_WEIGHTS)
JOINT_POSITION_WEIGHTS = 1.0                      # configs/danet_default.yaml:33 (cfg.DANET.JOINT_POSITION_WEIGHTS)


def _attr(mod, name):
    for part in name.split("."):
        mod = getattr(mod, part)
    return mod


def _pack(params, bufs, grads=None):
    p = _lib.GcnTrainParams()
    d = lambda t: t.data_ptr() if t is not None else None
    for l in range(5):
        p.W[l], p.b[l], p.bn_weight[l], p.bn_bias[l] = (d(t) for t in params[4 * l:4 * l + 4])
        p.running_mean[l], p.running_var[l] = d(bufs[l]), d(bufs[5 + l])
    p.r2p_A, p.p2r_A, p.I_n, p.A_mask, p.mean_pose = (d(t) for t in bufs[10:15])
    p.edge_importance = d(params[20])
    p.pose_w[0], p.pose_b[0], p.pose_w[1], p.pose_b[1] = (d(t) for t in params[21:25])
    p.coord_w[0], p.coord_b[0], p.coord_w[1], p.coord_b[1] = (d(t) for t in params[25:29])
    if grads is not None:
        for l in range(5):
            p.gW[l], p.gb[l], p.g_bn_weight[l], p.g_bn_bias[l] = (d(t) for t in grads[4 * l:4 * l + 4])
        p.g_edge_importance = d(grads[20])
        p.g_pose_w[0], p.g_pose_b[0], p.g_pose_w[1], p.g_pose_b[1] = (d(t) for t in grads[21:25])
        p.g_coord_w[0], p.g_coord_b[0], p.g_coord_w[1], p.g_coord_b[1] = (d(t) for t in grads[25:29])
    return p


def _empty(*shape, dev):
    return torch.empty(*shape, device=dev, dtype=torch.float32)


class _GcnHead(torch.autograd.Function):
    """(rot_feats, global_para, *29 parameters) -> para (eval) or (para, pose0, coord0, coord1) (training).  The
    forward keeps its saved activations in a workspace the backward reads."""

    @staticmethod
    def forward(ctx, training, bufs, new_stats, ws_bytes, rot_feats, global_para, *params):
        dev, B = rot_feats.device, rot_feats.shape[0]
        with torch.cuda.device(dev):
            ws = _lib.workspace(ws_bytes, dev)
            para = _empty(B, 229, dev=dev)
            pose0, c0, c1 = (_empty(B, 216, dev=dev), _empty(B, 24, 3, dev=dev), _empty(B, 24, 3, dev=dev)) if training \
                else (None, None, None)
            p = _pack(params, bufs)
            _lib.call("gcn_head_train_forward", B, ctypes.byref(p), int(training), _lib.ptr(rot_feats), _lib.ptr(global_para),
                      _lib.ptr(para), _lib.ptr(pose0), _lib.ptr(c0), _lib.ptr(c1), _lib.ptr(new_stats), _lib.ptr(ws),
                      device=dev)
        ctx.save_for_backward(rot_feats, *params)
        ctx.bufs, ctx.ws, ctx.training = bufs, ws, training
        return (para, pose0, c0, c1) if training else para

    @staticmethod
    @once_differentiable
    def backward(ctx, *g):
        rot_feats, *params = ctx.saved_tensors
        dev, B = rot_feats.device, rot_feats.shape[0]
        training = ctx.training
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        g_para = f32(g[0])
        g_pose0, g_c0, g_c1 = (f32(t) for t in g[1:4]) if training else (None, None, None)
        grads = [None if (not training and name in TRAINING_ONLY) else torch.empty_like(t)
                 for name, t in zip(PARAM_NAMES, params)]
        with torch.cuda.device(dev):
            g_rot, g_gp = torch.empty_like(rot_feats), _empty(B, 13, dev=dev)
            p = _pack(params, ctx.bufs, grads)
            _lib.call("gcn_head_train_backward", B, ctypes.byref(p), int(training), _lib.ptr(rot_feats), _lib.ptr(g_para),
                      _lib.ptr(g_pose0), _lib.ptr(g_c0), _lib.ptr(g_c1), _lib.ptr(g_rot), _lib.ptr(g_gp), _lib.ptr(ctx.ws),
                      device=dev)
        return (None, None, None, None, g_rot, g_gp, *grads)


def head_module(model):
    """The module that holds the head's parameters: model.iuv2smpl.smpl_para_Outs (DaNet) or the model itself."""
    iuv2smpl = getattr(model, "iuv2smpl", None)
    return iuv2smpl.smpl_para_Outs if iuv2smpl is not None else model


def gcn_head(model, rot_feats, global_para):
    """smpl_regressor.py:844-895 (+ the concatenation of :924) in model.training's BatchNorm mode.  rot_feats [B,24,128],
    global_para [B,13] on the model's CUDA device.  Returns {'para': [B,229], 'joint_rotation': [pose0] or [],
    'joint_position': [coord0, coord1] or []}; differentiable w.r.t. the inputs and the head's 29 parameters."""
    where = "danet_b200.regressor.gcn_head"
    mod = head_module(model)
    params = [_attr(mod, n) for n in PARAM_NAMES]
    dev = params[0].device
    _lib.require_cuda(rot_feats, "rot_feats")
    _lib.require_cuda(global_para, "global_para")
    if dev.type != "cuda":
        raise RuntimeError("danet_b200: move the model to a CUDA device (there is no CPU path)")
    if rot_feats.dim() != 3 or tuple(rot_feats.shape[1:]) != (24, 128) or rot_feats.shape[0] < 1:
        raise ValueError("%s: rot_feats must be [B,24,128] with B >= 1, got %s" % (where, tuple(rot_feats.shape)))
    B = rot_feats.shape[0]
    if tuple(global_para.shape) != (B, 13):
        raise ValueError("%s: global_para must be [B,13] = [%d,13], got %s" % (where, B, tuple(global_para.shape)))
    ws_bytes = _lib.load().danet_gcn_head_train_workspace_bytes(B)
    if ws_bytes <= 0:                                   # refused before anything is allocated or launched
        raise ValueError("%s: batch size %d is larger than the head's kernels take" % (where, B))
    _args.cuda(where, (("rot_feats", rot_feats), ("global_para", global_para)), dev)
    for (name, i), (di, do) in zip(LAYERS, DIMS):
        if tuple(_attr(mod, "%s.gc.%d.weight" % (name, i)).shape) != (di, do):
            raise ValueError("%s: %s.gc.%d.weight must be [%d,%d]" % (where, name, i, di, do))
    training = bool(model.training)
    bn = [_attr(mod, n) for n in BN_NAMES]
    bufs = [m.running_mean for m in bn] + [m.running_var for m in bn] + \
        [_attr(mod, k).reshape(-1) for k in ("r2p_A", "p2r_A", "I_n", "A_mask")] + [mod.mean_pose.reshape(-1)]
    if any(t.dtype != torch.float32 or not t.is_contiguous() for t in params + bufs):
        raise ValueError("%s: the head's parameters and buffers must be contiguous fp32" % where)
    new_stats = torch.empty(2, 5, 24, device=dev) if training else None
    out = _GcnHead.apply(training, bufs, new_stats, ws_bytes, rot_feats.float().contiguous(),
                         global_para.float().contiguous(), *params)
    if not training:
        return {"para": out, "joint_rotation": [], "joint_position": []}
    with torch.no_grad():                     # in-place: the tensors' versions move, so plans refold their BatchNorm
        for l, m in enumerate(bn):
            m.running_mean.copy_(new_stats[0, l])
            m.running_var.copy_(new_stats[1, l])
            m.num_batches_tracked.add_(1)
    para, pose0, c0, c1 = out
    return {"para": para, "joint_rotation": [pose0], "joint_position": [c0, c1]}


class _HeadLosses(torch.autograd.Function):
    """losses [3] = (joint_rotation0, joint_position0, joint_position1); one kernel writes the losses and the gradient
    of each w.r.t. its own prediction, the backward scales them by the incoming gradients."""

    @staticmethod
    def forward(ctx, pose0, coord0, coord1, target, gt, has, rot_w, pos_w):
        dev, B = pose0.device, pose0.shape[0]
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
        p_, c0_, c1_, t_, g_ = (f32(t) for t in (pose0, coord0, coord1, target, gt))
        grads = [torch.empty_like(t) for t in (p_, c0_, c1_)]
        with torch.cuda.device(dev):
            losses = _empty(3, dev=dev)
            _lib.call("gcn_head_losses", B, _lib.ptr(p_), _lib.ptr(c0_), _lib.ptr(c1_), _lib.ptr(t_), _lib.ptr(g_),
                      _lib.ptr(has), float(rot_w), float(pos_w), _lib.ptr(losses), *map(_lib.ptr, grads), device=dev)
        ctx.grads = grads
        ctx.dtypes = (pose0.dtype, coord0.dtype, coord1.dtype)
        return losses

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        out = [(t * g[k]).to(ctx.dtypes[k]) for k, t in enumerate(ctx.grads)]
        return (*out, None, None, None, None, None)


def gcn_head_losses(out, target, gt_smpl_joints, has_smpl, rot_weight=SMPL_POSE_WEIGHTS,
                    pos_weight=JOINT_POSITION_WEIGHTS):
    """smpl_regressor.py:147-166 for the head's intermediate outputs (training-mode `out` of gcn_head).
    target [B,229] (cam | betas | rotmats); gt_smpl_joints [B,24,3] (SMPL(target).smpl_joints, :158-162); has_smpl [B]
    (bool / uint8 / float; == 1 selects).  Returns {'joint_rotation0': rot_weight * MSE over the selected images,
    'joint_position0' / 'joint_position1': pos_weight * L1 sum / #selected} as 0-dim tensors (zeros with a zero gradient
    when nothing is selected)."""
    if len(out.get("joint_rotation", [])) != 1 or len(out.get("joint_position", [])) != 2:
        raise ValueError("gcn_head_losses: needs the training-mode output of gcn_head (one pose0, two coord outputs)")
    pose0 = out["joint_rotation"][0]
    coord0, coord1 = out["joint_position"]
    _lib.require_cuda(pose0, "pose0")
    B = pose0.shape[0]
    dev = pose0.device
    if tuple(pose0.shape) != (B, 216) or tuple(coord0.shape) != (B, 24, 3) or tuple(coord1.shape) != (B, 24, 3):
        raise ValueError("gcn_head_losses: expected pose0 [B,216] and coord0 / coord1 [B,24,3]")
    if tuple(target.shape) != (B, 229):
        raise ValueError("gcn_head_losses: target must be [B,229] = [%d,229], got %s" % (B, tuple(target.shape)))
    if tuple(gt_smpl_joints.shape) != (B, 24, 3):
        raise ValueError("gcn_head_losses: gt_smpl_joints must be [B,24,3], got %s" % (tuple(gt_smpl_joints.shape),))
    if has_smpl.dim() != 1 or has_smpl.shape[0] != B:
        raise ValueError("gcn_head_losses: has_smpl must hold one entry per image (%d), got %s" % (B, tuple(has_smpl.shape)))
    has = (has_smpl.to(dev) == 1).to(torch.uint8).contiguous()
    L = _HeadLosses.apply(pose0, coord0, coord1, target.to(dev), gt_smpl_joints.to(dev), has, rot_weight, pos_weight)
    return {"joint_rotation0": L[0], "joint_position0": L[1], "joint_position1": L[2]}


# ---------------------------------------------------------------------------------------------------------------------
# body_net, limb_net and limb_reslayer: the graph's regressor ops lowered into differentiable ops
# ---------------------------------------------------------------------------------------------------------------------
RP = "iuv2smpl.smpl_para_Outs."
BN_MOMENTUM, BN_EPS = 0.1, 1e-5                   # every BatchNorm2d of the branches (res_module.py:17, nn defaults)
BRANCHES = {"body": ("body_iuv", "global_para"), "limb": ("part_iuv_clean", "rot_feats")}
_BN_KEYS = ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")
_LOWERED = weakref.WeakKeyDictionary()


def _lower_op(op, where="lower_branches"):
    """One graph op -> training ops: dicts with the op name, input / output tensor names, their arguments and `keys`,
    the state_dict keys the op consumes.  `where` names the caller in refusals (danet_b200.estimator shares the conv
    rule)."""
    kind, x, y = op["op"], op["x"].name, op["y"].name
    if kind == "conv":
        (wkey, _, has_bias), = op["parts"]
        g = op["groups"]
        conv = dict(op="conv2d", x=x, y=y, weight=wkey + ".weight", bias=wkey + ".bias" if has_bias else None,
                    stride=op["stride"], padding=op["pad"], groups=g)
        conv["keys"] = tuple(k for k in (conv["weight"], conv["bias"]) if k)
        if not op["bn"]:
            if op["relu"] or op["res"] is not None:
                raise ValueError("%s: a residual or ReLU without BatchNorm (%s) has no training lowering" % (where, wkey))
            return [conv]
        conv["y"] = y + ":conv"
        bn = dict(op="batch_norm", x=conv["y"], y=y, bn=op["bn"], res=op["res"].name if op["res"] is not None else None,
                  relu=op["relu"], groups=g, keys=tuple("%s.%s" % (op["bn"], k) for k in _BN_KEYS))
        return [conv, bn]
    if kind == "maxpool":
        return [dict(op="max_pool2d", x=x, y=y, keys=())]
    if kind == "avgpool":
        return [dict(op="adaptive_avg_pool2d", x=x, y=y, keys=())]
    if kind == "body_fc":                         # SmplResNet's avg_pooling + final_layer, + mean_cam_shape (:696)
        w, b, add = RP + "body_net.3.final_layer.weight", RP + "body_net.3.final_layer.bias", RP + "mean_cam_shape"
        return [dict(op="adaptive_avg_pool2d", x=x, y=y + ":pool", keys=()),
                dict(op="linear", x=y + ":pool", y=y, weight=w, bias=b, add=add, keys=(w, b, add))]
    raise ValueError("%s: graph op %r has no training lowering" % (where, kind))


def _walk(graph, src, dst):
    live, out = {src}, []
    for op in graph.ops:
        x = op.get("x")
        if x is None or getattr(x, "name", None) not in live:
            continue
        if op.get("res") is not None and op["res"].name not in live:
            raise ValueError("lower_branches: residual %s of %s is not on the branch" % (op["res"].name, op["y"].name))
        out += _lower_op(op)
        live.add(op["y"].name)
        if op["y"].name == dst:
            return out
    raise ValueError("lower_branches: the graph has no path from %s to %s" % (src, dst))


def lower_branches(graph):
    """{'body': ops, 'limb': ops}: the ops of `graph` reachable from body_iuv up to global_para and from part_iuv_clean
    up to rot_feats, lowered once per graph (see _lower_op)."""
    low = _LOWERED.get(graph)
    if low is None:
        low = {name: dict(src=src, dst=dst, ops=_walk(graph, src, dst)) for name, (src, dst) in BRANCHES.items()}
        _LOWERED[graph] = low
    return low


def _grouped(t, g):
    """[N, C, H, W] -> [N / g, g C, H, W] (the same memory)"""
    return t if g == 1 else t.reshape(t.shape[0] // g, g * t.shape[1], t.shape[2], t.shape[3])


def _ungrouped(t, g):
    return t if g == 1 else t.reshape(t.shape[0] * g, t.shape[1] // g, t.shape[2], t.shape[3])


def run_branch(branch, state, x, training, ops):
    """Runs one lowered branch (lower_branches(graph)[name]) on x ([B,75,S,S] for 'body', [24B,21,S,S] for 'limb').
    `state` maps state_dict keys to tensors; `ops` provides conv2d, batch_norm, max_pool2d, adaptive_avg_pool2d and
    linear with the signatures of danet_b200.conv / danet_b200.layers.  Training mode adds 1 to num_batches_tracked.
    Returns the branch output: [B,13] or [24B,128,1,1]."""
    env = {branch["src"]: x}
    for op in branch["ops"]:
        kind, g, t = op["op"], op.get("groups", 1), env[op["x"]]
        if kind == "conv2d":
            bias = state[op["bias"]] if op["bias"] else None
            y = _ungrouped(ops.conv2d(_grouped(t, g), state[op["weight"]], bias, op["stride"], op["padding"], 1, g), g)
        elif kind == "batch_norm":
            p = lambda k: state["%s.%s" % (op["bn"], k)]
            res = _grouped(env[op["res"]], g) if op["res"] else None
            y = _ungrouped(ops.batch_norm(_grouped(t, g), p("running_mean"), p("running_var"), p("weight"), p("bias"),
                                          training, BN_MOMENTUM, BN_EPS, residual=res, relu=op["relu"]), g)
        elif kind == "max_pool2d":
            y = ops.max_pool2d(t, 3, 2, 1)
        elif kind == "adaptive_avg_pool2d":
            y = ops.adaptive_avg_pool2d(t, 1)
        else:
            y = ops.linear(t.reshape(t.shape[0], -1), state[op["weight"]], state[op["bias"]],
                           add=state[op["add"]].reshape(-1))
        env[op["y"]] = y
    if training:
        with torch.no_grad():
            for op in branch["ops"]:
                if op["op"] == "batch_norm":
                    state[op["bn"] + ".num_batches_tracked"].add_(1)
    return env[branch["dst"]]


def _cuda_ops():
    from . import conv, layers
    return types.SimpleNamespace(conv2d=conv.conv2d, batch_norm=layers.batch_norm, max_pool2d=layers.max_pool2d,
                                 adaptive_avg_pool2d=layers.adaptive_avg_pool2d, linear=layers.linear)


def _model_state(model, branch):
    graph = getattr(model, "graph", None)
    if graph is None:
        raise ValueError("danet_b200.regressor: model must be a danet_b200.DaNet (it has no network graph)")
    low = lower_branches(graph)[branch]
    state = {k: _attr(model, k) for op in low["ops"] for k in op["keys"]}
    dev = state[low["ops"][0]["weight"]].device
    if dev.type != "cuda":
        raise ValueError("danet_b200.regressor: move the model to a CUDA device (there is no CPU path)")
    return low, state, dev


def _branch_input(where, name, t, dev, shape_tail, desc):
    """t is fp32 on the model's device `dev`, of shape [B, *shape_tail, S, S] with B, S >= 1"""
    _args.tensor(where, name, t, contiguous=False)
    _args.cuda(where, [(name, t)], dev)
    n = len(shape_tail)
    if t.dim() != n + 3 or tuple(t.shape[1:n + 1]) != shape_tail or t.shape[0] < 1 or t.shape[-1] < 1 or \
            t.shape[-1] != t.shape[-2]:
        raise ValueError("%s: %s must be %s with B >= 1 (got %s)" % (where, name, desc, tuple(t.shape)))


def body_branch(model, body_iuv):
    """global_para [B,13] = body_net(body_iuv) + mean_cam_shape (smpl_regressor.py:688,696) in model.training's
    BatchNorm mode, differentiable w.r.t. body_iuv and body_net's parameters."""
    low, state, dev = _model_state(model, "body")
    _branch_input("danet_b200.regressor.body_branch", "body_iuv", body_iuv, dev, (75,), "[B,75,S,S]")
    return run_branch(low, state, body_iuv.contiguous(), bool(model.training), _cuda_ops())


def limb_branch(model, part_iuv):
    """rot_feats [B,24,128]: limb_net over the (batch, part) images, limb_reslayer over [B, 24 C, H, W] and the average
    pool (smpl_regressor.py:713-725) in model.training's BatchNorm mode, differentiable w.r.t. part_iuv and the
    parameters of limb_net and limb_reslayer."""
    low, state, dev = _model_state(model, "limb")
    _branch_input("danet_b200.regressor.limb_branch", "part_iuv", part_iuv, dev, (24, 3, 7), "[B,24,3,7,S,S]")
    B, S = part_iuv.shape[0], part_iuv.shape[-1]
    y = run_branch(low, state, part_iuv.reshape(B * 24, 21, S, S).contiguous(), bool(model.training), _cuda_ops())
    return y.reshape(B, 24, -1)


def predictor(model, body_iuv, part_iuv):
    """DecomposedPredictor.forward for the 'iuv' input and the 'gcn' strategy (smpl_regressor.py:676-928):
    gcn_head(model, limb_branch(model, part_iuv), body_branch(model, body_iuv)), i.e. {'para' [B,229],
    'joint_rotation', 'joint_position'}, which feed gcn_head_losses and smpl_losses unchanged."""
    if body_iuv.shape[0] != part_iuv.shape[0]:
        raise ValueError("danet_b200.regressor.predictor: body_iuv and part_iuv hold %d and %d images"
                         % (body_iuv.shape[0], part_iuv.shape[0]))
    global_para = body_branch(model, body_iuv)
    rot_feats = limb_branch(model, part_iuv)
    return gcn_head(model, rot_feats, global_para)
