"""SMPL layer with the reference's call surface (models/smpl.py:15-46 on top of smplx.SMPL),
executed by the fused CUDA kernels in csrc/lbs.cu through the C ABI.

    smpl = SMPL(model_dir, batch_size=B, create_transl=False).to(device)
    out = smpl(betas=betas, body_pose=rotmat[:, 1:], global_orient=rotmat[:, 0:1], pose2rot=False)
    out.vertices, out.joints, out.joints_J19, out.smpl_joints, ...

Inference only (the reference's hot path runs under torch.no_grad, danet.py:15-28).
"""
import ctypes
import os
import pickle
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from . import constants

# smplx.body_models.ModelOutput fields (smplx ~0.1.13) + the two the reference adds (models/smpl.py:24)
ModelOutput_ = namedtuple(
    "ModelOutput_", ["vertices", "joints", "full_pose", "betas", "global_orient", "body_pose",
                     "expression", "left_hand_pose", "right_hand_pose", "jaw_pose",
                     "smpl_joints", "joints_J19"])
ModelOutput_.__new__.__defaults__ = (None,) * len(ModelOutput_._fields)


class _ChStub(object):
    """Stand-in for chumpy.Ch objects inside the official SMPL pickles (chumpy is not required)."""

    def __setstate__(self, state):
        self.__dict__.update(state if isinstance(state, dict) else {"x": state})

    def as_array(self):
        for k in ("x", "r", "_x"):
            if k in self.__dict__:
                return np.asarray(self.__dict__[k])
        raise ValueError("cannot recover the array of a chumpy object with keys %s" % list(self.__dict__))


class _SmplUnpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if module.startswith("chumpy"):
            return _ChStub
        return super().find_class(module, name)


def _arr(v):
    if isinstance(v, _ChStub):
        return v.as_array()
    if hasattr(v, "toarray"):          # scipy.sparse J_regressor
        return v.toarray()
    return np.asarray(v)


def load_smpl_model(model_path, gender="neutral"):
    """dict of numpy arrays from (a) a dict (already loaded / synthetic), (b) an .npz written by
    `save_smpl_npz`, (c) the official SMPL_{GENDER}.pkl or a directory containing it
    (models/smpl.py -> smplx.SMPL.__init__; path_config.py:65 SMPL_MODEL_DIR = 'data/smpl')."""
    if isinstance(model_path, dict):
        return model_path
    if os.path.isdir(model_path):
        model_path = os.path.join(model_path, "SMPL_%s.pkl" % gender.upper())
    if not os.path.exists(model_path):
        raise ValueError("SMPL model file %s does not exist" % model_path)
    if model_path.endswith(".npz"):
        z = np.load(model_path)
        return {k: z[k] for k in z.files}
    with open(model_path, "rb") as f:
        raw = _SmplUnpickler(f, encoding="latin1").load()
    shapedirs = _arr(raw["shapedirs"])[:, :, :10]
    posedirs = _arr(raw["posedirs"])                      # [6890, 3, 207]
    parents = _arr(raw["kintree_table"])[0].astype(np.int64).copy()
    parents[0] = -1
    return {"v_template": _arr(raw["v_template"]).astype(np.float32),
            "shapedirs": shapedirs.astype(np.float32),
            "posedirs": posedirs.reshape(-1, posedirs.shape[-1]).T.astype(np.float32),   # smplx: [207, 20670]
            "J_regressor": _arr(raw["J_regressor"]).astype(np.float32),
            "lbs_weights": _arr(raw["weights"]).astype(np.float32),
            "parents": parents.astype(np.int32),
            "faces": _arr(raw["f"]).astype(np.int64)}


def _maybe_load(x, default_path):
    if x is None:
        x = default_path
    if isinstance(x, str):
        if not os.path.exists(x):
            raise ValueError("%s does not exist" % x)
        return np.load(x)
    return np.asarray(x)


class SMPL(nn.Module):
    """Extension of SMPL to 49 joints -- same constructor / call surface as models/smpl.py."""

    NUM_JOINTS = 23
    NUM_BODY_JOINTS = 23
    NUM_BETAS = 10

    def __init__(self, model_path, gender="neutral", batch_size=1, create_transl=False,
                 J_regressor_extra=None, J_regressor_h36m=None, dtype=torch.float32, **kwargs):
        super().__init__()
        m = load_smpl_model(model_path, gender)
        self.gender = gender
        self.batch_size = batch_size
        self.dtype = dtype
        self.faces = np.asarray(m["faces"])                                   # ndarray [13776,3] (part_utils.py:22)
        f32 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32)
        self.register_buffer("faces_tensor", torch.tensor(self.faces.astype(np.int64)))
        self.register_buffer("v_template", f32(m["v_template"]))
        self.register_buffer("shapedirs", f32(m["shapedirs"]))
        self.register_buffer("posedirs", f32(m["posedirs"]))
        self.register_buffer("J_regressor", f32(m["J_regressor"]))
        self.register_buffer("lbs_weights", f32(m["lbs_weights"]))
        self.register_buffer("parents", torch.tensor(np.asarray(m["parents"]).astype(np.int64)))
        # models/smpl.py:21-22 (path_config.py:64 JOINT_REGRESSOR_TRAIN_EXTRA)
        extra = m["J_regressor_extra"] if (J_regressor_extra is None and "J_regressor_extra" in m) else \
            _maybe_load(J_regressor_extra, "data/J_regressor_extra.npy")
        self.register_buffer("J_regressor_extra", f32(extra))
        # eval.py:78 (path_config.py:66 JOINT_REGRESSOR_H36M) -- optional, fused into the same pass
        if J_regressor_h36m is None and "J_regressor_h36m" in m:
            J_regressor_h36m = m["J_regressor_h36m"]
        elif J_regressor_h36m is None and os.path.exists("data/J_regressor_h36m.npy"):
            J_regressor_h36m = np.load("data/J_regressor_h36m.npy")
        if J_regressor_h36m is not None:
            self.register_buffer("J_regressor_h36m", f32(_maybe_load(J_regressor_h36m, None)))
        else:
            self.J_regressor_h36m = None
        self.selected_verts = np.asarray(m.get("selected_verts", constants.SMPLX_SELECTED_VERTS), dtype=np.int32)
        self.joint_map = torch.tensor(constants.JOINT_MAP_49, dtype=torch.long)       # models/smpl.py:23
        self.ModelOutput = ModelOutput_
        self._handles = {}
        self._ws = {}
        self.last_joints_h36m = None

    # -- C-ABI handle per device ------------------------------------------------------------
    def _handle(self, device):
        key = device.index if device.index is not None else torch.cuda.current_device()
        if key in self._handles:
            return self._handles[key]
        keep = []

        def host(t, dt):
            a = np.ascontiguousarray(t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t), dtype=dt)
            keep.append(a)
            return a.ctypes.data_as(ctypes.c_void_p)

        d = _lib.SmplDesc()
        d.num_verts = self.v_template.shape[0]
        d.num_joints = self.J_regressor.shape[0]
        d.num_betas = self.shapedirs.shape[-1]
        d.v_template = host(self.v_template, np.float32)
        d.shapedirs = host(self.shapedirs, np.float32)
        d.posedirs = host(self.posedirs, np.float32)
        d.J_regressor = host(self.J_regressor, np.float32)
        d.lbs_weights = host(self.lbs_weights, np.float32)
        d.parents = host(self.parents, np.int32)
        d.num_selected = len(self.selected_verts)
        d.selected_verts = host(self.selected_verts, np.int32)
        d.num_extra = self.J_regressor_extra.shape[0]
        d.J_regressor_extra = host(self.J_regressor_extra, np.float32)
        if self.J_regressor_h36m is not None:
            d.num_h36m = self.J_regressor_h36m.shape[0]
            d.J_regressor_h36m = host(self.J_regressor_h36m, np.float32)
        else:
            d.num_h36m = 0
            d.J_regressor_h36m = None
        d.num_out_joints = len(self.joint_map)
        d.joint_map = host(self.joint_map, np.int32)
        h = ctypes.c_void_p()
        with torch.cuda.device(key):
            _lib.check(_lib.load().danet_smpl_create(ctypes.byref(d), ctypes.byref(h)), "smpl_create")
        self._handles[key] = h
        return h

    def _drop_handles(self):
        """The device-side model (danet_smpl_t) snapshots the buffers: drop it whenever they may have changed."""
        try:
            lib = _lib.load()
            for h in self.__dict__.get("_handles", {}).values():
                lib.danet_smpl_destroy(h)
        except Exception:
            pass
        self.__dict__["_handles"] = {}                  # plain attribute: safe during interpreter shutdown too

    def __del__(self):
        self._drop_handles()

    def _apply(self, fn, *a, **k):
        self._drop_handles()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **kw):
        self._drop_handles()
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def _load_from_state_dict(self, *a, **k):
        self._drop_handles()
        return super()._load_from_state_dict(*a, **k)

    def _workspace(self, h, B, device):
        need = _lib.load().danet_smpl_workspace_bytes(h, B)
        key = (device.index, )
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need:
            ws = _lib.workspace(need, device)
            self._ws[key] = ws
        return ws

    # -- forward ----------------------------------------------------------------------------
    def forward(self, betas=None, body_pose=None, global_orient=None, transl=None, return_verts=True,
                return_full_pose=False, pose2rot=True, pose6d=None, bodies_per_cta=0, **kwargs):
        """betas [B,10]; body_pose [B,23,3,3] | [B,69]; global_orient [B,1,3,3] | [B,3].
        `pose6d` [B,24,6] (extension): feed the network's 6-d output directly (rot6d front-end).
        With autograd enabled and an input that requires grad, the rotation-matrix mode (pose2rot=False: what the
        training step feeds, smpl_regressor.py:170) is differentiable: vertices / joints / smpl_joints back-propagate into
        betas and the rotation matrices through danet_smpl_backward (csrc/lbs.cu)."""
        wants_grad = torch.is_grad_enabled() and any(
            t is not None and torch.is_tensor(t) and t.requires_grad for t in (betas, body_pose, global_orient, pose6d))
        if wants_grad:
            if pose2rot or pose6d is not None:
                raise NotImplementedError("danet_b200.SMPL: gradients are implemented for rotation-matrix inputs "
                                          "(pose2rot=False), the mode the reference trains with")
            return self._forward_autograd(betas, body_pose, global_orient, transl, return_verts, return_full_pose)
        with torch.no_grad():
            return self._forward_impl(betas, body_pose, global_orient, transl, return_verts, return_full_pose, pose2rot,
                                      pose6d, bodies_per_cta)

    def _forward_autograd(self, betas, body_pose, global_orient, transl, return_verts, return_full_pose):
        dev = self.v_template.device
        if dev.type != "cuda":
            raise RuntimeError("danet_b200.SMPL: move the module to a CUDA device first (no CPU path)")
        B = next(t for t in (betas, body_pose, global_orient) if t is not None).shape[0]
        f = lambda t: t.to(device=dev, dtype=torch.float32)
        eye = torch.eye(3, device=dev)
        betas = torch.zeros(B, self.shapedirs.shape[-1], device=dev) if betas is None else f(betas)
        go = eye.expand(B, 1, 3, 3) if global_orient is None else f(global_orient).reshape(B, 1, 3, 3)
        bp = eye.expand(B, 23, 3, 3) if body_pose is None else f(body_pose).reshape(B, 23, 3, 3)
        verts, joints, smpl_joints = _SmplLbs.apply(self, betas, torch.cat([go, bp], dim=1))
        if transl is not None:
            t = transl.to(dev, torch.float32).unsqueeze(1)
            joints, verts, smpl_joints = joints + t, verts + t, smpl_joints + t
        joints_J19 = joints[:, -24:, :][:, constants.J24_TO_J19, :]
        return self.ModelOutput(vertices=verts if return_verts else None, global_orient=go, body_pose=bp, joints=joints,
                                joints_J19=joints_J19, smpl_joints=smpl_joints, betas=betas,
                                full_pose=torch.cat([go, bp], dim=1) if return_full_pose else None)

    def _forward_impl(self, betas=None, body_pose=None, global_orient=None, transl=None, return_verts=True,
                      return_full_pose=False, pose2rot=True, pose6d=None, bodies_per_cta=0):
        dev = self.v_template.device
        if dev.type != "cuda":
            raise RuntimeError("danet_b200.SMPL: move the module to a CUDA device first (no CPU path)")
        B = None
        for t in (betas, body_pose, global_orient, pose6d):
            if t is not None:
                B = t.shape[0]
                break
        if B is None:
            B = self.batch_size
        f = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        betas = torch.zeros(B, self.shapedirs.shape[-1], device=dev) if betas is None else f(betas)
        if pose6d is not None:
            pose = f(pose6d).reshape(B, 24, 6)
            kind = 2
            go_in, bp_in = None, None
        elif pose2rot:
            go = torch.zeros(B, 3, device=dev) if global_orient is None else f(global_orient).reshape(B, 3)
            bp = torch.zeros(B, 69, device=dev) if body_pose is None else f(body_pose).reshape(B, 69)
            pose = torch.cat([go, bp], dim=1).contiguous()
            kind = 1
            go_in, bp_in = go, bp
        else:
            eye = torch.eye(3, device=dev)
            go = eye.expand(B, 1, 3, 3) if global_orient is None else f(global_orient).reshape(B, 1, 3, 3)
            bp = eye.expand(B, 23, 3, 3) if body_pose is None else f(body_pose).reshape(B, 23, 3, 3)
            pose = torch.cat([go, bp], dim=1).contiguous()
            kind = 0
            go_in, bp_in = go, bp
        if betas.shape[0] != B or pose.shape[0] != B:
            raise ValueError("SMPL.forward: inconsistent batch sizes")
        if B == 0:                                       # empty batch: empty outputs of the usual shapes, nothing to launch
            z = lambda *shape: torch.zeros(*shape, device=dev)
            self.last_joints_h36m = None if self.J_regressor_h36m is None else z(0, self.J_regressor_h36m.shape[0], 3)
            self.last_rotmats = z(0, 24, 3, 3)
            return self.ModelOutput(vertices=z(0, self.v_template.shape[0], 3) if return_verts else None, global_orient=go_in,
                                    body_pose=bp_in, joints=z(0, len(self.joint_map), 3), joints_J19=z(0, 19, 3),
                                    smpl_joints=z(0, 24, 3), betas=betas, full_pose=None)
        with torch.cuda.device(dev):
            h = self._handle(dev)
            V = self.v_template.shape[0]
            verts = torch.empty(B, V, 3, device=dev)
            joints = torch.empty(B, len(self.joint_map), 3, device=dev)
            smpl_joints = torch.empty(B, 24, 3, device=dev)
            nh = 0 if self.J_regressor_h36m is None else self.J_regressor_h36m.shape[0]
            jh = torch.empty(B, nh, 3, device=dev) if nh else None
            rot = torch.empty(B, 24, 3, 3, device=dev) if kind != 0 else None
            ws = self._workspace(h, B, dev)
            _lib.call("smpl_forward", h, B, _lib.ptr(betas), _lib.ptr(pose), kind, _lib.ptr(verts), _lib.ptr(joints),
                      _lib.ptr(smpl_joints), _lib.ptr(jh), _lib.ptr(rot), _lib.ptr(ws), int(bodies_per_cta))
        if transl is not None:
            # smplx adds the translation to joints and vertices; models/smpl.py:27-46 takes smpl_joints from the
            # translated joints, and eval.py regresses the H36M joints from the translated vertices
            t = transl.to(dev, torch.float32).unsqueeze(1)
            joints, verts, smpl_joints = joints + t, verts + t, smpl_joints + t
            if jh is not None:
                jh = jh + t
        self.last_joints_h36m = jh
        self.last_rotmats = rot if rot is not None else pose
        joints_J24 = joints[:, -24:, :]
        joints_J19 = joints_J24[:, constants.J24_TO_J19, :]                      # models/smpl.py:36-37
        if pose6d is not None:
            go_in, bp_in = rot[:, :1], rot[:, 1:]
        full_pose = None
        if return_full_pose:
            full_pose = torch.cat([go_in.reshape(B, -1, *go_in.shape[2:]) if kind == 0 else go_in,
                                   bp_in], dim=1)
        return self.ModelOutput(vertices=verts if return_verts else None,
                                global_orient=go_in, body_pose=bp_in, joints=joints,
                                joints_J19=joints_J19, smpl_joints=smpl_joints, betas=betas,
                                full_pose=full_pose)

    @torch.no_grad()
    def backward_lbs(self, betas, rotmats, grad_vertices, grad_smpl_joints=None):
        """dL/dbetas [B,10], dL/drotmats [B,24,3,3] from dL/dvertices [B,6890,3] (and dL/dsmpl_joints [B,24,3]) -- the
        SMPL-layer part of the reference's training back-propagation (train/trainer.py:148-215), for the rot-mat
        input mode.  Gradients w.r.t. vertex-regressed joints enter through grad_vertices (J_regressor^T g)."""
        _lib.require_cuda(betas, "betas")
        dev = betas.device
        B = betas.shape[0]
        f = lambda t: t.detach().to(dev, torch.float32).contiguous()
        betas, R, gv = f(betas), f(rotmats).reshape(B, 24, 3, 3), f(grad_vertices)
        gj = f(grad_smpl_joints) if grad_smpl_joints is not None else None
        with torch.cuda.device(dev):
            h = self._handle(dev)
            ws = _lib.workspace(_lib.load().danet_smpl_backward_workspace_bytes(h, B), dev)
            gb = torch.empty(B, betas.shape[1], device=dev)
            gR = torch.empty(B, 24, 3, 3, device=dev)
            _lib.call("smpl_backward", h, B, _lib.ptr(betas), _lib.ptr(R), _lib.ptr(gv), _lib.ptr(gj), _lib.ptr(gb),
                      _lib.ptr(gR), _lib.ptr(ws), device=dev)
        return gb, gR

    def joints_h36m(self):
        """[B,17,3] J_regressor_h36m joints of the last forward (eval.py:186,202 fused into the pass)."""
        return self.last_joints_h36m


class _SmplLbs(torch.autograd.Function):
    """vertices, joints (49), smpl_joints = SMPL(betas, rotmats) with the CUDA forward and backward of csrc/lbs.cu.
    joints = cat[posed skeleton 24 | selected vertices | J_regressor_extra . vertices][joint_map] (models/smpl.py:27-35),
    so their gradient folds into dL/dposed-joints and dL/dvertices before the LBS backward kernel runs."""

    @staticmethod
    def forward(ctx, module, betas, rotmats):
        with torch.no_grad():
            out = module._forward_impl(betas=betas, body_pose=rotmats[:, 1:], global_orient=rotmats[:, :1], pose2rot=False)
        ctx.module = module
        ctx.save_for_backward(betas.detach(), rotmats.detach())
        return out.vertices, out.joints, out.smpl_joints

    @staticmethod
    def backward(ctx, g_verts, g_joints, g_smpl_joints):
        m = ctx.module
        betas, rotmats = ctx.saved_tensors
        dev = betas.device
        B, V = betas.shape[0], m.v_template.shape[0]
        gv = torch.zeros(B, V, 3, device=dev) if g_verts is None else g_verts.to(torch.float32).clone()
        gs = torch.zeros(B, 24, 3, device=dev) if g_smpl_joints is None else g_smpl_joints.to(torch.float32).clone()
        if g_joints is not None:
            sel = torch.as_tensor(np.asarray(m.selected_verts), dtype=torch.long, device=dev)
            nsel, nextra = sel.numel(), m.J_regressor_extra.shape[0]
            gcat = torch.zeros(B, 24 + nsel + nextra, 3, device=dev)
            gcat.index_add_(1, m.joint_map.to(dev), g_joints.to(torch.float32))
            gs += gcat[:, :24]
            gv.index_add_(1, sel, gcat[:, 24:24 + nsel])
            gv += torch.einsum("jv,bjc->bvc", m.J_regressor_extra.to(dev), gcat[:, 24 + nsel:])
        gb, gR = m.backward_lbs(betas, rotmats, gv, gs)
        return None, gb, gR


def smpl_losses(smpl, para, target, target_kps, target_kps3d, target_verts, has_kp3d, has_smpl, focal_length=5000.0,
                img_size=224, openpose_weight=0.0, gt_weight=1.0, weights=None, outputs=None):
    """The SMPL-branch losses of the reference's training step (models/danet/smpl_regressor.py:170-215 with the
    criteria of :224-330: keypoint 2D / 3D, per-vertex, pose / betas regression, camera) on top of the differentiable
    SMPL layer.  para / target [B,229] = cam 3 | betas 10 | 24 rotation matrices; target_kps [B,49,3] (x, y in [-1,1],
    confidence); target_kps3d [B,24,4]; target_verts [B,6890,3]; has_kp3d / has_smpl [B] masks.  Returns a dict of
    scalar losses (already multiplied by their weights); the loss arithmetic is plain torch on the GPU -- the SMPL
    forward / backward underneath are the CUDA kernels.  A dict passed as `outputs` receives the predicted 'vertices'
    [B,V,3] and 'cam_t' [B,3] (smpl_regressor.py:183-188), attached to the graph."""
    w = {"keypoints_2d": 300.0, "keypoints_3d": 300.0, "smpl_pose": 60.0, "smpl_betas": 0.06, "smpl_verts": 0.0}      # configs/danet_default.yaml:25-29
    if weights:
        w.update(weights)
    B = para.shape[0]
    cam, betas, rot = para[:, :3], para[:, 3:13], para[:, 13:].reshape(B, 24, 3, 3)
    out = smpl(betas=betas, body_pose=rot[:, 1:], global_orient=rot[:, :1], pose2rot=False)
    verts, joints = out.vertices, out.joints
    cam_t = torch.stack([cam[:, 1], cam[:, 2], 2 * focal_length / (img_size * cam[:, 0] + 1e-9)], dim=-1)
    if outputs is not None:
        outputs.update(vertices=verts, cam_t=cam_t)
    pts = joints + cam_t.unsqueeze(1)                                       # rotation = identity, centre = 0
    kp2d = focal_length * pts[..., :2] / pts[..., 2:3] / (img_size / 2.0)
    conf = target_kps[:, :, -1:].clone()
    conf[:, :25] *= openpose_weight
    conf[:, 25:] *= gt_weight
    losses = {"keypoints_2d": w["keypoints_2d"] * (conf * (kp2d - target_kps[:, :, :-1]) ** 2).mean()}
    sel3 = has_kp3d.bool()
    if sel3.any():
        gt3, c3 = target_kps3d[sel3, :, :3], target_kps3d[sel3, :, 3:]
        pj = joints[sel3][:, 25:]
        gt3 = gt3 - (gt3[:, 2] + gt3[:, 3]).unsqueeze(1) / 2
        pj = pj - (pj[:, 2] + pj[:, 3]).unsqueeze(1) / 2
        losses["keypoints_3d"] = w["keypoints_3d"] * (c3 * (pj - gt3) ** 2).mean()
    else:
        losses["keypoints_3d"] = para.sum() * 0
    sels = has_smpl.bool()
    if sels.any():
        losses["smpl_verts"] = w["smpl_verts"] * (verts[sels] - target_verts[sels]).abs().mean()
        losses["smpl_pose"] = w["smpl_pose"] * ((rot[sels] - target[sels, 13:].reshape(-1, 24, 3, 3)) ** 2).mean()
        losses["smpl_betas"] = w["smpl_betas"] * ((betas[sels] - target[sels, 3:13]) ** 2).mean()
    else:
        losses["smpl_verts"] = losses["smpl_pose"] = losses["smpl_betas"] = para.sum() * 0
    losses["cam"] = (torch.exp(-cam[:, 0] * 10) ** 2).mean()
    return losses


def save_smpl_npz(path, model):
    np.savez(path, **{k: np.asarray(v) for k, v in model.items()})


@torch.no_grad()
def mpjpe_h36m(pred_j17, gt_j14):
    """eval.py:202-212: pred_j17 [B,17,3] from J_regressor_h36m; gt_j14 [B,14,3] pelvis-centred."""
    _lib.require_cuda(pred_j17, "pred_j17")
    B = pred_j17.shape[0]
    out = torch.empty(B, device=pred_j17.device)
    with torch.cuda.device(pred_j17.device):
        pred, gt = pred_j17.float().contiguous(), gt_j14.float().contiguous()      # locals: they must outlive the launch
        _lib.call("mpjpe_h36m", B, _lib.ptr(pred), _lib.ptr(gt), _lib.ptr(out))
    return out
