"""Differentiable restatement of the SMPL layer in torch -- TEST INFRASTRUCTURE (oracle/__init__.py).

The same arithmetic as ``oracle.lbs.lbs`` (smplx's ``lbs`` with pose2rot=False) followed by the reference wrapper's
49-joint assembly (models/smpl.py:27-35: cat[posed joints 24 | selected vertices | J_regressor_extra . vertices]
picked by JOINT_MAP_49, plus the optional translation), written with torch ops so that autograd gives dL/dbetas and
dL/dR for the 24 rotation matrices, taken as free 3x3 inputs.  Any model dict: any vertex count, 1 to 16 betas, any
kinematic tree whose parents precede their children.  Run it in float64 for the reference; float32 is allowed.

``absolute=True`` gives the magnitude of each gradient element.  Every model array and input is replaced by its
absolute value (the caller's upstream gradients too, in ``grads``), and every subtraction becomes an addition: the
pose feature R - I, the relative joints J_i - J_parent and the skinning transforms' tg - Rg J.  With rotation-matrix
input the layer is a polynomial in (betas, R), so the gradient of this absolute layer, M_e = dL_abs/dtheta_e at
|theta|, bounds the sum of the absolute values of the terms of each exact gradient element.
"""
import numpy as np
import torch

from .lbs import JOINT_MAP_49

_KEYS = ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights", "J_regressor_extra")


def prepare(model, dtype=torch.float64, device="cpu", absolute=False):
    """the model's arrays as tensors (absolute values with absolute=True), its parents and selected vertices"""
    if isinstance(model, dict) and model.get("_prepared") == (dtype, str(device), absolute):
        return model
    t = {k: torch.as_tensor(np.asarray(model[k], dtype=np.float64), device=device).to(dtype) for k in _KEYS}
    if absolute:
        t = {k: v.abs() for k, v in t.items()}
    t["parents"] = [int(p) for p in np.asarray(model["parents"])]
    t["selected_verts"] = torch.as_tensor(np.asarray(model["selected_verts"], dtype=np.int64), device=device)
    t["_prepared"] = (dtype, str(device), absolute)
    return t


def smpl_layer(model, betas, R, transl=None, absolute=False):
    """(vertices [B,nv,3], smpl_joints [B,24,3], joints [B,49,3]) of betas [B,nbetas] and R [B,24,3,3], in their
    dtype and on their device.  With absolute=True the inputs are expected non-negative (grads() takes care of it)."""
    m = prepare(model, betas.dtype, betas.device, absolute)
    sgn = 1.0 if absolute else -1.0                     # the sign of every subtraction
    B, nj = betas.shape[0], R.shape[1]
    parents = m["parents"]
    v_shaped = m["v_template"][None] + torch.einsum("bl,mkl->bmk", betas, m["shapedirs"])
    J = torch.einsum("bik,ji->bjk", v_shaped, m["J_regressor"])
    eye = torch.eye(3, dtype=betas.dtype, device=betas.device)
    pose_feature = (R[:, 1:] + sgn * eye).reshape(B, -1)
    v_posed = v_shaped + (pose_feature @ m["posedirs"]).reshape(B, -1, 3)
    # batch_rigid_transform: Rg_i = Rg_p R_i, tg_i = Rg_p (J_i - J_p) + tg_p
    Rg, tg = [R[:, 0]], [J[:, 0]]
    for i in range(1, nj):
        p = parents[i]
        rel = J[:, i] + sgn * J[:, p]
        Rg.append(Rg[p] @ R[:, i])
        tg.append(torch.einsum("brc,bc->br", Rg[p], rel) + tg[p])
    Rg, tg = torch.stack(Rg, 1), torch.stack(tg, 1)                              # [B,24,3,3], [B,24,3]
    At = tg + sgn * torch.einsum("bjrc,bjc->bjr", Rg, J)
    A = torch.cat([Rg, At[..., None]], -1)                                        # [B,24,3,4]
    T = torch.einsum("vj,bjrc->bvrc", m["lbs_weights"], A)
    verts = torch.einsum("bvrc,bvc->bvr", T[..., :3], v_posed) + T[..., 3]
    joints54 = torch.cat([tg, verts[:, m["selected_verts"]],
                          torch.einsum("jv,bvk->bjk", m["J_regressor_extra"], verts)], 1)
    joints = joints54[:, torch.as_tensor(JOINT_MAP_49, device=betas.device)]
    smpl_joints = tg
    if transl is not None:
        t = transl[:, None]
        verts, smpl_joints, joints = verts + t, smpl_joints + t, joints + t
    return verts, smpl_joints, joints


def grads(model, betas, R, grad_verts=None, grad_smpl_joints=None, grad_joints=None, transl=None, absolute=False):
    """(dL/dbetas, dL/dR) for L = <grad_verts, vertices> + <grad_smpl_joints, smpl_joints> + <grad_joints, joints>
    (None: no such term), in the dtype of betas.  absolute=True gives the magnitudes M of the module docstring."""
    f = (lambda a: a.abs()) if absolute else (lambda a: a)
    b = f(betas.detach()).clone().requires_grad_(True)
    r = f(R.detach()).clone().requires_grad_(True)
    t = None if transl is None else f(transl.detach())
    verts, smpl_joints, joints = smpl_layer(model, b, r, t, absolute)
    L = b.sum() * 0
    for g, y in ((grad_verts, verts), (grad_smpl_joints, smpl_joints), (grad_joints, joints)):
        if g is not None:
            L = L + (f(g.to(y.dtype)) * y).sum()
    db, dR = torch.autograd.grad(L, (b, r))
    return db, dR
