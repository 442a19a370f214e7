"""The covering sweep of the SMPL layer's backward (danet_smpl_backward, csrc/lbs.cu): the models, the case table, the
coverage classes and the per-element bound dL/dbetas and dL/dR are held to (tests/fp64_bound.py measures against it).

A case is (model, B, gradient source, pose regime, beta regime, gradient scale).  CLASSES states, as predicates over
a case, everything the table has to cover; tests/test_smpl_grad_sweep_cpu.py fails with the names of the uncovered
classes and shows that the bound catches a set of wrong backward passes, and tests/test_smpl_grad_sweep_gpu.py runs
every case on the GPU, through SMPL.backward_lbs and through autograd.

The bound: each element of dbeta and dR against the fp64 reference r of oracle/lbs_grad.py,

    |got - r| <= C * 2^-24 * M + 2^-24 * |r| + 2^-149

with M the element's magnitude (oracle.lbs_grad.grads with absolute=True: the gradient of the layer with every
array, input and upstream gradient made non-negative and every subtraction made an addition).  Each rounded fp32
operation a term of the exact gradient passes through moves the result by at most 2^-24 of that term, so C is the
largest number of rounded operations on any term's path through the kernels (see C below); a path counts every
element of a serial sum it enters before.
"""
import collections

import numpy as np
import torch

from oracle import lbs as olbs
from oracle import lbs_grad
from danet_b200 import synthetic

# ----------------------------------------------------------------------------------------------------------------------
# C: the longest serial fp32 chains of danet_smpl_backward, in rounded operations, for 6890 vertices, 16 betas and a
# tree of depth 23 (the largest counts any model here reaches)
# ----------------------------------------------------------------------------------------------------------------------
NBETAS_MAX = 16
DEPTH_MAX = 23
N_J = 2 + NBETAS_MAX                  # rest joints: Jt and Jsd rounded to fp32 on the host, then nbetas FMAs
N_CHAIN_FWD = 4 * DEPTH_MAX           # world transforms: per level a 3-term row product and the parent's translation
N_A = 4                               # A_t = tg - Rg J: a 3-term product and a subtraction
N_SKIN = 24 + 3                       # T = sum_j w_j A_j (24 FMAs with dense weights), dv_posed = T^T g (3 terms)
N_BLEND = 646 + 5                     # k_lbs_bwd_blend: a lane's strided dot over 20670 / 32 coordinates, 5 shuffles
N_BETA = 72                           # dbeta += dJ . Jsd over the 72 joint coordinates
N_VPOSED = 1 + NBETAS_MAX + 207       # pf = R - I, then v_posed = template + nbetas + 207 FMAs
N_GV = 1                              # g[r] * [v_posed; 1][c]
N_TILE = 128                          # a tile's partial of dA, summed over its 128 vertices in order
N_TILES = 54                          # the tile partials summed in tile order (6890 vertices)
N_DRG = 2                             # dRg = dA - dA_t J^T
N_CHAIN_BWD = 6 * DEPTH_MAX           # per level dRg_p += dRg_i R_i^T + dtg_i rel^T and dRi = Rg_p^T dRg_i
N_DJ = 3 + 2 * DEPTH_MAX              # dJ_i = -Rg_i^T dA_t, then += / -= drel at each level
# a term of dbeta or dR passes either through the pose-feature / shape blend (dv_posed -> dpf, dbeta_shape) or
# through dA (v_posed -> dA -> the reverse chain); both paths can end in the dbeta update
PATH_BLEND = N_J + N_CHAIN_FWD + N_A + N_SKIN + N_BLEND + 1 + N_BETA
PATH_DA = (N_VPOSED + N_J + N_CHAIN_FWD + N_A + N_GV + N_TILE + N_TILES + N_DRG + N_CHAIN_BWD + N_DJ + N_BETA + 1)
C = max(PATH_BLEND, PATH_DA)

# ----------------------------------------------------------------------------------------------------------------------
# models
# ----------------------------------------------------------------------------------------------------------------------
MODEL_NAMES = ("packed", "dense", "nbetas1", "nbetas16", "nv100", "nv128", "nv129", "chain", "star", "translated")


def _with_betas(m, nb, seed):
    m = dict(m)
    m["shapedirs"] = np.random.default_rng(seed).normal(0, 0.01, (m["v_template"].shape[0], 3, nb)).astype(np.float32)
    return m


def _submesh(m, nv, seed):
    """nv vertices spread over the synthetic mesh, with the joint, extra and H36M regressors rebuilt on them and 21
    selected vertices below nv, so that JOINT_MAP_49 stays valid"""
    rng = np.random.default_rng(seed)
    idx = np.round(np.linspace(0, synthetic.NV - 1, nv)).astype(np.int64)
    vt = m["v_template"][idx].astype(np.float64)
    P = m["posedirs"].reshape(207, synthetic.NV, 3)[:, idx].reshape(207, nv * 3)
    J_rest = m["J_regressor"].astype(np.float64) @ m["v_template"].astype(np.float64)
    rows = lambda targets: synthetic._sparse_rows(rng, targets, vt, 8).astype(np.float32)
    extra = J_rest[rng.integers(0, 24, 9)] + rng.normal(0, 0.05, (9, 3))
    h36m = J_rest[rng.integers(0, 24, 17)] + rng.normal(0, 0.05, (17, 3))
    return {"v_template": m["v_template"][idx].copy(), "shapedirs": m["shapedirs"][idx].copy(),
            "posedirs": np.ascontiguousarray(P), "J_regressor": rows(J_rest),
            "lbs_weights": m["lbs_weights"][idx].copy(), "parents": m["parents"].copy(),
            "faces": np.zeros((1, 3), dtype=np.int64), "J_regressor_extra": rows(extra), "J_regressor_h36m": rows(h36m),
            "selected_verts": np.sort(rng.choice(nv, 21, replace=False)).astype(np.int32)}


def make_model(name):
    """the model dict of a sweep model (float32 arrays, what danet_b200.SMPL takes)"""
    base = synthetic.make_smpl_model(0)
    if name == "packed":
        return base
    if name == "dense":
        return synthetic.make_smpl_model(0, dense_weights=True)
    if name in ("nbetas1", "nbetas16"):
        return _with_betas(base, int(name[6:]), 11)
    if name.startswith("nv"):
        return _submesh(base, int(name[2:]), 12)
    if name == "chain":
        return dict(base, parents=np.array([-1] + list(range(23)), dtype=np.int32))
    if name == "star":
        return dict(base, parents=np.array([-1] + [0] * 23, dtype=np.int32))
    if name == "translated":          # 3 m from the origin: |J| >> |v - J|, so dRg = dA - dA_t J^T cancels
        return dict(base, v_template=(base["v_template"] + np.array([2.0, 2.0, 1.0], dtype=np.float32)).astype(np.float32))
    raise KeyError(name)


_MODELS = {}


def model(name):
    if name not in _MODELS:
        _MODELS[name] = make_model(name)
    return _MODELS[name]


def depth(parents):
    d = [0] * len(parents)
    for i in range(1, len(parents)):
        d[i] = d[parents[i]] + 1
    return max(d)


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
Case = collections.namedtuple("Case", ["model", "B", "src", "pose", "beta", "scale"])

SOURCES = ("verts", "smpl_joints", "both", "no_smpl_joints", "joints49", "transl", "last_tile_vertex")
POSES = ("identity", "rot6d", "near180", "noisy", "gaussian")
BETAS = ("zero", "normal", "pm5")
SCALES = (1.0, 1e-6, 1e4)
BATCHES = (1, 2, 31, 32, 33, 64, 65)
BIG_B = 520
BIG_BODIES = (0, 31, 32, 511, 512, 519)     # the bodies of the B = 520 case compared to the reference

CASES = [
    Case("packed", 1, "verts", "identity", "zero", 1.0),
    Case("packed", 2, "both", "rot6d", "normal", 1.0),
    Case("packed", 31, "smpl_joints", "near180", "normal", 1.0),
    Case("packed", 32, "both", "noisy", "pm5", 1.0),
    Case("packed", 33, "no_smpl_joints", "gaussian", "normal", 1.0),
    Case("packed", 64, "both", "rot6d", "normal", 1e-6),
    Case("packed", 65, "both", "noisy", "normal", 1e4),
    Case("packed", 2, "joints49", "rot6d", "normal", 1.0),
    Case("packed", 3, "transl", "noisy", "pm5", 1.0),
    Case("packed", 2, "last_tile_vertex", "rot6d", "normal", 1.0),
    Case("packed", BIG_B, "both", "rot6d", "normal", 1.0),
    Case("dense", 2, "both", "rot6d", "normal", 1.0),
    Case("dense", 33, "verts", "gaussian", "pm5", 1.0),
    Case("dense", 1, "last_tile_vertex", "noisy", "normal", 1e4),
    Case("nbetas1", 2, "both", "rot6d", "normal", 1.0),
    Case("nbetas1", 33, "joints49", "noisy", "pm5", 1.0),
    Case("nbetas16", 2, "both", "near180", "normal", 1.0),
    Case("nbetas16", 65, "both", "gaussian", "pm5", 1.0),
    Case("nv100", 2, "both", "rot6d", "normal", 1.0),
    Case("nv100", 1, "last_tile_vertex", "noisy", "pm5", 1.0),
    Case("nv128", 2, "both", "rot6d", "normal", 1.0),
    Case("nv128", 1, "last_tile_vertex", "rot6d", "normal", 1.0),
    Case("nv129", 2, "joints49", "noisy", "normal", 1.0),
    Case("nv129", 1, "last_tile_vertex", "rot6d", "normal", 1e-6),
    Case("chain", 2, "both", "rot6d", "normal", 1.0),
    Case("chain", 33, "both", "near180", "pm5", 1.0),
    Case("chain", 1, "joints49", "gaussian", "zero", 1.0),
    Case("star", 2, "both", "rot6d", "normal", 1.0),
    Case("star", 33, "smpl_joints", "gaussian", "normal", 1.0),
    Case("translated", 2, "both", "rot6d", "normal", 1.0),
    Case("translated", 33, "verts", "noisy", "normal", 1.0),
    Case("translated", 1, "last_tile_vertex", "near180", "pm5", 1.0),
]


def case_id(c):
    return "%s-B%d-%s-%s-%s-%g" % c


def bodies(case):
    """the bodies of a case compared to the reference"""
    return list(BIG_BODIES) if case.B >= 512 else list(range(case.B))


def _classes():
    """[(name, predicate(case))]"""
    cl = []
    for n in MODEL_NAMES:
        cl.append(("model " + n, lambda c, n=n: c.model == n))
    for B in BATCHES:
        cl.append(("B = %d" % B, lambda c, B=B: c.B == B))
    for s in SOURCES:
        cl.append(("gradient source " + s, lambda c, s=s: c.src == s))
    for p in POSES:
        cl.append(("pose " + p, lambda c, p=p: c.pose == p))
    for b in BETAS:
        cl.append(("betas " + b, lambda c, b=b: c.beta == b))
    for s in SCALES:
        cl.append(("gradient scale %g" % s, lambda c, s=s: c.scale == s))
    cl.append(("body index >= 32 in the chain kernel", lambda c: c.B > 32))
    cl.append(("B >= 512 autograd (tensor-core forward route)", lambda c: c.B >= 512))
    return cl


CLASSES = _classes()


# ----------------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------------
def _rotations(rng, n, pose):
    if pose == "identity":
        return np.broadcast_to(np.eye(3), (n, 3, 3)).copy()
    if pose == "gaussian":
        return rng.normal(0, 1, (n, 3, 3))
    if pose == "near180":
        ax = rng.normal(0, 1, (n, 3))
        ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        th = (np.pi - 1e-3 * rng.random(n))[:, None, None]
        K = np.zeros((n, 3, 3))
        K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -ax[:, 2], ax[:, 1], -ax[:, 0]
        K = K - K.transpose(0, 2, 1)
        return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)
    R = olbs.rot6d_to_rotmat(rng.normal(0, 1, (n, 6)))
    if pose == "noisy":
        R = R + 0.05 * rng.normal(0, 1, R.shape)
    return R


Inputs = collections.namedtuple("Inputs", ["betas", "R", "gv", "gs", "gj", "transl"])


def make_inputs(case, seed=0):
    """float32 CPU tensors: betas [B,nb], R [B,24,3,3], and the upstream gradients of the case's source (None where
    the source has none): gv [B,nv,3], gs [B,24,3], gj [B,49,3]; transl [B,3] or None"""
    m = model(case.model)
    nv, nb, B = m["v_template"].shape[0], m["shapedirs"].shape[-1], case.B
    rng = np.random.default_rng(1000 + seed + 7 * CASES.index(case) if case in CASES else seed)
    betas = {"zero": np.zeros((B, nb)), "normal": rng.normal(0, 1, (B, nb)),
             "pm5": 5.0 * rng.choice([-1.0, 1.0], (B, nb))}[case.beta]
    R = _rotations(rng, B * 24, case.pose).reshape(B, 24, 3, 3)
    g = lambda *shape: rng.normal(0, 1, shape) * case.scale
    gv = gs = gj = transl = None
    if case.src in ("verts", "both", "no_smpl_joints", "transl"):
        gv = g(B, nv, 3)
    if case.src in ("smpl_joints", "both", "transl"):
        gs = g(B, 24, 3)
    if case.src == "verts":
        gs = np.zeros((B, 24, 3))
    if case.src == "smpl_joints":
        gv = np.zeros((B, nv, 3))
    if case.src == "joints49":
        gj = g(B, 49, 3)
    if case.src == "transl":
        transl = rng.normal(0, 1, (B, 3))
    if case.src == "last_tile_vertex":      # one nonzero vertex, the mesh's last, in the last (partial) vertex tile
        gv = np.zeros((B, nv, 3))
        gv[:, nv - 1] = g(B, 3)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return Inputs(t(betas), t(R), t(gv), t(gs), t(gj), t(transl))


def fold(mdl, inp):
    """(grad_verts, grad_smpl_joints) that backward_lbs takes for a case's upstream gradients: the 49-joint gradient
    folded into the posed joints, the selected vertices and the extra regressor's vertices in fp64, rounded to fp32"""
    B = inp.betas.shape[0]
    nv = mdl["v_template"].shape[0]
    gv = torch.zeros(B, nv, 3, dtype=torch.float64) if inp.gv is None else inp.gv.double()
    gs = None if inp.gs is None else inp.gs.double()
    if inp.gj is not None:
        sel = torch.as_tensor(np.asarray(mdl["selected_verts"], dtype=np.int64))
        extra = torch.as_tensor(np.asarray(mdl["J_regressor_extra"], dtype=np.float64))
        gcat = torch.zeros(B, 24 + sel.numel() + extra.shape[0], 3, dtype=torch.float64)
        gcat.index_add_(1, torch.as_tensor(olbs.JOINT_MAP_49), inp.gj.double())
        gs = gcat[:, :24] if gs is None else gs + gcat[:, :24]
        gv = gv.index_add(1, sel, gcat[:, 24:24 + sel.numel()])
        gv = gv + torch.einsum("jv,bjc->bvc", extra, gcat[:, 24 + sel.numel():])
    return gv.float(), (None if gs is None else gs.float())


def subset(inp, idx):
    return Inputs(*[None if a is None else a[idx] for a in inp])


# ----------------------------------------------------------------------------------------------------------------------
# the reference
# ----------------------------------------------------------------------------------------------------------------------
def reference(mdl, inp, device="cpu", dtype=torch.float64):
    """(ref, M) for dbeta and dR: [(r_beta, M_beta), (r_R, M_R)] on the device, in dtype"""
    pm = lbs_grad.prepare(mdl, dtype, device)
    pa = lbs_grad.prepare(mdl, dtype, device, absolute=True)
    a = [None if x is None else x.to(device=device, dtype=dtype) for x in inp]
    args = dict(grad_verts=a[2], grad_smpl_joints=a[3], grad_joints=a[4], transl=a[5])
    r = lbs_grad.grads(pm, a[0], a[1], **args)
    M = lbs_grad.grads(pa, a[0], a[1], absolute=True, **args)
    assert all(bool(torch.isfinite(t).all()) for t in r), "the sweep's inputs give finite gradients"
    return list(zip(r, M))

