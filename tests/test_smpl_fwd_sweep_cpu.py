"""CPU half of the SMPL forward sweep (tests/smpl_fwd_sweep_common.py): the coverage of the case table, the constants,
and the bound's power to tell a right forward pass from a wrong one.  An fp64 restatement in the kernels' structure
(host-rounded rest-joint tables, the split-fp16 GEMM of the tensor-core route, per-tile regressor partials) meets the
bound; a float32 evaluation of oracle/lbs_grad.py meets a quarter of it; and each of a set of restatements with one
plausible kernel bug built in (mutants) exceeds it somewhere in the table."""
import functools

import numpy as np
import pytest
import torch

from oracle import lbs as olbs
from oracle import lbs_grad
import fp64_bound as fb
import smpl_fwd_sweep_common as sc


def test_every_class_is_covered():
    missing = fb.uncovered(sc.CASES, sc.CLASSES)
    assert not missing, "uncovered classes: %s" % missing


def test_constants_are_derived_from_the_kernel_chains():
    assert sc.C_VERTS == sc.N_J + sc.N_REL + sc.N_CHAIN + sc.N_A + sc.N_VPOSED + sc.N_SKIN + sc.N_TRANSL
    assert sc.C_REGRESSED == sc.C_VERTS + sc.N_PARTIAL + sc.N_TILESUM
    assert sc.C_SMPL_JOINTS < sc.C_VERTS < sc.C_REGRESSED
    for name in sc.MODEL_NAMES:
        m = sc.model(name)
        assert sc.gsc.depth(m["parents"]) <= sc.DEPTH_MAX and m["shapedirs"].shape[-1] <= sc.NBETAS_MAX
        assert sc.ntiles(m) <= sc.NTILES_MAX
    # the routes the table reaches: k_smpl_skin needs packed weights and a tile count that is a multiple of 3
    assert sc.skin_path(sc.Case("packed", 512, "r6d", "typical", "normal", 0, "h36m")) == "skin"
    for name in sc.FALLBACK_MODELS:
        assert sc.skin_path(sc.Case(name, 512, "r6d", "typical", "normal", 0, "h36m")) == "fallback"


def test_rodrigues_magnitude_bounds_an_fp32_evaluation():
    """rodrigues_smplx's expression order in fp32 numpy meets C_AA against fp64 at every regime of the table"""
    rng = np.random.default_rng(0)
    aa = np.concatenate([sc._axis_angle(rng, 2000, p) for p in ("zero", "near", "typical", "large")])
    aa32 = aa.astype(np.float32)
    a = aa32.astype(np.float64)
    R = olbs.batch_rodrigues_smplx(a)
    v = aa32 + np.float32(1e-8)
    ang = np.sqrt(v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2])
    x, y, z = (aa32 / ang[:, None]).T
    s, c1 = np.sin(ang), np.float32(1) - np.cos(ang)
    one = np.float32(1)
    got = np.stack([one + c1 * (-(z * z) - y * y), s * (-z) + c1 * (x * y), s * y + c1 * (x * z),
                    s * z + c1 * (x * y), one + c1 * (-(z * z) - x * x), s * (-x) + c1 * (y * z),
                    s * (-y) + c1 * (x * z), s * x + c1 * (y * z), one + c1 * (-(y * y) - x * x)], 1).reshape(-1, 3, 3)
    M = sc.rodrigues_magnitude(a)
    excess = np.abs(got - R) - fb.U24 * np.abs(R)
    q = np.where(excess <= 0, -np.inf, excess / np.maximum(fb.U24 * M, 1e-300))
    print("fp32 rodrigues: worst ratio %.3g (C_AA = %d)" % (q.max(), sc.C_AA))
    assert q.max() <= sc.C_AA / 2


# ----------------------------------------------------------------------------------------------------------------------
# the kernels' structure in fp64, with optional defects
# ----------------------------------------------------------------------------------------------------------------------
MUTANTS = ("gemm_hi_features", "gemm_drop_weight_lo_mma", "rest_joints_float_sum", "pose_feature_R_not_R_minus_I",
           "regressor_partial_twice", "swapped_skinning_weights")


def _split(v):
    """split-fp16 planes (hi, lo) of float32 values, as k_smpl_pose and the weight packing write them"""
    v = np.asarray(v, dtype=np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


@functools.lru_cache(maxsize=None)
def _gemm_weights(name):
    """the packed GEMM weights [224, 3 nv] as split planes of W 2^s, and s"""
    m = sc.model(name)
    nv, nb = m["v_template"].shape[0], m["shapedirs"].shape[-1]
    W = np.zeros((224, nv * 3), dtype=np.float32)
    W[:207] = m["posedirs"]
    W[208:208 + nb] = m["shapedirs"].reshape(nv * 3, nb).T
    s = sc.weight_exponent(m)
    hi, lo = _split(W * np.float32(2.0 ** s))
    return hi, lo, s


def _rest_joint_tables(m, float_sum):
    """Jt [24,3], Jsd [24,3,nb] as danet_smpl_create builds them: double sums rounded to float32 (or, as a defect, a
    float32 sum in vertex order)"""
    Jr, vt, S = (np.asarray(m[k], dtype=np.float64) for k in ("J_regressor", "v_template", "shapedirs"))
    if not float_sum:
        return (Jr @ vt).astype(np.float32), np.einsum("jv,vkl->jkl", Jr, S).astype(np.float32)
    J32 = Jr.astype(np.float32)
    Jt = np.cumsum(J32[:, :, None] * vt.astype(np.float32)[None], axis=1, dtype=np.float32)[:, -1]
    Jsd = np.cumsum(J32[:, :, None, None] * S.astype(np.float32)[None], axis=1, dtype=np.float32)[:, -1]
    return Jt, Jsd


def _swap_vertex(W):
    """a vertex whose two largest skinning weights differ most"""
    top = -np.sort(-W, axis=1)[:, :2]
    return int(np.argmax(top[:, 0] - top[:, 1] - 1e9 * (top[:, 1] == 0)))


def manual_forward(case, m, inp, mutant=None):
    """{output: fp64 tensor} of the forward as the kernels compute it, in fp64"""
    R, _, _ = sc.rotations(case.front, inp.pose)
    betas = inp.betas.double().numpy()
    B, nv = betas.shape[0], m["v_template"].shape[0]
    vt, S, P, W = (np.asarray(m[k], dtype=np.float64) for k in ("v_template", "shapedirs", "posedirs", "lbs_weights"))
    parents = np.asarray(m["parents"])
    Jt, Jsd = _rest_joint_tables(m, mutant == "rest_joints_float_sum")
    J = Jt.astype(np.float64)[None] + np.einsum("jkl,bl->bjk", Jsd.astype(np.float64), betas)
    Rg, tg = [R[:, 0]], [J[:, 0]]
    for i in range(1, 24):
        p = parents[i]
        Rg.append(Rg[p] @ R[:, i])
        tg.append(np.einsum("brc,bc->br", Rg[p], J[:, i] - J[:, p]) + tg[p])
    Rg, tg = np.stack(Rg, 1), np.stack(tg, 1)
    A = np.concatenate([Rg, (tg - np.einsum("bjrc,bjc->bjr", Rg, J))[..., None]], -1)
    pf = (R[:, 1:] - np.eye(3)).reshape(B, 207)
    if mutant == "pose_feature_R_not_R_minus_I":
        pf[:, 36:45] = R[:, 5].reshape(B, 9)
    if sc.route(case) == "fused":
        vp = vt.reshape(1, -1) + betas @ S.reshape(nv * 3, -1).T + pf @ P
    else:
        feat = np.zeros((B, 224), dtype=np.float32)
        feat[:, :207] = pf
        feat[:, 208:208 + betas.shape[1]] = betas
        fh, fl = _split(feat)
        wh, wl, s = _gemm_weights(case.model)
        if mutant == "gemm_hi_features":
            fl = np.zeros_like(fl)
        prod = fh @ wh + fl @ wh + (0 if mutant == "gemm_drop_weight_lo_mma" else fh @ wl)
        vp = vt.reshape(1, -1) + prod * 2.0 ** -s
    vp = vp.reshape(B, nv, 3)
    if mutant == "swapped_skinning_weights":
        W = W.copy()
        v = _swap_vertex(W)
        a, b = np.argsort(-W[v])[:2]
        W[v, a], W[v, b] = W[v, b], W[v, a]
    T = np.einsum("vj,bjrc->bvrc", W, A)
    verts = np.einsum("bvrc,bvc->bvr", T[..., :3], vp) + T[..., 3]
    nt = sc.ntiles(m)
    vpad = np.zeros((B, nt * 128, 3))
    vpad[:, :nv] = verts

    def regress(rows):
        rp = np.zeros((rows.shape[0], nt * 128))
        rp[:, :nv] = rows
        part = np.einsum("jtv,btvk->bjtk", rp.reshape(-1, nt, 128), vpad.reshape(B, nt, 128, 3))
        out = part.sum(2)
        if mutant == "regressor_partial_twice":
            t = int(np.nonzero(np.abs(rp[0]).reshape(nt, 128).sum(1))[0][0])
            out[:, 0] += part[:, 0, t]
        return out
    extra = regress(np.asarray(m["J_regressor_extra"], dtype=np.float64))
    joints = np.concatenate([tg, verts[:, np.asarray(m["selected_verts"])], extra], 1)[:, olbs.JOINT_MAP_49]
    out = {"verts": verts, "smpl_joints": tg, "joints": joints, "joints_J19": joints[:, -24:][:, olbs.J24_TO_J19]}
    if case.out != "no_h36m":
        out["joints_h36m"] = regress(np.asarray(m["J_regressor_h36m"], dtype=np.float64))
    if inp.transl is not None:
        t = inp.transl.double().numpy()[:, None]
        out = {k: v + t for k, v in out.items()}
    if case.front != "rotmat":
        out["rotmats"] = R
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in out.items()}


@functools.lru_cache(maxsize=None)
def _case_data(i):
    """(model, inputs on the compared bodies, reference) of CASES[i]"""
    c = sc.CASES[i]
    m = sc.model(c.model)
    inp = sc.subset(sc.make_inputs(c), sc.bodies(c))
    return m, inp, sc.reference(c, m, inp, with_h36m=c.out != "no_h36m")


def _worst(got, ref):
    """the worst q / C over the outputs (<= 1 passes), and the output"""
    qs = {k: fb.worst(got[k], r, fb.U24 * M, fb.U24 * r.abs() + fb.TINY + slack)[0] / C for k, (r, M, slack, C) in ref.items()}
    k = max(qs, key=qs.get)
    return qs[k], k


def test_manual_forward_meets_the_bound():
    worst = {}
    for i, c in enumerate(sc.CASES):
        m, inp, ref = _case_data(i)
        q, k = _worst(manual_forward(c, m, inp), ref)
        worst[sc.route(c)] = max(worst.get(sc.route(c), -np.inf), q)
        assert q <= 1.0, (sc.case_id(c), k, q)
    print("fp64 restatement: worst error / bound per route %s" % worst)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_bound_catches_mutant(mutant):
    worst, where = -np.inf, None
    for i, c in enumerate(sc.CASES):
        m, inp, ref = _case_data(i)
        q, k = _worst(manual_forward(c, m, inp, mutant=mutant), ref)
        if q > worst:
            worst, where = q, "%s %s" % (sc.case_id(c), k)
    print("mutant %s: worst error / bound %.3g at %s" % (mutant, worst, where))
    assert worst > 1.0, (mutant, worst)


def _float32_forward(case, m, inp):
    """oracle/lbs_grad.py in float32, with oracle/lbs.py's front-ends in float32"""
    p = inp.pose.numpy()
    B = p.shape[0]
    if case.front == "rotmat":
        R = p
    elif case.front == "aa":
        R = olbs.batch_rodrigues_smplx(p.reshape(-1, 3)).reshape(B, 24, 3, 3)
    else:
        R = olbs.rot6d_to_rotmat(p.reshape(-1, 6)).reshape(B, 24, 3, 3)
    R = torch.from_numpy(np.ascontiguousarray(R, dtype=np.float32))
    pm = lbs_grad.prepare(m, torch.float32)
    v, sj, j = lbs_grad.smpl_layer(pm, inp.betas, R, inp.transl)
    h36m = None if case.out == "no_h36m" else torch.from_numpy(np.asarray(m["J_regressor_h36m"], dtype=np.float32))
    out = sc._outputs(m, v, sj, j, inp.transl, h36m)
    if case.front != "rotmat":
        out["rotmats"] = R
    return out


def test_float32_restatement_meets_a_quarter_of_the_bound():
    """the bound is not tighter than fp32 arithmetic allows"""
    worst = 0.0
    for i, c in enumerate(sc.CASES):
        if c.model == "jtail":          # its rest joints are the float32 sum the model is built to expose
            continue
        m, inp, _ = _case_data(i)
        ref = sc.reference(c, m, inp, with_h36m=c.out != "no_h36m", gemm=False)
        q, k = _worst(_float32_forward(c, m, inp), ref)
        worst = max(worst, q)
        assert q <= 0.25, (sc.case_id(c), k, q)
    print("float32 restatement: worst error / bound %.3g (<= 1/4)" % worst)
