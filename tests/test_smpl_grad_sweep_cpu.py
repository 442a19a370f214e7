"""CPU half of the SMPL backward sweep (tests/smpl_grad_sweep_common.py): the fp64 restatement of oracle/lbs_grad.py
against oracle/lbs.py, the coverage of the case table, and the bound's power to tell a right backward pass from a
wrong one.  The bound must fail each of a set of fp64 backward passes with one plausible kernel bug built in
(mutants), and must hold for a float32 evaluation of the restatement with a quarter of its constant."""
import functools

import numpy as np
import pytest
import torch

from oracle import lbs as olbs
from oracle import lbs_grad
import fp64_bound as fb
import smpl_grad_sweep_common as sc


def test_every_class_is_covered():
    missing = fb.uncovered(sc.CASES, sc.CLASSES)
    assert not missing, "uncovered classes: %s" % missing


def test_constant_is_derived_from_the_kernel_chains():
    assert sc.C == max(sc.PATH_BLEND, sc.PATH_DA)
    assert sc.N_BLEND == -(-20670 // 32) + 5 and sc.N_TILES == -(-6890 // 128)
    for name in sc.MODEL_NAMES:
        m = sc.model(name)
        assert sc.depth(m["parents"]) <= sc.DEPTH_MAX and m["shapedirs"].shape[-1] <= sc.NBETAS_MAX
        assert m["v_template"].shape[0] <= 6890


@pytest.mark.parametrize("name", sc.MODEL_NAMES)
def test_restatement_forward_matches_oracle(name):
    m = sc.model(name)
    c = sc.Case(name, 2, "both", "noisy", "normal", 1.0)
    inp = sc.make_inputs(c, seed=1)
    be, R = inp.betas.double().numpy(), inp.R.double().numpy()
    want = olbs.smpl_forward(m, be, R[:, 1:], R[:, :1], pose2rot=False, dtype=np.float64)
    v, sj, j = lbs_grad.smpl_layer(lbs_grad.prepare(m), inp.betas.double(), inp.R.double())
    for got, key in ((v, "vertices"), (sj, "smpl_joints"), (j, "joints")):
        w = want[key]
        assert got.shape == w.shape
        assert np.abs(got.numpy() - w).max() <= 1e-12 * np.abs(w).max(), key


@pytest.mark.parametrize("name", sc.MODEL_NAMES)
def test_restatement_gradient_matches_finite_differences(name):
    m = sc.model(name)
    c = sc.Case(name, 2, "both", "noisy", "normal", 1.0)
    inp = sc.make_inputs(c, seed=2)
    gj = torch.from_numpy(np.random.default_rng(3).normal(0, 1, (2, 49, 3)))
    gv, gs = inp.gv.double(), inp.gs.double()
    be, R = inp.betas.double(), inp.R.double()
    db, dR = lbs_grad.grads(lbs_grad.prepare(m), be, R, grad_verts=gv, grad_smpl_joints=gs, grad_joints=gj)

    def loss(b, r):
        o = olbs.smpl_forward(m, b, r[:, 1:], r[:, :1], pose2rot=False, dtype=np.float64)
        return (float((o["vertices"] * gv.numpy()).sum() + (o["smpl_joints"] * gs.numpy()).sum()
                      + (o["joints"] * gj.numpy()).sum()))
    rng = np.random.default_rng(4)
    nb = be.shape[1]
    picks = [("b", int(i), int(rng.integers(nb))) for i in range(2) for _ in range(4)]
    picks += [("R", int(rng.integers(2)), int(rng.integers(216))) for _ in range(24)]
    eps = 1e-6
    worst = 0.0
    scale = max(float(db.abs().max()), float(dR.abs().max()))
    for kind, i, k in picks:
        b0, r0 = be.numpy().copy(), R.numpy().copy()
        tgt = b0 if kind == "b" else r0.reshape(2, -1)
        tgt[i, k] += eps
        lp = loss(b0, r0)
        tgt[i, k] -= 2 * eps
        lm = loss(b0, r0)
        fd = (lp - lm) / (2 * eps)
        ad = float(db[i, k]) if kind == "b" else float(dR.reshape(2, -1)[i, k])
        worst = max(worst, abs(fd - ad) / scale)
    assert worst < 1e-6, worst


# ----------------------------------------------------------------------------------------------------------------------
# the bound discriminates: fp64 backward passes in the kernels' structure, each with one defect
# ----------------------------------------------------------------------------------------------------------------------
MUTANTS = ("drop_last_tile", "drop_pose_feature", "R_not_transposed", "drop_influence", "drop_Jsd", "neighbour_body",
           "drop_translation_column", "ignore_grad_smpl_joints", "vposed_fp16")


def _drop_fourth_influence(W):
    """the skinning weights without each vertex's 4th influence in joint order (the packed form's 4th slot)"""
    W = W.clone()
    nz = (W != 0).cumsum(1)
    W[(nz == 4) & (W != 0)] = 0
    return W


def manual_backward(mdl, betas, R, gv, gs, mutant=None):
    """dbeta, dR as danet_smpl_backward computes them (recompute, per-vertex dv_posed and dA over vertex tiles, the
    blend rows, the reverse chain), in fp64, with an optional defect"""
    pm = lbs_grad.prepare(mdl)
    vt, S, P, Jr, W = pm["v_template"], pm["shapedirs"], pm["posedirs"], pm["J_regressor"], pm["lbs_weights"]
    parents = pm["parents"]
    B, nv = betas.shape[0], vt.shape[0]
    Jt, Jsd = Jr @ vt, torch.einsum("jv,vkl->jkl", Jr, S)
    J = Jt + torch.einsum("jkl,bl->bjk", Jsd, betas)
    pf = (R[:, 1:] - torch.eye(3, dtype=R.dtype)).reshape(B, 207)
    vp = vt + torch.einsum("bl,vkl->bvk", betas, S) + (pf @ P).reshape(B, nv, 3)
    if mutant == "vposed_fp16":
        vp = vp.half().double()
    Rg, tg = [R[:, 0]], [J[:, 0]]
    for i in range(1, 24):
        p = parents[i]
        Rg.append(Rg[p] @ R[:, i])
        tg.append(torch.einsum("brc,bc->br", Rg[p], J[:, i] - J[:, p]) + tg[p])
    Rg, tg = torch.stack(Rg, 1), torch.stack(tg, 1)
    A = torch.cat([Rg, (tg - torch.einsum("bjrc,bjc->bjr", Rg, J))[..., None]], -1)
    if mutant == "drop_influence":
        W = _drop_fourth_influence(W)
    T = torch.einsum("vj,bjrc->bvrc", W, A)[..., :3]
    dvp = torch.einsum("bvrc,bvr->bvc", T, gv)
    vh = torch.cat([vp, torch.ones(B, nv, 1, dtype=vp.dtype)], -1)
    keep = torch.ones(nv, dtype=vp.dtype)
    if mutant == "drop_last_tile":
        keep[(nv - 1) // 128 * 128:] = 0
    dA = torch.einsum("vj,bvr,bvc,v->bjrc", W, gv, vh, keep)
    if mutant == "drop_translation_column":
        dA[..., 3] = 0
    dpf = dvp.reshape(B, -1) @ P.T
    dbeta = torch.einsum("bvk,vkl->bl", dvp, S)
    dRg = dA[..., :3] - dA[..., 3:] * J[:, :, None, :]
    dtg = dA[..., 3].clone()
    if gs is not None and mutant != "ignore_grad_smpl_joints":
        dtg = dtg + gs
    dJ = -torch.einsum("bjrc,bjr->bjc", Rg, dA[..., 3])
    out = torch.zeros(B, 24, 3, 3, dtype=R.dtype)
    for i in range(23, 0, -1):
        p = parents[i]
        rel = J[:, i] - J[:, p]
        dRi = Rg[:, p].transpose(1, 2) @ dRg[:, i]
        drel = torch.einsum("brc,br->bc", Rg[:, p], dtg[:, i])
        Ri = R[:, i] if mutant == "R_not_transposed" else R[:, i].transpose(1, 2)
        dRg[:, p] += dRg[:, i] @ Ri + dtg[:, i, :, None] * rel[:, None, :]
        dtg[:, p] += dtg[:, i]
        dJ[:, i] += drel
        dJ[:, p] -= drel
        out[:, i] = dRi + (0 if mutant == "drop_pose_feature" else dpf[:, (i - 1) * 9:i * 9].reshape(B, 3, 3))
    out[:, 0] = dRg[:, 0]
    dJ[:, 0] += dtg[:, 0]
    if mutant != "drop_Jsd":
        dbeta = dbeta + torch.einsum("bjk,jkl->bl", dJ, Jsd)
    if mutant == "neighbour_body" and B > 1:
        out[-1], dbeta[-1] = out[-2].clone(), dbeta[-2].clone()
    return dbeta, out


@functools.lru_cache(maxsize=None)
def _case_data(i):
    """(fp64 inputs as backward_lbs takes them, reference pairs) of CASES[i], on the bodies compared"""
    c = sc.CASES[i]
    m = sc.model(c.model)
    inp = sc.subset(sc.make_inputs(c), sc.bodies(c))
    gv, gs = sc.fold(m, inp)
    return m, inp, gv.double(), (None if gs is None else gs.double()), sc.reference(m, inp)


def _worst(got, ref):
    return max(fb.worst(g, r, fb.U24 * M, fb.U24 * r.abs() + fb.TINY)[0] for g, (r, M) in zip(got, ref))


def test_manual_backward_matches_the_reference():
    """the unmutated fp64 backward of the kernels' structure is the reference's gradient (so the mutants below differ
    from it by their defect alone)"""
    for i, c in enumerate(sc.CASES):
        m, inp, gv, gs, ref = _case_data(i)
        got = manual_backward(m, inp.betas.double(), inp.R.double(), gv, gs)
        assert _worst(got, ref) <= 1.0, sc.case_id(c)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_bound_catches_mutant(mutant):
    worst, where = -np.inf, None
    for i, c in enumerate(sc.CASES):
        m, inp, gv, gs, ref = _case_data(i)
        q = _worst(manual_backward(m, inp.betas.double(), inp.R.double(), gv, gs, mutant=mutant), ref)
        if q > worst:
            worst, where = q, sc.case_id(c)
    print("mutant %s: worst ratio %.3g (C = %d) at %s" % (mutant, worst, sc.C, where))
    assert worst > sc.C, (mutant, worst)


def test_float32_restatement_meets_a_quarter_of_the_bound():
    """fp32 CPU autograd of the same restatement: the bound is not tighter than fp32 arithmetic allows"""
    worst = 0.0
    for i, c in enumerate(sc.CASES):
        m, inp, _, _, ref = _case_data(i)
        got = lbs_grad.grads(lbs_grad.prepare(m, torch.float32), inp.betas, inp.R, grad_verts=inp.gv,
                             grad_smpl_joints=inp.gs, grad_joints=inp.gj, transl=inp.transl)
        q = _worst(got, ref)
        worst = max(worst, q)
        assert q <= sc.C / 4, (sc.case_id(c), q)
    print("float32 restatement: worst ratio %.3g, C / 4 = %.1f" % (worst, sc.C / 4))
