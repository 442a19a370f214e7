"""CPU restatement (numpy, fp64) of the decomposed regressor's head in training and eval mode, forward AND backward --
TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/ alone; the product path never touches it).

Follows models/danet/smpl_regressor.py:844-895 (the 'gcn' branch of DecomposedPredictor.forward), GCN.py:29-92,
utils/graph.py:232-261 (normalize_undigraph), utils/geometry.py rot6d_to_rotmat and the head losses of
smpl_regressor.py:144-166,233-238.  Pinned by tests/golden/gcn_head.npz, which oracle/gen_golden_gcn_head.py produces
with the reference's own modules under torch autograd (tests/test_gcn_head_cpu.py).

`torch_head` restates the same forward in torch (any dtype / device) for autograd: tools/gcn_head_bench.py times it
as the eager baseline on the GPU."""
import numpy as np

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
BUFFER_NAMES = ["r2p_A", "p2r_A", "A_mask", "I_n", "mean_pose"]
BN_EPS, BN_MOMENTUM = 1e-5, 0.1
SMPL_POSE_WEIGHTS, JOINT_POSITION_WEIGHTS = 60.0, 1.0          # configs/danet_default.yaml:25,33


def refine_adjacency(E, A_mask, I_n):
    """normalize_undigraph(I_n + A_mask * relu(E)) with column-sum degrees; returns (A_hat, M, d)."""
    M = I_n + A_mask * np.maximum(E, 0.0)
    s = M.sum(0)
    d = np.where(s > 0, np.abs(s) ** -0.5, 0.0)
    return d[:, None] * M * d[None, :], M, d


def _rot6d(x):
    """x [..., 6] -> R [..., 9] (geometry.py rot6d_to_rotmat: a1 = x[0::2], a2 = x[1::2]) and the saved state."""
    a1, a2 = x[..., 0::2], x[..., 1::2]
    n1 = np.maximum(np.linalg.norm(a1, axis=-1, keepdims=True), 1e-12)
    b1 = a1 / n1
    dd = (b1 * a2).sum(-1, keepdims=True)
    u = a2 - dd * b1
    n2 = np.maximum(np.linalg.norm(u, axis=-1, keepdims=True), 1e-12)
    b2 = u / n2
    b3 = np.cross(b1, b2)
    R = np.stack([b1, b2, b3], -1).reshape(x.shape[:-1] + (9,))
    return R, (a1, a2, n1, b1, dd, u, n2, b2)


def _normalize_bwd(v, n, b, g):
    """F.normalize(v) = v / max(|v|, 1e-12): d/dv of <g, b>."""
    big = np.linalg.norm(v, axis=-1, keepdims=True) > 1e-12
    return np.where(big, (g - b * (b * g).sum(-1, keepdims=True)) / n, g / n)


def _rot6d_bwd(st, gR):
    a1, a2, n1, b1, dd, u, n2, b2 = st
    gR = gR.reshape(gR.shape[:-1] + (3, 3))
    g1, g2, g3 = gR[..., 0], gR[..., 1], gR[..., 2]
    gb1 = g1 + np.cross(b2, g3)
    gb2 = g2 + np.cross(g3, b1)
    gu = _normalize_bwd(u, n2, b2, gb2)
    ga2 = gu - b1 * (gu * b1).sum(-1, keepdims=True)
    gb1 = gb1 - a2 * (gu * b1).sum(-1, keepdims=True) - dd * gu
    ga1 = _normalize_bwd(a1, n1, b1, gb1)
    out = np.empty(a1.shape[:-1] + (6,))
    out[..., 0::2], out[..., 1::2] = ga1, ga2
    return out


def _group_head(W, b, X, K):
    """grouped 1x1 conv, 24 groups of 128 -> K: W [24*K,128,1,1], X [B,24,128] -> [B,24,K]."""
    return np.einsum("jkf,bjf->bjk", W.reshape(24, K, -1), X) + b.reshape(24, K)


def forward(P, buf, bn, rot_feats, global_para, training=True):
    """P: the 29 parameters (PARAM_NAMES), buf: BUFFER_NAMES, bn: {BN_NAME: (running_mean, running_var)}.
    Returns (out, saved): out = para [B,229], pose0 [B,216], coord0 / coord1 [B,24,3] (training only) and the running
    statistics after the step (training only)."""
    f = lambda x: np.asarray(x, np.float64)
    X = f(rot_feats)
    B = X.shape[0]
    Ahat, M, d = refine_adjacency(f(P["edge_importance"])[0], f(buf["A_mask"])[0], f(buf["I_n"])[0])
    adjs = [f(buf["r2p_A"])[0], Ahat, Ahat, Ahat, f(buf["p2r_A"])[0]]
    sv = dict(X0=X, Ahat=Ahat, M=M, d=d, adjs=adjs, A_mask=f(buf["A_mask"])[0], layers=[])
    out = {}
    new_bn = {}
    mean_pose = f(buf["mean_pose"]).reshape(24, 6)
    if training:
        p6 = _group_head(f(P["pose_regressors.0.1.weight"]), f(P["pose_regressors.0.1.bias"]), X, 6) + mean_pose
        R0, sv["rot0"] = _rot6d(p6)
        out["pose0"] = R0.reshape(B, 216)
    h = X
    for l, (name, i) in enumerate(LAYERS):
        pre = "%s.gc.%d." % (name, i)
        bnk = BN_NAMES[l]
        AX = np.einsum("nk,bkf->bnf", adjs[l], h)
        Y = AX @ f(P[pre + "weight"]) + f(P[pre + "bias"])
        rm, rv = (f(t) for t in bn[bnk])
        if training:
            mean = Y.mean(axis=(0, 2))
            var = Y.var(axis=(0, 2))
            N = B * Y.shape[2]
            new_bn[bnk] = ((1 - BN_MOMENTUM) * rm + BN_MOMENTUM * mean,
                           (1 - BN_MOMENTUM) * rv + BN_MOMENTUM * var * N / (N - 1))
        else:
            mean, var = rm, rv
        invstd = 1.0 / np.sqrt(var + BN_EPS)
        xh = (Y - mean[None, :, None]) * invstd[None, :, None]
        Z = xh * f(P[bnk + ".weight"])[None, :, None] + f(P[bnk + ".bias"])[None, :, None]
        H = np.maximum(Z, 0.0)
        if l == 3:
            H = H + sv["layers"][0]["H"]                          # l_pos_feat = pos_feats_init + refine (:873)
        sv["layers"].append(dict(X=h, AX=AX, xh=xh, Z=Z, H=H, invstd=invstd))
        if training and l in (0, 3):
            k = 0 if l == 0 else 1
            out["coord%d" % k] = _group_head(f(P["coord_regressors.%d.1.weight" % k]),
                                             f(P["coord_regressors.%d.1.bias" % k]), H, 3)
        h = H
    p6 = _group_head(f(P["pose_regressors.1.1.weight"]), f(P["pose_regressors.1.1.bias"]), h, 6) + mean_pose
    R1, sv["rot1"] = _rot6d(p6)
    out["para"] = np.concatenate([f(global_para), R1.reshape(B, 216)], 1)
    out["bn"] = new_bn
    return out, sv


def _head_bwd(W, X, g, K):
    """grouped head backward: (dW [24*K,128,1,1], db [24*K], dX [B,24,128])."""
    Wr = W.reshape(24, K, -1)
    dW = np.einsum("bjk,bjf->jkf", g, X).reshape(W.shape)
    return dW, g.sum(0).reshape(-1), np.einsum("jkf,bjk->bjf", Wr, g)


def backward(P, sv, grads, training=True):
    """grads: 'para' [B,229] and, in training mode, 'pose0' [B,216], 'coord0' / 'coord1' [B,24,3].
    Returns {name: gradient} over PARAM_NAMES plus 'rot_feats' and 'global_para'."""
    f = lambda x: np.asarray(x, np.float64)
    gp = f(grads["para"])
    B = gp.shape[0]
    G = {"global_para": gp[:, :13].copy()}
    L = sv["layers"]
    g6 = _rot6d_bwd(sv["rot1"], gp[:, 13:].reshape(B, 24, 9))
    G["pose_regressors.1.1.weight"], G["pose_regressors.1.1.bias"], dH = _head_bwd(f(P["pose_regressors.1.1.weight"]),
                                                                                   L[4]["H"], g6, 6)
    dH0_extra = np.zeros_like(L[0]["H"])
    dAhat = np.zeros((24, 24))
    for l in range(4, -1, -1):
        name, i = LAYERS[l]
        pre, bnk = "%s.gc.%d." % (name, i), BN_NAMES[l]
        s = L[l]
        if training and l in (0, 3):
            k = 0 if l == 0 else 1
            gc = f(grads["coord%d" % k])
            G["coord_regressors.%d.1.weight" % k], G["coord_regressors.%d.1.bias" % k], dx = _head_bwd(
                f(P["coord_regressors.%d.1.weight" % k]), s["H"], gc, 3)
            dH = dH + dx
        if l == 3:
            dH0_extra = dH0_extra + dH                            # the residual's branch
        if l == 0:
            dH = dH + dH0_extra
        dZ = dH * (s["Z"] > 0)
        gamma = f(P[bnk + ".weight"])
        G[bnk + ".weight"] = (dZ * s["xh"]).sum(axis=(0, 2))
        G[bnk + ".bias"] = dZ.sum(axis=(0, 2))
        dxh = dZ * gamma[None, :, None]
        if training:
            N = B * dZ.shape[2]
            dY = s["invstd"][None, :, None] / N * (N * dxh - dxh.sum(axis=(0, 2))[None, :, None]
                                                   - s["xh"] * (dxh * s["xh"]).sum(axis=(0, 2))[None, :, None])
        else:
            dY = dxh * s["invstd"][None, :, None]
        W = f(P[pre + "weight"])
        G[pre + "weight"] = np.einsum("bni,bno->io", s["AX"], dY)
        G[pre + "bias"] = dY.sum(axis=(0, 1))
        dAX = dY @ W.T
        if 1 <= l <= 3:
            dAhat += np.einsum("bnf,bkf->nk", dAX, s["X"])
        dH = np.einsum("nk,bnf->bkf", sv["adjs"][l], dAX)
    G["rot_feats"] = dH
    # d A_hat -> d edge_importance (A_hat[i,j] = d_i M[i,j] d_j, d_j = (sum_i M[i,j])^-1/2)
    M, d = sv["M"], sv["d"]
    gd = (dAhat * M * d[None, :]).sum(1) + (dAhat * M * d[:, None]).sum(0)
    gs = np.where(d > 0, -0.5 * d ** 3 * gd, 0.0)
    dM = dAhat * d[:, None] * d[None, :] + gs[None, :]
    E = f(P["edge_importance"])
    G["edge_importance"] = (dM * sv["A_mask"] * (E[0] > 0))[None]
    if training:
        g6 = _rot6d_bwd(sv["rot0"], f(grads["pose0"]).reshape(B, 24, 9))
        G["pose_regressors.0.1.weight"], G["pose_regressors.0.1.bias"], dx = _head_bwd(
            f(P["pose_regressors.0.1.weight"]), sv["X0"], g6, 6)
        G["rot_feats"] = G["rot_feats"] + dx
    return G


def run(P, buf, bn, rot_feats, global_para, grads, training=True):
    out, sv = forward(P, buf, bn, rot_feats, global_para, training)
    return out, backward(P, sv, grads, training)


def losses(pose0, coord0, coord1, target, gt_joints, has, rot_w=SMPL_POSE_WEIGHTS, pos_w=JOINT_POSITION_WEIGHTS):
    """joint_rotation0 = rot_w * MSE over the selected images; joint_position{0,1} = pos_w * L1 sum / #selected
    (smpl_regressor.py:147-166,233-238).  Selected = has == 1; with none selected, zero losses and gradients.
    Returns (losses [3], (d/dpose0, d/dcoord0, d/dcoord1) of their sum)."""
    f = lambda x: np.asarray(x, np.float64)
    sel = (np.asarray(has, np.float64) == 1).astype(np.float64)
    n = sel.sum()
    if n == 0:
        z = np.zeros
        return np.zeros(3), (z(np.shape(pose0)), z(np.shape(coord0)), z(np.shape(coord1)))
    dr = (f(pose0) - f(target)[:, 13:]) * sel[:, None]
    L = [rot_w * (dr ** 2).sum() / (n * 216)]
    G = [rot_w * 2 * dr / (n * 216)]
    for c in (coord0, coord1):
        dc = (f(c) - f(gt_joints)) * sel[:, None, None]
        L.append(pos_w * np.abs(dc).sum() / n)
        G.append(pos_w * np.sign(dc) / n)
    return np.array(L), tuple(G)


def torch_head(P, buf, bn, rot_feats, global_para, training=True):
    """The same forward in torch for autograd (P / buf: tensors; bn: {name: (running_mean, running_var)} updated in
    place in training mode).  Returns (para, pose0, coord0, coord1); the last three are None in eval mode."""
    import torch
    import torch.nn.functional as F

    def rot6d(x):
        x = x.reshape(-1, 3, 2)
        b1 = F.normalize(x[:, :, 0], dim=1)
        a2 = x[:, :, 1]
        b2 = F.normalize(a2 - torch.einsum("bi,bi->b", b1, a2).unsqueeze(-1) * b1, dim=1)
        return torch.stack((b1, b2, torch.cross(b1, b2, dim=1)), dim=-1).reshape(rot_feats.shape[0], 216)

    def head(key, X, K):
        W = P[key + ".weight"].reshape(24, K, -1)
        return torch.einsum("jkf,bjf->bjk", W, X) + P[key + ".bias"].reshape(24, K)

    B = rot_feats.shape[0]
    M = buf["I_n"][0] + buf["A_mask"][0] * F.relu(P["edge_importance"][0])
    s = M.sum(0)
    d = torch.where(s > 0, s.clamp_min(1e-30) ** -0.5, torch.zeros_like(s))
    Ahat = d[:, None] * M * d[None, :]
    adjs = [buf["r2p_A"][0], Ahat, Ahat, Ahat, buf["p2r_A"][0]]
    mp = buf["mean_pose"].reshape(24, 6)
    pose0 = coord0 = coord1 = None
    if training:
        pose0 = rot6d(head("pose_regressors.0.1", rot_feats, 6) + mp)
    h = rot_feats
    h0 = None
    for l, (name, i) in enumerate(LAYERS):
        pre, bnk = "%s.gc.%d." % (name, i), BN_NAMES[l]
        y = torch.matmul(torch.matmul(adjs[l], h), P[pre + "weight"]) + P[pre + "bias"]
        rm, rv = bn[bnk]
        y = F.batch_norm(y, rm, rv, P[bnk + ".weight"], P[bnk + ".bias"], training, BN_MOMENTUM, BN_EPS)
        y = F.relu(y)
        if l == 0:
            h0 = y
            if training:
                coord0 = head("coord_regressors.0.1", y, 3)
        if l == 3:
            y = h0 + y
            if training:
                coord1 = head("coord_regressors.1.1", y, 3)
        h = y
    para = torch.cat([global_para, rot6d(head("pose_regressors.1.1", h, 6) + mp)], 1)
    return para, pose0, coord0, coord1
