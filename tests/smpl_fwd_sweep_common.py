"""The covering sweep of the SMPL layer's forward (danet_smpl_forward, csrc/lbs.cu): the case table, the coverage
classes, the inputs, the fp64 reference and the per-element bound every output is held to.

A case is (model, B, pose front-end, pose regime, beta regime, bodies_per_cta, outputs).  The route follows from B and
bodies_per_cta as in danet_smpl_forward: the fused fp32 route below 512 bodies or with bodies_per_cta = -1, the
tensor-core route otherwise, which skins with k_smpl_skin when the weights are packed and the 128-vertex tile count is
a multiple of 3, and with k_smpl_verts<8> otherwise.  CLASSES states, as predicates over a case, everything the table
has to cover; tests/test_smpl_fwd_sweep_cpu.py fails with the names of the uncovered classes and shows that the bound
catches a set of wrong forward passes, and tests/test_smpl_fwd_sweep_gpu.py runs every case on the GPU.  The models are
the SMPL backward sweep's (tests/smpl_grad_sweep_common.py) and one more, "jtail" (see make_model).

The reference of each output is oracle.lbs_grad.smpl_layer in fp64, with the rotations of oracle/lbs.py's
batch_rodrigues_smplx / rot6d_to_rotmat in fp64 for the axis-angle / rot6d front-ends.  The bound, per element:

    |got - r| <= C * 2^-24 * M + (M - M0) + G + 2^-24 * |r| + 2^-149

    M0   the element's magnitude: the same layer with absolute=True (every array and input made non-negative and every
         subtraction an addition) at |R|.
    M    the same at |R| + e, where e bounds the front-end's error on each rotation entry: 0 for rotation-matrix input,
         C_AA * 2^-24 * M_R for axis-angle and C_R6 * 2^-24 * M_R for rot6d (M_R below).  The layer is a polynomial in R
         whose absolute restatement bounds the sum of its terms' absolute values, so M - M0 bounds what the front-end's
         error moves the output, and C * 2^-24 * M covers the fp32 rounding of the layer at the kernel's rotations.
    C    the longest chain of rounded fp32 operations a term of the output passes through (the constants below).
    G    the tensor-core route's GEMM error on v_posed pushed through the absolute skinning transform and the absolute
         regressors (gemm_terms); 0 on the fused route.

The rotations the axis-angle and rot6d front-ends write (rotmats) are held to C_AA / C_R6 * 2^-24 * M_R + 2^-24 |r|.
"""
import collections
import math

import numpy as np
import torch

from oracle import lbs as olbs
from oracle import lbs_grad
from fp64_bound import U24
import gcn_head_sweep_common as gh
import smpl_grad_sweep_common as gsc

# ----------------------------------------------------------------------------------------------------------------------
# C: the longest serial fp32 chains of the forward, in rounded operations, for 16 betas, a tree of depth 23 and
# 54 vertex tiles (the largest counts any model here reaches)
# ----------------------------------------------------------------------------------------------------------------------
NBETAS_MAX = 16
DEPTH_MAX = 23
NTILES_MAX = 54
N_J = 2 + NBETAS_MAX                  # rest joints: Jt and Jsd rounded to fp32 on the host, then nbetas FMAs
N_REL = 1                             # J_i - J_parent
N_CHAIN = 4 * DEPTH_MAX               # world transforms: per level a 3-term row product and the parent's translation
N_A = 4                               # A_t = tg - Rg J: a 3-term product and a subtraction
N_VPOSED = 1 + NBETAS_MAX + 208       # pf = R - I, then v_posed = template + nbetas FMAs + 208 FMAs
N_SKIN = 24 + 4                       # T = sum_j w_j A_j (24 FMAs with dense weights), then T [v_posed; 1] (4 terms)
N_PARTIAL = 4 + 5                     # a 128-vertex tile partial: 4 FMAs per lane, 5 shuffle levels
N_TILESUM = NTILES_MAX                # k_smpl_joints: the tile partials summed in tile order
N_TRANSL = 1                          # + transl, added on the Python side
C_SMPL_JOINTS = N_J + N_REL + N_CHAIN + N_TRANSL
C_VERTS = N_J + N_REL + N_CHAIN + N_A + N_VPOSED + N_SKIN + N_TRANSL
C_REGRESSED = C_VERTS + N_PARTIAL + N_TILESUM

# front-ends.  Axis-angle (rodrigues_smplx): angle = sqrtf(|v + 1e-8|^2) has a relative error of at most 4 units
# (K_ANGLE) and x = v / angle 5 (K_UNIT); sinf and cosf are within 2 ulp (4 units) without fast-math, so
# s = sinf(angle) is within K_TRIG units of Ms = |s| + angle and c1 = 1 - cosf(angle) within K_TRIG units of
# Mc = 1 + |c1| + angle |s| (cosf's 2 ulp are absolute near 1; the angle's error moves sin and cos by 4 angle units at
# most).  The longest entry is the diagonal 1 + c1 (-(z z) - y y): a square (2 K_UNIT + 1), a subtraction, the product
# with c1 (K_TRIG + 1) and the addition; magnitudes M_R = 1 + Mc (y^2 + z^2) on the diagonal, Ms |z| + Mc |x y| off it.
K_ANGLE = 4
K_UNIT = K_ANGLE + 1
K_TRIG = 4
C_AA = (2 * K_UNIT + 1) + 1 + (K_TRIG + 1) + 1 + 1
# rot6d is common.cuh's, the one the regressor head runs: its constant and magnitudes are the GCN head sweep's
C_R6 = gh.C_R6

# the tensor-core route's split-fp16 exact-mode GEMM, with the terms of the convolution engine's parity sweep
# (tests/test_conv_sweep_gpu.py): relative unit 2^-22, subnormal floor 2^-25, constant 3
C_TC = 3.0
U_TC = 2.0 ** -22
FLOOR_TC = 2.0 ** -25

OUTPUTS = ("verts", "joints", "smpl_joints", "joints_J19", "joints_h36m", "rotmats")
C_OUT = {"verts": C_VERTS, "joints": C_REGRESSED, "smpl_joints": C_SMPL_JOINTS, "joints_J19": C_REGRESSED,
         "joints_h36m": C_REGRESSED}

GEMM_MIN_B = 512
GEMM_CHUNK = 512
SKIN_TL = 3                           # vertex tiles per CTA of k_smpl_skin

# ----------------------------------------------------------------------------------------------------------------------
# models: the backward sweep's zoo and "jtail"
# ----------------------------------------------------------------------------------------------------------------------
MODEL_NAMES = gsc.MODEL_NAMES + ("jtail",)
JTAIL = 2.0 ** -26


def make_model(name):
    """the model dict of a sweep model.  "jtail" is "translated" with every joint-regressor row given a tail of 2^-26 on
    each vertex outside its support (the real SMPL regressor has many small weights): past the support the running sum
    is ~2, so an fp32 sum of the rest-joint table drops every tail term, which a double sum keeps."""
    if name != "jtail":
        return gsc.model(name)
    m = dict(gsc.model("translated"))
    Jr = m["J_regressor"].astype(np.float64)
    Jr = np.where(Jr != 0, Jr * (1.0 - JTAIL * Jr.shape[1]), JTAIL)
    m["J_regressor"] = Jr.astype(np.float32)
    return m


_MODELS = {}


def model(name):
    if name not in _MODELS:
        _MODELS[name] = make_model(name)
    return _MODELS[name]


def without_h36m(m):
    return {k: v for k, v in m.items() if k != "J_regressor_h36m"}


def ntiles(m):
    return -(-m["v_template"].shape[0] // 128)


def packed(m):
    return int((np.asarray(m["lbs_weights"]) != 0).sum(1).max()) <= 4


def weight_exponent(m):
    """the exponent s of the scale 2^s k_pow2_scale gives the packed GEMM weights [posedirs ; shapedirs]: the largest
    finite |w| * 2^s lies in [2^13, 2^14), s clamped to [-126, 126]"""
    a = max(float(np.abs(m["posedirs"]).max()), float(np.abs(m["shapedirs"]).max()))
    return 0 if a == 0.0 else min(max(14 - math.frexp(a)[1], -126), 126)


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
Case = collections.namedtuple("Case", ["model", "B", "front", "pose", "beta", "nbc", "out"])

FRONTS = ("rotmat", "aa", "r6d")
POSES = ("identity", "near", "typical", "large", "zero", "nonortho", "collinear")
BETAS = ("zero", "normal", "large", "tiny")
OUTS = ("h36m", "no_h36m", "transl")
FUSED_AUTO_B = (1, 2, 3, 4, 31, 32, 33, 511)
GEMM_B = (512, 513, 1023, 1024, 1025)
FALLBACK_MODELS = ("dense", "nv100", "nv128", "nv129")
BLOCKINGS = (1, 2, 4, 8, 16)
BENCH_B = 8192

CASES = [
    # fused route, automatic blocking
    Case("packed", 1, "rotmat", "identity", "zero", 0, "h36m"),
    Case("packed", 2, "aa", "typical", "normal", 0, "h36m"),
    Case("packed", 3, "r6d", "typical", "normal", 0, "transl"),
    Case("packed", 4, "rotmat", "nonortho", "normal", 0, "no_h36m"),
    Case("packed", 31, "aa", "large", "large", 0, "h36m"),
    Case("packed", 32, "r6d", "collinear", "normal", 0, "h36m"),
    Case("packed", 33, "aa", "zero", "tiny", 0, "transl"),
    Case("packed", 511, "r6d", "typical", "normal", 0, "h36m"),
    Case("packed", 5, "rotmat", "near", "tiny", 0, "h36m"),
    Case("packed", 6, "aa", "near", "normal", 0, "h36m"),
    Case("packed", 3, "r6d", "identity", "large", 0, "h36m"),
    Case("packed", 2, "r6d", "near", "normal", 0, "h36m"),
    Case("packed", 2, "rotmat", "large", "normal", 0, "h36m"),
    Case("dense", 2, "r6d", "typical", "normal", 0, "h36m"),
    Case("nbetas1", 2, "aa", "typical", "normal", 0, "h36m"),
    Case("nbetas16", 33, "r6d", "typical", "large", 0, "h36m"),
    Case("nv100", 2, "rotmat", "typical", "normal", 0, "h36m"),
    Case("nv128", 3, "aa", "large", "normal", 0, "h36m"),
    Case("nv129", 2, "rotmat", "nonortho", "large", 0, "transl"),
    Case("chain", 4, "rotmat", "large", "normal", 0, "h36m"),
    Case("star", 2, "rotmat", "large", "normal", 0, "h36m"),
    Case("translated", 3, "rotmat", "typical", "normal", 0, "transl"),
    Case("jtail", 2, "rotmat", "typical", "normal", 0, "h36m"),
    # fused route, forced blockings with ragged batches, and forced at B >= 512
    Case("packed", 19, "rotmat", "typical", "normal", 1, "h36m"),
    Case("dense", 19, "rotmat", "typical", "normal", 2, "h36m"),
    Case("nv129", 19, "aa", "typical", "normal", 4, "h36m"),
    Case("packed", 37, "r6d", "typical", "large", 8, "h36m"),
    Case("chain", 37, "rotmat", "large", "normal", 16, "h36m"),
    Case("packed", 600, "aa", "typical", "normal", -1, "h36m"),
    # tensor-core route, k_smpl_skin
    Case("packed", 512, "r6d", "typical", "normal", 0, "h36m"),
    Case("packed", 513, "aa", "typical", "large", 0, "transl"),
    Case("packed", 1023, "rotmat", "nonortho", "normal", 0, "h36m"),
    Case("nbetas16", 1024, "rotmat", "typical", "large", 0, "h36m"),
    Case("packed", 1025, "aa", "near", "tiny", 0, "h36m"),
    Case("nbetas1", 600, "rotmat", "typical", "large", 0, "no_h36m"),
    Case("star", 520, "aa", "large", "normal", 0, "h36m"),
    Case("translated", 600, "r6d", "typical", "normal", 0, "h36m"),
    Case("chain", 600, "rotmat", "typical", "normal", 8, "h36m"),
    Case("jtail", 520, "rotmat", "typical", "large", 0, "h36m"),
    Case("packed", 520, "rotmat", "identity", "tiny", 0, "h36m"),
    Case("packed", BENCH_B, "r6d", "typical", "normal", 0, "h36m"),            # what bench.py's lbs_bench times
    # tensor-core route, k_smpl_verts<8> fallback, at every bodies_per_cta
    Case("dense", 520, "rotmat", "typical", "large", 0, "h36m"),
    Case("dense", 600, "r6d", "typical", "normal", 1, "h36m"),
    Case("nv100", 512, "aa", "typical", "normal", 2, "h36m"),
    Case("nv128", 530, "rotmat", "large", "large", 4, "h36m"),
    Case("nv129", 1025, "r6d", "collinear", "normal", 8, "h36m"),
    Case("dense", 513, "rotmat", "identity", "tiny", 16, "no_h36m"),
    Case("nv129", 600, "aa", "near", "large", 16, "transl"),
]


def case_id(c):
    return "%s-B%d-%s-%s-%s-nb%d-%s" % c


def route(c):
    return "gemm" if c.B >= GEMM_MIN_B and c.nbc >= 0 else "fused"


def skin_path(c):
    """which kernel skins the case's v_posed: verts (fused), skin or fallback (tensor-core route)"""
    if route(c) == "fused":
        return "fused"
    m = model(c.model)
    return "skin" if packed(m) and ntiles(m) % SKIN_TL == 0 else "fallback"


def bodies(case):
    """the bodies of a case compared to the reference: all of a small batch; of a large one a strided subset, the
    first and last body of every 512-body chunk and a few around warp and CTA edges"""
    B = case.B
    if B <= 64:
        return list(range(B))
    s = set(range(0, B, max(1, B // 48)))
    for off in range(0, B, GEMM_CHUNK):
        s |= {off, min(off + GEMM_CHUNK, B) - 1}
    s |= {1, 7, 8, 31, 32, 33, B - 2, B - 1}
    return sorted(s)


def _classes():
    cl = []
    for B in FUSED_AUTO_B:
        cl.append(("fused auto B = %d" % B, lambda c, B=B: route(c) == "fused" and c.nbc == 0 and c.B == B))
    for nb in BLOCKINGS:
        cl.append(("fused bodies_per_cta %d, ragged B" % nb,        # (one body per CTA: any batch of several)
                   lambda c, nb=nb: route(c) == "fused" and c.nbc == nb and (c.B % nb != 0 if nb > 1 else c.B > 1)))
    cl.append(("fused forced (-1) at B >= 512", lambda c: c.nbc == -1 and c.B >= GEMM_MIN_B))
    for B in GEMM_B:
        cl.append(("gemm B = %d" % B, lambda c, B=B: route(c) == "gemm" and c.B == B))
    cl.append(("gemm B not a multiple of 8", lambda c: route(c) == "gemm" and c.B % 8 != 0))
    cl.append(("gemm via k_smpl_skin", lambda c: skin_path(c) == "skin"))
    for n in FALLBACK_MODELS:
        cl.append(("gemm fallback model " + n, lambda c, n=n: skin_path(c) == "fallback" and c.model == n))
    for nb in (0,) + BLOCKINGS:
        cl.append(("gemm fallback bodies_per_cta %d" % nb, lambda c, nb=nb: skin_path(c) == "fallback" and c.nbc == nb))
    cl.append(("lbs_bench: gemm B = 8192 rot6d", lambda c: route(c) == "gemm" and c.B == BENCH_B and c.front == "r6d"))
    for f in FRONTS:
        cl.append(("front-end " + f, lambda c, f=f: c.front == f))
    for p in ("identity", "near", "typical", "large"):
        cl.append(("pose " + p, lambda c, p=p: c.pose == p))
    cl.append(("pose zero axis-angle vector", lambda c: c.front == "aa" and c.pose == "zero"))
    cl.append(("pose non-orthonormal matrices", lambda c: c.front == "rotmat" and c.pose == "nonortho"))
    cl.append(("pose rot6d nearly collinear", lambda c: c.front == "r6d" and c.pose == "collinear"))
    cl.append(("pose near-identity on the tensor-core route", lambda c: route(c) == "gemm" and c.pose == "near"))
    for b in BETAS:
        cl.append(("betas " + b, lambda c, b=b: c.beta == b))
    cl.append(("betas tiny on the tensor-core route", lambda c: route(c) == "gemm" and c.beta == "tiny"))
    cl.append(("betas large on the tensor-core route", lambda c: route(c) == "gemm" and c.beta == "large"))
    for nb in (1, 16):
        cl.append(("nbetas %d" % nb, lambda c, nb=nb: model(c.model)["shapedirs"].shape[-1] == nb))
    for n in MODEL_NAMES:
        cl.append(("model " + n, lambda c, n=n: c.model == n))
    for o in OUTS:
        cl.append(("outputs " + o, lambda c, o=o: c.out == o))
    for r in ("fused", "gemm"):
        cl.append(("outputs transl on the %s route" % r, lambda c, r=r: route(c) == r and c.out == "transl"))
    return cl


CLASSES = _classes()


# ----------------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------------
def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _axis_angle(rng, n, pose):
    if pose in ("zero", "identity"):
        return np.zeros((n, 3))
    if pose == "near":
        return _unit(rng, n) * rng.uniform(0.5e-4, 1.5e-4, (n, 1))
    if pose == "large":
        return _unit(rng, n) * rng.uniform(0.5 * np.pi, np.pi, (n, 1))
    return rng.normal(0, 0.3, (n, 3))


def _collinear6(rng, n):
    """6d pairs whose second column is 2^-10 off the first one's line"""
    a1 = _unit(rng, n) * rng.uniform(0.5, 2, (n, 1))
    b1 = a1 / np.linalg.norm(a1, axis=1, keepdims=True)
    perp = np.cross(b1, _unit(rng, n))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    a2 = b1 * rng.uniform(0.5, 2, (n, 1)) + 2.0 ** -10 * perp
    return np.stack([a1, a2], -1).reshape(n, 6)


Inputs = collections.namedtuple("Inputs", ["betas", "pose", "transl"])


def make_inputs(case, seed=0):
    """float32 CPU tensors: betas [B,nb], pose ([B,24,3,3] rotmat, [B,24,3] aa, [B,24,6] r6d), transl [B,3] or None"""
    m = model(case.model)
    nb, B, n = m["shapedirs"].shape[-1], case.B, case.B * 24
    rng = np.random.default_rng(2000 + seed + 7 * CASES.index(case) if case in CASES else seed)
    betas = {"zero": lambda: np.zeros((B, nb)), "normal": lambda: rng.normal(0, 1, (B, nb)),
             "large": lambda: rng.uniform(-50, 50, (B, nb)), "tiny": lambda: rng.normal(0, 1e-6, (B, nb))}[case.beta]()
    if case.front == "aa":
        pose = _axis_angle(rng, n, case.pose).reshape(B, 24, 3)
    elif case.front == "rotmat":
        if case.pose == "nonortho":
            R = olbs.rot6d_to_rotmat(rng.normal(0, 1, (n, 6))) + 0.05 * rng.normal(0, 1, (n, 3, 3))
        else:
            R = olbs.batch_rodrigues_smplx(_axis_angle(rng, n, case.pose))
        pose = R.reshape(B, 24, 3, 3)
    else:
        if case.pose == "typical":
            x = rng.normal(0, 1, (n, 6))
        elif case.pose == "collinear":
            x = _collinear6(rng, n)
        else:
            R = olbs.batch_rodrigues_smplx(_axis_angle(rng, n, case.pose))
            x = (R[:, :, :2] * rng.uniform(0.5, 2, (n, 1, 2))).reshape(n, 6)
        pose = x.reshape(B, 24, 6)
    transl = rng.normal(0, 1, (B, 3)) if case.out == "transl" else None
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return Inputs(t(betas), t(pose), t(transl))


def subset(inp, idx):
    return Inputs(*[None if a is None else a[idx] for a in inp])


# ----------------------------------------------------------------------------------------------------------------------
# front-ends: fp64 rotations and their magnitudes
# ----------------------------------------------------------------------------------------------------------------------
def rodrigues_magnitude(aa):
    """M_R [n,3,3] of rodrigues_smplx for axis-angle aa [n,3] fp64 (see C_AA)"""
    angle = np.linalg.norm(aa + 1e-8, axis=1)
    x, y, z = np.abs(aa / angle[:, None]).T
    s, c1 = np.sin(angle), 1.0 - np.cos(angle)
    Ms, Mc = np.abs(s) + angle, 1.0 + np.abs(c1) + angle * np.abs(s)
    M = np.empty((aa.shape[0], 3, 3))
    M[:, 0, 0], M[:, 1, 1], M[:, 2, 2] = 1 + Mc * (y * y + z * z), 1 + Mc * (z * z + x * x), 1 + Mc * (y * y + x * x)
    M[:, 0, 1] = M[:, 1, 0] = Ms * z + Mc * x * y
    M[:, 0, 2] = M[:, 2, 0] = Ms * y + Mc * x * z
    M[:, 1, 2] = M[:, 2, 1] = Ms * x + Mc * y * z
    return M


def rotations(front, pose):
    """(R [B,24,3,3], M_R [B,24,3,3] or None, C of the front-end) in fp64 numpy for a float32 pose tensor"""
    p = pose.double().numpy()
    B = p.shape[0]
    if front == "rotmat":
        return p, None, 0
    if front == "aa":
        a = p.reshape(-1, 3)
        return (olbs.batch_rodrigues_smplx(a).reshape(B, 24, 3, 3), rodrigues_magnitude(a).reshape(B, 24, 3, 3), C_AA)
    x = p.reshape(-1, 6)
    _, M = gh.rot6d_ref(torch.from_numpy(x))
    return olbs.rot6d_to_rotmat(x).reshape(B, 24, 3, 3), M.numpy().reshape(B, 24, 3, 3), C_R6


# ----------------------------------------------------------------------------------------------------------------------
# the reference and the bound
# ----------------------------------------------------------------------------------------------------------------------
def _outputs(mdl, verts, smpl_joints, joints, transl, h36m_rows):
    """{output: tensor} of one smpl_layer evaluation: the H36M joints regressed from the untranslated vertices, then
    translated, as SMPL.forward does"""
    out = {"verts": verts, "smpl_joints": smpl_joints, "joints": joints,
           "joints_J19": joints[:, -24:][:, olbs.J24_TO_J19]}
    if h36m_rows is not None:
        vu = verts if transl is None else verts - transl[:, None]
        out["joints_h36m"] = torch.einsum("jv,bvk->bjk", h36m_rows, vu) + (0 if transl is None else transl[:, None])
    return out


def _abs_transforms(pa, betas, R):
    """the absolute skinning transforms T [B,nv,3,4] (oracle/lbs_grad.py's absolute restatement, stopped before
    v_posed) at non-negative betas and R"""
    vs = pa["v_template"][None] + torch.einsum("bl,mkl->bmk", betas, pa["shapedirs"])
    J = torch.einsum("bik,ji->bjk", vs, pa["J_regressor"])
    Rg, tg = [R[:, 0]], [J[:, 0]]
    for i in range(1, R.shape[1]):
        p = pa["parents"][i]
        Rg.append(Rg[p] @ R[:, i])
        tg.append(torch.einsum("brc,bc->br", Rg[p], J[:, i] + J[:, p]) + tg[p])
    Rg, tg = torch.stack(Rg, 1), torch.stack(tg, 1)
    A = torch.cat([Rg, (tg + torch.einsum("bjrc,bjc->bjr", Rg, J))[..., None]], -1)
    return torch.einsum("vj,bjrc->bvrc", pa["lbs_weights"], A)


def gemm_terms(mdl, pa, betas, Rm, h36m_rows):
    """G of the tensor-core route per output, at absolute betas and rotations Rm (|R| + e): the split-fp16 GEMM's error
    on each v_posed coordinate,

        E = C_TC (2^-22 A + 2^-25 sum_k |W_kn| + 2^-25 2^-s sum_k |a_k|) + 2^-24 A,   A = |template| + sum_k |a_k| |W_kn|

    (the features a = [R - I | betas] are split unscaled, so a tiny one has a subnormal lo half: 2^-25 against the
    weights; the weights carry the scale 2^s: 2^-25 2^-s against the features; 2^-24 A is the fp32 output), pushed
    through the absolute skinning transform and the absolute regressors"""
    B, nv = betas.shape[0], pa["v_template"].shape[0]
    eye = torch.eye(3, dtype=Rm.dtype, device=Rm.device)
    feat = torch.cat([(Rm[:, 1:] + eye).reshape(B, 207), betas], 1)               # >= |R - I|, |betas|
    W = torch.cat([pa["posedirs"], pa["shapedirs"].reshape(nv * 3, -1).T], 0)      # [207 + nbetas, 3 nv], absolute
    A = pa["v_template"].reshape(1, -1) + feat @ W
    s = weight_exponent(mdl)
    E = (C_TC * (U_TC * A + FLOOR_TC * W.sum(0)[None] + FLOOR_TC * 2.0 ** -s * feat.sum(1, keepdim=True)) + U24 * A)
    T = _abs_transforms(pa, betas, Rm)
    gv = torch.einsum("bvrc,bvc->bvr", T[..., :3], E.reshape(B, nv, 3))
    cat = torch.cat([torch.zeros(B, 24, 3, dtype=gv.dtype, device=gv.device), gv[:, pa["selected_verts"]],
                     torch.einsum("jv,bvk->bjk", pa["J_regressor_extra"], gv)], 1)
    gj = cat[:, torch.as_tensor(olbs.JOINT_MAP_49, device=gv.device)]
    out = {"verts": gv, "smpl_joints": torch.zeros_like(gv[:, :24]), "joints": gj, "joints_J19": gj[:, -24:][:, olbs.J24_TO_J19]}
    if h36m_rows is not None:
        out["joints_h36m"] = torch.einsum("jv,bvk->bjk", h36m_rows.abs(), gv)
    return out


def reference(case, mdl, inp, device="cpu", with_h36m=True, gemm=None):
    """{output: (r, M, slack, C)} for the bodies of inp, fp64 on the device; slack = (M - M0) + G, with G on the
    case's route unless `gemm` says otherwise"""
    dev = torch.device(device)
    f64 = lambda a: None if a is None else torch.as_tensor(a, dtype=torch.float64).to(dev)
    R, MR, cfe = rotations(case.front, inp.pose)
    betas, transl, Rt = f64(inp.betas), f64(inp.transl), f64(R)
    h36m = f64(mdl["J_regressor_h36m"]) if with_h36m else None
    pm = lbs_grad.prepare(mdl, torch.float64, dev)
    pa = lbs_grad.prepare(mdl, torch.float64, dev, absolute=True)
    r = _outputs(mdl, *lbs_grad.smpl_layer(pm, betas, Rt, transl), transl, h36m)
    assert all(bool(torch.isfinite(t).all()) for t in r.values()), "the sweep's inputs give finite outputs"
    e = torch.zeros_like(Rt) if MR is None else cfe * U24 * f64(MR)
    ta = None if transl is None else transl.abs()
    habs = None if h36m is None else h36m.abs()
    M0 = _outputs(mdl, *lbs_grad.smpl_layer(pa, betas.abs(), Rt.abs(), ta, absolute=True), ta, habs)
    M = _outputs(mdl, *lbs_grad.smpl_layer(pa, betas.abs(), Rt.abs() + e, ta, absolute=True), ta, habs)
    gemm = route(case) == "gemm" if gemm is None else gemm
    G = gemm_terms(mdl, pa, betas.abs(), Rt.abs() + e, h36m) if gemm else None
    ref = {k: (r[k], M[k], (M[k] - M0[k]) + (0 if G is None else G[k]), C_OUT[k]) for k in r}
    if MR is not None:
        ref["rotmats"] = (Rt, f64(MR), torch.zeros_like(Rt), cfe)
    return ref

