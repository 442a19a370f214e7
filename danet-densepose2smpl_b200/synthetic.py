"""Seed-fixed synthetic stand-ins for the licensed assets the reference needs, and
deterministic random weights of the DaNet architecture (for benchmarks, smoke tests and parity
fixtures when no checkpoint is available).  The real files are absent here
(reference README.md:28-65 lists what a user must download):

* ``data/smpl/SMPL_NEUTRAL.pkl``          -> :func:`make_smpl_model`
* ``data/J_regressor_extra.npy``          -> ``J_regressor_extra`` of the same dict
* ``data/J_regressor_h36m.npy``           -> ``J_regressor_h36m``
* ``data/UV_data/UV_Processed.mat``       -> :func:`make_dp_mesh`
* ``data/smpl_mean_params.npz``           -> :func:`make_mean_params`

Array shapes and dtypes equal the real ones (6890 vertices, 13776 faces, 24
joints, 207x20670 pose-correctives, 7829-vertex / 13774-face DensePose mesh)
so the kernels run the same code paths; values are synthetic.

The surface is a body-sized ellipsoid sampled on a 65 x 106 latitude/longitude
grid (65*106 == 6890): 64 bands * 106 quads * 2 + two 104-triangle caps ==
13776 triangles == SMPL's face count.
"""
import numpy as np

NV = 6890
NF = 13776
NJ = 24
N_DP_V = 7829
N_DP_F = 13774

# kinematic tree of SMPL (reference utils/smpl_utlis.py:13 row 0, root = -1)
PARENTS = np.array([-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14,
                    16, 17, 18, 19, 20, 21], dtype=np.int32)

# rough rest-pose joint targets (metres, y up) so that the skeleton looks like a body
_JOINT_TARGETS = np.array([
    [0.00, -0.22, 0.02], [0.07, -0.31, 0.01], [-0.07, -0.31, 0.01], [0.00, -0.10, 0.00],
    [0.10, -0.69, 0.01], [-0.10, -0.69, 0.01], [0.00, 0.03, 0.02], [0.09, -1.09, -0.03],
    [-0.09, -1.09, -0.03], [0.00, 0.09, 0.03], [0.11, -1.15, 0.09], [-0.11, -1.15, 0.09],
    [0.00, 0.30, -0.01], [0.08, 0.21, 0.00], [-0.08, 0.21, 0.00], [0.00, 0.38, 0.04],
    [0.17, 0.24, -0.01], [-0.17, 0.24, -0.01], [0.43, 0.23, -0.03], [-0.43, 0.23, -0.03],
    [0.68, 0.24, -0.03], [-0.68, 0.24, -0.03], [0.76, 0.23, -0.04], [-0.76, 0.23, -0.04],
], dtype=np.float64)

# vertex ids smplx's VertexJointSelector appends (SURVEY Appendix B.1; ids from memory
# of smplx/vertex_ids.py -- they do not affect kernel-vs-oracle parity)
SELECTED_VERTS = np.array([332, 6260, 2800, 4071, 583,
                           3216, 3226, 3387, 6617, 6624, 6787,
                           2746, 2319, 2445, 2556, 2673,
                           6191, 5782, 5905, 6016, 6133], dtype=np.int32)


def _grid_surface():
    rows, cols = 65, 106
    lat = np.linspace(0.02 * np.pi, 0.98 * np.pi, rows)       # avoid degenerate poles
    lon = np.arange(cols) * (2 * np.pi / cols)
    la, lo = np.meshgrid(lat, lon, indexing="ij")
    # ellipsoid: ~1.7 m tall, arms-span bulge in x
    x = 0.30 * np.sin(la) * np.cos(lo) * (1.0 + 0.9 * np.exp(-((np.cos(la) - 0.55) / 0.12) ** 2))
    y = 0.85 * np.cos(la) - 0.35
    z = 0.14 * np.sin(la) * np.sin(lo)
    v = np.stack([x, y, z], -1).reshape(-1, 3)
    faces = []
    for r in range(rows - 1):
        for c in range(cols):
            a = r * cols + c
            b = r * cols + (c + 1) % cols
            d = (r + 1) * cols + c
            e = (r + 1) * cols + (c + 1) % cols
            faces.append((a, d, b))
            faces.append((b, d, e))
    top = [c for c in range(cols)]
    bot = [(rows - 1) * cols + c for c in range(cols)]
    for i in range(1, cols - 1):
        faces.append((top[0], top[i], top[i + 1]))
    for i in range(1, cols - 1):
        faces.append((bot[0], bot[i + 1], bot[i]))
    faces = np.asarray(faces, dtype=np.int64)
    assert v.shape == (NV, 3) and faces.shape == (NF, 3), (v.shape, faces.shape)
    return v, faces


def _sparse_rows(rng, targets, verts, k):
    """Non-negative rows summing to 1, supported on the k vertices nearest each target."""
    out = np.zeros((targets.shape[0], verts.shape[0]), dtype=np.float64)
    for j, t in enumerate(targets):
        d = np.linalg.norm(verts - t, axis=1)
        idx = np.argsort(d)[:k]
        w = rng.random(k) + 0.05
        out[j, idx] = w / w.sum()
    return out


def make_smpl_model(seed=0, dense_weights=False):
    """Synthetic SMPL-shaped model dict (float32 arrays, shapes of the real pkl)."""
    rng = np.random.default_rng(seed)
    v_template, faces = _grid_surface()
    v_template = v_template + rng.normal(0, 0.002, v_template.shape)
    shapedirs = rng.normal(0, 0.01, (NV, 3, 10))
    posedirs = rng.normal(0, 0.001, (207, NV * 3))             # stored [207, 20670] like smplx
    J_regressor = _sparse_rows(rng, _JOINT_TARGETS, v_template, 48)
    # skinning weights: <= 4 non-zeros per row (real SMPL has the same sparsity)
    J_rest = J_regressor @ v_template
    d = np.linalg.norm(v_template[:, None, :] - J_rest[None], axis=-1)        # [NV, 24]
    lbs_weights = np.zeros((NV, NJ))
    near = np.argsort(d, axis=1)[:, :4]
    rows = np.arange(NV)[:, None]
    w = np.exp(-(np.take_along_axis(d, near, 1) / 0.08) ** 2) + 1e-4
    # drop the 4th (and sometimes 3rd) influence on part of the mesh to exercise nnz < 4
    drop = rng.random((NV, 4)) < np.array([0.0, 0.0, 0.25, 0.5])
    w = np.where(drop, 0.0, w)
    lbs_weights[rows, near] = w / w.sum(1, keepdims=True)
    if dense_weights:
        lbs_weights = lbs_weights + 0.002 * rng.random((NV, NJ))
        lbs_weights /= lbs_weights.sum(1, keepdims=True)
    extra_targets = J_rest[rng.integers(0, NJ, 9)] + rng.normal(0, 0.05, (9, 3))
    h36m_targets = J_rest[rng.integers(0, NJ, 17)] + rng.normal(0, 0.05, (17, 3))
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return {
        "v_template": f32(v_template),
        "shapedirs": f32(shapedirs),
        "posedirs": f32(posedirs),
        "J_regressor": f32(J_regressor),
        "lbs_weights": f32(lbs_weights),
        "parents": PARENTS.copy(),
        "faces": faces.astype(np.int64),
        "J_regressor_extra": f32(_sparse_rows(rng, extra_targets, v_template, 32)),
        "J_regressor_h36m": f32(_sparse_rows(rng, h36m_targets, v_template, 32)),
        "selected_verts": SELECTED_VERTS.copy(),
    }


def make_dp_mesh(seed=0):
    """Synthetic DensePose-shaped UV mesh (what DensePoseMethods reads from UV_Processed.mat,
    reference utils/densepose_methods.py:16-29): 7829 vertices that map onto the 6890 SMPL
    vertices (seam duplicates), 13774 faces, per-face part id 1..24, per-vertex U/V in [0,1]."""
    rng = np.random.default_rng(seed + 1)
    _, faces = _grid_surface()
    # duplicate 939 vertices (the "seams"): new ids 6890..7828 alias random SMPL vertices
    dup_src = rng.choice(NV, N_DP_V - NV, replace=False)
    all_vertices = np.concatenate([np.arange(NV), dup_src]) + 1              # 1-based like the .mat
    remap = {int(s): NV + i for i, s in enumerate(dup_src)}
    f = faces[:N_DP_F].copy()
    # faces in the second half of the list use the duplicate ids where available
    half = N_DP_F // 2
    for i in range(half, N_DP_F):
        for k in range(3):
            f[i, k] = remap.get(int(f[i, k]), f[i, k])
    # part ids: 24 latitude/longitude patches, contiguous so that a render shows regions
    cent = (faces[:N_DP_F] // 106).mean(1)                                    # mean grid row
    lon = (faces[:N_DP_F] % 106).mean(1)
    band = np.minimum((cent / 65.0 * 12).astype(np.int64), 11)
    side = (lon >= 53).astype(np.int64)
    face_indices = (band * 2 + side + 1).astype(np.int64)                      # 1..24
    U = rng.random(N_DP_V)
    V = rng.random(N_DP_V)
    return {
        "All_vertices": all_vertices.astype(np.int64),      # [7829], 1-based SMPL ids
        "FacesDensePose": f.astype(np.int64),               # [13774, 3] into the 7829 list
        "FaceIndices": face_indices,                        # [13774] in 1..24
        "U_norm": U.astype(np.float64),
        "V_norm": V.astype(np.float64),
    }


def make_mean_params(seed=0):
    """Stand-in for data/smpl_mean_params.npz ('pose' [144] 6d, 'shape' [10], 'cam' [3])."""
    rng = np.random.default_rng(seed + 2)
    pose = np.tile(np.array([1, 0, 0, 1, 0, 0], dtype=np.float32), 24)
    pose = pose + rng.normal(0, 0.05, 144).astype(np.float32)
    return {"pose": pose.astype(np.float32),
            "shape": rng.normal(0, 0.3, 10).astype(np.float32),
            "cam": np.array([0.9, 0.0, 0.0], dtype=np.float32)}


def dp_textures(mesh):
    """Per-face constant texture (I/24, mean U, mean V) -- reference utils/renderer.py:243-249."""
    num_part = float(np.max(mesh["FaceIndices"]))
    f = mesh["FacesDensePose"]
    tex = np.stack([mesh["FaceIndices"] / num_part,
                    mesh["U_norm"][f].mean(1),
                    mesh["V_norm"][f].mean(1)], -1)
    return tex.astype(np.float32)


# ---------------------------------------------------------------------------------------------
# deterministic "keyed" weights: every tensor is a function of (state_dict key, seed) only, so
# the reference modules (oracle/gen_golden_net.py) and this package get identical parameters
# without shipping a checkpoint.
# ---------------------------------------------------------------------------------------------
def keyed_tensor(key, shape, seed=0, role=""):
    """role: 'bn_last' (last BatchNorm of a residual branch), 'bn_fuse' (cross-resolution fuse term)
    get a small gamma so that activations stay O(1) through ~100 residual / fuse stages while the
    input signal still reaches the heads (He-initialised convolutions everywhere)."""
    import zlib
    import torch
    g = torch.Generator().manual_seed((zlib.crc32(key.encode()) ^ (seed * 2654435761)) & 0x7FFFFFFF)
    leaf = key.rsplit(".", 1)[-1]
    shape = tuple(shape)
    if leaf == "num_batches_tracked":
        return torch.zeros(shape, dtype=torch.long)
    if leaf == "running_mean":
        return torch.randn(shape, generator=g) * 0.1
    if leaf == "running_var":
        return torch.rand(shape, generator=g) * 0.4 + 0.8
    if len(shape) == 1 and leaf == "weight":            # BatchNorm gamma
        if role == "bn_last":
            return torch.rand(shape, generator=g) * 0.15 + 0.15
        if role == "bn_fuse":
            return torch.rand(shape, generator=g) * 0.2 + 0.2
        return torch.rand(shape, generator=g) * 0.4 + 0.8
    if leaf == "bias":
        return torch.randn(shape, generator=g) * 0.1
    if len(shape) == 4:                                   # conv weight [co, ci, k, k]
        fan_in = shape[1] * shape[2] * shape[3]
        gain = 1.0
        if key.endswith("predict_hm.1.weight"):
            gain = 0.03          # keeps softmax(10*hm) soft (iuv_estimator.py:137)
        elif "final_pred.predict_" in key and "predict_hm" not in key:
            gain = 0.2
        return torch.randn(shape, generator=g) * gain * (2.0 / fan_in) ** 0.5
    if len(shape) == 2:                                   # linear [out,in] / GraphConv [in,out] weight
        fan_in = shape[0] if "gc." in key else shape[1]
        return torch.randn(shape, generator=g) * (1.0 / fan_in) ** 0.5
    if leaf == "edge_importance":
        return torch.rand(shape, generator=g) + 0.5
    return None


def _bn_role(key, template):
    if not key.endswith(".weight"):
        return ""
    prefix = key[:-len(".weight")]
    name = prefix.rsplit(".", 1)[-1]
    parent = prefix.rsplit(".", 1)[0] if "." in prefix else ""
    if name == "bn3":
        return "bn_last"
    if name == "bn2" and (parent + ".conv3.weight") not in template:
        return "bn_last"
    if "fuse_layers" in key and template[key].dim() == 1:
        return "bn_fuse"
    return ""


KEEP_KEYS = ("I_n", "A_link", "A_mask", "r2p_A", "p2r_A", "learned_ratio", "learned_offset", "mean_cam_shape",
             "mean_pose")


def keyed_state_dict(template, seed=0):
    """template: state_dict (key -> tensor) of either implementation.  Structural buffers, the
    learned STN ratios and the mean parameters are kept; everything else is regenerated."""
    out = {}
    for k, v in template.items():
        leaf = k.rsplit(".", 1)[-1]
        if k.startswith("iuv2smpl.smpl.") or leaf in KEEP_KEYS or (leaf == "A" and v.dim() == 3):
            out[k] = v.clone()
            continue
        t = keyed_tensor(k, v.shape, seed, _bn_role(k, template))
        out[k] = v.clone() if t is None else t.to(v.dtype)
    return out


# ---------------------------------------------------------------------------------------------
# evaluation stand-ins: the gendered SMPL models of 3DPW, PartRenderer's colour / part tables, and small caches
# ---------------------------------------------------------------------------------------------
def make_gendered_smpl_models(seed=0):
    """{'male', 'female'} stand-ins for SMPL_MALE.pkl / SMPL_FEMALE.pkl: synthetic models of their own seeds that carry
    the neutral model's J_regressor_h36m (eval.py uses one H36M regressor for every model)."""
    h36m = make_smpl_model(seed)["J_regressor_h36m"]
    out = {}
    for k, g in enumerate(("male", "female")):
        m = make_smpl_model(seed + 101 + k)
        m["J_regressor_h36m"] = h36m
        out[g] = m
    return out


def make_part_assets(seed=0):
    """PartRenderer's textures (VERTEX_TEXTURE_FILE: a colour per face, placed so that floor(100 * c) is unambiguous) and
    cube_parts (CUBE_PARTS_FILE: 100^3 part ids 0..6)."""
    rng = np.random.default_rng(seed + 3)
    tex = (rng.integers(0, 100, (NF, 3)).astype(np.float32) + 0.5) / 100.0
    return {"textures": tex, "cube_parts": rng.integers(0, 7, (100, 100, 100)).astype(np.float32)}


def make_eval_cache(dataset, n, seed=0):
    """A small cache in the format danet_b200.eval_h36m reads for `dataset` ('3dpw' or 'lsp'), with uint8 RGB crops."""
    rng = np.random.default_rng(seed + 4)
    yy, xx = np.mgrid[0:224, 0:224]
    img = ((np.sin(xx / 17.0)[None, :, :, None] + np.cos(yy / 23.0)[None, :, :, None]) * 60 + 128
           + rng.normal(0, 20, (n, 224, 224, 3))).clip(0, 255).astype(np.uint8)
    if dataset == "3dpw":
        return {"img": img, "pose": (rng.normal(0, 0.2, (n, 72))).astype(np.float32),
                "betas": rng.normal(0, 1, (n, 10)).astype(np.float32), "gender": rng.integers(-1, 2, n).astype(np.int32)}
    if dataset != "lsp":
        raise ValueError("make_eval_cache: '3dpw' or 'lsp' (got %r)" % (dataset,))
    shapes = np.stack([rng.integers(120, 400, n), rng.integers(120, 400, n)], 1).astype(np.int64)
    center = np.stack([rng.uniform(0.2, 0.8, n) * shapes[:, 1], rng.uniform(0.2, 0.8, n) * shapes[:, 0]], 1)
    scale = rng.uniform(0.4, 1.2, n) * shapes.min(1) / 200.0
    masks, parts = [], []
    for h, w in shapes:
        y, x = np.mgrid[0:h, 0:w]
        cy, cx, ry, rx = rng.uniform(0.3, 0.7) * h, rng.uniform(0.3, 0.7) * w, rng.uniform(0.2, 0.4) * h, rng.uniform(0.1, 0.3) * w
        inside = ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 < 1
        masks.append(np.where(inside, 255, 0).astype(np.uint8).ravel())
        p = np.where(inside, 1 + (y * 6) // h, 0).astype(np.uint8)
        p[rng.random((h, w)) < 0.02] = 255
        parts.append(p.ravel())
    return {"img": img, "center": center.astype(np.float32), "scale": scale.astype(np.float64), "orig_shape": shapes,
            "mask_gt": np.concatenate(masks), "parts_gt": np.concatenate(parts)}
