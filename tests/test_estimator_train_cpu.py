"""The IUV estimator's training driver without a GPU: the graph walk, driven through the fp64 test double, reproduces
the reference's IUV_Estimator (losses, outputs, running statistics, every gradient sketch) and its STN draws; the
lowering covers the graph from image to the part prediction and consumes every estimator key once; every convolution
the walk hands the conv engine is one it accepts, in all three roles; and the public function refuses bad arguments."""
import ctypes
import os

import numpy as np
import pytest
import torch

from estimator_train_common import EP, OUTPUTS, bn_names, golden, golden_image, golden_noise, golden_targets, step
from oracle import estimator_train as oet
from oracle import regressor_train as ort

TOL = 1e-9


@pytest.fixture(scope="module")
def gold():
    return golden()


@pytest.fixture(scope="module")
def keyed32():
    return oet.keyed_state(32)


def test_golden_layout(gold, keyed32):
    state, graph = keyed32
    np.testing.assert_allclose(ort.input_checksum(golden_image(gold)), gold["checksum_image"], rtol=1e-12)
    sk = {k[3:] for k in gold.files if k.startswith("sk_")}
    assert sk == set(oet.param_keys(state)) | {"image"}
    assert {k[4:] for k in gold.files if k.startswith("nbt_")} == set(bn_names(state))
    assert sorted(k[2:] for k in gold.files if k.startswith("L_")) == sorted(
        ["loss_U", "loss_V", "loss_IndexUV", "loss_segAnn", "loss_Udp", "loss_Vdp", "loss_IndexUVdp", "loss_segAnndp",
         "loss_roi", "loss_stnhm", "loss_pU", "loss_pV", "loss_pIndexUV"])
    assert list(gold["has_iuv"]) == [1, 0] and list(gold["has_dp"]) == [0, 1]       # a batch that mixes both
    assert float(gold["hm_weight"]) > 0 and float(gold["centre_margin"]) >= 1e-3
    assert os.path.getsize(os.path.join(os.path.dirname(__file__), "golden", "estimator_train.npz")) < 1100 << 10


def test_default_noise_draws_are_the_references(gold):
    from danet_b200.estimator import draw_noise
    torch.manual_seed(int(gold["noise_seed"]))
    cn, sn = draw_noise(int(gold["B"]))
    assert np.array_equal(cn.numpy(), gold["center_noise"]) and np.array_equal(sn.numpy(), gold["scale_noise"])


def test_double_walk_reproduces_reference_golden(gold, keyed32):
    """fp64 torch ops through the product's lowering and walk against the reference's own IUV_Estimator"""
    state = {k: v.clone() for k, v in keyed32[0].items()}
    dt = torch.float64
    out, L, grads, gx = step(state, keyed32[1], golden_image(gold).to(dt), True, oet.TorchEstimatorOps(),
                             golden_targets(gold, dt, "cpu"), golden_noise(gold, dt, "cpu"), float(gold["hm_weight"]))
    assert sorted(L) == sorted(k[2:] for k in gold.files if k.startswith("L_"))
    for k, v in L.items():
        assert abs(float(v.sum()) - float(gold["L_" + k])) <= TOL * max(1.0, abs(float(gold["L_" + k]))), k
    for k in OUTPUTS + ("part_iuv_gt",):
        t = out[k]
        assert ort.sketch_error(ort.sketch("out_" + k, t), gold["out_" + k], t.numel()) < TOL, k
    assert np.abs(out["thetas"].numpy() - gold["thetas"]).max() < TOL
    assert np.abs(out["centers"].numpy() - gold["stn_kps_pred"]).max() < TOL
    grads["image"] = gx
    worst = max((ort.sketch_error(ort.sketch(k, g), gold["sk_" + k], g.numel()), k) for k, g in grads.items())
    assert worst[0] < TOL, worst
    for n in bn_names(state):
        for s, key in (("rm1_", ".running_mean"), ("rv1_", ".running_var")):
            t = state[n + key]
            assert ort.sketch_error(ort.sketch(s + n, t), gold[s + n], t.numel()) < TOL, n + key
        assert int(state[n + ".num_batches_tracked"]) == int(gold["nbt_" + n])


def test_lowering_covers_the_graph_once(keyed32):
    from danet_b200 import netgraph
    from danet_b200.estimator import STOPS, lower_estimator
    for width in (32, 48):
        g = netgraph.danet_graph(width)
        low = lower_estimator(g)
        assert lower_estimator(g) is low                       # lowered once per graph
        ops = low["ops"]
        # every graph op from image to part_pred but the input and the cleaning is lowered, in graph order
        end = max(op["gop"] for op in ops)
        assert g.ops[end]["y"].name == g.outputs["part_pred"].name
        want = [i for i, op in enumerate(g.ops[:end + 1]) if op["op"] not in ("input",) + STOPS]
        assert sorted(set(op["gop"] for op in ops)) == want
        assert [op["gop"] for op in ops] == sorted(op["gop"] for op in ops)
        for i in want:                                          # conv + BatchNorm lowers to two ops, the rest to one
            n = sum(op["gop"] == i for op in ops)
            assert n == (2 if g.ops[i]["op"] == "conv" and g.ops[i]["bn"] else 1), (i, g.ops[i]["op"])
        used = [k for op in ops for k in op["keys"]]
        assert sorted(used) == sorted(k for k in g.params if k.startswith(EP))      # every estimator key, once
        heads = [op for op in ops if "split" in op]
        assert len(heads) == 1 and heads[0]["split"] == (25, 25, 25, 15) and len(heads[0]["weight"]) == 4
        part = ops[-1]
        assert part["op"] == "conv2d" and part["groups"] == 24 and part["y"] == g.outputs["part_pred"].name
        kinds = [op["op"] for op in ops]
        assert kinds.count("part_thetas") == 1 and kinds.count("part_crops") == 1
        assert kinds.count("hr_fuse") == sum(op["op"] == "fuse" for op in g.ops)


def test_unknown_op_kind_is_refused():
    from danet_b200 import netgraph
    from danet_b200.estimator import lower_estimator
    g = netgraph.danet_graph(32)
    xd = g.outputs["xd"]
    heads = next(i for i, op in enumerate(g.ops) if op.get("y") is g.outputs["heads"])
    g.ops.insert(heads, dict(op="mystery", x=xd, y=g.tensor(1, xd.H, xd.W, xd.C)))      # on the path
    with pytest.raises(ValueError, match="lower_estimator: graph op 'mystery' has no training lowering"):
        lower_estimator(g)


def test_eval_walk_leaves_statistics(keyed32):
    state = {k: v.clone() for k, v in keyed32[0].items()}
    img = oet.make_image(1, 3, size=64)
    from danet_b200 import netgraph
    g = netgraph.danet_graph(32, 64)
    out, _, _, _ = step(state, g, img.double(), False, oet.TorchEstimatorOps(), backward=False)
    assert tuple(out["part_pred"].shape) == (1, 24, 3, 7, 16, 16)
    for k, v in keyed32[0].items():
        assert torch.equal(state[k], v), k


# ---------------------------------------------------------------------------------------------------------------------
# conv engine census: every convolution of the walk, in its three roles
# ---------------------------------------------------------------------------------------------------------------------
class ShapeOps(object):
    """An op table on meta tensors that records every conv2d call"""

    def __init__(self):
        self.convs = []

    def conv2d(self, x, w, b, stride, padding, dilation, groups):
        B, _, H, W = x.shape
        self.convs.append((B, H, W, tuple(w.shape), stride, groups))
        Ho = (H - 1) // stride + 1
        return torch.empty(B, w.shape[0], Ho, (W - 1) // stride + 1, device="meta")

    def batch_norm(self, x, *a, **k):
        return torch.empty_like(x)

    def hr_fuse(self, terms, factors, relu=True):
        t, f = terms[0], factors[0]
        return torch.empty(t.shape[0], t.shape[1], t.shape[2] * f, t.shape[3] * f, device="meta")

    def part_thetas(self, hm, *a, **k):
        return torch.empty(hm.shape[0], 24, 2, device="meta"), torch.empty(hm.shape[0], 24, 2, 3, device="meta")

    def part_crops(self, xd, thetas):
        return torch.empty(xd.shape[0], 24 * xd.shape[1], xd.shape[2], xd.shape[3], device="meta")


@pytest.fixture(scope="module")
def lib():
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "danet-densepose2smpl_b200",
                      "libdanet_b200.so")
    if not os.path.exists(so):
        import __graft_entry__
        __graft_entry__.build()
    from danet_b200 import _lib
    return _lib.load()


def walk_convs(width, B):
    from danet_b200 import netgraph
    from danet_b200.estimator import lower_estimator, run_estimator
    g = netgraph.danet_graph(width)
    state = {k: torch.empty(s.shape, device="meta") for k, s in g.params.items()}
    ops = ShapeOps()
    run_estimator(lower_estimator(g), state, torch.empty(B, 3, 224, 224, device="meta"), False, ops)
    return ops.convs


@pytest.mark.parametrize("width", [32, 48])
@pytest.mark.parametrize("B", [1, 16])
def test_conv_engine_accepts_every_problem_of_the_walk(lib, width, B):
    from danet_b200 import conv
    convs = walk_convs(width, B)
    assert len(convs) == 304
    out = (ctypes.c_int64 * 32)()
    refused, seen = [], set()
    for (B_, H, W, (Cot, cin, k, _), stride, G) in convs:
        key = (B_, H, W, Cot, cin, k, stride, G)
        if key in seen:
            continue
        seen.add(key)
        cout, N = Cot // G, B_ * G
        Cinp, Coutp = conv._ceil8(cin), conv._ceil8(cout)
        Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
        fwd = conv._desc(N, H, W, Cinp, Coutp, k, stride, G)
        if lib.danet_conv_tc_dispatch(ctypes.byref(fwd), ctypes.cast(out, ctypes.c_void_p)) != 0 or \
                lib.danet_conv_tc_packed_bytes(ctypes.byref(fwd)) <= 0:
            refused.append(("forward", key))
        pieces, n = conv._pieces(k, stride)
        for i in range(n):
            d = conv._desc(N, Ho, Wo, Coutp, Cinp, pieces[i].K, 1, G)
            if lib.danet_conv_tc_dispatch(ctypes.byref(d), ctypes.cast(out, ctypes.c_void_p)) != 0 or \
                    lib.danet_conv_tc_packed_bytes(ctypes.byref(d)) <= 0:
                refused.append(("dgrad piece %d" % i, key))
        if lib.danet_conv_wgrad_workspace_bytes(ctypes.byref(fwd)) <= 0:
            refused.append(("wgrad", key))
    assert not refused, refused
    shapes = {(H, cin, Cot, k, stride, G) for (_, H, _, (Cot, cin, k, _), stride, G) in convs}
    assert (224, 3, 64, 3, 2, 1) in shapes                      # the stem
    assert (56, width, 90, 3, 1, 1) in shapes                   # the four heads as one convolution
    assert (56, width, 504, 3, 1, 24) in shapes                 # the grouped part prediction
    assert (14, width * 4, width * 8, 3, 2, 1) in shapes        # a fuse chain down to 7 x 7


# ---------------------------------------------------------------------------------------------------------------------
# argument refusals of the public function
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cpu_model():
    from danet_b200 import build_synthetic_danet
    return build_synthetic_danet(width=32, seed=0, device="cpu", keyed=False).train()


def test_iuv_estimator_refusals(cpu_model):
    from danet_b200 import iuv_estimator
    W = "danet_b200.estimator.iuv_estimator"
    m = cpu_model
    img = torch.zeros(2, 3, 224, 224)
    with pytest.raises(ValueError, match=W + ": model must be a danet_b200.DaNet"):
        iuv_estimator(torch.nn.Linear(2, 2), img)
    with pytest.raises(ValueError, match=W + ": image must be float32"):
        iuv_estimator(m, img.double())
    with pytest.raises(ValueError, match=W + r": image must be \[B,3,224,224\]"):
        iuv_estimator(m, torch.zeros(2, 3, 112, 112))
    with pytest.raises(ValueError, match=W + ": image must be 4-D"):
        iuv_estimator(m, torch.zeros(3, 224, 224))
    with pytest.raises(ValueError, match=W + ": center_noise needs smpl_kps_gt"):
        iuv_estimator(m, img, center_noise=torch.zeros(2, 24, 2))
    with pytest.raises(ValueError, match=W + r": scale_noise must have shape \(24, 2, 2\)"):
        iuv_estimator(m, img, scale_noise=torch.zeros(24, 2, 3))
    with pytest.raises(ValueError, match=W + r": iuv_image_gt must have shape \(2, 3, 56, 56\)"):
        iuv_estimator(m, img, iuv_image_gt=torch.zeros(2, 3, 224, 224))
    with pytest.raises(ValueError, match=W + r": smpl_kps_gt must be \[2,24,2\|3\]"):
        iuv_estimator(m, img, smpl_kps_gt=torch.zeros(2, 24, 4))
    with pytest.raises(ValueError, match=W + ": uvia_dp_gt must be a dict"):
        iuv_estimator(m, img, uvia_dp_gt=[torch.zeros(2)])
    with pytest.raises(ValueError, match=W + ": has_iuv must be a tensor with one entry per image"):
        iuv_estimator(m, img, has_iuv=torch.ones(3))
    with pytest.raises(ValueError, match=W + ": stn_hm_weight must be a number"):
        iuv_estimator(m, img, stn_hm_weight="1")
    with pytest.raises(ValueError, match=W + ": move the model to a CUDA device"):
        iuv_estimator(m, img)
    m.eval()
    try:
        with pytest.raises(ValueError, match=W + ": center_noise / scale_noise are training-mode jitter"):
            iuv_estimator(m, img, scale_noise=torch.zeros(24, 2, 2))
    finally:
        m.train()
