"""CPU tests of the host logic of the network half (graph wiring, BatchNorm folding, weight packing,
buffer planning, state_dict surface) using the torch test double of the kernel-level ops
(oracle/net_ops.py) against golden vectors produced by the reference's own modules."""
import os

import numpy as np
import pytest
import torch

from oracle.net_ops import TorchEmulOps
from net_common import GOLD, build, check_against_golden, infer_with_ops, make_image


def test_state_dict_surface_matches_reference():
    """Every key / shape of the reference's img2iuv + smpl_para_Outs state_dict exists here (W48)."""
    import danet_b200
    from danet_b200 import synthetic
    net = danet_b200.DaNet(None, synthetic.make_mean_params(0), pretrained=False, width=48,
                           smpl_model=synthetic.make_smpl_model(0), dp_mesh=synthetic.make_dp_mesh(0))
    mine = {k: tuple(v.shape) for k, v in net.state_dict().items() if not k.startswith("iuv2smpl.smpl.")}
    ref = {}
    for line in open(os.path.join(GOLD, "state_dict_keys_w48.txt")):
        k, shp = line.split()
        ref[k] = () if shp == "scalar" else tuple(int(d) for d in shp.split("x"))
    assert set(ref) == set(mine), (sorted(set(ref) - set(mine))[:5], sorted(set(mine) - set(ref))[:5])
    for k in ref:
        assert ref[k] == mine[k], (k, ref[k], mine[k])
    assert any(k.startswith("iuv2smpl.smpl.") for k in net.state_dict())
    assert net.img2iuv.dp2smpl_mapping[7] == [8, 10, 12, 14, 5, 5]
    assert hasattr(net, "iuv_renderer") and hasattr(net.iuv2smpl, "smpl")


@pytest.mark.parametrize("width", [32, 48])
def test_plan_with_emulated_kernels_matches_reference_golden(width):
    net = build(width)
    out = infer_with_ops(net, make_image(2, 100), TorchEmulOps())
    assert out["para"].shape == (2, 229)
    assert out["visualization"]["part_iuv_pred"].shape == (2, 24, 3, 7, 56, 56)
    check_against_golden(out, width, para_tol=5e-5, kps_tol=5e-5, margin_eps=1e-3)
    # rotation block of para is orthonormal (rot6d_to_rotmat)
    R = out["para"][:, 13:].reshape(-1, 3, 3)
    assert (R @ R.transpose(1, 2) - torch.eye(3)).abs().max() < 1e-5


def test_infer_net_requires_eval_mode_and_cuda():
    net = build(32)
    net.train()
    with pytest.raises(ValueError):
        net.infer_net(make_image(1, 1))
    net.eval()
    with pytest.raises(RuntimeError):                 # no CPU fallback in the product path
        net.infer_net(make_image(1, 1))
    with pytest.raises(NotImplementedError):
        net({"img": None})


def _views(a):
    import torch
    if torch.is_tensor(a):
        return [a]
    return [t for t in (a.f32, a.h) if t is not None]


@pytest.mark.parametrize("algo", ["simt", "tc"])
def test_step_records_reuse_memory_without_aliasing_live_tensors(algo):
    """Liveness-based reuse over the plan's step records: a step never reads and writes the same storage, and the
    convolutions that share one launch (tensor-core path) never write storage another member reads."""
    net = build(32, conv_algo=algo)
    plan = net.plan_for(1, "cpu", ops=TorchEmulOps())
    g = plan.g
    total = sum(t.nmult * t.H * t.W * t.Cp * 4 for t in g.tensors.values() if t.dtype == "f32")
    assert plan.bytes_alloc < 0.6 * total               # liveness-based reuse is effective
    for op in g.ops:
        y = op.get("y")
        if y is None:
            continue
        ins = [op.get(k) for k in ("x", "res", "hm", "gpara")] + [t for t, _ in op.get("terms", [])]
        for t in ins:
            if t is not None and t.dtype == "f32" and y.dtype == "f32":
                for a in _views(plan.buf[t.name]):
                    for b in _views(plan.buf[y.name]):
                        assert a.data_ptr() != b.data_ptr(), (op["op"], t, y)
    groups = [s.args[0] for s in plan.steps if s.name == "conv_group"]
    for convs in groups:
        reads, writes = set(), set()
        for cv in convs:
            for a in [cv["x"]] + ([cv["res"]] if cv["res"] is not None else []):
                reads.update(v.data_ptr() for v in _views(a))
            for v in _views(cv["y"]):
                assert v.data_ptr() not in writes, "two members of a launch write the same buffer"
                writes.add(v.data_ptr())
        assert not (reads & writes), "a member of a launch writes a buffer another member reads"
    if algo == "tc":
        n_convs = sum(1 for op in g.ops if op["op"] == "conv")
        assert len(groups) < 0.5 * n_convs, (len(groups), n_convs)  # HRNet's branches share launches
        assert max(len(convs) for convs in groups) >= 4


def test_tensor_core_plan_wiring_matches_reference_golden():
    """Host logic of the tensor-core plan (level scheduling, grouped launches, buffer reuse across groups) with the
    torch test double standing in for the kernels: same golden as the fp32 plan."""
    net = build(32, conv_algo="tc")
    out = infer_with_ops(net, make_image(2, 100), TorchEmulOps())
    check_against_golden(out, 32, para_tol=5e-5, kps_tol=5e-5, margin_eps=1e-3)


def test_tensor_formats_on_the_tensor_core_path():
    """plan._formats: convolutions / fuse sums / pools / STN exchange fp16 planes; the fp32 glue kernels and the
    tensors callers read keep an fp32 view."""
    from danet_b200.plan import Plan

    class PlaneOps(TorchEmulOps):
        def planes(self, precision):
            return 2 if precision == "exact" else 1

    net = build(48, conv_algo="tc")
    g = net.graph
    plan = Plan.__new__(Plan)
    plan.g, plan.B, plan.tc, plan.P, plan.ops = g, 2, True, 2, PlaneOps()
    plan._formats()
    fm = plan.fmt
    for op in g.ops:
        if op["op"] == "conv":
            assert "h" in fm[op["x"].name], op["x"]
    for k in ("heads", "hm", "para", "body_iuv", "rot_feats"):
        assert "f" in fm[g.outputs[k].name]
    assert fm[g.outputs["body_iuv"].name] == {"f", "h"}      # read by callers and by body_net.0
    assert fm[g.outputs["xd"].name] == {"h"}                   # conv input + STN source only
    crops = [op["y"].name for op in g.ops if op["op"] == "stn_sample"][0]
    assert fm[crops] == {"h"}
    n_h_only = sum(1 for v in fm.values() if v == {"h"})
    assert n_h_only > 300


def test_pretrained_flag_needs_files():
    import danet_b200
    from danet_b200 import synthetic
    with pytest.raises(ValueError):
        danet_b200.DaNet(None, synthetic.make_mean_params(0), pretrained=True, width=48,
                         smpl_model=synthetic.make_smpl_model(0), dp_mesh=synthetic.make_dp_mesh(0))
    with pytest.raises(ValueError):
        danet_b200.DaNet(None, "/nonexistent/smpl_mean_params.npz", pretrained=False)


def test_in_place_parameter_edit_invalidates_cached_plans():
    """Plans snapshot folded / packed weights; an in-place edit of a parameter or buffer (tensor version bump) must
    rebuild them (and the LRU keeps at most MAX_PLANS batch sizes)."""
    net = build(32)
    emul = TorchEmulOps()
    img = make_image(1, 3)
    a = infer_with_ops(net, img, emul)["para"].clone()
    p1 = net.plan_for(1, img.device, ops=emul)
    assert net.plan_for(1, img.device, ops=emul) is p1                 # cached
    with torch.no_grad():
        net.iuv2smpl.smpl_para_Outs.mean_cam_shape.add_(0.25)
    b = infer_with_ops(net, img, emul)["para"]
    assert net.plan_for(1, img.device, ops=emul) is not p1
    assert (b[:, :13] - a[:, :13] - 0.25).abs().max() < 1e-5            # cam/shape = linear head + mean_cam_shape
    for B in range(2, 2 + net.MAX_PLANS + 2):
        net.plan_for(B, img.device, ops=emul)
    assert len(net._plans) <= net.MAX_PLANS


def test_exported_step_records_are_well_formed():
    """Plan.export (the input of danet_net_load, csrc/net.cu): every reference stays inside its buffer / constant, the
    step list mirrors the plan's step records, the constants carry the packed weights byte for byte."""
    from netprog_common import parse_program
    net = build(32)
    image = make_image(1, 3)
    plan = net.plan_for(1, image.device, ops=TorchEmulOps())
    plan.run(image)
    blob = plan.export()
    prog = parse_program(blob)
    assert prog["version"] == 1 and prog["batch"] == 1 and prog["chw"] == (3, 224, 224) and prog["precision"] == 2
    n_expected = sum(2 if op["op"] == "body_fc" else 1 for op in plan.g.ops)       # fp32 path: one launch per op
    assert len(prog["steps"]) == len(plan.steps) == plan.n_launch == n_expected
    for s in prog["steps"]:
        assert 1 <= s["op"] <= 12
        for (kind, rid, roff) in s["refs"]:
            assert kind in (0, 1, 2, 3)
            if kind == 1:
                assert rid < len(prog["bufs"]) and roff < prog["bufs"][rid]
            if kind == 2:
                assert rid < len(prog["consts"]) and roff == 0
    names = [o["name"] for o in prog["outs"]]
    assert "para" in names and "centers" in names and "vis_u" in names and "part_iuv_raw" in names
    para = [o for o in prog["outs"] if o["name"] == "para"][0]
    assert para["elem_bytes"] == 4 and int(np.prod(para["dims"])) >= 229
    # a constant round-trips: the first conv step's weights
    conv = [s for s in prog["steps"] if s["op"] == 3][0]
    wref = conv["refs"][1]
    coff, cbytes = prog["consts"][wref[1]]
    w = [s.args[2] for s in plan.steps if s.name == "conv2d"][0]
    assert cbytes == w.numel() * 4
    assert np.array_equal(np.frombuffer(blob, dtype=np.float32, count=w.numel(), offset=coff), w.reshape(-1).numpy())


# (n_i, n_f, n_r) of each fixed-size step kind, as csrc/net.cu prepare() requires them
_FIXED_ARITY = {1: (4, 0, 4), 3: (11, 0, 5), 5: (4, 0, 6), 6: (3, 0, 4), 7: (8, 0, 9), 8: (4, 0, 5), 9: (4, 1, 6),
                10: (4, 0, 7), 11: (3, 0, 5), 12: (11, 0, 27)}


@pytest.mark.parametrize("algo", ["simt", "tc"])
def test_exported_steps_have_the_arity_the_loader_requires(algo):
    """Every step of an exported program carries the number of ints / floats / references that danet_net_load
    accepts for its opcode (and that danet_net_run_step accepts for each Python launch)."""
    from netprog_common import parse_program
    net = build(32, conv_algo=algo)
    plan = net.plan_for(2, "cpu", ops=TorchEmulOps())
    seen = set()
    for s in parse_program(plan.export())["steps"]:
        op, ints, nf, nr = s["op"], s["ints"], len(s["floats"]), len(s["refs"])
        seen.add(op)
        if op == 2:                       # conv group: n problems of 11 descriptor ints and 11 references
            n = ints[0]
            assert 1 <= n <= 6 and len(ints) == 1 + 11 * n and nf == 0 and nr == 11 * n, s
        elif op == 4:                     # fuse: n terms with one upsampling factor each, 3 references per activation
            n = ints[4]
            assert 1 <= n <= 4 and len(ints) == 6 + n and nf == 0 and nr == 3 * n + 3, s
        else:
            assert (len(ints), nf, nr) == _FIXED_ARITY[op], s
    assert seen == set(range(1, 13)) - {3 if algo == "tc" else 2}


class _PlaneOps(TorchEmulOps):
    """The test double with CudaOps' fp16 planes, so tensor-core plans carry the views they carry on the GPU."""

    def planes(self, precision):
        return 2 if precision == "exact" else 1


def _step_conditions(name, ints, ptrs):
    """Conditions of the launchers in csrc/glue.cu and csrc/conv_simt.cu beyond the loader's arity check, for one step
    record; returns the names of those it breaks."""
    bad = []
    if name in ("fuse_sum", "maxpool", "stn_sample"):
        C = ints[2] if name == "stn_sample" else ints[3]
        if C % 8:
            bad.append("C % 8 == 0")                       # the 8-channel kernels are the only ones
    if name == "clean_global":
        Chead, Cbody, heads = ints[2], ints[7], ptrs[0]
        if Chead % 4 or Cbody % 4:
            bad.append("Chead, Cbody % 4 == 0")
        if 64 * (Chead + 1 + Cbody + 1) * 4 > 48 * 1024:
            bad.append("64 staged pixels fit in 48 KB")
        if heads.data_ptr() % 16:
            bad.append("heads 16-byte aligned")
    if name == "clean_parts" and (min(ints[2], ints[3]) < 24 or ints[2] % 4 or ints[3] % 4):
        bad.append("Cx, Cy >= 24 and % 4 == 0")
    if name == "conv2d" and ints[10] != 0:
        bad.append("flags == 0")
    return bad


@pytest.mark.parametrize("width", [32, 48])
@pytest.mark.parametrize("algo,precision", [("simt", "exact"), ("tc", "exact"), ("tc", "fast")])
def test_plan_steps_meet_the_launchers_conditions(width, algo, precision):
    """Every step record a plan emits (B = 2 and 64) meets the conditions the executor's launchers check, so no plan
    step is refused: the fuse, pool and STN-sampler records carry C % 8 == 0, the global iuvmap_clean record fits the
    staged kernel and the part iuvmap_clean record has 24-channel rows.  The simt plan does not depend on precision."""
    from danet_b200.plan import wire
    net = build(width, conv_algo=algo, precision=precision)
    ops = _PlaneOps()
    for B in (2, 64):
        plan = net.plan_for(B, "cpu", ops=ops)
        assert plan.P == (0 if algo == "simt" else ops.planes(precision))
        names = set()
        for s in plan.steps:
            _op, ints, _floats, ptrs = wire(s.name, s.args)
            assert not _step_conditions(s.name, ints, ptrs), (B, s.name, ints, _step_conditions(s.name, ints, ptrs))
            names.add(s.name)
        assert {"fuse_sum", "maxpool", "stn_sample", "clean_global", "clean_parts"} <= names
