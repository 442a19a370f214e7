"""Execution plan of the DaNet network half: folds BatchNorm into the convolutions, packs the
weights into the kernels' layouts, schedules the graph into launch steps (independent convolutions --
HRNet's parallel branches, the body / limb regressors -- share one tensor-core launch), plans
activation buffers (liveness-based reuse) and replays the steps through the C ABI (optionally as one
CUDA graph)."""
import collections
import ctypes

import numpy as np
import torch

from . import _lib
from . import netgraph as ng

BN_EPS = 1e-5
MAX_GROUP = 6            # problems per tensor-core launch (csrc/conv_tc.cu kMaxProb)


class ActBuf(object):
    """One activation tensor of the plan (include/danet_b200.h danet_act): an fp32 NHWC view and/or
    split-fp16 planes h[P,N,H,W,C] (P = 2: hi + lo, exact mode; P = 1: hi only, fast mode)."""
    __slots__ = ("f32", "h")

    def __init__(self, f32=None, h=None):
        self.f32, self.h = f32, h

    def value(self):
        """fp32 torch tensor of the activation (tests / debugging)."""
        if self.f32 is not None:
            return self.f32
        v = self.h[0].float()
        return v + self.h[1].float() if self.h.shape[0] > 1 else v


# One launch of the plan: `name` is the CudaOps method that runs it, `args` its positional arguments.
Step = collections.namedtuple("Step", "name args")

# -- wire encoding ---------------------------------------------------------------------------------
# A launch as one step record of the network program (csrc/net.cu): opcode, ints, floats and a flat pointer list in
# the order net.cu's prepare / run_step decode it.  Plan.export writes these records and CudaOps runs them through
# danet_net_run_step, so the Python plan and the C executor decode every launch with the same code.
OPCODES = {"nchw_to_nhwc": 1, "conv_group": 2, "conv2d": 3, "fuse_sum": 4, "maxpool": 5, "avgpool": 6, "clean_global": 7,
           "clean_parts": 8, "stn_params": 9, "stn_sample": 10, "linear": 11, "gcn_head": 12}
_DESC_KEYS = ("N", "H", "W", "Cin", "Cout", "ksize", "stride", "pad", "wsets", "relu", "flags")


def _desc_ints(d):
    return [int(d.get(k, 0)) for k in _DESC_KEYS]


def _act(a):
    """danet_act pointers (f32, hi, lo) of an ActBuf; None is a null activation."""
    if a is None:
        return [None, None, None]
    h = a.h
    return [a.f32, h[0] if h is not None else None, h[1] if (h is not None and h.shape[0] > 1) else None]


def _wire_conv_group(convs):
    ints, ptrs = [len(convs)], []
    for cv in convs:
        ints += _desc_ints(cv["d"])
        ptrs += _act(cv["x"]) + _act(cv["res"]) + _act(cv["y"]) + [cv["w"], cv["b"]]
    return ints, [], ptrs


def _wire_conv2d(d, x, w, bias, res, y):
    return _desc_ints(d), [], [x.f32, w, bias, res.f32 if res is not None else None, y.f32]


def _wire_nchw_to_nhwc(x, y):
    N, C, H, W = x.shape
    t = y.f32 if y.f32 is not None else y.h[0]
    return [N, C, H * W, t.shape[-1]], [], [x] + _act(y)


def _wire_fuse_sum(terms, factors, relu, y, shape):
    N, H, W, C = shape
    ptrs = []
    for t in terms:
        ptrs += _act(t)
    return [N, H, W, C, len(terms), int(relu)] + [int(f) for f in factors], [], ptrs + _act(y)


def _wire_maxpool(x, y, shape):
    N, H, W, C = shape
    return [N, H, W, C], [], _act(x) + _act(y)


def _wire_avgpool(x, y, shape):
    N, H, W, C = shape
    return [N, H * W, C], [], _act(x) + [y]


def _wire_linear(x, w, b, add, y):
    return [x.shape[0], w.shape[1], w.shape[0]], [], [x, w, b, add, y]


def _wire_clean_global(heads, body, amax, vis, shape):
    B, H, W, Ch, Cb = shape
    vis = list(vis) if vis is not None else [None] * 4
    return [B, H * W, Ch, 0, 25, 50, 75, Cb], [], [heads.f32] + _act(body) + [amax] + vis


def _wire_clean_parts(x, y, raw, shape):
    N, H, W, Cx, Cy = shape
    return [N, H * W, Cx, Cy], [], [x.f32] + _act(y) + [raw]


def _wire_stn_params(hm, amax, ratio, offset, vis_thresh, align_corners, centers, theta):
    B, S, _, Chm = hm.f32.shape
    return [B, S, Chm, int(align_corners)], [float(vis_thresh)], [hm.f32, amax, ratio, offset, centers, theta]


def _wire_stn_sample(xd, theta, align_corners, crops, shape):
    B, S, C = shape
    return [B, S, C, int(align_corners)], [], _act(xd) + [theta] + _act(crops)


def _wire_gcn_head(gp, rot_feats, gpara, para):
    ints = [para.shape[0]] + [int(w.shape[0]) for w in gp["W"]] + [int(w.shape[1]) for w in gp["W"]]
    ptrs = [gp["adj"]] + gp["W"] + gp["b"] + gp["bn_scale"] + gp["bn_shift"] + \
           [gp["head_w"], gp["head_b"], gp["mean_pose"], rot_feats, gpara, para]
    return ints, [], ptrs


_WIRE = {"nchw_to_nhwc": _wire_nchw_to_nhwc, "conv_group": _wire_conv_group, "conv2d": _wire_conv2d,
         "fuse_sum": _wire_fuse_sum, "maxpool": _wire_maxpool, "avgpool": _wire_avgpool, "clean_global": _wire_clean_global,
         "clean_parts": _wire_clean_parts, "stn_params": _wire_stn_params, "stn_sample": _wire_stn_sample,
         "linear": _wire_linear, "gcn_head": _wire_gcn_head}


def wire(name, args):
    """(opcode, ints, floats, ptrs) of launch `name` with CudaOps arguments `args`; ptrs are tensors or None."""
    ints, floats, ptrs = _WIRE[name](*args)
    return OPCODES[name], ints, floats, ptrs


class CudaOps(object):
    """Thin tensor-level wrappers over libdanet_b200.so.  Fails loudly without the library / GPU."""

    def __init__(self, device):
        if not torch.cuda.is_available():
            raise RuntimeError("danet_b200: CUDA device required (there is no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device(device)

    def planes(self, precision):
        """fp16 planes per activation on the tensor-core path (0 would mean: fp32 buffers only)."""
        return 2 if precision == "exact" else 1

    def _sp(self):
        return _lib.stream_ptr(self.device)

    @staticmethod
    def _desc(d):
        c = _lib.ConvDesc()
        for k in ("N", "H", "W", "Cin", "Cout", "ksize", "stride", "pad", "wsets", "relu"):
            setattr(c, k, int(d[k]))
        c.flags = int(d.get("flags", 0))
        return c

    def tc_capable(self):
        """The wgmma kernels are sm_90a code: compute capability 9.0 only."""
        return torch.cuda.get_device_capability(self.device) == (9, 0)

    def conv_tc_supported(self, d):
        return bool(self.lib.danet_conv_tc_supported(ctypes.byref(self._desc(d))))

    def conv_tc_pack(self, d, w_simt):
        c = self._desc(d)
        nbytes = int(self.lib.danet_conv_tc_packed_bytes(ctypes.byref(c)))
        if nbytes <= 0:
            raise RuntimeError("danet_b200: convolution %r is not supported by the tensor-core path" % (d,))
        out = torch.empty(nbytes, dtype=torch.uint8, device=w_simt.device)
        _lib.check(self.lib.danet_conv_tc_pack(ctypes.byref(c), _lib.ptr(w_simt), _lib.ptr(out), self._sp()), "conv_tc_pack")
        return out

    # -- launches: each is one step record (`wire`) run by danet_net_run_step --------------------------
    def _run(self, name, *args):
        op, ints, floats, ptrs = wire(name, args)
        _lib.check(self.lib.danet_net_run_step(op, len(ints), (ctypes.c_int32 * len(ints))(*ints),
                                               len(floats), (ctypes.c_float * len(floats))(*floats),
                                               len(ptrs), (ctypes.c_void_p * len(ptrs))(*[_lib.ptr(p) for p in ptrs]),
                                               self._sp()), name)

    def conv_group(self, convs):
        """convs: list of dict(d, x, res, y (ActBuf), w (packed), b)."""
        self._run("conv_group", convs)

    def conv2d(self, d, x, w, bias, res, y):
        """fp32 FMA convolution on the fp32 views."""
        self._run("conv2d", d, x, w, bias, res, y)

    def nchw_to_nhwc(self, x, y):
        self._run("nchw_to_nhwc", x, y)

    def fuse_sum(self, terms, factors, relu, y, shape):
        self._run("fuse_sum", terms, factors, relu, y, shape)

    def maxpool(self, x, y, shape):
        self._run("maxpool", x, y, shape)

    def avgpool(self, x, y, shape):
        self._run("avgpool", x, y, shape)

    def linear(self, x, w, b, add, y):
        self._run("linear", x, w, b, add, y)

    def clean_global(self, heads, body, amax, vis, shape):
        self._run("clean_global", heads, body, amax, vis, shape)

    def clean_parts(self, x, y, raw, shape):
        self._run("clean_parts", x, y, raw, shape)

    def stn_params(self, hm, amax, ratio, offset, vis_thresh, align_corners, centers, theta):
        self._run("stn_params", hm, amax, ratio, offset, vis_thresh, align_corners, centers, theta)

    def stn_sample(self, xd, theta, align_corners, crops, shape):
        self._run("stn_sample", xd, theta, align_corners, crops, shape)

    def gcn_head(self, gp, rot_feats, gpara, para):
        self._run("gcn_head", gp, rot_feats, gpara, para)


def fold_bn(sd, prefix, cout):
    """(scale, shift) of an eval-mode BatchNorm (running stats), fp32 like the reference computes."""
    if prefix is None:
        return torch.ones(cout), torch.zeros(cout)
    g, b = sd[prefix + ".weight"].float().cpu(), sd[prefix + ".bias"].float().cpu()
    m, v = sd[prefix + ".running_mean"].float().cpu(), sd[prefix + ".running_var"].float().cpu()
    scale = g / torch.sqrt(v + BN_EPS)
    return scale, b - m * scale


def pack_conv(sd, op):
    """Conv(+BN) parameters -> SIMT layout: w [wsets][k*k*Cin_p][Cout_p], bias [wsets][Cout_p]."""
    x, y, k, G = op["x"], op["y"], op["k"], op["groups"]
    cin, cin_p, cout_p = x.C, x.Cp, y.Cp
    ws, bs = [], []
    for (wkey, co, has_bias) in op["parts"]:
        w = sd[wkey + ".weight"].float().cpu()                        # [G*co, cin, k, k]
        b = sd[wkey + ".bias"].float().cpu() if has_bias else torch.zeros(G * co)
        ws.append(w.reshape(G, co, cin, k, k))
        bs.append(b.reshape(G, co))
    w = torch.cat(ws, dim=1)                                           # [G, ctot, cin, k, k]
    b = torch.cat(bs, dim=1)
    ctot = w.shape[1]
    scale, shift = fold_bn(sd, op["bn"], G * ctot)
    w = w * scale.reshape(G, ctot, 1, 1, 1)
    b = b * scale.reshape(G, ctot) + shift.reshape(G, ctot)
    wp = torch.zeros(G, k, k, cin_p, cout_p)
    wp[:, :, :, :cin, :ctot] = w.permute(0, 3, 4, 2, 1)
    bp = torch.zeros(G, cout_p)
    bp[:, :ctot] = b
    return wp.reshape(G, k * k * cin_p, cout_p).contiguous(), bp.contiguous()


def refine_adjacency(sd, rp):
    """normalize_undigraph(I_n + A_mask * relu(edge_importance)) (smpl_regressor.py:870-871,
    utils/graph.py:232-261) -- parameter-only, so evaluated once per weight load."""
    I_n = sd[rp + "I_n"].float().cpu()[0]
    A = I_n + sd[rp + "A_mask"].float().cpu()[0] * torch.relu(sd[rp + "edge_importance"].float().cpu()[0])
    d = A.sum(0)
    dn = torch.zeros_like(d)
    dn[d > 0] = d[d > 0] ** (-0.5)
    return torch.matmul(torch.matmul(torch.diag(dn), A), torch.diag(dn))


def pack_gcn(sd, rp, device):
    layers = [("r2p_gcn", 0), ("refine_gcn", 0), ("refine_gcn", 1), ("refine_gcn", 2), ("p2r_gcn", 0)]
    gp = {"W": [], "b": [], "bn_scale": [], "bn_shift": []}
    for name, i in layers:
        gp["W"].append(sd["%s%s.gc.%d.weight" % (rp, name, i)].float().contiguous().to(device))
        gp["b"].append(sd["%s%s.gc.%d.bias" % (rp, name, i)].float().contiguous().to(device))
        s, t = fold_bn(sd, "%s%s.act.%d.0" % (rp, name, i), 24)
        gp["bn_scale"].append(s.contiguous().to(device)); gp["bn_shift"].append(t.contiguous().to(device))
    adj = torch.stack([sd[rp + "r2p_A"].float().cpu()[0], refine_adjacency(sd, rp), sd[rp + "p2r_A"].float().cpu()[0]])
    gp["adj"] = adj.contiguous().to(device)
    gp["head_w"] = sd[rp + "pose_regressors.1.1.weight"].float().reshape(144, 128).contiguous().to(device)
    gp["head_b"] = sd[rp + "pose_regressors.1.1.bias"].float().contiguous().to(device)
    gp["mean_pose"] = sd[rp + "mean_pose"].float().reshape(144).contiguous().to(device)
    return gp


# which views of its input tensors an op needs on the tensor-core path: "h" = fp16 planes, "f" = fp32
_F32_INPUTS = {("clean_global", "x"), ("clean_parts", "x"), ("stn_params", "hm"), ("gcn_head", "x"), ("gcn_head", "gpara"),
               ("stn_sample", "theta")}


def op_inputs(op):
    """(tensor, role) pairs an op reads (`amax` / `theta` are outputs of the op that makes them, inputs of the next)."""
    out = []
    keys = ["x", "res", "hm", "gpara"]
    if op["op"] == "stn_params":
        keys.append("amax")
    if op["op"] == "stn_sample":
        keys.append("theta")
    for key in keys:
        t = op.get(key)
        if t is not None:
            out.append((t, key))
    for (t, _f) in op.get("terms", []):
        out.append((t, "term"))
    return out


def op_outputs(op):
    out = []
    if op.get("y") is not None:
        out.append(op["y"])
    if op["op"] == "clean_global":
        out.append(op["amax"])
    if op["op"] == "stn_params":
        out += [op["theta"], op["centers"]]
    return out


class Plan(object):
    """Compiled forward for a fixed batch size B on one device."""

    RP = "iuv2smpl.smpl_para_Outs."

    def __init__(self, graph, state_dict, B, device, conv_algo="simt", precision="exact", align_corners=False,
                 vis_thresh=0.5, want_vis=True, ops=None, use_cuda_graph=False, group_convs=True, wcache=None,
                 keep_all=False):
        self.g, self.B, self.device = graph, B, torch.device(device)
        self.ops = ops if ops is not None else CudaOps(device)
        self.align_corners, self.vis_thresh, self.want_vis = align_corners, vis_thresh, want_vis
        if conv_algo not in ("simt", "tc"):
            raise ValueError("conv_algo must be 'simt' or 'tc'")
        if precision not in ("exact", "fast"):
            raise ValueError("precision must be 'exact' or 'fast'")
        self.conv_algo, self.precision = conv_algo, precision
        self.tc = conv_algo == "tc"
        if self.tc and hasattr(self.ops, "tc_capable") and not self.ops.tc_capable():
            raise RuntimeError("danet_b200: the tensor-core path is sm_90a code; device %s is not compute capability 9.0" % device)
        self.P = self.ops.planes(precision) if self.tc else 0          # fp16 planes per activation (0: fp32 buffers only)
        self.group_convs = group_convs and self.tc
        self.keep_all = keep_all                      # debugging: no buffer reuse, every intermediate stays readable
        self.wcache = wcache if wcache is not None else {}
        self.n_tc = 0
        self.consts = set()                           # data_ptr of every weight-like tensor a step reads (export: payload)
        sd = state_dict
        dev = self.device
        with self._guard():
            self._schedule()
            self._formats()
            self._plan_buffers()
            S = graph.outputs["heads"].H
            self.vis = None
            self.raw_parts = None
            if want_vis:
                self.vis = [torch.empty(B, c, S, S, device=dev) for c in (25, 25, 25, 15)]
                self.raw_parts = torch.empty(B * 24, 21, S, S, device=dev)
            self.steps = []
            for level_ops in self.schedule:
                group = []
                for op in level_ops:
                    if op["op"] == "conv":
                        cv = self._make_conv(op, sd)
                        if self.tc:
                            group.append(cv)
                        else:
                            self.steps.append(Step("conv2d", (cv["d"], cv["x"], cv["w"], cv["b"], cv["res"], cv["y"])))
                    else:
                        self.steps += self._lower_glue(op, sd)
                # tensor-core convolutions of one level: independent by construction, <= MAX_GROUP per launch,
                # most expensive tiles first (they start first inside the persistent grid)
                group.sort(key=lambda c: -c["cost"])
                for g in self._form_groups(group):
                    self.steps.append(Step("conv_group", (g,)))
        self.n_launch = len(self.steps)
        self.graph_exec = None
        self.use_cuda_graph = use_cuda_graph
        self.static_in = None

    def _form_groups(self, convs):
        """Partition one level's convolutions (cost-descending) into consecutive launches of <= MAX_GROUP."""
        if not self.group_convs:
            return [[c] for c in convs]
        return [convs[i:i + MAX_GROUP] for i in range(0, len(convs), MAX_GROUP)]

    def _guard(self):
        """Kernels, buffers and the stream handle must belong to the plan's device, whatever the caller's
        current device is."""
        if self.device.type == "cuda":
            return torch.cuda.device(self.device)
        import contextlib
        return contextlib.nullcontext()

    # tensors callers read after run() (infer_net, tests): never recycled, always with an fp32 view
    KEEP = ("para", "centers", "theta", "amax", "global_para", "rot_feats", "heads", "hm", "body_iuv")

    def _keep(self):
        return set(self.g.outputs[k].name for k in self.KEEP if k in self.g.outputs)

    # -- scheduling ---------------------------------------------------------------------------
    def _schedule(self):
        """ASAP levels of the op DAG: every op of a level depends only on earlier levels, so the convolutions
        of a level (HRNet's parallel branches, hr_module.py:165-166; the fuse layers' 1x1 and stride-2
        convolutions; the body and limb regressors) may share one launch."""
        level_of_tensor = {}
        levels = []
        for op in self.g.ops:
            lv = 0
            for (t, _role) in op_inputs(op):
                lv = max(lv, level_of_tensor.get(t.name, -1) + 1)
            for t in op_outputs(op):
                level_of_tensor[t.name] = lv
            while len(levels) <= lv:
                levels.append([])
            levels[lv].append(op)
        if not self.group_convs:
            # graph order (one op per step); still expressed as levels
            levels = [[op] for op in self.g.ops]
        self.schedule = [l for l in levels if l]
        self.step_of = {}
        for idx, l in enumerate(self.schedule):
            for op in l:
                self.step_of[id(op)] = idx

    # -- tensor formats -----------------------------------------------------------------------
    def _formats(self):
        """Views each tensor carries.  fp32 path: fp32 only.  Tensor-core path: convolutions, fuse sums, pools and
        the STN sampler exchange split-fp16 planes; the kernels that work on fp32 (iuvmap_clean, soft-argmax,
        GCN head) and the tensors callers read keep an fp32 view."""
        self.fmt = {}
        g = self.g
        for name in g.tensors:
            self.fmt[name] = set()
        keep = self._keep()
        for op in g.ops:
            for (t, role) in op_inputs(op):
                if t.dtype != "f32":
                    continue
                if not self.tc or self.P == 0 or (op["op"], role) in _F32_INPUTS or t.Cp % 8 != 0:
                    self.fmt[t.name].add("f")
                else:
                    self.fmt[t.name].add("h")
        for name in g.tensors:
            t = g.tensors[name]
            if t.dtype != "f32":
                continue
            if name in keep or not self.fmt[name]:
                self.fmt[name].add("f")
        # producers that can only write fp32
        for op in g.ops:
            if op["op"] in ("avgpool", "body_fc", "gcn_head", "stn_params"):
                for t in op_outputs(op):
                    if t.dtype == "f32":
                        if "h" in self.fmt[t.name]:
                            raise RuntimeError("plan: %s output %s is needed as fp16 planes" % (op["op"], t.name))

    # -- buffers ------------------------------------------------------------------------------
    def _plan_buffers(self):
        g, B, dev = self.g, self.B, self.device
        last_use, produced = {}, {}
        for op in g.ops:
            idx = self.step_of[id(op)]
            for (t, _r) in op_inputs(op):
                last_use[t.name] = max(last_use.get(t.name, -1), idx)
            for t in op_outputs(op):
                if t.name not in produced:
                    produced[t.name] = idx
        keep = self._keep()
        free = {}
        self.buf = {}
        release_at = {}
        for name, idx in last_use.items():
            if name not in keep and not self.keep_all:
                release_at.setdefault(idx, []).append(name)
        by_step = {}
        for name, idx in produced.items():
            by_step.setdefault(idx, []).append(name)

        def take(key, maker):
            pool = free.get(key)
            return pool.pop() if pool else maker()

        self._pool_key = {}
        for idx in range(len(self.schedule)):
            for name in by_step.get(idx, []):
                t = g.tensors[name]
                shape = (B * t.nmult, t.H, t.W, t.Cp)
                numel = int(np.prod(shape))
                if t.dtype == "u8":
                    self.buf[name] = torch.empty(shape[:3], dtype=torch.uint8, device=dev)
                    continue
                fm = self.fmt[name]
                f32 = h = None
                if "f" in fm:
                    if name in keep:
                        f32 = torch.empty(shape, device=dev)
                    else:
                        f32 = take(("f", numel), lambda: torch.empty(numel, device=dev)).view(shape)
                if "h" in fm:
                    h = take(("h", numel), lambda: torch.empty(self.P * numel, dtype=torch.float16, device=dev)).view((self.P,) + shape)
                    if name in keep:
                        h = torch.empty((self.P,) + shape, dtype=torch.float16, device=dev)
                self.buf[name] = ActBuf(f32, h)
            for name in release_at.get(idx, []):
                a = self.buf.get(name)
                if not isinstance(a, ActBuf):
                    continue
                if a.f32 is not None:
                    free.setdefault(("f", a.f32.numel()), []).append(a.f32.reshape(-1))
                if a.h is not None:
                    free.setdefault(("h", a.h.numel() // self.P), []).append(a.h.reshape(-1))
        seen = {}
        for a in self.buf.values():
            for t in ([a] if torch.is_tensor(a) else [a.f32, a.h]):
                if t is not None:
                    seen[t.untyped_storage().data_ptr()] = t.untyped_storage().nbytes()
        self.bytes_alloc = sum(seen.values())

    def T(self, t):
        return self.buf[t.name]

    def shape(self, t):
        return (self.B * t.nmult, t.H, t.W, t.Cp)

    # -- conv ---------------------------------------------------------------------------------
    def _conv_desc(self, op):
        x, y = op["x"], op["y"]
        return dict(N=self.B * x.nmult, H=x.H, W=x.W, Cin=x.Cp, Cout=y.Cp, ksize=op["k"], stride=op["stride"],
                    pad=op["pad"], wsets=op["groups"], relu=int(op["relu"]),
                    flags=4 if (self.tc and self.precision == "exact") else 0)

    def _make_conv(self, op, sd):
        x, y = op["x"], op["y"]
        d = self._conv_desc(op)
        dev = self.device
        key = (op["parts"][0][0], "tc" if self.tc else "simt", d["flags"], x.Cp, y.Cp)
        if key not in self.wcache:
            w, b = pack_conv(sd, op)
            w, b = w.to(dev), b.to(dev)
            if self.tc:
                if not self.ops.conv_tc_supported(d):
                    raise RuntimeError("plan: convolution %r is not supported by the tensor-core path" % (d,))
                w = self.ops.conv_tc_pack(d, w)
            self.wcache[key] = (w, b)
        w, b = self.wcache[key]
        self._const(w, b)
        if self.tc:
            self.n_tc += 1
        Ho, Wo = y.H, y.W
        cost = float(d["N"]) * Ho * Wo * d["ksize"] ** 2 * d["Cin"] * d["Cout"]
        return dict(d=d, w=w, b=b, x=self.T(x), y=self.T(y), res=self.T(op["res"]) if op["res"] is not None else None,
                    cost=cost, op=op)

    def _const(self, *ts):
        """Marks weight-like tensors: an exported program carries them in its payload."""
        self.consts.update(t.data_ptr() for t in ts)

    def _lower_glue(self, op, sd):
        """Step records of one op that is not a convolution."""
        kind, T, dev, B = op["op"], self.T, self.device, self.B
        x, y = op.get("x"), op.get("y")
        if kind == "input":
            # `run` puts the caller's image in place of this placeholder; export refers to the program's input
            self.image = torch.empty(B, 3, y.H, y.W, device="meta")
            return [Step("nchw_to_nhwc", (self.image, T(y)))]
        if kind == "fuse":
            terms = op["terms"]
            return [Step("fuse_sum", ([T(t) for t, _ in terms], [f for _, f in terms], op["relu"], T(y), self.shape(y)))]
        if kind == "maxpool":
            return [Step("maxpool", (T(x), T(y), self.shape(x)))]
        if kind == "avgpool":
            return [Step("avgpool", (T(x), T(y).f32, self.shape(x)))]
        if kind == "clean_global":
            return [Step("clean_global", (T(x), T(y), T(op["amax"]), self.vis, (B, x.H, x.W, x.Cp, y.Cp)))]
        if kind == "stn_params":
            ratio = sd["img2iuv.learned_ratio"].float().contiguous().to(dev)
            offset = sd["img2iuv.learned_offset"].float().contiguous().to(dev)
            self._const(ratio, offset)
            return [Step("stn_params", (T(op["hm"]), T(op["amax"]), ratio, offset, self.vis_thresh, self.align_corners,
                                        T(op["centers"]).f32, T(op["theta"]).f32))]
        if kind == "stn_sample":
            return [Step("stn_sample", (T(x), T(op["theta"]).f32, self.align_corners, T(y), (B, x.H, x.Cp)))]
        if kind == "clean_parts":
            return [Step("clean_parts", (T(x), T(y), self.raw_parts, (B * x.nmult, x.H, x.W, x.Cp, y.Cp)))]
        if kind == "body_fc":
            fc_w = sd[self.RP + "body_net.3.final_layer.weight"].float().contiguous().to(dev)
            fc_b = sd[self.RP + "body_net.3.final_layer.bias"].float().contiguous().to(dev)
            fc_add = sd[self.RP + "mean_cam_shape"].float().reshape(13).contiguous().to(dev)
            self._const(fc_w, fc_b, fc_add)
            self.pooled = torch.empty(B, 512, device=dev)
            return [Step("avgpool", (T(x), self.pooled, self.shape(x))),
                    Step("linear", (self.pooled, fc_w, fc_b, fc_add, T(y).f32))]
        if kind == "gcn_head":
            gp = self.gcn = pack_gcn(sd, self.RP, dev)
            self._const(gp["adj"], *gp["W"], *gp["b"], *gp["bn_scale"], *gp["bn_shift"], gp["head_w"], gp["head_b"],
                        gp["mean_pose"])
            return [Step("gcn_head", (gp, T(x).f32, T(op["gpara"]).f32, T(y).f32))]
        raise ValueError("unknown op %s" % kind)

    # -- run ----------------------------------------------------------------------------------
    def _run_steps(self, image):
        for s in self.steps:
            args = (image,) + s.args[1:] if s.args[0] is self.image else s.args
            getattr(self.ops, s.name)(*args)

    def run(self, image):
        """image [B,3,H,W] fp32 NCHW on the plan's device.  Results stay in the plan's buffers."""
        if image.shape[0] != self.B:
            raise ValueError("plan compiled for batch %d, got %d" % (self.B, image.shape[0]))
        image = image.detach().to(self.device, torch.float32).contiguous()
        with self._guard():
            if not self.use_cuda_graph:
                self._run_steps(image)
                return
            cur = torch.cuda.current_stream(self.device)
            if self.graph_exec is None:
                self.static_in = image.clone()
                s = torch.cuda.Stream(device=self.device)
                s.wait_stream(cur)
                with torch.cuda.stream(s):
                    self._run_steps(self.static_in)          # warm-up outside capture
                cur.wait_stream(s)
                self.graph_exec = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph_exec):
                    self._run_steps(self.static_in)
            self.static_in.copy_(image, non_blocking=True)
            self.graph_exec.replay()

    # -- export ---------------------------------------------------------------------------------
    def export(self, path=None):
        """Serialise this plan as a network program for danet_net_load (csrc/net.cu, include/danet_b200.h): the launch
        steps with their arguments, the activation buffer table and the folded / packed weights.  Returns the bytes
        (and writes them to `path` when given).  The program is tied to this plan's batch size and precision."""
        import struct
        bufs, consts = {}, {}                          # storage ptr -> (id, nbytes) ; tensor ptr -> (id, tensor)

        def ref(t):
            """(kind, id, offset) of one pointer: 0 null, 1 activation buffer, 2 constant, 3 the input image."""
            if t is None:
                return (0, 0, 0)
            if t is self.image:
                return (3, 0, 0)
            key = t.data_ptr()
            if key in self.consts:
                if not t.is_contiguous():
                    raise RuntimeError("export: constant tensors must be contiguous")
                if key not in consts:
                    consts[key] = (len(consts), t)
                return (2, consts[key][0], 0)
            st = t.untyped_storage()
            key = st.data_ptr()
            if key not in bufs:
                bufs[key] = (len(bufs), st.nbytes())
            return (1, bufs[key][0], t.data_ptr() - key)

        step_bytes = b""
        for s in self.steps:
            code, ints, floats, ptrs = wire(s.name, s.args)
            step_bytes += struct.pack("<4I", code, len(ints), len(floats), len(ptrs))
            step_bytes += struct.pack("<%di" % len(ints), *ints) + struct.pack("<%df" % len(floats), *floats)
            for p in ptrs:
                step_bytes += struct.pack("<IIQ", *ref(p))

        outs = []                                       # (name, ref, elem_bytes, dims)
        for k in self.KEEP:
            if k not in self.g.outputs:
                continue
            a = self.T(self.g.outputs[k])
            t = a if torch.is_tensor(a) else a.f32
            outs.append((k, ref(t), t.element_size(), list(t.shape)))
        if self.vis is not None:
            for nm, t in zip(("vis_u", "vis_v", "vis_i", "vis_a"), self.vis):
                outs.append((nm, ref(t), 4, list(t.shape)))
            outs.append(("part_iuv_raw", ref(self.raw_parts), 4, list(self.raw_parts.shape)))

        def pad16(b):
            return b + b"\0" * (-len(b) % 16)

        buf_list = sorted(bufs.values())
        const_list = sorted(consts.values(), key=lambda c: c[0])
        hdr_size = 8 + 12 * 4 + 4 * 8
        tables_size = 8 * len(buf_list) + 16 * len(const_list) + 72 * len(outs)
        steps_off = (hdr_size + tables_size + 15) // 16 * 16
        payload_off = (steps_off + len(step_bytes) + 15) // 16 * 16
        crecs, off = [], payload_off
        for (_i, t) in const_list:
            n = t.numel() * t.element_size()
            crecs.append((off, n))
            off += (n + 15) // 16 * 16
        payload_bytes = off - payload_off
        prec = 2 if not self.tc else (1 if self.precision == "exact" else 0)
        blob = bytearray()
        blob += b"DANETPRG" + struct.pack("<12I", 1, *self.image.shape, len(buf_list), len(const_list), len(outs), len(self.steps), prec,
                                             0, 0)
        blob += struct.pack("<4Q", steps_off, len(step_bytes), payload_off, payload_bytes)
        for (_i, nbytes) in buf_list:
            blob += struct.pack("<Q", nbytes)
        for (o, n) in crecs:
            blob += struct.pack("<QQ", o, n)
        for (name, r, eb, dims) in outs:
            d = (list(dims) + [1, 1, 1, 1])[:4]
            if len(dims) > 4:
                raise RuntimeError("export: output %s has more than 4 dims" % name)
            blob += name.encode()[:31].ljust(32, b"\0") + struct.pack("<IIQ", *r) + struct.pack("<Ii4i", eb, len(dims), *d)
        blob += b"\0" * (steps_off - len(blob))
        blob += step_bytes
        blob += b"\0" * (payload_off - len(blob))
        with self._guard():
            for (_i, t), (o, n) in zip(const_list, crecs):
                assert len(blob) == o
                blob += pad16(t.detach().reshape(-1).view(torch.uint8).cpu().numpy().tobytes())
        blob = bytes(blob)
        if path is not None:
            with open(path, "wb") as f:
                f.write(blob)
        return blob

    def out(self, name):
        """fp32 tensor of a graph output."""
        a = self.T(self.g.outputs[name])
        return a if torch.is_tensor(a) else a.value()
