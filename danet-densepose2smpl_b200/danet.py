"""DaNet with the reference's call surface (models/danet/danet.py:31-131):

    model = DaNet(options, smpl_mean_params, pretrained=False).to(device)
    model.load_state_dict(checkpoint['model'], strict=False); model.eval()
    pred = model.infer_net(image)            # {'para': [B,229], 'visualization': {...}}

Parameters live under the reference's state_dict key names (img2iuv.iuv_est.*,
img2iuv.learned_{ratio,offset}, iuv2smpl.smpl_para_Outs.*, iuv2smpl.smpl.*); the forward is an
execution plan over the CUDA kernels of libdanet_b200.so (plan.py), not torch modules.
"""
import math
import os

import numpy as np
import torch
import torch.nn as nn

from . import constants
from . import netgraph as ng
from .plan import Plan
from .renderer import IUV_Renderer
from .smpl import SMPL

# configs/danet_default.yaml values the inference path reads (SURVEY section 5)
DEFAULT_CFG = dict(INIMG_SIZE=224, HEATMAP_SIZE=56, STN_PART_VIS_SCORE=0.5, WIDTH=48,
                   PRETRAINED_COCO="data/pretrained_model/pose_hrnet_w48_256x192.pth",
                   PRETRAINED_18="data/pretrained_model/resnet18-5c106cde.pth",
                   SMPL_MODEL_DIR="data/smpl")


class ParamTree(nn.Module):
    """Container that registers tensors under dotted reference key names."""

    def add(self, key, tensor, kind="param"):
        head, _, rest = key.partition(".")
        if rest:
            if head not in self._modules:
                self.add_module(head, ParamTree())
            self._modules[head].add(rest, tensor, kind)
        elif kind == "param":
            self.register_parameter(head, nn.Parameter(tensor, requires_grad=tensor.is_floating_point()))
        else:
            self.register_buffer(head, tensor)


def _init_tensor(spec, mean_params, gbuf):
    shape, init = spec.shape, spec.init
    if init == "ones":
        return torch.ones(shape)
    if init == "zeros":
        return torch.zeros(shape)
    if init == "long0":
        return torch.zeros(shape, dtype=torch.long)
    if init == "conv" or init == "linear":
        fan_in = int(np.prod(shape[1:]))
        return (torch.rand(shape) * 2 - 1) / math.sqrt(fan_in)
    if init.startswith("conv_bias:"):
        return (torch.rand(shape) * 2 - 1) / math.sqrt(int(init.split(":")[1]))
    if init == "xavier_relu":
        bound = math.sqrt(2.0) * math.sqrt(6.0 / (shape[0] + shape[1]))
        return (torch.rand(shape) * 2 - 1) * bound
    if init == "xavier_small":
        bound = 0.01 * math.sqrt(6.0 / (shape[0] + shape[1]))
        return (torch.rand(shape) * 2 - 1) * bound
    if init == "learned_ratio":
        return torch.from_numpy(constants.LEARNED_RATIO.copy())
    if init == "learned_offset":
        return torch.from_numpy(constants.LEARNED_OFFSET.copy())
    if init == "mean_cam_shape":
        return torch.cat([torch.as_tensor(mean_params["cam"], dtype=torch.float32).reshape(1, 3),
                          torch.as_tensor(mean_params["shape"], dtype=torch.float32).reshape(1, 10)], dim=1)
    if init == "mean_pose":
        return torch.as_tensor(mean_params["pose"], dtype=torch.float32).reshape(1, 144)
    if init.startswith("graph:"):
        return torch.from_numpy(gbuf[init.split(":")[1]].copy())
    raise ValueError(init)


def load_mean_params(smpl_mean_params):
    if isinstance(smpl_mean_params, dict):
        return smpl_mean_params
    if not os.path.exists(smpl_mean_params):
        raise ValueError("%s does not exist (smpl_mean_params, reference README.md:44-48)" % smpl_mean_params)
    z = np.load(smpl_mean_params)
    return {k: z[k] for k in ("pose", "shape", "cam")}


class DaNet(nn.Module):
    """Decompose-and-aggregate network, inference path (INPUT_MODE='iuv', DECOMPOSED, 'gcn')."""

    def __init__(self, options, smpl_mean_params, pretrained=True, width=None, smpl_model=None, dp_mesh=None,
                 conv_algo="auto", precision="exact", legacy_align_corners=False, cfg=None, use_cuda_graph=False,
                 want_vis=True, group_convs=True):
        super().__init__()
        self.options = options
        self.cfg = dict(DEFAULT_CFG)
        if cfg:
            self.cfg.update(cfg)
        self.width = width or self.cfg["WIDTH"]
        # conv_algo: 'auto' / 'tc' = wgmma tensor-core convolutions (sm_90a), 'simt' = fp32 FMA kernels (an
        # independent fp32 check path).  precision (tensor-core path): 'exact' = split-fp16 operands, three MMAs per
        # K step, fp32-grade results (the reference computes in fp32; this is the default and what parity is
        # stated for); 'fast' = single fp16 pass (~1e-3 on para), about twice the throughput.
        self.conv_algo = conv_algo
        self.precision = precision
        self.legacy_align_corners = legacy_align_corners
        self.use_cuda_graph = use_cuda_graph
        self.group_convs = group_convs               # independent convolutions of one graph level share a launch
        self.want_vis = want_vis
        self.graph = ng.danet_graph(self.width, self.cfg["INIMG_SIZE"])
        mean_params = load_mean_params(smpl_mean_params)
        gbuf = ng.graph_buffers()
        self.img2iuv = ParamTree()
        self.iuv2smpl = ParamTree()
        for key, spec in self.graph.params.items():
            root, rest = key.split(".", 1)
            getattr(self, root).add(rest, _init_tensor(spec, mean_params, gbuf), spec.kind)
        self.img2iuv.dp2smpl_mapping = constants.DP2SMPL_MAPPING                    # demo.py:139
        bs = getattr(options, "batch_size", 1) if options is not None else 1
        self.iuv2smpl.smpl = SMPL(smpl_model if smpl_model is not None else self.cfg["SMPL_MODEL_DIR"],
                                  batch_size=bs, create_transl=False)                   # smpl_regressor.py:64
        self.iuv_renderer = IUV_Renderer(self.cfg["INIMG_SIZE"], self.cfg["HEATMAP_SIZE"], mesh=dp_mesh)  # danet.py:59
        self._plans = {}
        self._wcache = {}                              # packed weights, shared by the plans of every batch size
        if pretrained:
            self._load_pretrained()
        self.train()                                     # nn.Module default; callers call .eval()

    # -- pretrained backbones (iuv_estimator.py:46-54, smpl_regressor.py:438-439,501-502) --------
    def _load_pretrained(self):
        hr = self.cfg["PRETRAINED_COCO"]
        if not os.path.isfile(hr):
            raise ValueError("{} is not exist!".format(hr))                           # hr_module.py:408-410
        sd = torch.load(hr, map_location="cpu")
        self.img2iuv.iuv_est.load_state_dict(sd, strict=False)
        r18 = self.cfg["PRETRAINED_18"]
        if not os.path.isfile(r18):
            raise ValueError("imagenet pretrained model does not exist")             # res_module.py:493-497
        sd = torch.load(r18, map_location="cpu")
        for net in (self.iuv2smpl.smpl_para_Outs.body_net._modules["3"], self.iuv2smpl.smpl_para_Outs.limb_net._modules["3"]):
            own = net.state_dict()
            net.load_state_dict({k: v for k, v in sd.items() if k in own and own[k].shape == v.shape}, strict=False)

    # -- plan cache -----------------------------------------------------------------------------
    MAX_PLANS = 4                                      # batch sizes kept compiled (LRU)
    MAX_BATCH = 256                                    # images per plan; larger batches are chunked (infer_net)

    def _invalidate(self):
        self._plans = {}
        self._wcache = {}
        self.__dict__["_vt"] = None                      # tensors may have been replaced (.to(), load_state_dict)

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **kw):
        self._invalidate()
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def _algo(self):
        if self.conv_algo == "auto":
            return "tc"
        return self.conv_algo

    def plan_for(self, B, device, ops=None):
        """Compiled plan for batch size B (cached, LRU over MAX_PLANS batch sizes; packed weights are shared).
        `ops` replaces the kernel layer (plan.CudaOps) -- used by the host-logic tests, which drive a Plan directly."""
        # plans snapshot the (folded, packed) weights: in-place parameter edits bump tensor versions and invalidate them
        # (flat tensor list cached: walking the module tree costs 3 ms per call, the flat sum 0.13 ms)
        vt = self.__dict__.get("_vt")
        if vt is None:
            vt = [t for t in list(self.parameters()) + list(self.buffers())]
            self.__dict__["_vt"] = vt
        ver = sum(t._version for t in vt)
        if ver != self.__dict__.get("_param_version"):
            self._plans = {}
            self._wcache = {}
            self.__dict__["_param_version"] = ver
        key = (B, str(device), id(ops) if ops is not None else 0)
        if key in self._plans:
            self._plans[key] = self._plans.pop(key)            # most recently used last
            return self._plans[key]
        sd = {k: v for k, v in self.state_dict().items() if not k.startswith("iuv2smpl.smpl.")}
        wc = self._wcache.setdefault((str(device), self._algo(), self.precision, id(ops) if ops is not None else 0), {})
        plan = Plan(self.graph, sd, B, device, conv_algo=self._algo(), precision=self.precision,
                    align_corners=self.legacy_align_corners, vis_thresh=self.cfg["STN_PART_VIS_SCORE"],
                    want_vis=self.want_vis, ops=ops, use_cuda_graph=self.use_cuda_graph,
                    group_convs=self.group_convs, wcache=wc)
        while len(self._plans) >= self.MAX_PLANS:
            self._plans.pop(next(iter(self._plans)))
        self._plans[key] = plan
        return plan

    def outputs_of(self, plan, B):
        """The reference's infer_net return value (danet.py:118-131) from a plan that has run.  `para` and
        `stn_kps_pred` are fresh tensors; the visualisation maps are VIEWS of the plan's buffers (404 MB at
        B = 64: not copied per call) and are overwritten by the next infer_net of the same batch size."""
        S = self.cfg["HEATMAP_SIZE"]
        ret = {"visualization": {}}
        ret["para"] = plan.out("para").reshape(-1)[:B * 229].view(B, 229).clone()
        if plan.vis is not None:
            ret["visualization"]["iuv_pred"] = list(plan.vis)
            ret["visualization"]["part_iuv_pred"] = plan.raw_parts.view(B, 24, 3, 7, S, S)
        ret["stn_kps_pred"] = plan.out("centers").reshape(-1)[:B * 48].view(B, 24, 2).clone()
        return ret

    # -- inference ------------------------------------------------------------------------------
    @torch.no_grad()
    def infer_net(self, image):
        """image [B,3,224,224] fp32 -> {'para': [B,229] = cam(3)|shape(10)|24 rot-mats, 'visualization': ...}"""
        if self.training:
            raise ValueError('You should call this function only on inference.'
                             'Set the network in inference mode by net.eval().')        # danet.py:24-26
        dev = self.img2iuv.learned_ratio.device
        if dev.type != "cuda":
            raise RuntimeError("danet_b200.DaNet: move the model to a CUDA device (there is no CPU path)")
        B = image.shape[0]
        S = self.cfg["HEATMAP_SIZE"]
        if B == 0:                                       # what the reference's modules return for an empty batch
            z = lambda *shape: torch.zeros(*shape, device=dev)
            vis = {"iuv_pred": [z(0, c, S, S) for c in (25, 25, 25, 15)], "part_iuv_pred": z(0, 24, 3, 7, S, S)} if self.want_vis else {}
            return {"para": z(0, 229), "visualization": vis, "stn_kps_pred": z(0, 24, 2)}
        if B > self.MAX_BATCH:
            # the kernels index activations with 32-bit element offsets (the 24 x B part crops are the largest tensor):
            # larger batches run as chunks; their visualisation maps are copied (a plan's buffers are reused per chunk)
            outs = []
            for lo in range(0, B, self.MAX_BATCH):
                o = self.infer_net(image[lo:lo + self.MAX_BATCH])
                o["visualization"] = {k: ([t.clone() for t in v] if isinstance(v, list) else v.clone())
                                      for k, v in o["visualization"].items()}
                outs.append(o)
            ret = {"para": torch.cat([o["para"] for o in outs]), "stn_kps_pred": torch.cat([o["stn_kps_pred"] for o in outs]),
                   "visualization": {}}
            if self.want_vis:
                ret["visualization"]["iuv_pred"] = [torch.cat([o["visualization"]["iuv_pred"][i] for o in outs]) for i in range(4)]
                ret["visualization"]["part_iuv_pred"] = torch.cat([o["visualization"]["part_iuv_pred"] for o in outs])
            return ret
        plan = self.plan_for(B, dev)
        plan.run(image)
        return self.outputs_of(plan, B)

    def export_program(self, batch_size, path=None):
        """Network program of this model for one batch size (bytes; also written to `path`): what the C entry
        danet_net_load / danet_net_infer replays without Python (include/danet_b200.h, INTEGRATION.md)."""
        dev = self.img2iuv.learned_ratio.device
        if dev.type != "cuda":
            raise RuntimeError("danet_b200.DaNet: move the model to a CUDA device (there is no CPU path)")
        return self.plan_for(batch_size, dev).export(path)

    def forward(self, in_dict):
        raise NotImplementedError("danet_b200.DaNet implements the inference path (infer_net); the training "
                                  "forward (danet.py:133-366) is out of scope (SURVEY section 8f)")


def build_synthetic_danet(width=48, seed=0, device="cuda:0", conv_algo="auto", keyed=True, **kw):
    """Random-weight DaNet on synthetic assets (no licensed files / checkpoints needed)."""
    from . import synthetic
    net = DaNet(None, synthetic.make_mean_params(seed), pretrained=False, width=width,
                smpl_model=synthetic.make_smpl_model(seed), dp_mesh=synthetic.make_dp_mesh(seed),
                conv_algo=conv_algo, **kw)
    if keyed:
        net.load_state_dict(synthetic.keyed_state_dict(net.state_dict(), seed), strict=True)
    return net.to(device).eval()
