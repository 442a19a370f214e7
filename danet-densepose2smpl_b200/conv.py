"""Differentiable convolution on the tensor-core engine, exact (split-fp16, fp32-grade) precision:

    from danet_b200.conv import conv2d
    y = conv2d(x, weight, bias, stride, padding, dilation, groups)    # instead of torch.nn.functional.conv2d

Same meaning and argument order as torch.nn.functional.conv2d, for fp32 NCHW CUDA tensors and the shapes the tensor-core
path accepts: kernel size 1 or 3 with stride 1 or 2, or 7 with stride 2; padding k // 2, dilation 1, any groups.  These
cover every convolution of the network.  Anything else raises ValueError; there is no fall-back to torch.  Channel counts
need not be multiples of 8: the op pads them internally.

- Forward: x becomes scaled split-fp16 NHWC planes (danet_conv_grad_split), the current weights are packed on every
  call (danet_conv_tc_pack: they change every optimiser step), danet_conv_tc_group runs the convolution without the
  bias, and danet_conv_dgrad_scatter writes the fp32 NCHW result: x's scale removed, then the bias added.
- Input gradient: forward problems of the same engine.  Stride 1 is conv(dy, W') with W' the rotated filter.  Stride 2
  splits each output-parity class of dx into 1x1 / 3x3 stride-1 pieces (a 4-tap 7x7/s2 parity becomes a centred 3-tap
  window plus a 1-tap piece read back shifted by one pixel), runs them as multi-problem launches and sums them into dx.
- Weight and bias gradients: danet_conv_wgrad, a wgmma implicit GEMM over the pixels with split K and a fixed-order
  finishing sum (csrc/conv_wgrad.cu).

`backward` computes only the gradients in ctx.needs_input_grad.  Results repeat bit for bit, nothing synchronises with the
host, and forward + backward can be captured in a CUDA graph.  `groups = G` maps onto the engine's weight sets over the
(batch, group)-flattened image axis, the lowering the inference plan uses for the reference's grouped convolutions.

Precision: x and dy are each scaled by a power of two found on the device from their max |v| before the fp16 hi + lo
split (the weights are too, when they are packed), and the scales are removed exactly afterwards, so operands of any
magnitude keep fp32-grade precision.  The bias never enters a scaled sum.  db sums the fp32 dy.  NaN and +-inf in x, dy
or the weights stay non-finite in every output they reach."""
import ctypes

import torch
from torch.autograd.function import once_differentiable

from . import _args, _lib

EXACT = 4                         # DANET_CONV_EXACT
_MAX_PROBLEMS = 6                 # problems per danet_conv_tc_group launch


def _ceil8(c):
    return (c + 7) // 8 * 8


def _desc(N, H, W, Cin, Cout, k, stride, wsets):
    d = _lib.ConvDesc()
    d.N, d.H, d.W, d.Cin, d.Cout, d.ksize, d.stride, d.pad, d.wsets, d.relu, d.flags = \
        N, H, W, Cin, Cout, k, stride, k // 2, wsets, 0, EXACT
    return d


def _planes(shape, dev):
    return (torch.empty(shape, dtype=torch.float16, device=dev), torch.empty(shape, dtype=torch.float16, device=dev))


def _split_scaled(t, N, C, HW, Cp, shape, dev):
    """fp32 NCHW [N, C, HW] -> split-fp16 NHWC planes [shape] of t * 2^s with Cp >= C channels (pad channels zero), and
    the scale [2^s, 2^-s, -, -] (danet_conv_grad_split)"""
    hi, lo = _planes(shape, dev)
    scale = torch.empty(4, dtype=torch.float32, device=dev)
    _lib.call("conv_grad_split", N, C, HW, Cp, _lib.ptr(t), _lib.ptr(hi), _lib.ptr(lo), _lib.ptr(scale), device=dev)
    return (hi, lo), scale


def _pack(d, w_simt, dev):
    nbytes = int(_lib.load().danet_conv_tc_packed_bytes(ctypes.byref(d)))
    if nbytes <= 0:
        raise ValueError("danet_b200.conv.conv2d: shape not supported by the tensor-core path")
    pk = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.call("conv_tc_pack", ctypes.byref(d), _lib.ptr(w_simt), _lib.ptr(pk), device=dev)
    return pk


def _problem(d, x_planes, pk, bias, y):
    p = _lib.ConvProblem()
    p.d = d
    p.x = _lib.Act(None, x_planes[0].data_ptr(), x_planes[1].data_ptr())
    p.res = _lib.Act(None, None, None)
    p.y = _lib.Act(y.data_ptr(), None, None)
    p.w_packed = pk.data_ptr()
    p.bias = bias.data_ptr() if bias is not None else None
    return p


_PIECES = {}


def _pieces(k, stride):
    """the input-gradient pieces of a (k, stride) convolution (danet_conv_dgrad_pieces), cached"""
    key = (k, stride)
    if key not in _PIECES:
        arr = (_lib.DgradPiece * 9)()
        n = int(_lib.load().danet_conv_dgrad_pieces(k, stride, arr))
        if n < 0:
            raise ValueError("danet_b200.conv.conv2d: no input gradient for k=%d stride=%d" % (k, stride))
        _PIECES[key] = ((_lib.DgradPiece * max(n, 1))(*arr[:n]), n)
    return _PIECES[key]


def _scatter(pieces, n, maps, N, C, H, W, Cp, stride, Hc, Wc, scale, dev, bias=None, G=1):
    """NHWC piece maps -> fp32 NCHW [N, C, H, W] (summed per class, shifted, cropped, scale removed, then the bias
    [G * C] of image n's group n % G added)"""
    y = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
    arr = (ctypes.c_void_p * max(n, 1))(*[m.data_ptr() for m in maps])
    _lib.call("conv_dgrad_scatter", N, C, H, W, Cp, stride, Hc, Wc, n, pieces, arr, _lib.ptr(scale), _lib.ptr(bias), G,
              _lib.ptr(y), device=dev)
    return y


class _Conv2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, stride, groups):
        dev = x.device
        B, Ct, H, W = x.shape
        Cot, cin, k, _ = weight.shape
        G = groups
        cout, N = Cot // G, B * G
        Cinp, Coutp = _ceil8(cin), _ceil8(cout)
        Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
        d = _desc(N, H, W, Cinp, Coutp, k, stride, G)
        with torch.cuda.device(dev):
            xp, x_scale = _split_scaled(x, N, cin, H * W, Cinp, (N, H, W, Cinp), dev)
            w_simt = torch.empty(G * k * k * Cinp * Coutp, dtype=torch.float32, device=dev)
            _lib.call("conv_weights_simt", G, cout, cin, k, Coutp, Cinp, _lib.ptr(weight), _lib.ptr(w_simt), device=dev)
            pk = _pack(d, w_simt, dev)
            # the engine's sum is of x * 2^s: the bias joins after the scatter has removed 2^s
            y_nhwc = torch.empty(N, Ho, Wo, Coutp, dtype=torch.float32, device=dev)
            arr = (_lib.ConvProblem * 1)(_problem(d, xp, pk, None, y_nhwc))
            _lib.call("conv_tc_group", 1, arr, device=dev)
            one = (_lib.DgradPiece * 1)(_lib.DgradPiece(0, 0, k, 0, 0, 0, 0, 0, 0))
            y = _scatter(one, 1, [y_nhwc], N, cout, Ho, Wo, Coutp, 1, Ho, Wo, x_scale, dev, bias, G)
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        ctx.save_for_backward(weight if need_dx else None, xp[0] if need_dw else None, xp[1] if need_dw else None,
                              x_scale if need_dw else None)
        ctx.geom = (B, Ct, H, W, Cot, cin, cout, k, stride, G, Ho, Wo)
        return y.view(B, Cot, Ho, Wo)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        weight, x_hi, x_lo, x_scale = ctx.saved_tensors
        B, Ct, H, W, Cot, cin, cout, k, stride, G, Ho, Wo = ctx.geom
        need_dx, need_dw, need_db = ctx.needs_input_grad[:3]
        N, Cinp, Coutp = B * G, _ceil8(cin), _ceil8(cout)
        dev = gy.device
        dx = dw = db = None
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            if need_dx or need_dw:
                # dy * 2^s as split planes, 2^s from max |dy| on the device: small gradients keep their 22 bits
                dyp, scale = _split_scaled(gy, N, cout, Ho * Wo, Coutp, (N, Ho, Wo, Coutp), dev)
            if need_dx:
                pieces, n = _pieces(k, stride)
                probs, outs, keep = [], [], []
                for i in range(n):
                    pc = pieces[i]
                    dd = _desc(N, Ho, Wo, Coutp, Cinp, pc.K, 1, G)
                    wc = torch.empty(G * pc.K * pc.K * Coutp * Cinp, dtype=torch.float32, device=dev)
                    _lib.call("conv_dgrad_weights", G, cout, cin, k, stride, ctypes.byref(pc), Coutp, Cinp, _lib.ptr(weight),
                              _lib.ptr(wc), device=dev)
                    pk = _pack(dd, wc, dev)
                    o = torch.empty(N, Ho, Wo, Cinp, dtype=torch.float32, device=dev)
                    probs.append(_problem(dd, dyp, pk, None, o))
                    outs.append(o)
                    keep += [wc, pk]
                for i in range(0, n, _MAX_PROBLEMS):          # the engine runs up to 6 problems per launch
                    grp = probs[i:i + _MAX_PROBLEMS]
                    arr = (_lib.ConvProblem * len(grp))(*grp)
                    _lib.call("conv_tc_group", len(grp), arr, device=dev)
                dx = _scatter(pieces, n, outs, N, cin, H, W, Cinp, stride, Ho, Wo, scale, dev).view(B, Ct, H, W)
            if need_dw:
                d = _desc(N, H, W, Cinp, Coutp, k, stride, G)
                ws = _lib.workspace(_lib.load().danet_conv_wgrad_workspace_bytes(ctypes.byref(d)), dev)
                dw = torch.empty(Cot, cin, k, k, dtype=torch.float32, device=dev)
                xa = _lib.Act(None, x_hi.data_ptr(), x_lo.data_ptr())
                da = _lib.Act(None, dyp[0].data_ptr(), dyp[1].data_ptr())
                _lib.call("conv_wgrad", ctypes.byref(d), cout, cin, ctypes.byref(xa), ctypes.byref(da), _lib.ptr(scale),
                          _lib.ptr(x_scale), _lib.ptr(dw), _lib.ptr(ws), device=dev)
            if need_db:
                # from the fp32 dy itself
                ws = _lib.workspace(_lib.load().danet_conv_bias_grad_workspace_bytes(B, Cot, Ho * Wo), dev)
                db = torch.empty(Cot, dtype=torch.float32, device=dev)
                _lib.call("conv_bias_grad", B, Cot, Ho * Wo, _lib.ptr(gy), _lib.ptr(db), _lib.ptr(ws), device=dev)
        return dx, dw, db, None, None


def conv2d(x, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    """torch.nn.functional.conv2d on the tensor-core engine (exact mode), differentiable.  See the module docstring."""
    where = "danet_b200.conv.conv2d"
    stride = _args.int_pair(where, "stride", stride)
    padding = _args.int_pair(where, "padding", padding)
    dilation = _args.int_pair(where, "dilation", dilation)
    if isinstance(groups, bool) or not isinstance(groups, int) or groups < 1:
        raise ValueError("%s: groups must be a positive int (got %r)" % (where, groups))
    tensors = [(name, t) for name, t in (("x", x), ("weight", weight), ("bias", bias)) if t is not None]
    for name, t in tensors:                     # each tensor in turn: type, CUDA, dtype
        _args.cuda(where, [(name, t)])
        _args.tensor(where, name, t, contiguous=False)
    if x.dim() != 4 or weight.dim() != 4:
        raise ValueError("danet_b200.conv.conv2d: x and weight must be 4-D (NCHW, OIHW)")
    _args.cuda(where, tensors)                  # one device
    Cot, cin, kh, kw = weight.shape
    if kh != kw or kh not in (1, 3, 7):
        raise ValueError("danet_b200.conv.conv2d: kernel size must be 1, 3 or 7 and square (got %dx%d)" % (kh, kw))
    if padding != kh // 2:
        raise ValueError("danet_b200.conv.conv2d: padding must be k // 2 = %d (got %d)" % (kh // 2, padding))
    if stride not in (1, 2):
        raise ValueError("danet_b200.conv.conv2d: stride must be 1 or 2 (got %d)" % stride)
    if kh == 7 and stride != 2:
        raise ValueError("danet_b200.conv.conv2d: a 7x7 convolution must have stride 2 (the engine's limit)")
    if dilation != 1:
        raise ValueError("danet_b200.conv.conv2d: dilation must be 1 (got %d)" % dilation)
    if x.shape[1] != groups * cin or Cot % groups != 0:
        raise ValueError("danet_b200.conv.conv2d: channels do not match groups=%d (x %s, weight %s)"
                         % (groups, tuple(x.shape), tuple(weight.shape)))
    if bias is not None and tuple(bias.shape) != (Cot,):
        raise ValueError("danet_b200.conv.conv2d: bias must have shape (%d,)" % Cot)
    if x.shape[0] < 1 or x.shape[2] < 1 or x.shape[3] < 1:
        raise ValueError("danet_b200.conv.conv2d: empty input")
    return _Conv2d.apply(x.contiguous(), weight.contiguous(), bias.contiguous() if bias is not None else None, stride, groups)
