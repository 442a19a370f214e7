"""Training layers of the regressor's ResNet blocks (body_net, limb_net, limb_reslayer), differentiable, on the GPU
(csrc/bn_train.cu):

    from danet_b200.layers import batch_norm, max_pool2d
    y = batch_norm(x, running_mean, running_var, weight, bias, training, momentum, eps,
                   residual=None, relu=False)      # relu(F.batch_norm(...) + residual)
    y = max_pool2d(x, 3, 2, 1)                     # F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    y = adaptive_avg_pool2d(x, 1)                  # F.adaptive_avg_pool2d(x, 1)
    y = linear(x, weight, bias, add=None)          # F.linear(x, weight, bias) + add (add: a constant [Out] term)
    y = hr_fuse([t0, t1, ...], [f0, f1, ...])      # relu(up(t0, f0) + up(t1, f1) + ...), nearest upsampling

`batch_norm` has the meaning and argument order of torch.nn.functional.batch_norm.  Training mode normalises with the
biased batch variance over (N, H, W) and updates running_mean / running_var in place with `momentum` and the unbiased
variance (the kernel writes the new statistics to a scratch tensor, copied in under no_grad, so the buffers' _version
moves and DaNet.plan_for refolds).  num_batches_tracked belongs to the module and is left alone, as F.batch_norm does.
Eval mode normalises with the running statistics and is still differentiable.  The keyword-only options fuse the
ResNet forms: bn + relu (bn1, the stems), bn + residual + relu (bn2), bn alone (the downsample).  The batch statistics
are sums of x - x[0, c, 0] in double, so the variance keeps its precision at any |mean| / std.  The ReLU is torch's:
NaN stays NaN, and its backward passes dy except where the output is <= 0, so a NaN output passes dy.

`max_pool2d` takes only kernel 3, stride 2, padding 1 (the SmplResNet stem pool).  Ties and NaN pick the window slot
torch picks, and the backward is a gather, so results match torch's CUDA max_pool2d bit for bit.

Inputs are fp32, contiguous NCHW CUDA tensors with any C and H x W; anything else raises ValueError (there is no
fall-back to torch).  weight, bias and the running statistics must be given and momentum must be a number: every
BatchNorm2d of the network is affine, tracks its statistics and uses momentum 0.1 (res_module.py:17).  The backward
computes only the gradients in ctx.needs_input_grad.  Nothing synchronises with the host and no float atomics are used:
results repeat bit for bit, and forward + backward can be captured in a CUDA graph."""
import ctypes

import torch
from torch.autograd.function import once_differentiable

from . import _args, _lib


class _BatchNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, new_running, training, momentum, eps, relu):
        dev = x.device
        N, C, H, W = x.shape
        nbytes = int(_lib.load().danet_bn2d_workspace_bytes(N, C, H * W))
        if nbytes <= 0:
            raise ValueError("danet_b200.layers.batch_norm: unsupported size N=%d C=%d HW=%d" % (N, C, H * W))
        with torch.cuda.device(dev):
            y = torch.empty_like(x)
            save = torch.empty(2, C, dtype=torch.float64, device=dev)
            ws = _lib.workspace(nbytes, dev)
            _lib.call("bn2d_forward", N, C, H * W, _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(running_mean),
                      _lib.ptr(running_var), int(training), momentum, eps, _lib.ptr(residual), int(relu), _lib.ptr(y),
                      _lib.ptr(save), _lib.ptr(new_running), _lib.ptr(ws), device=dev)
        ctx.save_for_backward(x, weight, save, y if relu else None)
        ctx.training, ctx.relu = training, relu
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, weight, save, y = ctx.saved_tensors
        need_x, need_w, need_b, need_r = ctx.needs_input_grad[:4]
        dev = x.device
        N, C, H, W = x.shape
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty_like(x) if need_x else None
            dr = torch.empty_like(x) if need_r else None
            dw = torch.empty_like(weight) if need_w else None
            db = torch.empty_like(weight) if need_b else None
            ws = _lib.workspace(_lib.load().danet_bn2d_workspace_bytes(N, C, H * W), dev)
            _lib.call("bn2d_backward", N, C, H * W, _lib.ptr(x), _lib.ptr(y), _lib.ptr(gy), _lib.ptr(weight), _lib.ptr(save),
                      int(ctx.training), int(ctx.relu), _lib.ptr(dx), _lib.ptr(dw), _lib.ptr(db), _lib.ptr(dr), _lib.ptr(ws),
                      device=dev)
        return dx, dw, db, dr, None, None, None, None, None, None, None


def batch_norm(input, running_mean, running_var, weight=None, bias=None, training=False, momentum=0.1, eps=1e-5, *,
               residual=None, relu=False):
    """relu(F.batch_norm(input, running_mean, running_var, weight, bias, training, momentum, eps) + residual) on the GPU,
    differentiable w.r.t. input, weight, bias and residual.  See the module docstring."""
    where = "danet_b200.layers.batch_norm"
    params = (("running_mean", running_mean), ("running_var", running_var), ("weight", weight), ("bias", bias))
    for name, t in params:
        if t is None:
            raise ValueError("%s: %s must be given (every BatchNorm2d of the network is affine and tracks its "
                             "statistics)" % (where, name))
    if momentum is None:
        raise ValueError("%s: momentum must be a number (the cumulative average of momentum=None is not supported)"
                         % where)
    momentum, eps = _args.number(where, "momentum", momentum), _args.number(where, "eps", eps)
    _args.tensor(where, "input", input)
    if input.dim() != 4:
        raise ValueError("%s: input must be 4-D NCHW (got %d-D)" % (where, input.dim()))
    N, C, H, W = input.shape
    if N < 1 or C < 1 or H < 1 or W < 1:
        raise ValueError("%s: empty input %s" % (where, tuple(input.shape)))
    for name, t in params:
        _args.tensor(where, name, t, shape=(C,))
    if residual is not None:
        _args.tensor(where, "residual", residual, shape=input.shape)
    training, relu = bool(training), bool(relu)
    if training and N * H * W == 1:
        raise ValueError("%s: expected more than 1 value per channel when training, got input size %s"
                         % (where, tuple(input.shape)))
    _args.cuda(where, (("input", input),) + params + ((("residual", residual),) if residual is not None else ()))
    new_running = torch.empty(2, C, dtype=torch.float32, device=input.device) if training else None
    y = _BatchNorm.apply(input, weight, bias, residual, running_mean, running_var, new_running, training, momentum, eps,
                         relu)
    if training:
        with torch.no_grad():                 # in place: the buffers' versions move, so plans refold their BatchNorm
            running_mean.copy_(new_running[0])
            running_var.copy_(new_running[1])
    return y


def _pool_shape(x):
    N, C, H, W = x.shape
    return N, C, H, W, (H - 1) // 2 + 1, (W - 1) // 2 + 1


def max_pool_forward(x):
    """(y, slot): the forward of max_pool2d(x, 3, 2, 1) and, per output, the row-major slot (uint8, 0..8) of the input
    pixel its 3x3 window took: input row 2 * oh - 1 + slot // 3, column 2 * ow - 1 + slot % 3."""
    dev = x.device
    N, C, H, W, Ho, Wo = _pool_shape(x)
    with torch.cuda.device(dev):
        y = torch.empty(N, C, Ho, Wo, dtype=torch.float32, device=dev)
        slot = torch.empty(N, C, Ho, Wo, dtype=torch.uint8, device=dev)
        _lib.call("maxpool3x3s2_nchw_forward", N, C, H, W, _lib.ptr(x), _lib.ptr(y), _lib.ptr(slot), device=dev)
    return y, slot


class _MaxPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y, slot = max_pool_forward(x)
        ctx.save_for_backward(slot)
        ctx.shape = tuple(x.shape)
        ctx.mark_non_differentiable(slot)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        (slot,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        dev = slot.device
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
            _lib.call("maxpool3x3s2_nchw_backward", N, C, H, W, _lib.ptr(gy), _lib.ptr(slot), _lib.ptr(dx), device=dev)
        return dx


def max_pool2d(input, kernel_size, stride=None, padding=0, dilation=1, ceil_mode=False, return_indices=False):
    """F.max_pool2d for kernel_size 3, stride 2, padding 1 (nn.MaxPool2d(3, 2, 1) of SmplResNet) on the GPU,
    differentiable.  See the module docstring."""
    where = "danet_b200.layers.max_pool2d"
    k = _args.int_pair(where, "kernel_size", kernel_size)
    s = k if stride is None or (isinstance(stride, (tuple, list)) and len(stride) == 0) else \
        _args.int_pair(where, "stride", stride)
    p, d = _args.int_pair(where, "padding", padding), _args.int_pair(where, "dilation", dilation)
    if (k, s, p, d) != (3, 2, 1, 1) or ceil_mode or return_indices:
        raise ValueError("%s: only kernel_size=3, stride=2, padding=1, dilation=1 without ceil_mode or return_indices "
                         "is supported (got k=%d s=%d p=%d d=%d ceil_mode=%r return_indices=%r)"
                         % (where, k, s, p, d, ceil_mode, return_indices))
    _args.tensor(where, "input", input)
    if input.dim() != 4:
        raise ValueError("%s: input must be 4-D NCHW (got %d-D)" % (where, input.dim()))
    if min(input.shape) < 1:
        raise ValueError("%s: empty input %s" % (where, tuple(input.shape)))
    _args.cuda(where, [("input", input)])
    return _MaxPool.apply(input)


class _AvgPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        dev = x.device
        N, C, H, W = x.shape
        with torch.cuda.device(dev):
            y = torch.empty(N, C, 1, 1, dtype=torch.float32, device=dev)
            act = _lib.Act(x.data_ptr(), None, None)          # NCHW [N, C, HW] is NHWC [N * C, HW, 1]
            _lib.call("global_avgpool", N * C, H * W, 1, ctypes.byref(act), _lib.ptr(y), device=dev)
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        N, C, H, W = ctx.shape
        dev = gy.device
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
            _lib.call("global_avgpool_backward", N * C, H * W, _lib.ptr(gy), _lib.ptr(dx), device=dev)
        return dx


def adaptive_avg_pool2d(input, output_size):
    """F.adaptive_avg_pool2d for output size 1 (nn.AdaptiveAvgPool2d(1) of SmplResNet and LimbResLayers) on the GPU,
    differentiable: [N, C, H, W] -> [N, C, 1, 1]."""
    where = "danet_b200.layers.adaptive_avg_pool2d"
    size = tuple(output_size) if isinstance(output_size, (tuple, list)) else (output_size, output_size)
    if size != (1, 1):
        raise ValueError("%s: only output_size=1 is supported (got %r)" % (where, output_size))
    _args.tensor(where, "input", input)
    if input.dim() != 4:
        raise ValueError("%s: input must be 4-D NCHW (got %d-D)" % (where, input.dim()))
    if min(input.shape) < 1:
        raise ValueError("%s: empty input %s" % (where, tuple(input.shape)))
    _args.cuda(where, [("input", input)])
    return _AvgPool.apply(input)


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, add):
        dev = x.device
        (N, In), Out = x.shape, weight.shape[0]
        with torch.cuda.device(dev):
            y = torch.empty(N, Out, dtype=torch.float32, device=dev)
            _lib.call("linear", N, In, Out, _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(add), _lib.ptr(y),
                      device=dev)
        need_x, need_w = ctx.needs_input_grad[:2]
        ctx.save_for_backward(x if need_w else None, weight if need_x else None)
        ctx.shape = (N, In, Out)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        N, In, Out = ctx.shape
        dev = gy.device
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty(N, In, dtype=torch.float32, device=dev) if need_x else None
            dw = torch.empty(Out, In, dtype=torch.float32, device=dev) if need_w else None
            db = torch.empty(Out, dtype=torch.float32, device=dev) if need_b else None
            if need_x or need_w or need_b:
                _lib.call("linear_backward", N, In, Out, _lib.ptr(x), _lib.ptr(weight), _lib.ptr(gy), _lib.ptr(dx),
                          _lib.ptr(dw), _lib.ptr(db), device=dev)
        return dx, dw, db, None


def linear(input, weight, bias=None, *, add=None):
    """F.linear(input, weight, bias) + add on the GPU, differentiable w.r.t. input, weight and bias.  input [N, In],
    weight [Out, In], bias and add [Out]; `add` is a constant term with no gradient (body_net's tail adds
    mean_cam_shape there)."""
    where = "danet_b200.layers.linear"
    _args.tensor(where, "input", input)
    if input.dim() != 2:
        raise ValueError("%s: input must be 2-D [N, In] (got %d-D)" % (where, input.dim()))
    _args.tensor(where, "weight", weight)
    if weight.dim() != 2 or weight.shape[1] != input.shape[1]:
        raise ValueError("%s: weight must be [Out, %d] (got %s)" % (where, input.shape[1], tuple(weight.shape)))
    if min(input.shape) < 1 or weight.shape[0] < 1:
        raise ValueError("%s: empty input or weight (%s, %s)" % (where, tuple(input.shape), tuple(weight.shape)))
    tensors = [("input", input), ("weight", weight)]
    for name, t in (("bias", bias), ("add", add)):
        if t is not None:
            _args.tensor(where, name, t, shape=(weight.shape[0],))
            tensors.append((name, t))
    _args.cuda(where, tensors)
    return _Linear.apply(input, weight, bias, add.detach() if add is not None else None)


class _HrFuse(torch.autograd.Function):
    @staticmethod
    def forward(ctx, relu, factors, *terms):
        t0, f0 = terms[0], factors[0]
        dev = t0.device
        N, C, H, W = t0.shape[0], t0.shape[1], t0.shape[2] * f0, t0.shape[3] * f0
        n = len(terms)
        with torch.cuda.device(dev):
            y = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
            ptrs = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in terms])
            facs = (ctypes.c_int32 * 4)(*factors)
            _lib.call("hr_fuse_forward", N, C, H, W, n, ptrs, facs, int(relu), _lib.ptr(y), device=dev)
        ctx.save_for_backward(y if relu else None)
        ctx.factors, ctx.shape = factors, (N, C, H, W)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        (y,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        dev = gy.device
        grads = []
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            for f, need in zip(ctx.factors, ctx.needs_input_grad[2:]):
                if not need:
                    grads.append(None)
                    continue
                dt = torch.empty(N, C, H // f, W // f, dtype=torch.float32, device=dev)
                _lib.call("hr_fuse_backward", N, C, H, W, f, _lib.ptr(gy), _lib.ptr(y), _lib.ptr(dt), device=dev)
                grads.append(dt)
        return (None, None) + tuple(grads)


def hr_fuse(terms, factors, relu=True):
    """One HRNet fuse output (hr_module.py:161-179) on the GPU, differentiable w.r.t. every term:
    relu(up(terms[0], factors[0]) + up(terms[1], factors[1]) + ...), up = nearest upsampling by 1, 2, 4 or 8.

    terms: 1 to 4 fp32 contiguous NCHW CUDA tensors [N, C, H / f, W / f] with t.H * f == H and t.W * f == W for one
    (H, W).  The terms are added in list order, the reference's `y = y + ...` order, so the forward is bit-identical
    to the fp32 sequence F.interpolate(t, scale_factor=f, mode='nearest') + ... + relu.  The backward of a term is
    the sum of dy over each f x f block, except where y <= 0 (an exact 0 gets no gradient, a NaN passes dy), in row-major order,
    in fp32: within (f^2 - 1) 2^-24 sum |dy| of the exact block sum."""
    where = "danet_b200.layers.hr_fuse"
    if not isinstance(terms, (list, tuple)) or not 1 <= len(terms) <= 4:
        raise ValueError("%s: terms must be a list of 1 to 4 tensors" % where)
    if not isinstance(factors, (list, tuple)) or len(factors) != len(terms):
        raise ValueError("%s: factors must be a list with one factor per term" % where)
    for f in factors:
        if isinstance(f, bool) or not isinstance(f, int) or f not in (1, 2, 4, 8):
            raise ValueError("%s: factors must be 1, 2, 4 or 8 (got %r)" % (where, f))
    named = [("terms[%d]" % j, t) for j, t in enumerate(terms)]
    for name, t in named:
        _args.tensor(where, name, t)
        if t.dim() != 4 or min(t.shape) < 1:
            raise ValueError("%s: %s must be a non-empty 4-D NCHW tensor (got %s)" % (where, name, tuple(t.shape)))
    N, C = terms[0].shape[:2]
    H, W = terms[0].shape[2] * factors[0], terms[0].shape[3] * factors[0]
    for j, (t, f) in enumerate(zip(terms, factors)):
        if tuple(t.shape) != (N, C, H // f, W // f) or H % f or W % f:
            raise ValueError("%s: terms[%d] %s upsampled by %d is not [%d, %d, %d, %d]"
                             % (where, j, tuple(t.shape), f, N, C, H, W))
    _args.cuda(where, named)
    return _HrFuse.apply(bool(relu), tuple(int(f) for f in factors), *terms)
