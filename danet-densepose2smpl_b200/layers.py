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
ResNet forms: bn + relu (bn1, the stems), bn + residual + relu (bn2), bn alone (the downsample).

`max_pool2d` takes only kernel 3, stride 2, padding 1 (the SmplResNet stem pool).  Ties and NaN pick the window slot
torch picks, and the backward is a gather, so results match torch's CUDA max_pool2d bit for bit.

Inputs are fp32, contiguous NCHW CUDA tensors with any C and H x W; anything else raises ValueError (there is no
fall-back to torch).  weight, bias and the running statistics must be given and momentum must be a number: every
BatchNorm2d of the network is affine, tracks its statistics and uses momentum 0.1 (res_module.py:17).  The backward
computes only the gradients in ctx.needs_input_grad.  Nothing synchronises with the host and no float atomics are used:
results repeat bit for bit, and forward + backward can be captured in a CUDA graph."""
import ctypes
import numbers

import torch
from torch.autograd.function import once_differentiable

from . import _lib


def _workspace(lib, N, C, HW, dev):
    nbytes = int(lib.danet_bn2d_workspace_bytes(N, C, HW))
    if nbytes <= 0:
        raise ValueError("danet_b200.layers.batch_norm: unsupported size N=%d C=%d HW=%d" % (N, C, HW))
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


class _BatchNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, new_running, training, momentum, eps, relu):
        lib = _lib.load()
        dev = x.device
        N, C, H, W = x.shape
        with torch.cuda.device(dev):
            y = torch.empty_like(x)
            save = torch.empty(2, C, dtype=torch.float64, device=dev)
            ws = _workspace(lib, N, C, H * W, dev)
            _lib.check(lib.danet_bn2d_forward(N, C, H * W, _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias),
                                              _lib.ptr(running_mean), _lib.ptr(running_var), int(training), float(momentum),
                                              float(eps), _lib.ptr(residual), int(relu), _lib.ptr(y), _lib.ptr(save),
                                              _lib.ptr(new_running), _lib.ptr(ws), _lib.stream_ptr(dev)), "bn2d_forward")
        ctx.save_for_backward(x, weight, save, y if relu else None)
        ctx.training, ctx.relu = training, relu
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, weight, save, y = ctx.saved_tensors
        need_x, need_w, need_b, need_r = ctx.needs_input_grad[:4]
        lib = _lib.load()
        dev = x.device
        N, C, H, W = x.shape
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty_like(x) if need_x else None
            dr = torch.empty_like(x) if need_r else None
            dw = torch.empty_like(weight) if need_w else None
            db = torch.empty_like(weight) if need_b else None
            ws = _workspace(lib, N, C, H * W, dev)
            _lib.check(lib.danet_bn2d_backward(N, C, H * W, _lib.ptr(x), _lib.ptr(y), _lib.ptr(gy), _lib.ptr(weight),
                                               _lib.ptr(save), int(ctx.training), int(ctx.relu), _lib.ptr(dx), _lib.ptr(dw),
                                               _lib.ptr(db), _lib.ptr(dr), _lib.ptr(ws), _lib.stream_ptr(dev)),
                       "bn2d_backward")
        return dx, dw, db, dr, None, None, None, None, None, None, None


def _check_tensor(fn, name, t, shape=None):
    if not isinstance(t, torch.Tensor):
        raise ValueError("danet_b200.layers.%s: %s must be a tensor (got %s)" % (fn, name, type(t).__name__))
    if t.dtype != torch.float32:
        raise ValueError("danet_b200.layers.%s: %s must be float32 (got %s)" % (fn, name, t.dtype))
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError("danet_b200.layers.%s: %s must have shape %s (got %s)" % (fn, name, tuple(shape), tuple(t.shape)))
    if not t.is_contiguous():
        raise ValueError("danet_b200.layers.%s: %s must be contiguous" % (fn, name))


def _check_cuda(fn, tensors, dev):
    for name, t in tensors:
        if not t.is_cuda:
            raise ValueError("danet_b200.layers.%s: %s must be a CUDA tensor (there is no CPU path)" % (fn, name))
        if t.device != dev:
            raise ValueError("danet_b200.layers.%s: %s is on %s, x on %s" % (fn, name, t.device, dev))


def batch_norm(input, running_mean, running_var, weight=None, bias=None, training=False, momentum=0.1, eps=1e-5, *,
               residual=None, relu=False):
    """relu(F.batch_norm(input, running_mean, running_var, weight, bias, training, momentum, eps) + residual) on the GPU,
    differentiable w.r.t. input, weight, bias and residual.  See the module docstring."""
    fn = "batch_norm"
    for name, t in (("running_mean", running_mean), ("running_var", running_var), ("weight", weight), ("bias", bias)):
        if t is None:
            raise ValueError("danet_b200.layers.batch_norm: %s must be given (every BatchNorm2d of the network is affine "
                             "and tracks its statistics)" % name)
    if momentum is None:
        raise ValueError("danet_b200.layers.batch_norm: momentum must be a number (the cumulative average of "
                         "momentum=None is not supported)")
    if isinstance(momentum, bool) or not isinstance(momentum, numbers.Real):
        raise ValueError("danet_b200.layers.batch_norm: momentum must be a number (got %r)" % (momentum,))
    if isinstance(eps, bool) or not isinstance(eps, numbers.Real):
        raise ValueError("danet_b200.layers.batch_norm: eps must be a number (got %r)" % (eps,))
    _check_tensor(fn, "input", input)
    if input.dim() != 4:
        raise ValueError("danet_b200.layers.batch_norm: input must be 4-D NCHW (got %d-D)" % input.dim())
    N, C, H, W = input.shape
    if N < 1 or C < 1 or H < 1 or W < 1:
        raise ValueError("danet_b200.layers.batch_norm: empty input %s" % (tuple(input.shape),))
    for name, t in (("running_mean", running_mean), ("running_var", running_var), ("weight", weight), ("bias", bias)):
        _check_tensor(fn, name, t, (C,))
    if residual is not None:
        _check_tensor(fn, "residual", residual, input.shape)
    training, relu = bool(training), bool(relu)
    if training and N * H * W == 1:
        raise ValueError("danet_b200.layers.batch_norm: expected more than 1 value per channel when training, got input "
                         "size %s" % (tuple(input.shape),))
    tensors = [("input", input), ("running_mean", running_mean), ("running_var", running_var), ("weight", weight),
               ("bias", bias)] + ([("residual", residual)] if residual is not None else [])
    _check_cuda(fn, tensors, input.device)
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
    lib = _lib.load()
    dev = x.device
    N, C, H, W, Ho, Wo = _pool_shape(x)
    with torch.cuda.device(dev):
        y = torch.empty(N, C, Ho, Wo, dtype=torch.float32, device=dev)
        slot = torch.empty(N, C, Ho, Wo, dtype=torch.uint8, device=dev)
        _lib.check(lib.danet_maxpool3x3s2_nchw_forward(N, C, H, W, _lib.ptr(x), _lib.ptr(y), _lib.ptr(slot),
                                                       _lib.stream_ptr(dev)), "maxpool3x3s2_nchw_forward")
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
        lib = _lib.load()
        dev = slot.device
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
            _lib.check(lib.danet_maxpool3x3s2_nchw_backward(N, C, H, W, _lib.ptr(gy), _lib.ptr(slot), _lib.ptr(dx),
                                                            _lib.stream_ptr(dev)), "maxpool3x3s2_nchw_backward")
        return dx


def _int_pair(v, name):
    if isinstance(v, (tuple, list)):
        if len(v) != 2 or v[0] != v[1]:
            raise ValueError("danet_b200.layers.max_pool2d: %s must be one int or an equal pair (got %r)" % (name, v))
        v = v[0]
    if isinstance(v, bool) or not isinstance(v, int):
        raise ValueError("danet_b200.layers.max_pool2d: %s must be an int (got %r)" % (name, v))
    return v


def max_pool2d(input, kernel_size, stride=None, padding=0, dilation=1, ceil_mode=False, return_indices=False):
    """F.max_pool2d for kernel_size 3, stride 2, padding 1 (nn.MaxPool2d(3, 2, 1) of SmplResNet) on the GPU,
    differentiable.  See the module docstring."""
    k = _int_pair(kernel_size, "kernel_size")
    s = k if stride is None or (isinstance(stride, (tuple, list)) and len(stride) == 0) else _int_pair(stride, "stride")
    p, d = _int_pair(padding, "padding"), _int_pair(dilation, "dilation")
    if (k, s, p, d) != (3, 2, 1, 1) or ceil_mode or return_indices:
        raise ValueError("danet_b200.layers.max_pool2d: only kernel_size=3, stride=2, padding=1, dilation=1 without "
                         "ceil_mode or return_indices is supported (got k=%d s=%d p=%d d=%d ceil_mode=%r "
                         "return_indices=%r)" % (k, s, p, d, ceil_mode, return_indices))
    _check_tensor("max_pool2d", "input", input)
    if input.dim() != 4:
        raise ValueError("danet_b200.layers.max_pool2d: input must be 4-D NCHW (got %d-D)" % input.dim())
    if min(input.shape) < 1:
        raise ValueError("danet_b200.layers.max_pool2d: empty input %s" % (tuple(input.shape),))
    _check_cuda("max_pool2d", [("input", input)], input.device)
    return _MaxPool.apply(input)


class _AvgPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        lib = _lib.load()
        dev = x.device
        N, C, H, W = x.shape
        with torch.cuda.device(dev):
            y = torch.empty(N, C, 1, 1, dtype=torch.float32, device=dev)
            act = _lib.Act(x.data_ptr(), None, None)          # NCHW [N, C, HW] is NHWC [N * C, HW, 1]
            _lib.check(lib.danet_global_avgpool(N * C, H * W, 1, ctypes.byref(act), _lib.ptr(y), _lib.stream_ptr(dev)),
                       "global_avgpool")
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        N, C, H, W = ctx.shape
        lib = _lib.load()
        dev = gy.device
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
            _lib.check(lib.danet_global_avgpool_backward(N * C, H * W, _lib.ptr(gy), _lib.ptr(dx), _lib.stream_ptr(dev)),
                       "global_avgpool_backward")
        return dx


def adaptive_avg_pool2d(input, output_size):
    """F.adaptive_avg_pool2d for output size 1 (nn.AdaptiveAvgPool2d(1) of SmplResNet and LimbResLayers) on the GPU,
    differentiable: [N, C, H, W] -> [N, C, 1, 1]."""
    size = tuple(output_size) if isinstance(output_size, (tuple, list)) else (output_size, output_size)
    if size != (1, 1):
        raise ValueError("danet_b200.layers.adaptive_avg_pool2d: only output_size=1 is supported (got %r)" % (output_size,))
    _check_tensor("adaptive_avg_pool2d", "input", input)
    if input.dim() != 4:
        raise ValueError("danet_b200.layers.adaptive_avg_pool2d: input must be 4-D NCHW (got %d-D)" % input.dim())
    if min(input.shape) < 1:
        raise ValueError("danet_b200.layers.adaptive_avg_pool2d: empty input %s" % (tuple(input.shape),))
    _check_cuda("adaptive_avg_pool2d", [("input", input)], input.device)
    return _AvgPool.apply(input)


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, add):
        lib = _lib.load()
        dev = x.device
        (N, In), Out = x.shape, weight.shape[0]
        with torch.cuda.device(dev):
            y = torch.empty(N, Out, dtype=torch.float32, device=dev)
            _lib.check(lib.danet_linear(N, In, Out, _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(add), _lib.ptr(y),
                                        _lib.stream_ptr(dev)), "linear")
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
        lib = _lib.load()
        dev = gy.device
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            dx = torch.empty(N, In, dtype=torch.float32, device=dev) if need_x else None
            dw = torch.empty(Out, In, dtype=torch.float32, device=dev) if need_w else None
            db = torch.empty(Out, dtype=torch.float32, device=dev) if need_b else None
            if need_x or need_w or need_b:
                _lib.check(lib.danet_linear_backward(N, In, Out, _lib.ptr(x), _lib.ptr(weight), _lib.ptr(gy), _lib.ptr(dx),
                                                     _lib.ptr(dw), _lib.ptr(db), _lib.stream_ptr(dev)), "linear_backward")
        return dx, dw, db, None


def linear(input, weight, bias=None, *, add=None):
    """F.linear(input, weight, bias) + add on the GPU, differentiable w.r.t. input, weight and bias.  input [N, In],
    weight [Out, In], bias and add [Out]; `add` is a constant term with no gradient (body_net's tail adds
    mean_cam_shape there)."""
    fn = "linear"
    _check_tensor(fn, "input", input)
    if input.dim() != 2:
        raise ValueError("danet_b200.layers.linear: input must be 2-D [N, In] (got %d-D)" % input.dim())
    _check_tensor(fn, "weight", weight)
    if weight.dim() != 2 or weight.shape[1] != input.shape[1]:
        raise ValueError("danet_b200.layers.linear: weight must be [Out, %d] (got %s)" % (input.shape[1], tuple(weight.shape)))
    if min(input.shape) < 1 or weight.shape[0] < 1:
        raise ValueError("danet_b200.layers.linear: empty input or weight (%s, %s)" % (tuple(input.shape), tuple(weight.shape)))
    tensors = [("input", input), ("weight", weight)]
    for name, t in (("bias", bias), ("add", add)):
        if t is not None:
            _check_tensor(fn, name, t, (weight.shape[0],))
            tensors.append((name, t))
    _check_cuda(fn, tensors, input.device)
    return _Linear.apply(input, weight, bias, add.detach() if add is not None else None)


class _HrFuse(torch.autograd.Function):
    @staticmethod
    def forward(ctx, relu, factors, *terms):
        lib = _lib.load()
        t0, f0 = terms[0], factors[0]
        dev = t0.device
        N, C, H, W = t0.shape[0], t0.shape[1], t0.shape[2] * f0, t0.shape[3] * f0
        n = len(terms)
        with torch.cuda.device(dev):
            y = torch.empty(N, C, H, W, dtype=torch.float32, device=dev)
            ptrs = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in terms])
            facs = (ctypes.c_int32 * 4)(*factors)
            _lib.check(lib.danet_hr_fuse_forward(N, C, H, W, n, ptrs, facs, int(relu), _lib.ptr(y), _lib.stream_ptr(dev)),
                       "hr_fuse_forward")
        ctx.save_for_backward(y if relu else None)
        ctx.factors, ctx.shape = factors, (N, C, H, W)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        (y,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        lib = _lib.load()
        dev = gy.device
        grads = []
        with torch.cuda.device(dev):
            gy = gy.to(torch.float32).contiguous()
            for f, need in zip(ctx.factors, ctx.needs_input_grad[2:]):
                if not need:
                    grads.append(None)
                    continue
                dt = torch.empty(N, C, H // f, W // f, dtype=torch.float32, device=dev)
                _lib.check(lib.danet_hr_fuse_backward(N, C, H, W, f, _lib.ptr(gy), _lib.ptr(y), _lib.ptr(dt),
                                                      _lib.stream_ptr(dev)), "hr_fuse_backward")
                grads.append(dt)
        return (None, None) + tuple(grads)


def hr_fuse(terms, factors, relu=True):
    """One HRNet fuse output (hr_module.py:161-179) on the GPU, differentiable w.r.t. every term:
    relu(up(terms[0], factors[0]) + up(terms[1], factors[1]) + ...), up = nearest upsampling by 1, 2, 4 or 8.

    terms: 1 to 4 fp32 contiguous NCHW CUDA tensors [N, C, H / f, W / f] with t.H * f == H and t.W * f == W for one
    (H, W).  The terms are added in list order, the reference's `y = y + ...` order, so the forward is bit-identical
    to the fp32 sequence F.interpolate(t, scale_factor=f, mode='nearest') + ... + relu.  The backward of a term is
    the sum of dy * [y > 0] over each f x f block in row-major order (torch's ReLU rule: an exact 0 gets no gradient),
    in fp32: within (f^2 - 1) 2^-24 sum |dy| of the exact block sum."""
    fn = "hr_fuse"
    if not isinstance(terms, (list, tuple)) or not 1 <= len(terms) <= 4:
        raise ValueError("danet_b200.layers.hr_fuse: terms must be a list of 1 to 4 tensors")
    if not isinstance(factors, (list, tuple)) or len(factors) != len(terms):
        raise ValueError("danet_b200.layers.hr_fuse: factors must be a list with one factor per term")
    for f in factors:
        if isinstance(f, bool) or not isinstance(f, int) or f not in (1, 2, 4, 8):
            raise ValueError("danet_b200.layers.hr_fuse: factors must be 1, 2, 4 or 8 (got %r)" % (f,))
    for j, t in enumerate(terms):
        _check_tensor(fn, "terms[%d]" % j, t)
        if t.dim() != 4 or min(t.shape) < 1:
            raise ValueError("danet_b200.layers.hr_fuse: terms[%d] must be a non-empty 4-D NCHW tensor (got %s)"
                             % (j, tuple(t.shape)))
    N, C = terms[0].shape[:2]
    H, W = terms[0].shape[2] * factors[0], terms[0].shape[3] * factors[0]
    for j, (t, f) in enumerate(zip(terms, factors)):
        if tuple(t.shape) != (N, C, H // f, W // f) or H % f or W % f:
            raise ValueError("danet_b200.layers.hr_fuse: terms[%d] %s upsampled by %d is not [%d, %d, %d, %d]"
                             % (j, tuple(t.shape), f, N, C, H, W))
    _check_cuda(fn, [("terms[%d]" % j, t) for j, t in enumerate(terms)], terms[0].device)
    return _HrFuse.apply(bool(relu), tuple(int(f) for f in factors), *terms)
