"""The training step's optimizer: train/trainer.py:42-44's torch.optim.Adam(params, lr, weight_decay=0) as one CUDA pass.

    from danet_b200.optim import Adam
    optimizer = Adam(model.parameters(), lr=cfg.SOLVER.BASE_LR, weight_decay=0)

torch's CUDA default for that optimizer is the foreach implementation (_multi_tensor_adam): seven elementwise passes
over every parameter and a temporary the size of the model.  `Adam.step()` makes one danet_adam_step call
(csrc/optim.cu) per (param group, step count), which reads p, grad, exp_avg and exp_avg_sq once and writes p, exp_avg
and exp_avg_sq once, with torch's roundings: the parameters, moments and step counts stay bit-identical to
torch.optim.Adam's.  The state per parameter is torch's own ('step' a CPU 0-dim tensor, 'exp_avg' and 'exp_avg_sq'
created on the first step with a gradient), so state dicts move both ways between the two classes.

Only the options the reference uses are provided: weight_decay, amsgrad, maximize, foreach, fused, capturable,
differentiable and decoupled_weight_decay set, a Tensor lr or beta, sparse gradients, and parameters that are not
contiguous fp32 CUDA tensors on one device raise ValueError.  There is no CPU path."""
import ctypes

import numpy as np
import torch

from . import _args, _lib

WHERE = "danet_b200.optim.Adam"
_OFF = ("amsgrad", "maximize", "capturable", "differentiable", "decoupled_weight_decay")   # must be False
_UNSET = ("foreach", "fused")                                                               # must be None


def _scalar_dtype():
    """torch.optim's dtype of 'step' for a non-capturable, non-fused optimizer"""
    return torch.float64 if torch.get_default_dtype() == torch.float64 else torch.float32


def _check_device(where, name, t):
    """the kernel layer's device check (a CUDA tensor; there is no CPU path)"""
    if not t.is_cuda:
        raise ValueError("%s: %s must be a CUDA tensor (there is no CPU path)" % (where, name))


def _launch(device, params, grads, exp_avgs, exp_avg_sqs, lerp_weight, beta2, one_minus_beta2, bias_correction2_sqrt,
            eps, step_size):
    """one danet_adam_step call on `device`'s current stream: host tables of the tensors' addresses and sizes"""
    ptrs = np.array([[t.data_ptr() for t in ts] for ts in (params, grads, exp_avgs, exp_avg_sqs)], dtype=np.uint64)
    numels = np.array([t.numel() for t in params], dtype=np.int64)
    addr = lambda a: ctypes.c_void_p(a.ctypes.data)
    with torch.cuda.device(device):
        _lib.call("adam_step", len(params), addr(ptrs[0]), addr(ptrs[1]), addr(ptrs[2]), addr(ptrs[3]), addr(numels),
                  lerp_weight, beta2, one_minus_beta2, bias_correction2_sqrt, eps, step_size, device=device)


def _check_group(where, group):
    for k in _OFF:
        if group.get(k, False):
            raise ValueError("%s: %s=True is not provided (the reference's Adam does not use it)" % (where, k))
    for k in _UNSET:
        if group.get(k) is not None:
            raise ValueError("%s: %s must be None (the step is always danet_adam_step)" % (where, k))
    if group.get("weight_decay", 0) != 0:
        raise ValueError("%s: weight_decay must be 0 (got %r)" % (where, group["weight_decay"]))
    if isinstance(group["lr"], torch.Tensor):
        raise ValueError("%s: lr must be a number, not a Tensor" % where)
    lr = _args.number(where, "lr", group["lr"])
    eps = _args.number(where, "eps", group["eps"])
    betas = group["betas"]
    if not isinstance(betas, (tuple, list)) or len(betas) != 2:
        raise ValueError("%s: betas must be a pair of numbers (got %r)" % (where, betas))
    b1, b2 = (_args.number(where, "betas[%d]" % i, b) for i, b in enumerate(betas))
    if lr < 0 or eps < 0 or not (0 <= b1 < 1 and 0 <= b2 < 1):
        raise ValueError("%s: need lr >= 0, eps >= 0 and 0 <= betas < 1 (got lr=%r, eps=%r, betas=%r)"
                         % (where, lr, eps, betas))


def _check_param(where, p, name):
    if not isinstance(p, torch.Tensor):
        raise ValueError("%s: %s must be a tensor (got %s)" % (where, name, type(p).__name__))
    if p.dtype != torch.float32:
        raise ValueError("%s: %s must be float32 (got %s)" % (where, name, p.dtype))
    _check_device(where, name, p)
    if not p.is_contiguous():
        raise ValueError("%s: %s must be contiguous" % (where, name))


class Adam(torch.optim.Optimizer):
    """torch.optim.Adam(params, lr, betas, eps, weight_decay=0) with torch's defaults for the other options, whose step
    is danet_adam_step; see the module docstring.  `lr` is read from param_groups on every step, so an in-place decay
    (the reference's, danet_b200.training.LRDecay) takes effect on the next step."""

    def __init__(self, params, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None,
                 maximize=False, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False):
        # torch.optim.Adam's defaults, key for key, so that state dicts load both ways
        defaults = {"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay, "amsgrad": amsgrad,
                    "maximize": maximize, "foreach": foreach, "capturable": capturable,
                    "differentiable": differentiable, "fused": fused, "decoupled_weight_decay": decoupled_weight_decay}
        _check_group(WHERE, defaults)
        defaults["betas"] = tuple(float(b) for b in betas)
        super().__init__(params, defaults)

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        _check_group(WHERE, group)
        for i, p in enumerate(group["params"]):
            _check_param(WHERE, p, "param_groups[%d]['params'][%d]" % (len(self.param_groups) - 1, i))

    @torch.no_grad()
    def step(self, closure=None):
        """One Adam step of every parameter that has a gradient (the others and their state are left as they are).
        Parameters are grouped by (param group, step count) and each group is one danet_adam_step call; nothing waits
        for the GPU.  Returns closure's loss when a closure is given."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        where = WHERE + ".step"
        device = None
        work = []
        for gi, group in enumerate(self.param_groups):
            _check_group(where, group)
            stepped = [p for p in group["params"] if p.grad is not None]
            for p in stepped:
                if device is None:
                    _check_param(where, p, "a parameter")
                    device = p.device
                # one cheap test per parameter; the messages are built only for a parameter that fails it
                g, st = p.grad, self.state.get(p)
                ok = (p.dtype == g.dtype == torch.float32 and p.device == g.device == device and not g.is_sparse
                      and p.is_contiguous() and g.is_contiguous() and g.shape == p.shape)
                if ok and st:
                    m, v = st["exp_avg"], st["exp_avg_sq"]
                    ok = (m.dtype == v.dtype == torch.float32 and m.device == v.device == device and m.is_contiguous()
                          and v.is_contiguous() and m.shape == v.shape == p.shape)
                if not ok:
                    self._refuse(where, gi, group, p, device)
            work.append(stepped)
        calls, steps = {}, []
        for stepped in work:
            for p in stepped:
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=_scalar_dtype())
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                steps.append(st["step"])
        if steps:
            torch._foreach_add_(steps, torch.tensor(1.0), alpha=1.0)      # _multi_tensor_adam's count update
        for gi, stepped in enumerate(work):
            for p in stepped:
                st = self.state[p]
                lists = calls.setdefault((gi, st["step"].item()), ([], [], [], []))
                for lst, t in zip(lists, (p, p.grad, st["exp_avg"], st["exp_avg_sq"])):
                    lst.append(t)
        for (gi, t), (ps, gs, ms, vs) in calls.items():
            group = self.param_groups[gi]
            lr, (beta1, beta2), eps = group["lr"], group["betas"], group["eps"]
            # torch/optim/adam.py _multi_tensor_adam (capturable=False): the same Python expressions, so the same doubles
            bias_correction1 = 1 - beta1 ** t
            bias_correction2 = 1 - beta2 ** t
            step_size = (lr / bias_correction1) * -1
            bias_correction2_sqrt = bias_correction2 ** 0.5
            _launch(device, ps, gs, ms, vs, 1 - beta1, beta2, 1 - beta2, bias_correction2_sqrt, eps, step_size)
            # the kernel wrote through raw pointers: tell autograd (a saved parameter is now stale) and DaNet.plan_for
            # (it refolds its inference weights when a parameter's version moves)
            torch.autograd.graph.increment_version(ps + ms + vs)
        return loss

    def _refuse(self, where, gi, group, p, device):
        """raise the ValueError that says why `p` (in param group gi) cannot be stepped"""
        name = "param_groups[%d]['params'][%d]" % (gi, next(i for i, q in enumerate(group["params"]) if q is p))
        _check_param(where, p, name)
        g = p.grad
        if g.is_sparse:
            raise ValueError("%s: %s has a sparse gradient (Adam does not support sparse gradients)" % (where, name))
        _check_param(where, g, name + ".grad")
        named = [(name + ".grad", g)]
        st = self.state.get(p)
        if st:
            for k in ("exp_avg", "exp_avg_sq"):
                _check_param(where, st[k], "state[%s][%r]" % (name, k))
                named.append(("state[%s][%r]" % (name, k), st[k]))
        if p.device != device:
            raise ValueError("%s: parameters on more than one device (%s and %s)" % (where, device, p.device))
        for n, t in named:
            if t.device != device or t.shape != p.shape:
                raise ValueError("%s: %s must match its parameter's device and shape" % (where, n))
        raise AssertionError("%s: %s was refused without a reason" % (where, name))
