"""Argument checks of the differentiable ops.  Each raises ValueError with a message of the form
`<where>: <name> must ...`, where `where` is the op's public name (e.g. "danet_b200.layers.batch_norm").  `tensor` and
`cuda` are separate so that each op keeps its own order of checks."""
import numbers

import torch


def tensor(where, name, t, dim=None, shape=None, contiguous=True):
    """t is a float32 tensor with `dim` dimensions and shape `shape` (when given), contiguous unless contiguous=False."""
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s: %s must be a tensor (got %s)" % (where, name, type(t).__name__))
    if t.dtype != torch.float32:
        raise ValueError("%s: %s must be float32 (got %s)" % (where, name, t.dtype))
    if dim is not None and t.dim() != dim:
        raise ValueError("%s: %s must be %d-D (got %s)" % (where, name, dim, tuple(t.shape)))
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError("%s: %s must have shape %s (got %s)" % (where, name, tuple(shape), tuple(t.shape)))
    if contiguous and not t.is_contiguous():
        raise ValueError("%s: %s must be contiguous" % (where, name))


def cuda(where, named_tensors, dev=None):
    """Each (name, t) of named_tensors is a tensor on the CUDA device `dev` (default: the first tensor's device)."""
    for name, t in named_tensors:
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: %s must be a tensor (got %s)" % (where, name, type(t).__name__))
        if not t.is_cuda:
            raise ValueError("%s: %s must be a CUDA tensor (there is no CPU path)" % (where, name))
        dev = t.device if dev is None else dev
        if t.device != dev:
            raise ValueError("%s: %s is on %s, expected %s" % (where, name, t.device, dev))


def number(where, name, v):
    """v as a float; v must be a real number and not a bool."""
    if isinstance(v, bool) or not isinstance(v, numbers.Real):
        raise ValueError("%s: %s must be a number (got %r)" % (where, name, v))
    return float(v)


def int_pair(where, name, v):
    """v as an int; v must be an int or a pair of equal ints (torch's size arguments)."""
    if isinstance(v, (tuple, list)):
        if len(v) != 2 or v[0] != v[1]:
            raise ValueError("%s: %s must be one int or an equal pair (got %r)" % (where, name, v))
        v = v[0]
    if isinstance(v, bool) or not isinstance(v, int):
        raise ValueError("%s: %s must be an int (got %r)" % (where, name, v))
    return v


def mask(where, name, t, shape):
    """t is a bool or uint8 tensor of shape `shape` (a per-image flag; nonzero = true), contiguous."""
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s: %s must be a tensor (got %s)" % (where, name, type(t).__name__))
    if t.dtype not in (torch.bool, torch.uint8):
        raise ValueError("%s: %s must be bool or uint8 (got %s)" % (where, name, t.dtype))
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s: %s must have shape %s (got %s)" % (where, name, tuple(shape), tuple(t.shape)))
    if not t.is_contiguous():
        raise ValueError("%s: %s must be contiguous" % (where, name))
