"""The per-element bound every fp64 sweep holds its outputs to, and the coverage of a sweep's case table.

Each output element of a kernel is checked against its fp64 reference r:

    |got - r| <= floor + C * scale

scale is the size of one unit of C (usually U24 * M, with M the element's magnitude: the sum of the absolute values of
the terms of its accumulation chain) and floor the error allowed outright (usually U24 * |r| for the final rounding
and a multiple of TINY for roundings in the subnormal range).  Each sweep derives its C, M and floor where it states
its kernels' chains; this module only measures against them.

The non-finite rule: a NaN reference needs a NaN result, a +-inf reference the same infinity and a finite reference a
finite result.  A break counts as infinitely far off.  worst(..., finiteness_only=True) holds a non-finite reference to
a non-finite result of either kind; the training-layer sweep's batch_norm running mean needs it (see there).
"""
import math

import torch

U24 = 2.0 ** -24          # one fp32 rounding, relative
TINY = 2.0 ** -149        # the spacing of fp32's subnormals: one rounding in that range, absolute


def worst(got, r, scale, floor, finiteness_only=False):
    """(worst, index): the max over the elements of (|got - r| - floor) / scale, <= C passes, and the index of the
    element where it is reached.  -inf when every element is within the floor; +inf where the error passes the floor
    and scale is 0, or where the non-finite rule breaks.  finiteness_only relaxes that rule for a non-finite reference
    to any non-finite result."""
    r = r.double()
    g = got.to(r.device, torch.float64).reshape(r.shape)
    broke = torch.where(torch.isnan(r), ~torch.isnan(g), torch.where(torch.isinf(r), g != r, ~torch.isfinite(g)))
    if finiteness_only:
        broke = torch.isfinite(r) != torch.isfinite(g)
    excess = (g - r).abs() - floor
    q = torch.where(excess <= 0, -math.inf, excess / scale)
    q = torch.where(torch.isfinite(r), torch.where(torch.isnan(q), math.inf, q), -math.inf)
    q = torch.where(broke, math.inf, q)
    if q.numel() == 0:
        return -math.inf, None
    i = int(q.argmax())
    return float(q.flatten()[i]), tuple(int(v) for v in torch.unravel_index(torch.tensor(i), q.shape))


def err_ratio(got, r, scale):
    """the worst |got - r| / scale over the elements where both are finite (0 where both the error and scale are 0):
    the figure the sweeps print"""
    r = r.double()
    g = got.to(r.device, torch.float64).reshape(r.shape)
    scale = torch.as_tensor(scale, dtype=torch.float64, device=r.device).expand_as(r)
    fin = torch.isfinite(r) & torch.isfinite(g)
    e = (g - r).abs()[fin]
    if e.numel() == 0:
        return 0.0
    return float(torch.where(e == 0, 0.0, e / scale[fin]).max())


def coverage(cases, classes):
    """{class name: [indices of the cases in it]} for classes given as [(name, predicate(case))]"""
    return {name: [i for i, c in enumerate(cases) if fn(c)] for name, fn in classes}


def uncovered(cases, classes):
    """the names of the classes no case is in"""
    return [name for name, fn in classes if not any(fn(c) for c in cases)]
