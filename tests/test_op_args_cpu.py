"""Argument refusals of every public differentiable op, with CPU tensors: the exception type and the message of each
refusal that is reachable without a GPU (wrong type, dtype, rank or shape, non-contiguous input, a bad number or int
pair, a CPU tensor).  The cases also pin each entry point's check order: `layers` checks every tensor's dtype, shape
and layout before any CUDA check, `stn` checks CUDA right after the tensor's own checks, and `conv2d` checks CUDA
before dtype."""
import re

import pytest
import torch

BN = "danet_b200.layers.batch_norm: "
MP = "danet_b200.layers.max_pool2d: "
AP = "danet_b200.layers.adaptive_avg_pool2d: "
LIN = "danet_b200.layers.linear: "
HR = "danet_b200.layers.hr_fuse: "
PC = "danet_b200.stn.part_crops: "
PT = "danet_b200.stn.part_thetas: "
CV = "danet_b200.conv.conv2d: "
NO_CPU = "must be a CUDA tensor (there is no CPU path)"


def _refuses(exc, pattern, fn):
    with pytest.raises(exc, match=pattern):
        fn()


def _t(*shape, dtype=torch.float32):
    return torch.zeros(shape, dtype=dtype)


def _noncontig(*shape):
    return torch.zeros(*shape[:-2], shape[-1], shape[-2]).transpose(-1, -2)


def _cases(prefix, cases):
    """(id, exception, message, call) -> pytest params; the raised message must contain `prefix` + message"""
    return [pytest.param(exc, re.escape(prefix + text), fn, id=i) for i, exc, text, fn in cases]


def _bn(x=None, rm=None, rv=None, w=None, b=None, training=True, momentum=0.1, eps=1e-5, **kw):
    from danet_b200.layers import batch_norm
    x = _t(2, 3, 4, 4) if x is None else x
    C = 3
    p = [_t(C) if t is None else t for t in (rm, rv, w, b)]
    return lambda: batch_norm(x, *p, training, momentum, eps, **kw)


def _bn_missing(i):
    from danet_b200.layers import batch_norm
    p = [_t(3) for _ in range(4)]
    p[i] = None
    return lambda: batch_norm(_t(2, 3, 4, 4), *p, True, 0.1, 1e-5)


BATCH_NORM = _cases(BN, [
    ("running_mean-none", ValueError, "running_mean must be given", _bn_missing(0)),
    ("running_var-none", ValueError, "running_var must be given", _bn_missing(1)),
    ("weight-none", ValueError, "weight must be given", _bn_missing(2)),
    ("bias-none", ValueError, "bias must be given", _bn_missing(3)),
    ("momentum-none", ValueError, "momentum must be a number", _bn(momentum=None)),
    ("momentum-bool", ValueError, "momentum must be a number (got True)", _bn(momentum=True)),
    ("momentum-str", ValueError, "momentum must be a number (got '0.1')", _bn(momentum="0.1")),
    ("eps-none", ValueError, "eps must be a number (got None)", _bn(eps=None)),
    ("input-type", ValueError, "input must be a tensor (got list)", _bn(x=[1.0])),
    ("input-dtype", ValueError, "input must be float32 (got torch.float64)", _bn(x=_t(2, 3, 4, 4, dtype=torch.float64))),
    ("input-layout", ValueError, "input must be contiguous", _bn(x=_noncontig(2, 3, 4, 5))),
    ("input-rank", ValueError, "input must be 4-D NCHW (got 3-D)", _bn(x=_t(2, 3, 16))),
    ("input-layout-before-rank", ValueError, "input must be contiguous", _bn(x=_noncontig(2, 3, 16))),
    ("input-empty", ValueError, "empty input (0, 3, 4, 4)", _bn(x=_t(0, 3, 4, 4))),
    ("stat-shape", ValueError, "running_mean must have shape (3,) (got (2,))", _bn(rm=_t(2))),
    ("stat-dtype", ValueError, "running_var must be float32 (got torch.float16)", _bn(rv=_t(3, dtype=torch.float16))),
    ("weight-layout", ValueError, "weight must be contiguous", _bn(w=_t(6)[::2])),
    ("bias-type", ValueError, "bias must be a tensor (got float)", _bn(b=0.0)),
    ("residual-shape", ValueError, "residual must have shape (2, 3, 4, 4) (got (1, 3, 4, 4))",
     _bn(residual=_t(1, 3, 4, 4))),
    ("residual-dtype", ValueError, "residual must be float32", _bn(residual=_t(2, 3, 4, 4, dtype=torch.float64))),
    ("residual-layout", ValueError, "residual must be contiguous", _bn(residual=_noncontig(2, 3, 4, 4))),
    ("one-value", ValueError, "expected more than 1 value per channel when training", _bn(x=_t(1, 3, 1, 1))),
    ("cpu", ValueError, "input " + NO_CPU, _bn()),
    ("cpu-eval", ValueError, "input " + NO_CPU, _bn(training=False, x=_t(1, 3, 1, 1))),
])


@pytest.mark.parametrize("exc,pattern,fn", BATCH_NORM)
def test_batch_norm_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


def _mp(*args, x=None, **kw):
    from danet_b200.layers import max_pool2d
    x = _t(2, 3, 9, 9) if x is None else x
    return lambda: max_pool2d(x, *args, **kw)


MAX_POOL = _cases(MP, [
    ("kernel-pair", ValueError, "kernel_size must be one int or an equal pair (got (3, 2))", _mp((3, 2), 2, 1)),
    ("kernel-triple", ValueError, "kernel_size must be one int or an equal pair (got (3, 3, 3))", _mp((3, 3, 3), 2, 1)),
    ("kernel-float", ValueError, "kernel_size must be an int (got 3.0)", _mp(3.0, 2, 1)),
    ("kernel-bool", ValueError, "kernel_size must be an int (got True)", _mp(True, 2, 1)),
    ("stride-pair", ValueError, "stride must be one int or an equal pair (got (2, 1))", _mp(3, (2, 1), 1)),
    ("padding-str", ValueError, "padding must be an int (got '1')", _mp(3, 2, "1")),
    ("dilation-pair", ValueError, "dilation must be one int or an equal pair (got [1, 2])", _mp(3, 2, 1, [1, 2])),
    ("kernel", ValueError, "only kernel_size=3, stride=2, padding=1, dilation=1", _mp(2, 2, 1)),
    ("stride-default", ValueError, "only kernel_size=3, stride=2, padding=1, dilation=1", _mp(3, None, 1)),
    ("ceil", ValueError, "only kernel_size=3, stride=2, padding=1, dilation=1", _mp(3, 2, 1, ceil_mode=True)),
    ("indices", ValueError, "only kernel_size=3, stride=2, padding=1, dilation=1", _mp(3, 2, 1, return_indices=True)),
    ("input-type", ValueError, "input must be a tensor (got ndarray)", _mp(3, 2, 1, x=_t(2, 3, 9, 9).numpy())),
    ("input-dtype", ValueError, "input must be float32 (got torch.float64)", _mp(3, 2, 1, x=_t(2, 3, 9, 9, dtype=torch.float64))),
    ("input-layout", ValueError, "input must be contiguous", _mp(3, 2, 1, x=_noncontig(2, 3, 9, 8))),
    ("input-rank", ValueError, "input must be 4-D NCHW (got 3-D)", _mp(3, 2, 1, x=_t(3, 9, 9))),
    ("input-layout-before-rank", ValueError, "input must be contiguous", _mp(3, 2, 1, x=_noncontig(3, 9, 8))),
    ("input-empty", ValueError, "empty input (2, 0, 9, 9)", _mp(3, 2, 1, x=_t(2, 0, 9, 9))),
    ("cpu", ValueError, "input " + NO_CPU, _mp(3, 2, 1)),
    ("cpu-pairs", ValueError, "input " + NO_CPU, _mp((3, 3), [2, 2], (1, 1), (1, 1))),
])


@pytest.mark.parametrize("exc,pattern,fn", MAX_POOL)
def test_max_pool2d_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


def _ap(x, size=1):
    from danet_b200.layers import adaptive_avg_pool2d
    return lambda: adaptive_avg_pool2d(x, size)


AVG_POOL = _cases(AP, [
    ("size", ValueError, "only output_size=1 is supported (got 2)", _ap(_t(2, 3, 4, 4), 2)),
    ("size-pair", ValueError, "only output_size=1 is supported (got (1, 2))", _ap(_t(2, 3, 4, 4), (1, 2))),
    ("input-type", ValueError, "input must be a tensor (got NoneType)", _ap(None)),
    ("input-dtype", ValueError, "input must be float32 (got torch.int64)", _ap(_t(2, 3, 4, 4, dtype=torch.int64))),
    ("input-layout", ValueError, "input must be contiguous", _ap(_noncontig(2, 3, 4, 5))),
    ("input-rank", ValueError, "input must be 4-D NCHW (got 3-D)", _ap(_t(2, 3, 16))),
    ("input-layout-before-rank", ValueError, "input must be contiguous", _ap(_noncontig(2, 3, 16))),
    ("input-empty", ValueError, "empty input (2, 3, 0, 4)", _ap(_t(2, 3, 0, 4))),
    ("cpu", ValueError, "input " + NO_CPU, _ap(_t(2, 3, 4, 4))),
    ("cpu-pair", ValueError, "input " + NO_CPU, _ap(_t(2, 3, 4, 4), (1, 1))),
])


@pytest.mark.parametrize("exc,pattern,fn", AVG_POOL)
def test_adaptive_avg_pool2d_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


def _lin(x=None, w=None, b=None, add=None, bias=True):
    from danet_b200.layers import linear
    x = _t(2, 5) if x is None else x
    w = _t(3, 5) if w is None else w
    b = (_t(3) if b is None else b) if bias else None
    return lambda: linear(x, w, b, add=add)


LINEAR = _cases(LIN, [
    ("input-type", ValueError, "input must be a tensor (got int)", _lin(x=3)),
    ("input-dtype", ValueError, "input must be float32 (got torch.float64)", _lin(x=_t(2, 5, dtype=torch.float64))),
    ("input-layout", ValueError, "input must be contiguous", _lin(x=_t(5, 2).t())),
    ("input-rank", ValueError, "input must be 2-D [N, In] (got 3-D)", _lin(x=_t(2, 5, 1))),
    ("input-layout-before-rank", ValueError, "input must be contiguous", _lin(x=_noncontig(2, 5, 3))),
    ("weight-type", ValueError, "weight must be a tensor (got list)", _lin(w=[[0.0] * 5] * 3)),
    ("weight-dtype", ValueError, "weight must be float32 (got torch.float16)", _lin(w=_t(3, 5, dtype=torch.float16))),
    ("weight-layout", ValueError, "weight must be contiguous", _lin(w=_t(5, 3).t())),
    ("weight-shape", ValueError, "weight must be [Out, 5] (got (3, 4))", _lin(w=_t(3, 4))),
    ("weight-rank", ValueError, "weight must be [Out, 5] (got (3, 5, 1))", _lin(w=_t(3, 5, 1))),
    ("empty", ValueError, "empty input or weight ((0, 5), (3, 5))", _lin(x=_t(0, 5))),
    ("empty-weight", ValueError, "empty input or weight ((2, 5), (0, 5))", _lin(w=_t(0, 5), bias=False)),
    ("bias-shape", ValueError, "bias must have shape (3,) (got (2,))", _lin(b=_t(2))),
    ("bias-dtype", ValueError, "bias must be float32 (got torch.float64)", _lin(b=_t(3, dtype=torch.float64))),
    ("add-shape", ValueError, "add must have shape (3,) (got (4,))", _lin(add=_t(4))),
    ("add-layout", ValueError, "add must be contiguous", _lin(add=_t(6)[::2])),
    ("cpu", ValueError, "input " + NO_CPU, _lin()),
    ("cpu-no-bias", ValueError, "input " + NO_CPU, _lin(bias=False, add=_t(3))),
])


@pytest.mark.parametrize("exc,pattern,fn", LINEAR)
def test_linear_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


def _hr(terms, factors, relu=True):
    from danet_b200.layers import hr_fuse
    return lambda: hr_fuse(terms, factors, relu)


_T = _t(1, 4, 8, 8)
HR_FUSE = _cases(HR, [
    ("no-terms", ValueError, "terms must be a list of 1 to 4 tensors", _hr([], [])),
    ("five-terms", ValueError, "terms must be a list of 1 to 4 tensors", _hr([_T] * 5, [1] * 5)),
    ("terms-tensor", ValueError, "terms must be a list of 1 to 4 tensors", _hr(_T, [1])),
    ("factor-count", ValueError, "factors must be a list with one factor per term", _hr([_T, _T], [1])),
    ("factor-int", ValueError, "factors must be a list with one factor per term", _hr([_T], 1)),
    ("factor-3", ValueError, "factors must be 1, 2, 4 or 8 (got 3)", _hr([_T], [3])),
    ("factor-bool", ValueError, "factors must be 1, 2, 4 or 8 (got True)", _hr([_T], [True])),
    ("factor-float", ValueError, "factors must be 1, 2, 4 or 8 (got 2.0)", _hr([_T, _t(1, 4, 4, 4)], [1, 2.0])),
    ("term-type", ValueError, "terms[1] must be a tensor (got float)", _hr([_T, 0.0], [1, 2])),
    ("term-dtype", ValueError, "terms[0] must be float32 (got torch.float64)", _hr([_T.double()], [1])),
    ("term-layout", ValueError, "terms[0] must be contiguous", _hr([_noncontig(1, 4, 8, 8)], [1])),
    ("term-rank", ValueError, "terms[0] must be a non-empty 4-D NCHW tensor (got (4, 8, 8))", _hr([_t(4, 8, 8)], [1])),
    ("term-layout-before-rank", ValueError, "terms[0] must be contiguous", _hr([_noncontig(4, 8, 8)], [1])),
    ("term-empty", ValueError, "terms[1] must be a non-empty 4-D NCHW tensor (got (1, 4, 0, 4))",
     _hr([_T, _t(1, 4, 0, 4)], [1, 2])),
    ("term-size", ValueError, "terms[1] (1, 4, 3, 4) upsampled by 2 is not [1, 4, 8, 8]",
     _hr([_T, _t(1, 4, 3, 4)], [1, 2])),
    ("term-channels", ValueError, "terms[1] (1, 2, 4, 4) upsampled by 2 is not [1, 4, 8, 8]",
     _hr([_T, _t(1, 2, 4, 4)], [1, 2])),
    ("cpu", ValueError, "terms[0] " + NO_CPU, _hr([_T], [1])),
    ("cpu-two", ValueError, "terms[0] " + NO_CPU, _hr([_T, _t(1, 4, 2, 2)], [1, 4], relu=False)),
])


@pytest.mark.parametrize("exc,pattern,fn", HR_FUSE)
def test_hr_fuse_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


def _pc(xd, th=None):
    from danet_b200.stn import part_crops
    th = _t(2, 24, 2, 3) if th is None else th
    return lambda: part_crops(xd, th)


PART_CROPS = _cases(PC, [
    ("xd-type", ValueError, "xd must be a tensor (got tuple)", _pc((1, 2))),
    ("xd-dtype", ValueError, "xd must be float32 (got torch.float64)", _pc(_t(2, 4, 8, 8, dtype=torch.float64))),
    ("xd-rank", ValueError, "xd must be 4-D (got (2, 4, 8))", _pc(_t(2, 4, 8))),
    ("xd-layout", ValueError, "xd must be contiguous", _pc(_noncontig(2, 4, 8, 8))),
    ("cpu", ValueError, "xd " + NO_CPU, _pc(_t(2, 4, 8, 8))),
    # the CUDA check of xd comes before xd's shape and before every check of thetas
    ("cpu-before-shape", ValueError, "xd " + NO_CPU, _pc(_t(2, 4, 8, 6))),
    ("cpu-before-thetas", ValueError, "xd " + NO_CPU, _pc(_t(2, 4, 8, 8), _t(2, 23, 2, 3, dtype=torch.float64))),
])


@pytest.mark.parametrize("exc,pattern,fn", PART_CROPS)
def test_part_crops_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


def _pt(hm, **kw):
    from danet_b200.stn import part_thetas
    r = _t(24)
    return lambda: part_thetas(hm, _t(2, 25, 8, 8), r, r, **kw)


PART_THETAS = _cases(PT, [
    ("hm-type", ValueError, "hm must be a tensor (got NoneType)", _pt(None)),
    ("hm-dtype", ValueError, "hm must be float32 (got torch.float16)", _pt(_t(2, 24, 8, 8, dtype=torch.float16))),
    ("hm-rank", ValueError, "hm must be 4-D (got (2, 24, 64))", _pt(_t(2, 24, 64))),
    ("hm-layout", ValueError, "hm must be contiguous", _pt(_noncontig(2, 24, 8, 8))),
    ("cpu", ValueError, "hm " + NO_CPU, _pt(_t(2, 24, 8, 8))),
    ("cpu-before-shape", ValueError, "hm " + NO_CPU, _pt(_t(2, 23, 8, 8))),
    ("cpu-before-numbers", ValueError, "hm " + NO_CPU, _pt(_t(2, 24, 8, 8), vis_score="x", center_jitter=None)),
])


@pytest.mark.parametrize("exc,pattern,fn", PART_THETAS)
def test_part_thetas_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


def _cv(x=None, w=None, b=None, *args, **kw):
    from danet_b200.conv import conv2d
    x = _t(2, 8, 6, 6) if x is None else x
    w = _t(8, 8, 3, 3) if w is None else w
    return lambda: conv2d(x, w, b, *args, **kw)


CONV2D = _cases(CV, [
    ("stride-pair", ValueError, "stride must be one int or an equal pair (got (1, 2))", _cv(None, None, None, (1, 2), 1)),
    ("stride-float", ValueError, "stride must be an int (got 1.0)", _cv(None, None, None, 1.0, 1)),
    ("padding-pair", ValueError, "padding must be one int or an equal pair (got [1])", _cv(None, None, None, 1, [1])),
    ("padding-bool", ValueError, "padding must be an int (got True)", _cv(None, None, None, 1, True)),
    ("dilation-str", ValueError, "dilation must be an int (got '1')", _cv(None, None, None, 1, 1, "1")),
    ("groups-zero", ValueError, "groups must be a positive int (got 0)", _cv(None, None, None, 1, 1, 1, 0)),
    ("groups-bool", ValueError, "groups must be a positive int (got True)", _cv(None, None, None, 1, 1, 1, True)),
    ("groups-float", ValueError, "groups must be a positive int (got 1.0)", _cv(None, None, None, 1, 1, 1, 1.0)),
    ("x-type", ValueError, "x must be a tensor", _cv([0.0])),
    ("cpu", ValueError, "x " + NO_CPU, _cv(None, None, None, 1, 1)),
    ("cpu-bias", ValueError, "x " + NO_CPU, _cv(None, None, _t(8), (1, 1), (1, 1), (1, 1), 1)),
    # CUDA before dtype, rank and shape
    ("cpu-before-dtype", ValueError, "x " + NO_CPU, _cv(_t(2, 8, 6, 6, dtype=torch.float64))),
    ("cpu-before-rank", ValueError, "x " + NO_CPU, _cv(_t(8, 6, 6), _t(8, 8, 5))),
    ("cpu-before-weight-type", ValueError, "x " + NO_CPU, _cv(None, [[0.0]])),
    ("cpu-before-layout", ValueError, "x " + NO_CPU, _cv(_noncontig(2, 8, 6, 6), _noncontig(8, 8, 3, 3))),
])


@pytest.mark.parametrize("exc,pattern,fn", CONV2D)
def test_conv2d_refusals(exc, pattern, fn):
    _refuses(exc, pattern, fn)


@pytest.fixture(scope="module")
def cpu_net():
    from danet_b200.danet import build_synthetic_danet
    return build_synthetic_danet(width=32, device="cpu", keyed=False)


def test_branches_refuse_a_model_without_graph_or_on_the_cpu(cpu_net):
    from danet_b200.regressor import body_branch, limb_branch
    body, part = _t(1, 75, 8, 8), _t(1, 24, 3, 7, 8, 8)
    for fn, x in ((body_branch, body), (limb_branch, part)):
        _refuses(ValueError, re.escape("danet_b200.regressor: model must be a danet_b200.DaNet (it has no network graph)"),
                 lambda: fn(object(), x))
        _refuses(ValueError, re.escape("danet_b200.regressor: move the model to a CUDA device (there is no CPU path)"),
                 lambda: fn(cpu_net, x))
        # the model's device is checked before the input
        _refuses(ValueError, re.escape("danet_b200.regressor: move the model to a CUDA device"), lambda: fn(cpu_net, None))


def test_gcn_head_refuses_cpu_tensors_with_runtime_error(cpu_net):
    from danet_b200.regressor import gcn_head
    rot, gp = _t(2, 24, 128), _t(2, 13)
    _refuses(RuntimeError, re.escape("danet_b200: rot_feats " + NO_CPU), lambda: gcn_head(cpu_net, rot, gp))
    # before any shape check
    _refuses(RuntimeError, re.escape("danet_b200: rot_feats " + NO_CPU), lambda: gcn_head(cpu_net, _t(2, 23, 128), gp))
    _refuses(RuntimeError, re.escape("danet_b200: rot_feats " + NO_CPU),
             lambda: gcn_head(cpu_net, rot.double(), _t(3, 13)))
