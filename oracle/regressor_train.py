"""fp64 torch test double of the regressor branches' training ops -- TEST INFRASTRUCTURE (oracle/__init__.py).

danet_b200.regressor.run_branch walks the lowered network graph through a table of ops; TorchTrainOps is that table
restated with torch.nn.functional (conv2d, batch_norm, max_pool2d, adaptive_avg_pool2d, linear) in the inputs' dtype.
Driven by the product's own walk in float64, it reproduces the reference's DecomposedPredictor (the golden
tests/golden/regressor_train.npz, oracle/gen_golden_regressor.py), which pins the wiring; the GPU tests then use it as
the oracle at batch and map sizes the golden does not cover.

Also here: the synthetic cleaned IUV inputs of the golden and the tests, the keyed fp64 state of the branches, and the
gradient sketch the golden stores instead of 33 M gradient values."""
import zlib

import numpy as np
import torch
import torch.nn.functional as F

RP = "iuv2smpl.smpl_para_Outs."
SKETCH_EDGE = 16                                  # first and last entries kept per tensor


class TorchTrainOps(object):
    """Same interface as the CUDA op table of danet_b200.regressor (conv.conv2d and danet_b200.layers)."""

    @staticmethod
    def conv2d(x, w, b, stride, padding, dilation, groups):
        return F.conv2d(x, w, b, stride, padding, dilation, groups)

    @staticmethod
    def batch_norm(x, rm, rv, w, b, training, momentum, eps, residual=None, relu=False):
        y = F.batch_norm(x, rm, rv, w, b, training, momentum, eps)
        if residual is not None:
            y = y + residual
        return torch.relu(y) if relu else y

    @staticmethod
    def max_pool2d(x, k, s, p):
        return F.max_pool2d(x, k, s, p)

    @staticmethod
    def adaptive_avg_pool2d(x, size):
        return F.adaptive_avg_pool2d(x, size)

    @staticmethod
    def linear(x, w, b, add=None):
        y = F.linear(x, w, b)
        return y + add if add is not None else y


def make_inputs(B, S, seed):
    """Cleaned-looking IUV maps (fp32, CPU): per pixel a one-hot part index (0 = background) with U and V in [0, 1) only
    on the chosen channel.  body_iuv [B,75,S,S] = cat[U,V,I] over 25 parts; part_iuv [B,24,3,7,S,S] per part over
    7 channels."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, 25, (B, S, S), generator=g)
    f32 = dict(generator=g, dtype=torch.float32)
    u, v = torch.rand(B, 1, S, S, **f32), torch.rand(B, 1, S, S, **f32)
    oh = F.one_hot(idx, 25).permute(0, 3, 1, 2).to(torch.float32)
    body = torch.cat([oh * u, oh * v, oh], 1)
    pidx = torch.randint(0, 7, (B, 24, S, S), generator=g)
    pu, pv = torch.rand(B, 24, 1, S, S, **f32), torch.rand(B, 24, 1, S, S, **f32)
    poh = F.one_hot(pidx, 7).permute(0, 1, 4, 2, 3).to(torch.float32)
    part = torch.stack([poh * pu, poh * pv, poh], 2)
    return body.contiguous(), part.contiguous()


def input_checksum(t):
    """(sum, sum of x * (i mod 97)) over the flat tensor, in float64"""
    a = t.detach().double().reshape(-1)
    return np.array([a.sum().item(), (a * (torch.arange(a.numel(), dtype=torch.float64) % 97)).sum().item()])


def keyed_state(seed=0, dtype=torch.float64):
    """The keyed state of the whole regressor (danet_b200.synthetic.keyed_state_dict over the graph's keys, mean
    parameters of make_mean_params(seed)): what build_synthetic_danet loads, and the golden's weights."""
    from danet_b200 import netgraph, synthetic
    g = netgraph.danet_graph(32)
    template = {k: torch.zeros(s.shape, dtype=torch.long if s.init == "long0" else torch.float32) for k, s in g.params.items()
                if k.startswith(RP)}
    mp = synthetic.make_mean_params(seed)
    template[RP + "mean_cam_shape"] = torch.cat([torch.as_tensor(mp["cam"]).reshape(1, 3),
                                                 torch.as_tensor(mp["shape"]).reshape(1, 10)], 1).float()
    sd = synthetic.keyed_state_dict(template, seed)
    return {k: (v.to(dtype) if v.is_floating_point() else v.clone()) for k, v in sd.items()}, g


def _probes(key, shape):
    g = torch.Generator().manual_seed(zlib.crc32(key.encode()) & 0x7FFFFFFF)
    return torch.randn(shape, generator=g, dtype=torch.float64), torch.randn(shape, generator=g, dtype=torch.float64)


def sketch(key, grad):
    """float64 [4 + 2 m]: Frobenius norm, sum, inner products with two tensors seeded from `key`, then the first and
    last m = min(16, numel) entries of the flat gradient."""
    gr = torch.as_tensor(np.asarray(grad, np.float64) if not isinstance(grad, torch.Tensor) else grad.detach().double().cpu())
    r1, r2 = _probes(key, gr.shape)
    f = gr.reshape(-1)
    m = min(SKETCH_EDGE, f.numel())
    head = [f.norm().item(), f.sum().item(), (gr * r1).sum().item(), (gr * r2).sum().item()]
    return np.concatenate([np.array(head), f[:m].numpy(), f[-m:].numpy()])


def sketch_error(got, ref, numel):
    """Largest relative error of a sketch against the reference's, each part scaled by the bound a relative Frobenius
    error e implies (Cauchy-Schwarz): |d norm| <= e |g|; |d sum|, |d <g, r>| <= e |g| |r| (|r| ~ sqrt(numel)); any entry
    |d g_i| <= e |g|.  So sketch_error <= e whenever the full gradients agree to e."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    n = max(abs(ref[0]), 1e-300)
    s = n * np.sqrt(numel)
    return max(abs(got[0] - ref[0]) / n, abs(got[1] - ref[1]) / s, abs(got[2] - ref[2]) / s, abs(got[3] - ref[3]) / s,
               np.abs(got[4:] - ref[4:]).max() / n)


def rel_norm(a, b):
    a = np.asarray(a.detach().double().cpu() if isinstance(a, torch.Tensor) else a, np.float64)
    b = np.asarray(b.detach().double().cpu() if isinstance(b, torch.Tensor) else b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
