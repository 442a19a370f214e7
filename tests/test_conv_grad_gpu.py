"""GPU tests of the differentiable convolution (danet_b200.conv.conv2d) beyond its numbers: repeatability, CUDA-graph
replay, batch independence of dx, needs_input_grad subsets, the input-gradient pieces against the restatement and
argument errors.  y, dx, dW and db against fp64 autograd, element by element, are the sweep's
(tests/test_conv_grad_sweep_gpu.py)."""
import pytest
import torch

from conv_grad_sweep_common import NET_SHAPES as SHAPES

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def make(shape, B, bias, seed=0):
    _, cin, cout, H, k, s, G = shape
    g = torch.Generator(device="cpu").manual_seed(seed + 1000 * B + 7 * H + k)
    x = torch.randn(B, G * cin, H, H, generator=g)
    w = torch.randn(G * cout, cin, k, k, generator=g) * (1.0 / (cin * k * k)) ** 0.5
    b = torch.randn(G * cout, generator=g) * 0.1 if bias else None
    Ho = (H - 1) // s + 1
    gy = torch.randn(B, G * cout, Ho, Ho, generator=g)
    return [t.to(DEV) if t is not None else None for t in (x, w, b, gy)]


def run(x, w, b, gy, s, G, need=(True, True, True)):
    from danet_b200.conv import conv2d
    x = x.clone().requires_grad_(need[0])
    w = w.clone().requires_grad_(need[1])
    b = b.clone().requires_grad_(need[2]) if b is not None else None
    y = conv2d(x, w, b, s, w.shape[-1] // 2, 1, G)
    y.backward(gy)
    return y.detach(), x.grad, w.grad, (b.grad if b is not None else None)


def test_pieces_match_the_restatement():
    import ctypes
    from danet_b200 import _lib
    from oracle import conv_bwd as cb
    lib = _lib.load()
    for k, s in [(1, 1), (3, 1), (1, 2), (3, 2), (7, 2)]:
        arr = (_lib.DgradPiece * 9)()
        n = lib.danet_conv_dgrad_pieces(k, s, arr)
        got = [(p.a, p.b, p.K, p.tr, p.tc, (p.jr0, p.jr1), (p.jc0, p.jc1)) for p in arr[:n]]
        assert got == cb.dgrad_pieces(k, s), (k, s)
    assert lib.danet_conv_dgrad_pieces(7, 1, (_lib.DgradPiece * 9)()) == -1


REP = [SHAPES[2], SHAPES[7], SHAPES[13]]


@pytest.mark.parametrize("shape", REP, ids=[s[0] for s in REP])
def test_bit_repeatable(shape):
    x, w, b, gy = make(shape, 4, True)
    r1 = run(x, w, b, gy, shape[5], shape[6])
    r2 = run(x, w, b, gy, shape[5], shape[6])
    for a, c in zip(r1, r2):
        assert torch.equal(a, c)


@pytest.mark.parametrize("shape", REP, ids=[s[0] for s in REP])
def test_needs_input_grad_subsets(shape):
    x, w, b, gy = make(shape, 4, True)
    full = run(x, w, b, gy, shape[5], shape[6])
    for need in [(True, False, False), (False, True, False), (False, False, True), (False, True, True)]:
        got = run(x, w, b, gy, shape[5], shape[6], need)
        assert torch.equal(got[0], full[0])
        for i in range(3):
            if need[i]:
                assert torch.equal(got[i + 1], full[i + 1]), (need, i)
            else:
                assert got[i + 1] is None


@pytest.mark.parametrize("shape", REP, ids=[s[0] for s in REP])
def test_dx_does_not_depend_on_the_batch(shape):
    s, G = shape[5], shape[6]
    x, w, b, gy = make(shape, 5, False)
    full = run(x, w, b, gy, s, G, (True, False, False))
    for i in (0, 3):
        one = run(x[i:i + 1], w, b, gy[i:i + 1], s, G, (True, False, False))
        assert torch.equal(one[0], full[0][i:i + 1])
        assert torch.equal(one[1], full[1][i:i + 1])


def test_cuda_graph_replays_eager_bits():
    from danet_b200.conv import conv2d
    shape = SHAPES[7]
    s, G = shape[5], shape[6]
    x0, w0, b0, gy = make(shape, 4, True)
    eager = run(x0, w0, b0, gy, s, G)
    x, w, b = x0.clone().requires_grad_(), w0.clone().requires_grad_(), b0.clone().requires_grad_()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            x.grad = w.grad = b.grad = None
            conv2d(x, w, b, s, shape[4] // 2, 1, G).backward(gy)
    torch.cuda.current_stream().wait_stream(side)
    x.grad = w.grad = b.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = conv2d(x, w, b, s, shape[4] // 2, 1, G)
        y.backward(gy)
    graph.replay()
    torch.cuda.synchronize()
    for a, c in zip((y, x.grad, w.grad, b.grad), eager):
        assert torch.equal(a.detach(), c)
    # new weights, same graph: the packing inside the graph follows them
    with torch.no_grad():
        w.mul_(0.5)
    graph.replay()
    torch.cuda.synchronize()
    again = run(x0, w0 * 0.5, b0, gy, s, G)
    for a, c in zip((y, x.grad, w.grad, b.grad), again):
        assert torch.equal(a.detach(), c)


def test_argument_errors():
    from danet_b200.conv import conv2d
    x = torch.randn(2, 8, 8, 8, device=DEV)
    w = torch.randn(8, 8, 3, 3, device=DEV)
    with pytest.raises(ValueError):
        conv2d(x.cpu(), w.cpu(), None, 1, 1)
    with pytest.raises(ValueError):
        conv2d(x.double(), w.double(), None, 1, 1)
    with pytest.raises(ValueError):
        conv2d(x, w, None, 1, 1, dilation=2)
    with pytest.raises(ValueError):
        conv2d(x, torch.randn(8, 8, 5, 5, device=DEV), None, 1, 2)
    with pytest.raises(ValueError):
        conv2d(x, w, None, 1, 0)
    with pytest.raises(ValueError):
        conv2d(x, w, None, 3, 1)
    w7 = torch.randn(8, 8, 7, 7, device=DEV)
    with pytest.raises(ValueError):
        conv2d(x, w7, None, 1, 3)                                  # 7x7 stride 1: not an engine shape
    # each tensor in turn (type, CUDA, dtype), then rank, then one device
    with pytest.raises(ValueError, match="x must be float32"):
        conv2d(x.double(), w.cpu(), None, 1, 1)
    with pytest.raises(ValueError, match="weight must be a CUDA tensor"):
        conv2d(x, w.cpu().double(), None, 1, 1)
    with pytest.raises(ValueError, match="bias must be float32"):
        conv2d(x, w, torch.zeros(8, dtype=torch.float64, device=DEV), 1, 1)
    with pytest.raises(ValueError, match="4-D"):
        conv2d(x[0], w, None, 1, 1)
