"""Exact mode's tile pairs on the GPU: two tiles share one weight stream (tile rows 2q, 2q + 1 of a tall map, or image
groups 2q, 2q + 1 of one weight set on a one-row map), and a pair without a partner computes a second tile past the map
that stores nothing.  Pairing must not change a bit: every image's output is the same whether it runs in the full batch
or alone, in single- and multi-problem launches; and the results match the fp32 SIMT path."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

CASES = [
    # N, H, W, Cin, Cout, k, stride, wsets, relu, residual
    (3, 56, 56, 48, 48, 3, 1, 1, 1, 1),           # 4 tile rows: row pairs
    (3, 40, 40, 64, 64, 3, 1, 1, 1, 0),           # 3 tile rows: the last row has no partner
    (3, 56, 56, 64, 64, 7, 2, 1, 1, 0),           # the limb stem: stride 2, 2 tile rows
    (5, 14, 14, 64, 96, 3, 1, 1, 1, 1),           # one tile row: image pairs, odd image count
    (3, 7, 7, 64, 64, 3, 1, 1, 1, 1),             # stacked small maps (2 per tile): 2 groups, then 1 unpaired
    (7, 7, 7, 128, 64, 3, 2, 1, 0, 1),            # stacked stride 2 (3 per tile), 3 groups
    (264, 2, 2, 32, 48, 3, 1, 24, 1, 1),          # 24 weight sets, 11 images per set: 5 + 5 + 1 per tile, 3 groups
    (72, 4, 4, 64, 32, 3, 2, 24, 1, 0),           # weight sets, stacked stride 2: one group per set, unpaired
    (48, 28, 28, 48, 24, 3, 1, 24, 0, 0),         # weight sets on tall maps: row pairs of one image
]


def _run(problems_inputs):
    """[(case, x, w, b, res)] -> one exact-mode launch; [(y_f32, merged planes)] on the CPU"""
    from conv_tc_common import desc, launch, merge, pack, problem, split
    probs, outs, keep = [], [], []
    for case, x, w, b, res in problems_inputs:
        N, H, W, Cin, Cout, k, s, G, relu, has_res = case
        Ho, Wo = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
        d = desc(case, True)
        xp = split(x.to(DEV))
        wpk = pack(d, w.to(DEV))
        bc = b.to(DEV)
        rc = res.to(DEV) if res is not None else None
        y = torch.full((N, Ho, Wo, Cout), float("nan"), device=DEV)
        yh = torch.full((N, Ho, Wo, Cout), float("nan"), dtype=torch.float16, device=DEV)
        yl = torch.full((N, Ho, Wo, Cout), float("nan"), dtype=torch.float16, device=DEV)
        probs.append(problem(d, xp, wpk, bc, res=rc, y_f32=y, y_planes=(yh, yl)))
        outs.append((y, yh, yl))
        keep += [xp, wpk, bc, rc]
    launch(probs)
    torch.cuda.synchronize()
    return [(y.cpu(), merge(yh, yl).cpu()) for y, yh, yl in outs]


def _alone(case, x, res, j):
    """batch entry j alone: image j, or with weight sets the wsets images of entry j"""
    G = case[7]
    sub = (G,) + case[1:] if G > 1 else (1,) + case[1:]
    sl = slice(j * G, (j + 1) * G) if G > 1 else slice(j, j + 1)
    return sub, x[sl], (res[sl] if res is not None else None), sl


@pytest.mark.parametrize("case", CASES)
def test_pair_outputs_do_not_depend_on_the_batch(case):
    from conv_tc_common import make_case
    x, w, b, res = make_case(case, seed=7)
    (y, ym), = _run([(case, x, w, b, res)])
    assert not torch.isnan(y).any() and not torch.isnan(ym).any()
    N, G = case[0], case[7]
    for j in range(N // G if G > 1 else N):
        sub, xs, rs, sl = _alone(case, x, res, j)
        (y1, ym1), = _run([(sub, xs, w, b, rs)])
        assert torch.equal(y[sl], y1) and torch.equal(ym[sl], ym1), (case, j)


@pytest.mark.parametrize("case", CASES)
def test_pair_matches_simt(case):
    from conv_tc_common import make_case
    from danet_b200.plan import ActBuf, CudaOps
    N, H, W, Cin, Cout, k, s, G, relu, has_res = case
    x, w, b, res = make_case(case, seed=11)
    (y, ym), = _run([(case, x, w, b, res)])
    d = dict(N=N, H=H, W=W, Cin=Cin, Cout=Cout, ksize=k, stride=s, pad=k // 2, wsets=G, relu=relu)
    ys = torch.full(y.shape, float("nan"), device=DEV)
    CudaOps(DEV).conv2d(d, ActBuf(f32=x.to(DEV)), w.to(DEV), b.to(DEV), ActBuf(f32=res.to(DEV)) if has_res else None,
                        ActBuf(f32=ys))
    torch.cuda.synchronize()
    # the exact mode's tolerance against fp64 (tests/test_kernels_gpu.py) plus the SIMT path's own
    tol = 2e-5 + 1.5e-8 * k * k * Cin + 2e-5
    e1, e2 = (y - ys.cpu()).abs().max().item(), (ym - ys.cpu()).abs().max().item()
    assert e1 < tol and e2 < tol, (case, e1, e2)


def test_multi_problem_launch_pairs_each_problem():
    """row pairs, image pairs, an unpaired image group and weight sets in one launch == each problem alone, and each
    batch entry alone, bit for bit"""
    from conv_tc_common import make_case
    cases = [CASES[1], CASES[3], CASES[4], CASES[6]]
    inputs = []
    for c in cases:
        x, w, b, res = make_case(c, seed=3)
        inputs.append((c, x, w, b, res))
    together = _run(inputs)
    for (c, x, w, b, res), (y, ym) in zip(inputs, together):
        (y1, ym1), = _run([(c, x, w, b, res)])
        assert torch.equal(y, y1) and torch.equal(ym, ym1), c
        sub, xs, rs, sl = _alone(c, x, res, (c[0] // c[7] if c[7] > 1 else c[0]) - 1)     # the last entry: unpaired
        (y2, ym2), = _run([(sub, xs, w, b, rs)])
        assert torch.equal(y[sl], y2) and torch.equal(ym[sl], ym2), c
