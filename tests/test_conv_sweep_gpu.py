"""The covering parity sweep of the tensor-core convolution engine on the GPU (the table and its coverage classes are in
tests/conv_sweep_common.py; tests/test_conv_sweep_cpu.py proves the table covers every class).

Every output element is held to a scale-free bound against an fp64 reference r of the same convolution:

    |y - r| <= c * (u * A + f * conv(1, |w|)) + u_out * |r| + f_out,      A = conv(|x|, |w|) + |b| + |res|

    exact mode: u = 2^-22 (split-fp16 operands), f = 2^-25 (an activation below 0.25 has a subnormal lo half, so its
                split has an absolute error of up to 2^-25 instead of 22 relative bits)
    fast mode:  u = 2^-10 (two fp16 operands), f = 2^-25 (fp16 subnormals)
    output:     u_out = 2^-24 for the fp32 view, 2^-22 (exact) / 2^-11 (fast) for the planes, which also have the
                absolute floor f_out = 2^-25

A residual given as planes carries the same absolute floor f on its own, so it adds f beside conv(1, |w|).

The constants c are calibrated, not derived: on an NVIDIA H100 80GB HBM3 (700 W power limit) the worst ratio
|error| / bound over every test of this file was 0.95 in exact mode and 0.51 in fast mode; C is 3.0 and 2.0.  The mean
signed error of long sums of non-negative data (test_long_sums_of_non_negative_data_are_not_biased) measured -1.7 u to
-1.9 u on the same card for chains of 98 to 392 main-chain MMAs: the truncation inside one K segment of 8 MMAs, which
does not grow with K; C_BIAS is 4.0 (an unsegmented chain of these lengths sits tens of u below the reference).
"""
import pytest
import torch

from conv_sweep_common import CASES, base, out_hw, report
import fp64_bound as fb

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

U_MMA = {"exact": 2.0 ** -22, "fast": 2.0 ** -10}
FLOOR = 2.0 ** -25
U_PLANES = {"exact": 2.0 ** -22, "fast": 2.0 ** -11}
C = {"exact": 3.0, "fast": 2.0}
C_BIAS = 4.0


def _inputs(case, seed, dist="randn"):
    """x, w, b, res of a case (CPU fp32); b is None for a NULL bias, res None without a residual"""
    from conv_tc_common import make_case
    bc = base(case)
    x, w, b, res = make_case(bc, seed=seed)
    if dist == "uniform":
        g = torch.Generator().manual_seed(seed)
        x, w = torch.rand(x.shape, generator=g), torch.rand(w.shape, generator=g)
    if len(case) > 11 and not case[11]:
        b = None
    return x, w, b, res


def _reference(case, x, w, b, res):
    """fp64: the reference r, the magnitude A and conv(1, |w|)"""
    from conv_tc_common import reference
    bc = base(case)
    zb = torch.zeros(w.shape[0], w.shape[2])
    r = reference(bc, x, w, zb if b is None else b, res)
    lin = bc[:8] + (0, bc[9])                                     # no ReLU on the magnitudes
    A = reference(lin, x.abs(), w.abs(), zb if b is None else b.abs(), res.abs() if res is not None else None)
    Ws = reference(lin[:9] + (0,), torch.ones_like(x), w.abs(), zb, None)
    return r, A, Ws


def _worst(y, view, prec, r, A, Ws, res_planes=False):
    """the worst error of one output view in units of the bound's c (<= C[prec] passes), and where"""
    u_out, f_out = (fb.U24, 0.0) if view == "f32" else (U_PLANES[prec], FLOOR)
    assert torch.isfinite(y).all(), "%s output has NaN / inf (unwritten or overflowed elements)" % view
    return fb.worst(y, r, U_MMA[prec] * A + FLOOR * (Ws + (1.0 if res_planes else 0.0)), u_out * r.abs() + f_out)


def _run(case, x, w, b, res):
    from conv_tc_common import collect, launch, prepare
    exact = case[12] == "exact"
    p, outs, keep = prepare(base(case), exact, x, w, b, res, res_kind=case[9], out_kind=case[10])
    launch([p])
    torch.cuda.synchronize()
    return collect(outs)


def _check(case, x, w, b, res, out=None, what=""):
    """run (unless out is given) and hold every output view to the bound; returns the worst ratio"""
    prec = case[12]
    out = _run(case, x, w, b, res) if out is None else out
    r, A, Ws = _reference(case, x, w, b, res)
    worst = 0.0
    for view in ("f32", "planes"):
        if view not in out:
            continue
        q, at = _worst(out[view], view, prec, r, A, Ws, res_planes=case[9] == "planes")
        print("RATIO %s %s %.3f %s %s" % (prec, view, q, what, case))
        assert q <= C[prec], ("%s view off by %.2f x the %s bound at (n, oh, ow, co) = %s" % (view, q / C[prec], prec, at),
                              what, case, report(case))
        worst = max(worst, q)
    return worst


# ------------------------------------------------------------------------------------------------------------------
# a. the sweep
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(CASES)), ids=lambda i: "%d-%s" % (i, "x".join(str(v) for v in CASES[i][:8]) + "-" + CASES[i][12]))
def test_sweep(i):
    case = CASES[i]
    _check(case, *_inputs(case, seed=1000 + i))


# ------------------------------------------------------------------------------------------------------------------
# b. the K segments keep the tensor core's truncating accumulation from biasing long sums
# ------------------------------------------------------------------------------------------------------------------
BIAS_CASES = [
    (2, 14, 14, 384, 64, 3, 1, 1, 0, "none", "f32", 0, "exact"),
    (4, 7, 7, 512, 64, 3, 1, 1, 0, "none", "f32", 0, "exact"),
    (1, 56, 56, 64, 64, 7, 2, 1, 0, "none", "f32", 0, "exact"),
    (2, 16, 16, 2048, 32, 1, 1, 1, 0, "none", "f32", 0, "exact"),
]


@pytest.mark.parametrize("case", BIAS_CASES, ids=lambda c: "x".join(str(v) for v in c[:8]))
def test_long_sums_of_non_negative_data_are_not_biased(case):
    """x, w uniform in [0, 1): every product is positive, so an accumulation that truncates drifts below the reference
    in proportion to the chain length; the mean signed relative error shows it where a max-error bound does not."""
    x, w, b, res = _inputs(case, seed=77, dist="uniform")
    out = _run(case, x, w, b, res)
    r, A, Ws = _reference(case, x, w, b, res)
    _check(case, x, w, b, res, out=out, what="uniform")
    mean = float(((out["f32"].double() - r) / A).mean())
    print("BIAS %.4f u %s" % (mean / U_MMA["exact"], case))
    assert abs(mean) <= C_BIAS * U_MMA["exact"], ("mean signed error %.3f u" % (mean / U_MMA["exact"]), case, report(case))


# ------------------------------------------------------------------------------------------------------------------
# c. operand range
# ------------------------------------------------------------------------------------------------------------------
RANGE_SHAPES = [
    (2, 12, 10, 48, 32, 3, 1, 1, 1, "f32", "both", 1),
    (3, 7, 7, 64, 24, 3, 2, 1, 0, "planes", "both", 1),
    (2, 9, 9, 16, 16, 1, 1, 1, 0, "f32", "both", 1),
    (1, 20, 12, 24, 40, 7, 2, 1, 1, "planes", "both", 1),
]


@pytest.mark.parametrize("prec", ["exact", "fast"])
@pytest.mark.parametrize("e", [-16, -8, -4, 0, 4, 8])
def test_activation_scale(e, prec):
    """forward activations carry no scale: the bound holds with its absolute floor term at every magnitude"""
    for j, shape in enumerate(RANGE_SHAPES):
        case = shape + (prec,)
        x, w, b, res = _inputs(case, seed=300 + j)
        # bias and residual follow the activations' magnitude, so that the small results stay visible
        sc = 2.0 ** e
        _check(case, x * sc, w, b * sc, res * sc, what="x * 2^%d" % e)


@pytest.mark.parametrize("prec", ["exact", "fast"])
@pytest.mark.parametrize("ew,eb", [(20, 0), (-20, 0), (0, 8), (0, -8), (20, 8), (-20, -8)])
def test_weight_bias_residual_scale(ew, eb, prec):
    """the packed weights' power-of-two scale: bias and residual enter the sum times 2^s and leave it times 2^-s"""
    for j, shape in enumerate(RANGE_SHAPES):
        # weights of 2^20 put the outputs beyond the planes' range: the fp32 view alone
        case = shape[:10] + ("f32" if ew > 0 else "both", 1, prec)
        x, w, b, res = _inputs(case, seed=400 + j)
        _check(case, x, w * 2.0 ** ew, b * 2.0 ** eb, res * 2.0 ** eb, what="w * 2^%d, b, res * 2^%d" % (ew, eb))


@pytest.mark.parametrize("prec", ["exact", "fast"])
def test_weights_of_mixed_magnitude(prec):
    """one scale per packed tensor: output channels whose weights are 2^-12 of the largest still meet the bound"""
    case = RANGE_SHAPES[0] + (prec,)
    x, w, b, res = _inputs(case, seed=500)
    w = w * (2.0 ** -torch.arange(w.shape[2]).remainder(13).float())
    _check(case, x, w, b, res, what="mixed weight magnitudes")


@pytest.mark.parametrize("prec", ["exact", "fast"])
def test_outputs_beyond_the_planes_range(prec):
    """|y| past 65504: the fp32 view is finite and within the bound, the planes are beyond fp16's range exactly there"""
    case = (2, 16, 8, 64, 32, 1, 1, 1, 0, "none", "both", 1, prec)
    x, w, b, res = _inputs(case, seed=600)
    x, w = x * 64.0, w * 512.0                                    # y ~ N(0, 32768^2)
    from conv_tc_common import collect, launch, prepare
    p, outs, keep = prepare(base(case), prec == "exact", x, w, b, None, res_kind="none", out_kind="both")
    launch([p])
    torch.cuda.synchronize()
    out = collect(outs)
    r, A, Ws = _reference(case, x, w, b, None)
    q, at = _worst(out["f32"], "f32", prec, r, A, Ws)
    assert q <= C[prec], (q, at)
    over = out["f32"].abs() >= 65520.0                            # rn_f16 overflows from here
    assert over.any() and (r.abs() > 65504).float().mean() > 0.01
    assert (out["hi"][over].float().abs() >= 65504.0).all()       # no finite value of the wrong magnitude
    inside = out["f32"].abs() < 65504.0
    err = (out["planes"].double() - r).abs()[inside]
    lim = (C[prec] * (U_MMA[prec] * A + FLOOR * Ws) + U_PLANES[prec] * r.abs() + FLOOR)[inside]
    assert (err <= lim).all()


@pytest.mark.parametrize("prec", ["exact", "fast"])
@pytest.mark.parametrize("zero", [0.0, -0.0])
def test_zero_activations_give_bias_plus_residual_exactly(zero, prec):
    for j, shape in enumerate(RANGE_SHAPES):
        case = shape + (prec,)
        x, w, b, res = _inputs(case, seed=700 + j)
        x = torch.full_like(x, zero)
        out = _run(case, x, w, b, res)
        bb = b[torch.arange(case[0]) % case[7]][:, None, None, :]
        if case[9] == "planes":                                   # the planes of the residual are added one after the other
            hi = res.half().float()
            want = bb + hi + ((res - hi).half().float() if prec == "exact" else 0.0)
        else:
            want = bb + res
        want = torch.relu(want) if case[8] else want
        assert torch.equal(out["f32"], want), (case, zero)
        assert torch.equal(out["hi"], want.half()), (case, zero)


# ------------------------------------------------------------------------------------------------------------------
# d. impulses: one input element, every output is one weight tap or the bias
# ------------------------------------------------------------------------------------------------------------------
def _impulse_positions(H, W, Cin):
    pix = [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (0, W // 2), (H // 2, 0), (H - 1, W // 2), (H // 2, W // 2)]
    pix = sorted(set(pix))
    KCH = 64 if Cin >= 40 else (32 if Cin > 16 else 16)
    last0 = (Cin - 1) // KCH * KCH                                # first channel of the last chunk
    ch = sorted({0, min(KCH, Cin) - 1, last0, Cin - 1})
    return [(py, px, ci) for py, px in pix for ci in ch]


def _check_impulses(shape, prec, images=None):
    """image n of the batch carries impulse n (a 1.0 at one pixel and channel).  images: which images of a larger
    batch carry one (the others stay zero and must come out as the bias exactly)."""
    N, H, W, Cin, Cout, k, s, G = shape
    pos = _impulse_positions(H, W, Cin)
    images = list(range(len(pos))) if images is None else images
    N = max(N, len(images)) if G == 1 else N
    case = (N, H, W, Cin, Cout, k, s, G, 0, "none", "both", 1, prec)
    g = torch.Generator().manual_seed(900)
    w = torch.randn(G, k * k * Cin, Cout, generator=g)
    b = torch.randn(G, Cout, generator=g)
    x = torch.zeros(N, H, W, Cin)
    Ho, Wo = out_hw(case)
    want = b.double()[torch.arange(N) % G][:, None, None, :].repeat(1, Ho, Wo, 1)
    tap_at = {}
    for n, (py, px, ci) in zip(images, pos):
        x[n, py, px, ci] = 1.0
        for r in range(k):
            for c in range(k):
                oh, ow = py + k // 2 - r, px + k // 2 - c          # oh * s - pad + r == py
                if oh % s or ow % s or not (0 <= oh // s < Ho and 0 <= ow // s < Wo):
                    continue
                want[n, oh // s, ow // s] += w[n % G, (r * k + c) * Cin + ci].double()
                tap_at[(n, oh // s, ow // s)] = (r, c, ci)
    out = _run(case, x, w, b, None)
    for view, u in (("f32", U_MMA[prec]), ("planes", U_MMA[prec] + U_PLANES[prec])):
        y = out[view].double()
        tol = torch.zeros_like(want)
        for (n, oh, ow) in tap_at:
            tol[n, oh, ow] = 2.0 * u * (want[n, oh, ow].abs() + b[n % G].abs().double()) + FLOOR
        if view == "planes":                                      # elsewhere: the bias, to the planes' precision
            tol = torch.maximum(tol, U_PLANES[prec] * want.abs() + FLOOR)
        bad = ((y - want).abs() > tol).any(-1).nonzero()
        if len(bad):
            n, oh, ow = (int(v) for v in bad[0])
            co = int(((y - want).abs() > tol)[n, oh, ow].nonzero()[0])
            pytest.fail("%s view: %d wrong pixels; first at image %d, output pixel (%d, %d), channel %d: got %r, want %r; "
                        "the pixel %s; impulses %s; %s %s" % (
                            view, len(bad), n, oh, ow, co, float(y[n, oh, ow, co]), float(want[n, oh, ow, co]),
                            ("sees tap (r, s, cin) = %s" % (tap_at[(n, oh, ow)],)) if (n, oh, ow) in tap_at else "sees no impulse: bias only",
                            list(zip(images, pos)), case, report(case)))


@pytest.mark.parametrize("prec", ["exact", "fast"])
@pytest.mark.parametrize("k,s", [(1, 1), (1, 2), (3, 1), (3, 2), (7, 2)])
@pytest.mark.parametrize("hw", [(11, 9), (20, 12)])
def test_impulse_response(k, s, hw, prec):
    _check_impulses((1, hw[0], hw[1], 72, 24, k, s, 1), prec)      # 72 channels: a full chunk and one of 8 channels


@pytest.mark.parametrize("prec", ["exact", "fast"])
@pytest.mark.parametrize("shape,images", [
    ((120, 2, 2, 32, 16, 3, 1, 24), [0, 23, 24, 49, 95, 96, 119, 30, 55, 5, 77, 100, 47, 71, 25, 1]),   # 5 images per set: one tile
    ((264, 2, 2, 32, 48, 3, 1, 24), [0, 24, 120, 121, 144, 240, 263, 239, 119, 47, 26, 168, 215, 192, 25, 1]),
    ((72, 4, 4, 64, 32, 3, 2, 24), list(range(0, 72, 3))),
    ((7, 7, 7, 48, 16, 3, 1, 1), None),
    ((35, 1, 1, 16, 16, 1, 1, 1), None),
])
def test_impulse_in_stacked_images(shape, images, prec):
    """an impulse in one image of a tile must leave every other image of the tile at the bias, exactly"""
    _check_impulses(shape, prec, images)


# ------------------------------------------------------------------------------------------------------------------
# e. launches
# ------------------------------------------------------------------------------------------------------------------
def _mixed_launch(prec):
    t = lambda *c: c + (prec,)
    return [
        t(2, 56, 56, 64, 64, 7, 2, 1, 1, "none", "both", 1),        # the largest halo and box of any problem
        t(3, 16, 8, 16, 16, 1, 1, 1, 0, "f32", "planes", 0),         # 32-byte rows, one K step: runs with the stem's A slot
        t(48, 2, 2, 32, 48, 3, 1, 24, 1, "planes", "both", 1),       # stacked 2x2 maps, 24 weight sets
        t(2, 13, 9, 24, 40, 3, 1, 1, 1, "f32", "f32", 1),            # 64-byte rows, ragged Cout
        t(2, 14, 14, 192, 200, 3, 1, 1, 0, "none", "both", 1),       # several chunks, N tiles; fast: NT 208 ragged
        t(5, 7, 7, 128, 64, 3, 2, 1, 1, "f32", "both", 0),           # stacked stride 2
    ]


@pytest.mark.parametrize("prec", ["exact", "fast"])
def test_mixed_six_problem_launch(prec):
    from conv_tc_common import collect, launch, prepare
    cases = _mixed_launch(prec)
    assert len({report(c)["NT"] for c in cases}) >= 3 and {report(c)["SWB"] for c in cases} == {32, 64, 128}
    inputs = [_inputs(c, seed=800 + j) for j, c in enumerate(cases)]
    prep = [prepare(base(c), prec == "exact", *inp, res_kind=c[9], out_kind=c[10]) for c, inp in zip(cases, inputs)]
    launch([p for p, _, _ in prep])
    torch.cuda.synchronize()
    for c, inp, (_, outs, _) in zip(cases, inputs, prep):
        together, alone = collect(outs), _run(c, *inp)
        for view in alone:
            if view != "planes":
                assert torch.equal(together[view], alone[view]), (view, c)
        _check(c, *inp, out=together, what="six-problem launch")


@pytest.mark.parametrize("prec", ["exact", "fast"])
def test_fewer_work_units_than_sms(prec):
    case = (1, 16, 8, 64, 32, 3, 1, 1, 1, "f32", "both", 1, prec)
    rep = report(case)
    assert rep["tiles_h"] * rep["tiles_w"] * rep["ntn"] == 1
    _check(case, *_inputs(case, seed=810))
    case = (3, 20, 20, 64, 32, 3, 1, 1, 1, "f32", "both", 1, prec)  # a handful of units
    _check(case, *_inputs(case, seed=811))


@pytest.mark.parametrize("prec", ["exact", "fast"])
def test_dynamic_scheduler_and_its_reset(prec):
    """more than 3 work units per CTA, so the global counter hands out tiles; a captured launch keeps its counter slot,
    so the second replay only sees every tile if the first one re-armed the counter"""
    from conv_tc_common import collect, launch, prepare
    case = (32, 56, 56, 16, 16, 3, 1, 1, 1, "f32", "both", 1, prec)
    rep = report(case)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    units = rep["pairs"] if prec == "exact" else case[0] * rep["tiles_h"] * rep["tiles_w"] * rep["ntn"]
    assert units > 3 * sms, (units, sms)
    x, w, b, res = _inputs(case, seed=820)
    p, outs, keep = prepare(base(case), prec == "exact", x, w, b, res, res_kind=case[9], out_kind=case[10])
    launch([p])
    torch.cuda.synchronize()
    first = collect(outs)
    _check(case, x, w, b, res, out=first, what="eager")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch([p])
    replays = []
    for _ in (1, 2):                                              # two replays of one captured argument block
        for t in outs:
            if t is not None:
                t.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        replays.append(collect(outs))
    for rp in replays:
        for view in ("f32", "hi") + (("lo",) if prec == "exact" else ()):
            assert torch.equal(rp[view], first[view]), view


# ------------------------------------------------------------------------------------------------------------------
# f. outputs of more than 2^30 elements: fp32 byte offsets past 4 GiB
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [
    (1, 2056, 2056, 8, 256, 1, 1, 1, 0, "none", "both", 1, "fast"),
    (4, 2056, 2056, 8, 64, 1, 1, 1, 0, "none", "both", 1, "exact"),
], ids=["fast-1x2056x2056x256", "exact-4x2056x2056x64"])
def test_output_offsets_past_4_gib(case):
    from conv_tc_common import desc, launch, pack, problem, split
    free, _ = torch.cuda.mem_get_info()
    if free < 16 << 30:
        pytest.skip("needs 16 GB of free device memory (%.1f GB free)" % (free / 2 ** 30))
    N, H, W, Cin, Cout = case[:5]
    prec, exact = case[12], case[12] == "exact"
    assert N * H * W * Cout > 2 ** 30
    g = torch.Generator().manual_seed(930)
    w = torch.randn(1, Cin, Cout, generator=g)
    b = torch.randn(1, Cout, generator=g)
    x = torch.randn(N, H, W, Cin, generator=g).to(DEV)
    d = desc(base(case), exact)
    xp, wpk, bc = split(x, want_lo=exact), pack(d, w.to(DEV)), b.to(DEV)
    y = torch.full((N, H, W, Cout), float("nan"), device=DEV)
    yh = torch.full((N, H, W, Cout), float("nan"), dtype=torch.float16, device=DEV)
    yl = torch.full((N, H, W, Cout), float("nan"), dtype=torch.float16, device=DEV) if exact else None
    try:
        launch([problem(d, xp, wpk, bc, y_f32=y, y_planes=(yh, yl))])
        torch.cuda.synchronize()
        flat = y.view(-1)
        step = 1 << 28
        for o in range(0, flat.numel(), step):                    # every element was written
            assert not bool(torch.isnan(flat[o:o + step]).any()), "unwritten outputs near element %d" % o
        # the first and last rows and 4096 sampled pixels against an fp64 matmul
        idx = torch.randint(0, N * H * W, (4096,), generator=g)
        idx = torch.cat([torch.arange(W), torch.arange(N * H * W - W, N * H * W), idx]).to(DEV)
        xs = x.view(-1, Cin)[idx].cpu().double()
        r = xs @ w[0].double() + b[0].double()
        A = xs.abs() @ w[0].abs().double() + b[0].abs().double()
        Ws = w[0].abs().double().sum(0).expand_as(r)
        got = {"f32": y.view(-1, Cout)[idx].cpu(),
               "planes": yh.view(-1, Cout)[idx].float().cpu() + (yl.view(-1, Cout)[idx].float().cpu() if exact else 0.0)}
        for view in got:
            q, at = _worst(got[view], view, prec, r, A, Ws)
            assert q <= C[prec], (view, q, at, int(idx[at[0]]))
    finally:
        del y, yh, yl, x, xp
        torch.cuda.empty_cache()
