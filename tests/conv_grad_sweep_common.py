"""The covering sweep of the differentiable convolution (danet_b200.conv.conv2d): the case table, the coverage classes,
the weight-gradient geometry restated from csrc/conv_wgrad.cu, and the per-element bound its outputs are held to.

A case is (B, cin, cout, H, W, k, stride, groups, bias), channel counts per group as in torch.nn.functional.conv2d.
What a case exercises in the backward is not visible in its shape: the weight gradient's split K (pixel chunks, stage
counts) comes from make_geo in conv_wgrad.cu, which wgrad_geo restates (tests/test_conv_grad_sweep_cpu.py holds it to
the library's own workspace size), and the input gradient's pieces come from oracle/conv_bwd.dgrad_pieces.  CLASSES
states, as predicates over a case and its geometry, everything the table has to cover; tests/test_conv_grad_sweep_cpu.py
fails with the names of the uncovered classes, and tests/test_conv_grad_sweep_gpu.py runs every case on the GPU.

The bound (see bounds()): each output element against an fp64 reference r,

    |out - r| <= c * (u * A + phi_a * P_a + phi_b * P_b) + 2^-24 |r| + 2^-149

with u = 2^-22 (split-fp16 operands), A the output's sum of absolute products, and for each of the two operands a, b
of the product phi = 2^-25 * 2^-s, where 2^s is the power-of-two scale that operand's split applies (pow2_scale: the
largest finite |v| * 2^s lies in [2^13, 2^14), s clamped to [-126, 126]): below 2^-12 of the largest value the lo half
of a scaled split is an fp16 subnormal, an absolute error of up to 2^-25 in scaled units.  P_a is the same product with
|b| and a replaced by ones.  db, a sum of the fp32 dy in double, has 2^-24 |r| + 2^-50 sum |dy|."""
import math

import torch
import torch.nn.functional as F

import fp64_bound as fb

U_SPLIT = 2.0 ** -22

# the 18 network convolutions of body_net, limb_net, limb_reslayer and two HRNet shapes:
# (name, cin, cout, H, k, stride, groups), channel counts per group, square maps
NET_SHAPES = [
    ("body_in_1x1_75-64", 75, 64, 56, 1, 1, 1),
    ("limb_in_1x1_21-64", 21, 64, 56, 1, 1, 1),
    ("stem_7x7s2_64-64", 64, 64, 56, 7, 2, 1),
    ("layer1_3x3_64-64", 64, 64, 14, 3, 1, 1),
    ("layer2_3x3s2_64-128", 64, 128, 14, 3, 2, 1),
    ("layer2_down_1x1s2_64-128", 64, 128, 14, 1, 2, 1),
    ("layer2_3x3_128-128", 128, 128, 7, 3, 1, 1),
    ("layer3_3x3s2_128-256_7to4", 128, 256, 7, 3, 2, 1),
    ("layer3_down_1x1s2_128-256_7to4", 128, 256, 7, 1, 2, 1),
    ("layer3_3x3_256-256", 256, 256, 4, 3, 1, 1),
    ("layer4_3x3s2_256-512_4to2", 256, 512, 4, 3, 2, 1),
    ("layer4_down_1x1s2_256-512", 256, 512, 4, 1, 2, 1),
    ("layer4_3x3_512-512", 512, 512, 2, 3, 1, 1),
    ("limb_reslayer_3x3s2_g24", 256, 128, 4, 3, 2, 24),
    ("limb_reslayer_3x3_g24", 128, 128, 2, 3, 1, 24),
    ("limb_reslayer_down_1x1s2_g24", 256, 128, 4, 1, 2, 24),
    ("hrnet_3x3_96-96", 96, 96, 28, 3, 1, 1),
    ("hrnet_3x3s2_48-96", 48, 96, 56, 3, 2, 1),
]


def net_case(shape, B, bias):
    _, cin, cout, H, k, s, G = shape
    return (B, cin, cout, H, H, k, s, G, bias)


# (B, cin, cout, H, W, k, stride, groups, bias): the class cases, then the network rows
CASES = [
    (2, 5, 21, 13, 10, 1, 1, 1, 1),        # 1x1: H != W, cin < 8, Ho % 8 and Wo % 8 over two patches
    (3, 8, 3, 1, 37, 1, 1, 1, 0),          # 1x1, H = 1, W = 37: a ragged scatter column tile, cout < 8
    (2, 21, 8, 9, 1, 3, 1, 1, 1),          # 3x3, W = 1, cout = 8
    (1, 64, 25, 11, 7, 3, 1, 1, 0),        # 3x3: H != W, cout 25 (an IUV head), B = 1
    (2, 3, 64, 1, 1, 3, 1, 1, 1),          # 1x1 map, cout = 64
    (2, 72, 15, 10, 12, 1, 2, 1, 0),       # 1x1/s2 even x even, cin 72: a ragged last wgrad block, cout 15
    (2, 25, 136, 9, 11, 1, 2, 1, 1),       # 1x1/s2 odd x odd, cout 136, a ragged scatter channel tile of y
    (1, 40, 128, 12, 7, 1, 2, 1, 1),       # 1x1/s2 even x odd
    (3, 16, 4, 7, 10, 1, 2, 1, 0),         # 1x1/s2 odd x even, cout 4 (an IUV head)
    (2, 136, 72, 14, 10, 3, 2, 1, 1),      # 3x3/s2 even x even, cin 136
    (2, 24, 40, 13, 9, 3, 2, 1, 0),        # 3x3/s2 odd x odd
    (3, 1, 24, 10, 17, 3, 2, 1, 1),        # 3x3/s2 even x odd, cin = 1
    (2, 128, 64, 9, 16, 3, 2, 1, 0),       # 3x3/s2 odd x even, cin 128
    (2, 16, 24, 20, 22, 7, 2, 1, 1),       # 7x7/s2 even x even, two patches per direction
    (2, 8, 16, 21, 15, 7, 2, 1, 0),        # 7x7/s2 odd x odd
    (1, 3, 8, 12, 9, 7, 2, 1, 1),          # 7x7/s2 even x odd, cin 3 (an image stem), B = 1
    (2, 24, 16, 3, 2, 7, 2, 1, 0),         # 7x7/s2 on a 3 x 2 map
    (2, 16, 8, 1, 1, 7, 2, 1, 1),          # 7x7/s2 on a 1 x 1 map
    (2, 5, 7, 9, 8, 3, 1, 2, 1),           # 2 groups, per-group channels padded to 8
    (2, 3, 5, 8, 9, 3, 2, 3, 0),           # 3 groups, padded, stride 2
    (2, 21, 15, 6, 5, 1, 1, 3, 1),         # 3 groups, padded, 1x1
    (2, 72, 136, 5, 3, 3, 1, 24, 1),       # 24 groups: units0 = 24 * 9 * 2 * 3 > 8 * 132
    (4, 200, 64, 6, 6, 1, 1, 1, 0),        # nchunk = 1 (four tiles: the cap is 1)
    (13, 64, 64, 8, 290, 3, 1, 1, 1),      # 481 tiles: nchunk 97 from the 8-wave target, a last chunk of one stage
    (2, 64, 64, 72, 40, 1, 1, 1, 0),       # nchunk capped at tiles_set / 4 (22), chunks of 5 stages
    (1, 16, 16, 72, 40, 3, 1, 1, 1),       # nchunk capped at tiles_set / 4 (11), chunks of 5 stages
]
CASES += [net_case(s, B, bias) for s in NET_SHAPES for B in (2, 16) for bias in (0, 1)]

# make_geo's constants (conv_wgrad.cu)
_BOX, _CH, _TARGET, _MIN_STAGES = 8, 64, 8 * 132, 4


def ceil8(c):
    return (c + 7) // 8 * 8


def out_hw(case):
    H, W, k, s = case[3], case[4], case[5], case[6]
    return (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1


def desc_fields(case):
    """the danet_conv_desc fields (N, H, W, Cin, Cout, ksize, stride, pad, wsets) conv2d gives danet_conv_wgrad"""
    B, cin, cout, H, W, k, s, G = case[:8]
    return (B * G, H, W, ceil8(cin), ceil8(cout), k, s, k // 2, G)


def make_geo(N, H, W, Cin, Cout, k, s, pad, wsets):
    """make_geo of conv_wgrad.cu: a dict, or None where it refuses the shape"""
    if s not in (1, 2) or k not in (1, 3, 7) or pad != k // 2:
        return None
    if Cin % 8 or Cout % 8 or H < 1 or W < 1 or N < 1 or wsets < 1 or N % wsets:
        return None
    g = {"Ho": (H + 2 * pad - k) // s + 1, "Wo": (W + 2 * pad - k) // s + 1, "taps": k * k,
         "ncib": -(-Cin // _CH), "ncob": -(-Cout // _CH)}
    g["tiles_w"], g["tiles_h"] = -(-g["Wo"] // _BOX), -(-g["Ho"] // _BOX)
    ts = N // wsets * g["tiles_w"] * g["tiles_h"]
    u0 = wsets * g["taps"] * g["ncib"] * g["ncob"]
    if ts >= 1 << 30 or u0 >= 1 << 24:
        return None
    if N * H * W * Cin >= 1 << 31 or N * g["Ho"] * g["Wo"] * Cout >= 1 << 31:
        return None
    g["tiles_set"], g["units0"] = ts, u0
    g["target"] = -(-_TARGET // u0)
    g["cap"] = ts // _MIN_STAGES if ts // _MIN_STAGES > 1 else 1
    nchunk = min(g["target"], g["cap"])
    g["tpc"] = -(-ts // nchunk)
    g["nchunk"] = -(-ts // g["tpc"])
    g["stages_first"] = min(g["tpc"], ts)
    g["stages_last"] = ts - (g["nchunk"] - 1) * g["tpc"]
    return g


def wgrad_geo(case):
    """the weight-gradient geometry conv2d's backward gives danet_conv_wgrad for a case"""
    g = make_geo(*desc_fields(case))
    assert g is not None, ("make_geo refuses this case", case)
    return g


def _classes():
    """[(name, predicate((case, geo)))]"""
    cl = []

    def add(name, fn):
        cl.append((name, lambda cg: fn(*cg)))

    # filter x stride x map parity; a non-square map for every (k, s)
    for k, s in ((1, 1), (3, 1), (1, 2), (3, 2), (7, 2)):
        add("%dx%d/s%d, H != W" % (k, k, s), lambda c, g, k=k, s=s: c[5] == k and c[6] == s and c[3] != c[4])
        if s == 2:
            for ph in (0, 1):
                for pw in (0, 1):
                    add("%dx%d/s2, %s H x %s W" % (k, k, ("even", "odd")[ph], ("even", "odd")[pw]),
                        lambda c, g, k=k, ph=ph, pw=pw: c[5] == k and c[6] == 2 and c[3] > 1 and c[4] > 1
                        and c[3] % 2 == ph and c[4] % 2 == pw)
    # map edges
    add("1x1 map", lambda c, g: c[3] == 1 and c[4] == 1)
    add("H = 1, W > 1", lambda c, g: c[3] == 1 and c[4] > 1)
    add("W = 1, H > 1", lambda c, g: c[4] == 1 and c[3] > 1)
    add("7x7/s2 on a map no larger than 3", lambda c, g: c[5] == 7 and c[3] <= 3 and c[4] <= 3)
    add("W > 32, W % 32 != 0: a ragged scatter column tile of dx", lambda c, g: c[4] > 32 and c[4] % 32 != 0)
    add("Wo > 32, Wo % 32 != 0: a ragged scatter column tile of y", lambda c, g: g["Wo"] > 32 and g["Wo"] % 32 != 0)
    add("Ho % 8 != 0 over two or more wgrad patches", lambda c, g: g["Ho"] % 8 != 0 and g["tiles_h"] >= 2)
    add("Wo % 8 != 0 over two or more wgrad patches", lambda c, g: g["Wo"] % 8 != 0 and g["tiles_w"] >= 2)
    # channels, per group
    for name, i in (("cin", 1), ("cout", 2)):
        add("%s < 8" % name, lambda c, g, i=i: c[i] < 8)
        add("%s = 8" % name, lambda c, g, i=i: c[i] == 8)
        add("8 < %s < 64, not a multiple of 8" % name, lambda c, g, i=i: 8 < c[i] < 64 and c[i] % 8 != 0)
        add("%s = 64" % name, lambda c, g, i=i: c[i] == 64)
        add("%s > 64, not a multiple of 64: a ragged last wgrad block" % name, lambda c, g, i=i: c[i] > 64 and c[i] % 64 != 0)
        add("%s >= 128, a multiple of 64" % name, lambda c, g, i=i: c[i] >= 128 and c[i] % 64 == 0)
    add("cout > 32, cout % 32 != 0: a ragged scatter channel tile of y", lambda c, g: c[2] > 32 and c[2] % 32 != 0)
    add("cin > 32, cin % 32 != 0: a ragged scatter channel tile of dx", lambda c, g: c[1] > 32 and c[1] % 32 != 0)
    # groups
    add("groups = 1", lambda c, g: c[7] == 1)
    add("groups 2 or 3, per-group cin and cout padded", lambda c, g: c[7] in (2, 3) and c[1] % 8 != 0 and c[2] % 8 != 0)
    add("groups = 24", lambda c, g: c[7] == 24)
    # the weight gradient's split K
    add("wgrad nchunk = 1", lambda c, g: g["nchunk"] == 1)
    add("wgrad nchunk capped at tiles_set / 4", lambda c, g: g["cap"] > 1 and g["target"] > g["cap"])
    add("wgrad nchunk from the 8-wave target, uncapped, > 1", lambda c, g: 1 < g["target"] <= g["cap"])
    add("wgrad ragged last chunk", lambda c, g: g["tiles_set"] % g["tpc"] != 0)
    add("wgrad chunk of an odd stage count: a last K segment of one stage",
        lambda c, g: g["stages_first"] % 2 == 1 or g["stages_last"] % 2 == 1)
    add("wgrad units0 > 8 * 132", lambda c, g: g["units0"] > _TARGET)
    # the input gradient: nine 7x7/s2 pieces in two launches, shifted pieces
    add("dgrad 7x7/s2 on an odd map", lambda c, g: c[5] == 7 and c[3] % 2 == 1 and c[4] % 2 == 1 and c[3] > 1)
    add("dgrad 7x7/s2 on an even map", lambda c, g: c[5] == 7 and c[3] % 2 == 0 and c[4] % 2 == 0)
    # other
    add("bias", lambda c, g: c[8] == 1)
    add("no bias", lambda c, g: c[8] == 0)
    add("B = 1", lambda c, g: c[0] == 1)
    # the network rows
    for s in NET_SHAPES:
        for B in (2, 16):
            for bias in (0, 1):
                add("network %s B=%d bias=%d" % (s[0], B, bias), lambda c, g, nc=net_case(s, B, bias): c == nc)
    return cl


CLASSES = _classes()


def coverage(cases=None):
    """{class name: [indices of the cases in it]}"""
    cases = CASES if cases is None else cases
    return fb.coverage([(c, wgrad_geo(c)) for c in cases], CLASSES)


# ----------------------------------------------------------------------------------------------------------------------
# inputs and the bound
# ----------------------------------------------------------------------------------------------------------------------
def make_inputs(case, seed):
    """x, w, b (None without bias), dy of a case: fp32 on the CPU, unit-scale data"""
    B, cin, cout, H, W, k, s, G, bias = case
    Ho, Wo = out_hw(case)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, G * cin, H, W, generator=g)
    w = torch.randn(G * cout, cin, k, k, generator=g) * (1.0 / (cin * k * k)) ** 0.5
    b = torch.randn(G * cout, generator=g) * 0.1 if bias else None
    dy = torch.randn(B, G * cout, Ho, Wo, generator=g)
    return x, w, b, dy


def split_exp(v):
    """the exponent s of the power-of-two scale pow2_scale gives v: max finite |v| * 2^s in [2^13, 2^14), clamped to
    [-126, 126]; 0 when v has no finite nonzero value"""
    f = v[torch.isfinite(v)]
    a = float(f.abs().max()) if f.numel() else 0.0
    if a == 0.0:
        return 0
    return min(max(14 - math.frexp(a)[1], -126), 126)


def phi(v):
    return 2.0 ** (-25 - split_exp(v))


class Ops:
    """the convolution C, its input gradient Ct and its weight gradient Wg in fp64 for one case's geometry"""

    def __init__(self, case, x_shape, w_shape):
        self.s, self.p, self.G = case[6], case[5] // 2, case[7]
        self.x_shape, self.w_shape = x_shape, w_shape

    def C(self, x, w):
        return F.conv2d(x, w, stride=self.s, padding=self.p, groups=self.G)

    def Ct(self, dy, w):
        return torch.nn.grad.conv2d_input(self.x_shape, w, dy, stride=self.s, padding=self.p, groups=self.G)

    def Wg(self, x, dy):
        return torch.nn.grad.conv2d_weight(x, self.w_shape, dy, stride=self.s, padding=self.p, groups=self.G)


def reference(case, x, w, b, dy):
    """fp64 torch autograd of F.conv2d: (y, dx, dW, db) on the inputs' device (db None without bias)"""
    xd, wd = x.double().requires_grad_(), w.double().requires_grad_()
    bd = b.double().requires_grad_() if b is not None else None
    y = F.conv2d(xd, wd, bd, stride=case[6], padding=case[5] // 2, groups=case[7])
    y.backward(dy.double())
    return y.detach(), xd.grad, wd.grad, (bd.grad if bd is not None else None)


def bounds(case, x, w, b, dy):
    """{output: (r, base, floor)}: the reference r and the bound's terms, |out - r| <= c * base + floor, in fp64 on the
    inputs' device.  The operand scales are those of the whole tensors (a dgrad piece packs with its own, finer scale)."""
    r = dict(zip(("y", "dx", "dW", "db"), reference(case, x, w, b, dy)))
    xd, wd, dyd = x.double(), w.double(), dy.double()
    ax, aw, ady = xd.abs(), wd.abs(), dyd.abs()
    ox, ow, ody = torch.ones_like(xd), torch.ones_like(wd), torch.ones_like(dyd)
    fx, fw, fdy = phi(x), phi(w), phi(dy)
    op = Ops(case, x.shape, w.shape)
    A = op.C(ax, aw)
    if b is not None:
        A = A + b.double().abs()[None, :, None, None]
    out = {"y": U_SPLIT * A + fx * op.C(ox, aw) + fw * op.C(ax, ow),
           "dx": U_SPLIT * op.Ct(ady, aw) + fdy * op.Ct(ody, aw) + fw * op.Ct(ady, ow),
           "dW": U_SPLIT * op.Wg(ax, ady) + fdy * op.Wg(ax, ody) + fx * op.Wg(ox, ady)}
    res = {}
    for name in ("y", "dx", "dW"):
        res[name] = (r[name], out[name], fb.U24 * r[name].abs() + fb.TINY)
    if b is not None:
        res["db"] = (r["db"], torch.zeros_like(r["db"]), fb.U24 * r["db"].abs() + 2.0 ** -50 * ady.sum(dim=(0, 2, 3)))
    return res


# operand magnitudes (x * 2^ex, w * 2^ew, dy * 2^edy; the bias follows y's magnitude 2^(ex + ew)): every fp64 reference
# value stays a finite fp32 value
RANGE = ([(e, 0, 0) for e in (-120, -40, -16, -8, 8, 16, 40)] + [(0, e, 0) for e in (-120, -40, 20, 40)]
         + [(0, 0, e) for e in (-120, -60, -30, 30, 60)]
         + [(40, -40, -60), (-40, 40, 60), (-120, 20, 60), (16, 20, -30), (-16, -40, 30)])


def scaled(x, w, b, dy, ex, ew, edy):
    return x * 2.0 ** ex, w * 2.0 ** ew, (b * 2.0 ** (ex + ew) if b is not None else None), dy * 2.0 ** edy
