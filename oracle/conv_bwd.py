"""numpy fp64 restatement of the convolution backward of csrc/conv_wgrad.cu and danet_b200.conv:

- conv_fwd: torch.nn.functional.conv2d (padding k // 2, stride 1 or 2, groups) by taps;
- dgrad_pieces / dgrad_piece_weights: the output-parity decomposition of the input gradient.  Class (a, b) of dx
  (rows a mod stride, columns b mod stride) is a stride-1 correlation of dy with the taps of W of that parity, Cin and
  Cout swapped; it is split into 1x1 / 3x3 pieces (padding K // 2), each read back shifted by (tr, tc) output pixels;
  for stride 1 the one piece is W rotated by 180 degrees;
- dgrad: the pieces run as stride-1 convolutions, then are shifted, interleaved, cropped and summed into dx;
- wgrad: dW[g][co][ci][r][s] = sum over the images of group g and the output pixels of dy * x at tap (r, s); db = the
  channel sums of dy.

Every array is NCHW / OIHW as torch has them; groups follow nn.Conv2d."""
import numpy as np


def _out_size(n, k, stride):
    return (n + 2 * (k // 2) - k) // stride + 1


def conv_fwd(x, w, stride=1, groups=1):
    """x [B, G*cin, H, W], w [G*cout, cin, k, k] -> y [B, G*cout, Ho, Wo] (padding k // 2), fp64"""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    B, Ct, H, W = x.shape
    Cot, cin, k, _ = w.shape
    G, p = groups, k // 2
    cout = Cot // G
    Ho, Wo = _out_size(H, k, stride), _out_size(W, k, stride)
    xp = np.zeros((B, Ct, H + 2 * p + stride, W + 2 * p + stride))
    xp[:, :, p:p + H, p:p + W] = x
    y = np.zeros((B, Cot, Ho, Wo))
    for g in range(G):
        xg, wg = xp[:, g * cin:(g + 1) * cin], w[g * cout:(g + 1) * cout]
        for r in range(k):
            for s in range(k):
                patch = xg[:, :, r:r + stride * Ho:stride, s:s + stride * Wo:stride]
                y[:, g * cout:(g + 1) * cout] += np.einsum("bchw,oc->bohw", patch, wg[:, :, r, s])
    return y


def parity_taps(k, stride, a):
    """(r0, T, c): taps r = r0 + stride*j (j < T) of dimension parity a; dx[stride*u + a] gets W[r] * dy[u + c - j]"""
    pad = k // 2
    r0 = (a + pad) % stride
    T = (k - 1 - r0) // stride + 1 if r0 <= k - 1 else 0
    return r0, T, (a + pad - r0) // stride


def pieces_1d(k, stride, a):
    """[(K, t, j0, j1)]: the taps whose dy offset c - j lies in [-1, 1] form one centred window (K = 1 for a single
    centred tap, else 3); every other tap is a K = 3 piece with its one tap at the window's edge, read back shifted by
    t = offset - 1 (or offset + 1) output pixels"""
    r0, T, c = parity_taps(k, stride, a)
    if T == 0:
        return []
    jlo, jhi = max(0, c - 1), min(T - 1, c + 1)
    out = [(1 if (jlo == jhi == c) else 3, 0, jlo, jhi)] if jlo <= jhi else []
    for j in range(T):
        if not jlo <= j <= jhi:
            o = c - j
            out.append((3, o - 1 if o > 0 else o + 1, j, j))
    return out


def dgrad_pieces(k, stride):
    """[(a, b, K, tr, tc, (jr0, jr1), (jc0, jc1))] in the order of danet_conv_dgrad_pieces"""
    res = []
    for a in range(stride):
        for b in range(stride):
            for (Kr, tr, r0, r1) in pieces_1d(k, stride, a):
                for (Kc, tc, c0, c1) in pieces_1d(k, stride, b):
                    res.append((a, b, max(Kr, Kc), tr, tc, (r0, r1), (c0, c1)))
    return res


def dgrad_piece_weights(w, k, stride, piece, groups=1):
    """w [G*cout, cin, k, k] -> the piece's kernel as an nn.Conv2d weight of its stride-1 problem: [G*cin, cout, K, K].
    Its output at u + t is dx[stride*u + a], so tap q holds the tap j = K//2 + c - q - t of the parity (if in range)."""
    a, b, K, tr, tc, (jr0, jr1), (jc0, jc1) = piece
    w = np.asarray(w, np.float64)
    Cot, cin = w.shape[:2]
    G = groups
    cout = Cot // G
    out = np.zeros((G * cin, cout, K, K))
    (r0a, _, ca), (r0b, _, cb) = parity_taps(k, stride, a), parity_taps(k, stride, b)
    for qr in range(K):
        jr = K // 2 + ca - qr - tr
        if not jr0 <= jr <= jr1:
            continue
        for qs in range(K):
            js = K // 2 + cb - qs - tc
            if not jc0 <= js <= jc1:
                continue
            r, s = r0a + stride * jr, r0b + stride * js
            for g in range(G):
                out[g * cin:(g + 1) * cin, :, qr, qs] = w[g * cout:(g + 1) * cout, :, r, s].T
    return out


def dgrad(dy, w, H, W, stride=1, groups=1):
    """dy [B, G*cout, Ho, Wo], w [G*cout, cin, k, k] -> dx [B, G*cin, H, W] through the pieces: each a stride-1
    convolution of dy, its map read at [u + tr][v + tc] (0 outside) and summed into its class's entries of dx"""
    dy = np.asarray(dy, np.float64)
    B, _, Ho, Wo = dy.shape
    Cot, cin, k, _ = w.shape
    dx = np.zeros((B, groups * cin, H, W))
    for piece in dgrad_pieces(k, stride):
        a, b, K, tr, tc = piece[:5]
        m = conv_fwd(dy, dgrad_piece_weights(w, k, stride, piece, groups), 1, groups)
        pad = np.zeros((B, groups * cin, Ho + 2 * abs(tr) + 2, Wo + 2 * abs(tc) + 2))
        oy, ox = abs(tr) + 1, abs(tc) + 1
        pad[:, :, oy:oy + Ho, ox:ox + Wo] = m
        sub = dx[:, :, a::stride, b::stride]
        hu, wv = sub.shape[2], sub.shape[3]
        sub += pad[:, :, oy + tr:oy + tr + hu, ox + tc:ox + tc + wv]     # classes without taps have no piece: 0
    return dx


def wgrad(x, dy, k, stride=1, groups=1):
    """x [B, G*cin, H, W], dy [B, G*cout, Ho, Wo] -> (dW [G*cout, cin, k, k], db [G*cout])"""
    x, dy = np.asarray(x, np.float64), np.asarray(dy, np.float64)
    B, Ct, H, W = x.shape
    Cot, Ho, Wo = dy.shape[1:]
    G, p = groups, k // 2
    cin, cout = Ct // G, Cot // G
    xp = np.zeros((B, Ct, H + 2 * p + stride, W + 2 * p + stride))
    xp[:, :, p:p + H, p:p + W] = x
    dW = np.zeros((Cot, cin, k, k))
    for g in range(G):
        xg, dg = xp[:, g * cin:(g + 1) * cin], dy[:, g * cout:(g + 1) * cout]
        for r in range(k):
            for s in range(k):
                patch = xg[:, :, r:r + stride * Ho:stride, s:s + stride * Wo:stride]
                dW[g * cout:(g + 1) * cout, :, r, s] = np.einsum("bohw,bchw->oc", dg, patch)
    return dW, dy.sum(axis=(0, 2, 3))


def executed_taps(k, stride):
    """filter taps the dgrad pieces execute per output pixel of dy (needed: k*k)"""
    return sum(p[2] ** 2 for p in dgrad_pieces(k, stride))
