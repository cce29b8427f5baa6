"""Restatements of main.lua's training path (arch 'fast', KITTI) -- TEST INFRASTRUCTURE.

* :func:`warp_affine`: OpenCV's ``warpAffine(src, M, (ws, ws), INTER_CUBIC, BORDER_CONSTANT, 0)`` on a float32 image
  (what cv.cpp:19-45 calls through ``cvWarpAffine(.., CV_INTER_CUBIC + CV_WARP_FILL_OUTLIERS)``), in numpy, one
  operation at a time: M inverted in double, source coordinates on AB_BITS = 10 fixed point rounded to the 1/32 grid,
  the float cubic table (A = -0.75), interior taps summed row by row, border taps summed one by one onto 0.
* :func:`make_patch`: main.lua:607-619 (mul32 in double, the matrix stored as float, then ``mul(contrast):add(brightness)``
  in float).
* :func:`sample_params`: main.lua:791-818 line by line on ``preprocess.MT19937``, one sample at a time.
* :func:`step64`: one training step of net_tr + Margin2 (main.lua:726-749, 852-874) in float64 torch autograd.
"""
import math

import numpy as np

AB_BITS, INTER_BITS = 10, 5
AB_SCALE, TAB = 1 << AB_BITS, 1 << INTER_BITS
ROUND_DELTA = AB_SCALE // TAB // 2


def cubic_coeffs(x):
    """OpenCV's interpolateCubic in float32, A = -0.75"""
    f = np.float32
    A, x = f(-0.75), f(x)
    t = x + f(1)
    c0 = ((A * t - f(5) * A) * t + f(8) * A) * t - f(4) * A
    c1 = ((A + f(2)) * x - (A + f(3))) * x * x + f(1)
    u = f(1) - x
    c2 = ((A + f(2)) * u - (A + f(3))) * u * u + f(1)
    c3 = f(1) - c0 - c1 - c2
    return [f(c0), f(c1), f(c2), f(c3)]


_TAB1 = [cubic_coeffs(np.float32(1.0 / TAB) * np.float32(i)) for i in range(TAB)]


def invert(m):
    """warpAffine's inversion of the forward matrix, in double"""
    M = [float(v) for v in np.asarray(m, np.float32).reshape(6)]
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    M[0] = A11
    M[1] *= -D
    M[3] *= -D
    M[4] = A22
    b1 = -M[0] * M[2] - M[1] * M[5]
    b2 = -M[3] * M[2] - M[4] * M[5]
    M[2], M[5] = b1, b2
    return M


def _round(v):
    """cvRound: round half to even"""
    return int(np.rint(v))


def _short(v):
    return max(-32768, min(32767, v))


def warp_affine(src, m, ws):
    """(H, W) float32 source, forward 2x3 matrix `m` (float32) -> (ws, ws) float32"""
    src = np.asarray(src, np.float32)
    H, W = src.shape
    M = invert(m)
    out = np.zeros((ws, ws), np.float32)
    f32 = np.float32
    for y in range(ws):
        X0 = _round((M[1] * y + M[2]) * AB_SCALE) + ROUND_DELTA
        Y0 = _round((M[4] * y + M[5]) * AB_SCALE) + ROUND_DELTA
        for x in range(ws):
            X = (X0 + _round(M[0] * x * AB_SCALE)) >> (AB_BITS - INTER_BITS)
            Y = (Y0 + _round(M[3] * x * AB_SCALE)) >> (AB_BITS - INTER_BITS)
            sx, sy = _short(X >> INTER_BITS) - 1, _short(Y >> INTER_BITS) - 1
            ty, tx = _TAB1[Y & (TAB - 1)], _TAB1[X & (TAB - 1)]
            w = [[f32(ty[i] * tx[j]) for j in range(4)] for i in range(4)]
            if 0 <= sx < max(W - 3, 0) and 0 <= sy < max(H - 3, 0):
                s = f32(0)
                for i in range(4):
                    r = src[sy + i, sx:sx + 4]
                    row = f32(f32(f32(r[0] * w[i][0]) + f32(r[1] * w[i][1])) + f32(r[2] * w[i][2])) + f32(r[3] * w[i][3])
                    s = f32(row) if i == 0 else f32(s + row)
                out[y, x] = s
            elif sx >= W or sx + 4 <= 0 or sy >= H or sy + 4 <= 0:
                out[y, x] = 0
            else:
                s = f32(0)
                for i in range(4):
                    if not 0 <= sy + i < H:
                        continue
                    for j in range(4):
                        if 0 <= sx + j < W:
                            s = f32(s + f32(src[sy + i, sx + j] * w[i][j]))
                out[y, x] = s
    return out


def mul32(a, b):
    """main.lua:603-605"""
    return [a[0] * b[0] + a[1] * b[3], a[0] * b[1] + a[1] * b[4], a[0] * b[2] + a[1] * b[5] + a[2],
            a[3] * b[0] + a[4] * b[3], a[3] * b[1] + a[4] * b[4], a[3] * b[2] + a[4] * b[5] + a[5]]


def patch_matrix(ws, dim3, dim4, scale, phi, trans, hshear):
    """make_patch's matrix (main.lua:608-616) as float32"""
    m = [1, 0, -dim4, 0, 1, -dim3]
    m = mul32([1, 0, trans[0], 0, 1, trans[1]], m)
    m = mul32([scale[0], 0, 0, 0, scale[1], 0], m)
    c, s = math.cos(phi), math.sin(phi)
    m = mul32([c, s, 0, -s, c, 0], m)
    m = mul32([1, hshear, 0, 0, 1, 0], m)
    m = mul32([1, 0, (ws - 1) / 2, 0, 1, (ws - 1) / 2], m)
    return np.asarray(m, np.float64).astype(np.float32)


def make_patch(src, ws, dim3, dim4, scale, phi, trans, hshear, brightness, contrast):
    """main.lua:607-619"""
    dst = warp_affine(src, patch_matrix(ws, dim3, dim4, scale, phi, trans, hshear), ws)
    return (dst * np.float32(contrast) + np.float32(brightness)).astype(np.float32)


def uniform(g, a=0.0, b=1.0):
    """torch.uniform(a, b): THRandom_random / 2^32 * (b - a) + a in double"""
    return g.random() * (1.0 / 4294967296.0) * (b - a) + a


def sample_params(g, o):
    """main.lua:791-818 for one sample: the draws of `g` (an MT19937) under options `o` (a dict) -> dict"""
    u = lambda a=0.0, b=1.0: uniform(g, a, b)
    d_pos = u(-o["true1"], o["true1"])
    d_neg = u(o["false1"], o["false2"])
    if u() < 0.5:
        d_neg = -d_neg
    s = u(o["scale"], 1)
    scale = [s * u(o["hscale"], 1), s]
    if o["hflip"] == 1 and u() < 0.5:
        scale[0] = -scale[0]
    if o["vflip"] == 1 and u() < 0.5:
        scale[1] = -scale[1]
    hshear = u(-o["hshear"], o["hshear"])
    trans = [u(-o["trans"], o["trans"]), u(-o["trans"], o["trans"])]
    phi = u(-o["rotate"] * math.pi / 180, o["rotate"] * math.pi / 180)
    brightness = u(-o["brightness"], o["brightness"])
    contrast = u(1 / o["contrast"], o["contrast"])
    scale_ = [scale[0] * u(o["d_hscale"], 1), scale[1]]
    hshear_ = hshear + u(-o["d_hshear"], o["d_hshear"])
    trans_ = [trans[0], trans[1] + u(-o["d_vtrans"], o["d_vtrans"])]
    phi_ = phi + u(-o["d_rotate"] * math.pi / 180, o["d_rotate"] * math.pi / 180)
    brightness_ = brightness + u(-o["d_brightness"], o["d_brightness"])
    contrast_ = contrast * u(1 / o["d_contrast"], o["d_contrast"])
    return dict(d_pos=d_pos, d_neg=d_neg, scale=scale, hshear=hshear, trans=trans, phi=phi, brightness=brightness,
                contrast=contrast, scale_=scale_, hshear_=hshear_, trans_=trans_, phi_=phi_, brightness_=brightness_,
                contrast_=contrast_)


def sample_patches(p, row, x0, x1, ws):
    """main.lua:820-846: the four patches of one sample from its parameters `p` and nnz row (img, dim3, dim4, d)"""
    _, dim3, dim4, d = (float(v) for v in row)
    a = (p["scale"], p["phi"], p["trans"], p["hshear"], p["brightness"], p["contrast"])
    b = (p["scale_"], p["phi_"], p["trans_"], p["hshear_"], p["brightness_"], p["contrast_"])
    return [make_patch(x0, ws, dim3, dim4, *a), make_patch(x1, ws, dim3, dim4 - d + p["d_pos"], *b),
            make_patch(x0, ws, dim3, dim4, *a), make_patch(x1, ws, dim3, dim4 - d + p["d_neg"], *b)]


def init_weights(g, l1, fm, n_in=1, ks=3):
    """nn.SpatialConvolution:reset() of each layer in order: weight then bias, U(-1/sqrt(ks*ks*cin), +..) in double,
    stored as float -> [(W (fm, cin, ks, ks), b (fm,))]"""
    out = []
    for i in range(l1):
        cin = n_in if i == 0 else fm
        stdv = 1 / math.sqrt(ks * ks * cin)
        w = np.array([uniform(g, -stdv, stdv) for _ in range(fm * cin * ks * ks)]).astype(np.float32)
        b = np.array([uniform(g, -stdv, stdv) for _ in range(fm)]).astype(np.float32)
        out.append((w.reshape(fm, cin, ks, ks), b))
    return out


def step64(patches, layers, margin, pow_, inter=False, device=None):
    """One forward / backward of net_tr + Margin2 in float64 autograd: patches (2 bs, 1, ws, ws); layers [(W, b)] ->
    (loss, [(gW, gb)]) as float64 numpy.  With `inter`, a third item: a dict of float64 numpy arrays, "z" and "dz" (each
    layer's convolution output, before its ReLU, and dLoss/dz), "norm" (N,), "normalized" (N, fm), "join" (bs,), "hinge"
    (bs / 2,): the per-sample terms before the mean.  `device` is where torch computes (default the CPU)."""
    import torch

    x = torch.as_tensor(np.asarray(patches), dtype=torch.float64, device=device)
    ps = []
    for w, b in layers:
        ps.append(torch.tensor(np.asarray(w, np.float64), requires_grad=True, device=device))
        ps.append(torch.tensor(np.asarray(b, np.float64), requires_grad=True, device=device))
    h, zs = x, []
    for i in range(len(layers)):
        h = torch.nn.functional.conv2d(h, ps[2 * i], ps[2 * i + 1])
        zs.append(h)
        if i < len(layers) - 1:
            h = torch.relu(h)
    norm = (h * h).sum(1, keepdim=True) + 1e-5                  # Normalize2: x / sqrt(sum x^2 + 1e-5)
    h = h / norm.sqrt()
    s = (h[0::2] * h[1::2]).sum(1).reshape(-1)                 # StereoJoin1: (bs,)
    f = s[1::2] - s[0::2] + margin                             # Margin2: neg - pos + m
    f = torch.clamp(f, min=0)
    terms = f if pow_ == 1 else 0.5 * f * f
    loss = terms.mean()
    grads = torch.autograd.grad(loss, ps + (zs if inter else []))
    g = [t.cpu().numpy() for t in grads]
    out = float(loss.detach()), [(g[2 * i], g[2 * i + 1]) for i in range(len(layers))]
    if not inter:
        return out
    np64 = lambda t: t.detach().cpu().numpy()
    return out + (dict(z=[np64(t) for t in zs], dz=g[len(ps):], norm=np64(norm).reshape(-1),
                       normalized=np64(h).reshape(len(h), -1), join=np64(s), hinge=np64(terms)),)


def update32(p, v, g, mom, lr):
    """main.lua:871-874 in float32: v = v * mom; v = v + (-lr) * g; p = p + v (each operation rounded)"""
    f = np.float32
    v = (np.asarray(v, f) * f(mom)).astype(f)
    v = (v + (f(-lr) * np.asarray(g, f)).astype(f)).astype(f)
    p = (np.asarray(p, f) + v).astype(f)
    return p, v
