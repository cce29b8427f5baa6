"""CPU restatement of preprocess_mb.py -- TEST INFRASTRUCTURE.

* ``read_im``: the script's read_im on decoded bytes: cv2's BGR2GRAY written out as its fused multiply-adds (every product of
  a byte and a float32 coefficient, and every sum below, is exact in float64, so one rounding to float32 per step is the
  fma's), then numpy's own ``(x - x.mean()) / x.std()``;
* ``pairwise_sum``: numpy's float32 pairwise summation (the order csrc/preprocess_mb.cu reproduces), to be pinned against
  numpy itself;
* ``half_image``: the Lanczos-3 halving that replaces ``convert -resize 50%``, in float64 (``half_image_f64`` keeps the values
  before rounding);
* ``half_disp``: load_pfm(.., True) as np.sort over each 2x2 block;
* ``mask``: the computemask rule, in float64;
* ``preprocess_mb``: the whole script, in the script's own order, on top of them.
"""
import os
import re

import numpy as np

F32 = np.float32
LEAF = 128


# ---- views --------------------------------------------------------------------------------------------------------

def cv_grey(rgb):
    """cv2.cvtColor(float32 BGR, BGR2GRAY) of (..., 3) R, G, B bytes: fma(R, .299, fma(B, .114, G * .587)) in float32"""
    rgb = np.asarray(rgb)
    r, g, b = (rgb[..., k].astype(np.float64) for k in range(3))
    inner = (g.astype(F32) * F32(0.587)).astype(F32)
    inner = (b * np.float64(F32(0.114)) + inner.astype(np.float64)).astype(F32)
    return (r * np.float64(F32(0.299)) + inner.astype(np.float64)).astype(F32)


def read_im(rgb, color):
    """read_im(fname, ..) of preprocess_mb.py:85-97 from the decoded (H, W, 3) R, G, B bytes -> (1, C, H, W) float32"""
    rgb = np.asarray(rgb, dtype=np.uint8)
    if color == "rgb":
        x = rgb.astype(F32).transpose(2, 0, 1)              # a view: memory order stays H, W, C
    else:
        x = cv_grey(rgb)[None]
    x = (x - x.mean()) / x.std()
    return x[None]


def pairwise_sum(a):
    """numpy's float32 pairwise_sum of a 1-D array: < 8 elements in turn; <= 128 with eight strided accumulators; else the
    halves [0, n2) and [n2, n), n2 = n // 2 rounded down to a multiple of 8"""
    a = np.asarray(a, dtype=F32)
    n = len(a)
    if n < 8:
        r = F32(0)
        for v in a:
            r = F32(r + v)
        return r
    if n <= LEAF:
        body = n - n % 8
        r = a[:8].copy()
        for i in range(8, body, 8):
            r = (r + a[i:i + 8]).astype(F32)
        res = F32(F32(F32(r[0] + r[1]) + F32(r[2] + r[3])) + F32(F32(r[4] + r[5]) + F32(r[6] + r[7])))
        for i in range(body, n):
            res = F32(res + a[i])
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return F32(pairwise_sum(a[:n2]) + pairwise_sum(a[n2:]))


def mean_std(flat):
    """np.mean and np.std of a float32 array in memory order `flat`, through pairwise_sum"""
    flat = np.asarray(flat, dtype=F32).ravel()
    n = flat.size
    m = F32(np.float64(pairwise_sum(flat)) / n)
    d = (flat - m).astype(F32)
    return m, F32(np.sqrt(F32(np.float64(pairwise_sum((d * d).astype(F32))) / n)))


# ---- halving ------------------------------------------------------------------------------------------------------

def lanczos_weights():
    t = (np.arange(12) - 5.5) / 2
    return np.sinc(t) * np.sinc(t / 3)


def _half_axis(a, axis):
    a = np.moveaxis(np.asarray(a, dtype=np.float64), axis, 0)
    n = a.shape[0]
    w = lanczos_weights()
    out = np.empty((n // 2,) + a.shape[1:])
    for x in range(n // 2):
        j = np.arange(2 * x - 5, 2 * x + 7)
        keep = (j >= 0) & (j < n)
        ww = w[keep]
        out[x] = np.tensordot(ww, a[j[keep]], axes=1) / ww.sum()
    return np.moveaxis(out, 0, axis)


def half_image_f64(img):
    """(H, W, C) bytes, H and W even -> the (H/2, W/2, C) float64 values before rounding: rows first, then columns"""
    img = np.asarray(img)
    if img.shape[0] % 2 or img.shape[1] % 2:
        raise ValueError("odd image size %s" % (img.shape[:2],))
    return _half_axis(_half_axis(img, 1), 0)


def half_image(img):
    return np.clip(np.floor(half_image_f64(img) + 0.5), 0, 255).astype(np.uint8)


def half_disp(d):
    """load_pfm(.., True) on a top-down map: the second smallest of each 2x2 block of d / 2 in np.sort's order"""
    x = np.asarray(d, dtype=F32) / 2
    H, W = x.shape
    if H % 2 or W % 2:
        raise ValueError("odd map size %s" % (x.shape,))
    blocks = x.reshape(H // 2, 2, W // 2, 2).transpose(0, 2, 1, 3).reshape(H // 2, W // 2, 4)
    return np.sort(blocks, axis=-1)[..., 1].astype(F32)


# ---- mask ---------------------------------------------------------------------------------------------------------

def mask(d0, d1, d0y=None):
    """the computemask rule: 0 where d0 is not finite; x1 = floor(x - d0 + .5), y1 = floor(y + d0y + .5) in float64; 128 if
    (x1, y1) is outside the frame (or d0y is not finite) or not |d0 - d1[y1, x1]| <= 1; else 255"""
    d0 = np.asarray(d0, dtype=F32).astype(np.float64)
    d1 = np.asarray(d1, dtype=F32).astype(np.float64)
    H, W = d0.shape
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    dy = np.zeros_like(d0) if d0y is None else np.asarray(d0y, dtype=F32).astype(np.float64)
    fin = np.isfinite(d0)
    with np.errstate(invalid="ignore"):
        x1 = np.floor(x - d0 + 0.5)
        y1 = np.floor(y + dy + 0.5)
        inside = fin & (x1 >= 0) & (x1 < W) & (y1 >= 0) & (y1 < H)
        r = np.full_like(d0, np.nan)
        r[inside] = d1[y1[inside].astype(np.int64), x1[inside].astype(np.int64)]
        ok = inside & (np.abs(d0 - r) <= 1)
    m = np.where(fin, np.uint8(128), np.uint8(0)).astype(np.uint8)
    m[ok] = 255
    return m


def clean(d0, m, image):
    """dispnoc (d0 where m == 255, else 0) and the (image, y, x, d0) float32 rows of the m == 255 pixels, row-major"""
    d0 = np.asarray(d0, dtype=F32).copy()
    d0[m != 255] = 0
    y, x = np.nonzero(m == 255)
    return d0, np.column_stack((np.zeros_like(y) + image, y, x, d0[y, x])).astype(F32)


# ---- the script -----------------------------------------------------------------------------------------------------

def imread_rgb(path):
    """cv2.imread(path) as R, G, B bytes (H, W, 3); a grey file is replicated"""
    from PIL import Image

    with Image.open(path) as im:
        return np.asarray(im.convert("RGB"), dtype=np.uint8)


def imread_grey(path):
    from PIL import Image

    with Image.open(path) as im:
        assert im.mode == "L", "%s: grey 8-bit expected" % path
        return np.asarray(im, dtype=np.uint8)


def read_pfm(path):
    """the script's load_pfm(path, False): the map flipped to top-down rows"""
    from mccnn_b200 import dataio

    return np.ascontiguousarray(np.flipud(dataio.read_pfm(path)))


def _view(path, color, downsample, half=None):
    if downsample:
        cache = path + ".H.png"
        return read_im(imread_rgb(cache) if os.path.isfile(cache) else (half or half_image)(imread_rgb(path)), color)
    return read_im(imread_rgb(path), color)


def _disp_half(path):
    cache = path + ".H.pfm"
    return read_pfm(cache) if os.path.isfile(cache) else half_disp(read_pfm(path))


EXPOSURES = {8: [1, 3, 5], 7: [1, 3, 5], 6: [0, 2, 4], 5: [0, 2, 4], 3: [0, 1, 2], 2: [0, 1]}
_EXP = re.compile(r"^im([01])e(\d)\.png$")
MB = "data.mb/unzip/vision.middlebury.edu/stereo/data"


def preprocess_mb(data_root, rect, color, half=None):
    """preprocess_mb.py: dict(X = [[array or None per view file]], dispnoc, meta, nnz_tr, nnz_te, te, fname_submit).
    `half` replaces half_image for the 2014 views without a cache (tests pass a checked device result)."""
    C = 3 if color == "rgb" else 1
    X, dispnoc, meta, nnz_tr, nnz_te = [], [], [], [], []
    te = np.arange(1, 11)
    root = lambda *p: os.path.join(data_root, *p)

    base1 = root(MB, "scenes2014", "datasets")
    for d in sorted(os.listdir(base1)):
        if not d.endswith("imperfect"):
            continue
        b_imp = os.path.join(base1, d)
        b_perf = b_imp.replace("imperfect", "perfect")
        ndisp = int(re.search("ndisp=(.*)", open(os.path.join(b_imp, "calib.txt")).read()).group(1)) // 2
        views = [_view(os.path.join(b_imp, f), color, True, half) for f in ("im0.png", "im1.png", "im1E.png", "im1L.png")]
        XX = [np.concatenate(views)]
        base3 = os.path.join(b_perf if rect == "perfect" else b_imp, "ambient")
        num_exp = [], []
        for f in os.listdir(os.path.join(base3, "L1")):
            m = _EXP.match(f)
            if m:
                num_exp[int(m.group(1))].append(int(m.group(2)) + 1)
        num_exp = min(max(num_exp[0]), max(num_exp[1]))
        for light in range(len(os.listdir(base3))):
            imgs = [_view(os.path.join(base3, "L%d" % (light + 1), "im%de%d.png" % (cam, e)), color, True, half)
                    for e in EXPOSURES[num_exp] for cam in range(2)]
            _, _, h, w = imgs[0].shape
            XX.append(np.concatenate(imgs).reshape(len(imgs) // 2, 2, C, h, w))
        d0, d1, dy = (_disp_half(os.path.join(b_imp, f)) for f in ("disp0.pfm", "disp1.pfm", "disp0y.pfm"))
        X.append(XX)
        dn, rows = clean(d0, mask(d0, d1, dy), len(X))
        (nnz_te if len(X) in te else nnz_tr).append(rows)
        dispnoc.append(dn)
        meta.append((views[0].shape[2], views[0].shape[3], ndisp))

    def pair(base, f0, f1, fd0, fd1, div, tsukuba=False, ndisp_rule="ceil"):
        x0, x1 = _view(os.path.join(base, f0), color, False), _view(os.path.join(base, f1), color, False)
        _, _, h, w = x0.shape
        d0 = imread_grey(os.path.join(base, fd0)).astype(F32) / div
        if tsukuba:
            m = imread_grey(os.path.join(base, "nonocc.png"))
            ndisp = -1
        else:
            d1 = imread_grey(os.path.join(base, fd1)).astype(F32) / div
            if ndisp_rule == "ceil":
                ndisp = int(np.ceil(d0.max()))
                d0[d0 == 0] = np.inf
                d1[d1 == 0] = np.inf
            else:
                ndisp = -1
            m = mask(d0, d1)
        return x0, x1, d0, m, ndisp, h, w

    for year in (2006, 2005):
        base1 = root(MB, "scenes%d" % year, "HalfSize")
        for d in sorted(os.listdir(base1)):
            base2 = os.path.join(base1, d)
            if not os.path.isfile(base2 + "/disp1.png"):
                continue
            XX = [None]
            for light in range(3):
                imgs = []
                for e in (0, 1, 2):
                    b3 = os.path.join(base2, "Illum%d/Exp%d" % (light + 1, e))
                    imgs += [_view(os.path.join(b3, "view1.png"), color, False), _view(os.path.join(b3, "view5.png"), color, False)]
                _, _, h, w = imgs[0].shape
                XX.append(np.concatenate(imgs).reshape(3, 2, C, h, w))
            d0 = imread_grey(base2 + "/disp1.png").astype(F32) / 2
            d1 = imread_grey(base2 + "/disp5.png").astype(F32) / 2
            ndisp = int(np.ceil(d0.max()))
            d0[d0 == 0] = np.inf
            d1[d1 == 0] = np.inf
            X.append(XX)
            dn, rows = clean(d0, mask(d0, d1), len(X))
            nnz_tr.append(rows)
            dispnoc.append(dn)
            meta.append((h, w, ndisp))

    for d in ("conesH", "teddyH"):
        base1 = root(MB, "scenes2003", d)
        x0, x1, d0, m, ndisp, h, w = pair(base1, "im2.ppm", "im6.ppm", "disp2.pgm", "disp6.pgm", 2)
        X.append([None, np.concatenate((x0, x1)).reshape(1, 2, C, h, w)])
        dn, rows = clean(d0, m, len(X))
        nnz_tr.append(rows)
        dispnoc.append(dn)
        meta.append((h, w, ndisp))

    base1 = root(MB, "scenes2001", "data")
    for d in sorted(os.listdir(base1)):
        if d == "tsukuba":
            f = ("scene1.row3.col3.ppm", "scene1.row3.col4.ppm", "truedisp.row3.col3.pgm", "", 16)
        elif d == "map":
            f = ("im0.pgm", "im1.pgm", "disp0.pgm", "disp1.pgm", 8)
        else:
            f = ("im2.ppm", "im6.ppm", "disp2.pgm", "disp6.pgm", 8)
        base2 = os.path.join(base1, d)
        if not os.path.isfile(os.path.join(base2, f[2])):
            continue
        x0, x1, d0, m, _, h, w = pair(base2, *f, tsukuba=d == "tsukuba", ndisp_rule="none")
        X.append([None, np.concatenate((x0, x1)).reshape(1, 2, C, h, w)])
        dn, rows = clean(d0, m, len(X))
        nnz_tr.append(rows)
        dispnoc.append(dn)
        meta.append((h, w, -1))

    fname_submit = []
    for d1 in ("trainingH", "testH"):
        base2 = root("data.mb/unzip/MiddEval3", d1)
        for d2 in sorted(os.listdir(base2)):
            base3 = os.path.join(base2, d2)
            ndisp = int(re.search("ndisp=(.*)", open(os.path.join(base3, "calib.txt")).read()).group(1))
            x0, x1 = _view(os.path.join(base3, "im0.png"), color, False), _view(os.path.join(base3, "im1.png"), color, False)
            X.append([np.concatenate((x0, x1)).astype(F32)])
            meta.append((x0.shape[2], x0.shape[3], ndisp))
            fname_submit.append(os.path.join(d1, d2))

    return dict(X=X, dispnoc=dispnoc, meta=np.array(meta, dtype=np.int32), nnz_tr=np.vstack(nnz_tr), nnz_te=np.vstack(nnz_te),
                te=te, fname_submit="\n".join(fname_submit))
