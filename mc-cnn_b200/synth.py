"""Seeded synthetic stereo pairs (numpy only): the tower output and the two images.

There is no network for KITTI/Middlebury or trained nets, so tests and bench.py
feed the hot path with data of the right shape and statistics:
unit-norm C-channel features where the left map is the right map shifted by a
piecewise-constant ground-truth disparity plus noise, so that argmin / LR check /
interpolation / sub-pixel all see realistic structure, and two standardised
grey images with the same shift (they drive cross() and the SGM penalties).
"""
import numpy as np


def _gauss_blur(a, sigma):
    """separable Gaussian blur (reflect padding), numpy only"""
    r = int(np.ceil(3 * sigma))
    k = np.exp(-0.5 * (np.arange(-r, r + 1) / sigma) ** 2)
    k = (k / k.sum()).astype(np.float32)
    for axis in (0, 1):
        pad = [(0, 0), (0, 0)]
        pad[axis] = (r, r)
        p = np.pad(a, pad, mode="reflect")
        a = np.apply_along_axis(lambda v: np.convolve(v, k, mode="valid"), axis, p).astype(np.float32)
    return a


def natural_image(rng, H, W):
    """Piecewise-smooth grey image whose gradient statistics match the KITTI sample pair of the
    reference (standardised samples/input/kittiL.png: median |dx| 0.026, 77% of |dx| below
    tau_so = 0.08, mean cross arm 4.1 of L1 = 5 at tau1 = 0.13, mean CBCA support ~52 taps; this
    generator gives ~0.028 / 90% / 4.1 / ~50).  The roughness of the image decides how much work
    cross-based aggregation does, so white noise would understate it five-fold."""
    base = _gauss_blur(rng.standard_normal((H, W), dtype=np.float32), 15.0)
    base /= base.std()
    by, bx = 16, 48
    blk = np.kron(rng.standard_normal(((H + by - 1) // by, (W + bx - 1) // bx)).astype(np.float32),
                  np.ones((by, bx), np.float32))[:H, :W]
    tex = _gauss_blur(rng.standard_normal((H, W), dtype=np.float32), 1.0)
    tex /= tex.std()
    mask = (_gauss_blur(rng.standard_normal((H, W), dtype=np.float32), 20.0) > 0.02).astype(np.float32)
    return base + 0.8 * blk + 0.3 * tex * mask + 0.008 * rng.standard_normal((H, W), dtype=np.float32)


def make_pair(H, W, C, D, seed=0, noise=0.1, block=(16, 48)):
    """Returns dict(featL, featR (C,H,W), imgL, imgR (H,W), gt (H,W)) as float32 arrays."""
    rng = np.random.default_rng(seed)
    dmax = max(1, min(D, max(2, W // 3)))
    by, bx = block
    gy, gx = (H + by - 1) // by, (W + bx - 1) // bx
    gt_blocks = rng.integers(0, dmax, size=(gy, gx))
    gt = np.kron(gt_blocks, np.ones((by, bx), dtype=np.int64))[:H, :W]

    ext = W + D
    scene = rng.standard_normal((C, H, ext), dtype=np.float32)
    cols = np.arange(W)[None, :] + D
    rows = np.arange(H)[:, None]
    featR = scene[:, :, D:D + W].copy()
    featL = scene[:, rows, cols - gt] + noise * rng.standard_normal((C, H, W), dtype=np.float32)

    def unit(f):  # Normalize2 (adcensus.cu:1284-1308)
        return (f / np.sqrt((f * f).sum(0, keepdims=True) + 1e-5)).astype(np.float32)

    img_scene = natural_image(rng, H, ext)
    imgR = img_scene[:, D:D + W].copy()
    imgL = img_scene[rows, cols - gt] + 0.004 * rng.standard_normal((H, W), dtype=np.float32)

    def standardise(x):  # main.lua:1095-1096 (unbiased std, as torch's :std())
        return ((x - x.mean()) / x.std(ddof=1)).astype(np.float32)

    return dict(featL=unit(featL), featR=unit(featR), imgL=standardise(imgL), imgR=standardise(imgR),
                gt=gt.astype(np.float32))


def _standardise(x):
    return ((x - x.mean()) / x.std(ddof=1)).astype(np.float32)


def _scene_views(rng, H, W, D, n_views=2):
    """(views (n_views, H, W), gt (H, W)): standardised grey views of one natural scene, view 0 the left image, every other
    view the right image (views 2, 3 ... with their own brightness and noise, like Middlebury's extra exposures / lights).
    Left pixel x matches right pixel x - gt; gt is piecewise constant in [1, D) and 0 (invalid) on about 10% of the pixels."""
    dmax = max(2, min(D, W // 3))
    gy, gx = (H + 15) // 16, (W + 47) // 48
    gt = np.kron(rng.integers(1, dmax, size=(gy, gx)), np.ones((16, 48), np.int64))[:H, :W]
    ext = W + D
    scene = natural_image(rng, H, ext)
    cols = np.arange(W)[None, :] + D
    rows = np.arange(H)[:, None]
    views = [_standardise(scene[rows, cols - gt] + 0.004 * rng.standard_normal((H, W), dtype=np.float32))]
    for k in range(1, n_views):
        gain = 1.0 if k == 1 else 0.7 + 0.2 * k
        views.append(_standardise(gain * scene[:, D:D + W] + 0.004 * k * rng.standard_normal((H, W), dtype=np.float32)))
    gt = gt.astype(np.float32)
    gt[rng.random((H, W)) < 0.1] = 0
    return np.stack(views), gt


def write_kitti_set(root, dataset="kitti", n_tr=4, n_te=2, H=48, width=130, widths=(130, 117), seed=0):
    """A small seeded KITTI set in preprocess_kitti.lua's layout under ``root/data.kitti`` (or ``data.kitti2015``):
    x0.bin, x1.bin (n, 1, H, width) with row i's first widths[i % len(widths)] columns filled, dispnoc.bin (n_tr, 1, H, width),
    metadata.bin (n, 3) int32 (img_height = H + 25, img_width, id), tr.bin / te.bin (1-based int64 split of the training
    rows, te first).  Returns the directory."""
    from . import dataio
    import os

    rng = np.random.default_rng(seed)
    d = os.path.join(root, "data.kitti" if dataset == "kitti" else "data.kitti2015")
    os.makedirs(d, exist_ok=True)
    n = n_tr + n_te
    x0 = np.zeros((n, 1, H, width), np.float32)
    x1 = np.zeros_like(x0)
    dispnoc = np.zeros((n_tr, 1, H, width), np.float32)
    meta = np.zeros((n, 3), np.int32)
    for i in range(n):
        w = int(widths[i % len(widths)])
        assert 1 <= w <= width
        views, gt = _scene_views(rng, H, w, 32)
        x0[i, 0, :, :w], x1[i, 0, :, :w] = views
        if i < n_tr:
            dispnoc[i, 0, :, :w] = gt
        meta[i] = (H + 25, w, i if i < n_tr else i - n_tr)
    perm = rng.permutation(n_tr) + 1
    n_val = max(1, n_tr // 3)
    for name, x in (("x0", x0), ("x1", x1), ("dispnoc", dispnoc), ("metadata", meta),
                    ("te", perm[:n_val].astype(np.int64)), ("tr", perm[n_val:].astype(np.int64))):
        dataio.tofile(os.path.join(d, name + ".bin"), x)
    return d


def write_kitti_raw(root, dataset="kitti", n_tr=41, n_te=2, H=375, widths=(1242, 1241, 1224), seed=0, D=64):
    """A seeded raw KITTI tree as the archives unpack, under ``root/data.kitti/unzip`` (or ``data.kitti2015``):
    ``{training,testing}/<left>|<right>/%06d_10.png`` (8-bit grey image_0 / image_1 for 'kitti', RGB image_2 / image_3 for
    'kitti2015') and ``training/<disp_noc>/%06d_10.png`` (disp_noc / disp_noc_0), 16-bit maps of disparity * 256.  Image k
    of a directory is H x widths[k % len(widths)].  The maps are _scene_views' ground truth (piecewise constant in [1, D),
    so there are real occlusions where a nearer block lies to the right, and entries d >= x at the left border) plus a
    per-block slant quantised to 1/256, with about 10% zero (invalid) pixels.  Returns the unzip directory."""
    import os

    from PIL import Image

    from . import dataio

    rgb = dataset == "kitti2015"
    names = ("image_2", "image_3", "disp_noc_0") if rgb else ("image_0", "image_1", "disp_noc")
    unzip = os.path.join(root, "data.kitti2015" if rgb else "data.kitti", "unzip")
    rng = np.random.default_rng(seed)
    for sub, n in (("training", n_tr), ("testing", n_te)):
        for name in names[:2] + ((names[2],) if sub == "training" else ()):
            os.makedirs(os.path.join(unzip, sub, name), exist_ok=True)
        for k in range(n):
            W = int(widths[k % len(widths)])
            views, gt = _scene_views(rng, H, W, D)
            fname = "%06d_10.png" % k
            for v, name in zip(views, names[:2]):
                byte = lambda a: np.clip(np.rint(128 + 40 * a), 0, 255).astype(np.uint8)
                if rgb:
                    tint = rng.uniform(0.8, 1.2, 3)
                    im = Image.fromarray(np.stack([byte(v * t) for t in tint], axis=2), "RGB")
                else:
                    im = Image.fromarray(byte(v), "L")
                im.save(os.path.join(unzip, sub, name, fname), format="PNG")
            if sub == "training":
                slant = np.kron(rng.integers(0, 256, size=((H + 15) // 16, (W + 47) // 48)), np.ones((16, 48), np.int64))
                frac = (slant[:H, :W] * (np.arange(W)[None, :] % 48) // 48) / np.float32(256)
                dataio.write_png16(np.where(gt > 0, gt + frac, 0).astype(np.float32), os.path.join(unzip, sub, names[2], fname))
    return unzip


def write_mb_set(root, n=6, shapes=((40, 96, 24), (48, 130, 32)), seed=0, rect="imperfect", color="gray"):
    """A small seeded Middlebury set in preprocess_mb.py's layout under ``root/data.mb.<rect>_<color>``: per image k = 1..n
    x_<k>_1.bin (views, 1, H, W) (4 views for image 5, else 2) and dispnoc<k>.bin (H, W), meta.bin (n, 3) int32 (H, W,
    ndisp) with (H, W, ndisp) = shapes[(k - 1) % len(shapes)], te.bin (1-based int64: images 1 .. n // 2) and
    fname_submit.txt naming the last min(n, 30) images.  Returns the directory."""
    from . import dataio
    import os

    assert n >= 5, "the test action reads views 3 and 4 of image 5"
    rng = np.random.default_rng(seed)
    d = os.path.join(root, "data.mb.%s_%s" % (rect, color))
    os.makedirs(d, exist_ok=True)
    meta = np.zeros((n, 3), np.int32)
    for k in range(1, n + 1):
        H, W, ndisp = shapes[(k - 1) % len(shapes)]
        views, gt = _scene_views(rng, H, W, ndisp, n_views=4 if k == 5 else 2)
        dataio.tofile(os.path.join(d, "x_%d_1.bin" % k), np.ascontiguousarray(views[:, None]))
        dataio.tofile(os.path.join(d, "dispnoc%d.bin" % k), gt)
        meta[k - 1] = (H, W, ndisp)
    dataio.tofile(os.path.join(d, "meta.bin"), meta)
    dataio.tofile(os.path.join(d, "te.bin"), np.arange(1, n // 2 + 1, dtype=np.int64))
    n_sub = min(n, 30)
    with open(os.path.join(d, "fname_submit.txt"), "w") as f:
        f.write("\n".join("%s/Synth%d" % ("trainingH" if j < n_sub // 2 else "testH", j) for j in range(n_sub)))
    return d
