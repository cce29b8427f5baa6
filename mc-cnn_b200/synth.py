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


def _scene_views(rng, H, W, D, n_views=2, levels=None):
    """(views (n_views, H, W), gt (H, W)): standardised grey views of one natural scene, view 0 the left image, every other
    view the right image (views 2, 3 ... with their own brightness and noise, like Middlebury's extra exposures / lights).
    Left pixel x matches right pixel x - gt; gt is piecewise constant in [1, D) (or drawn from the integers `levels`) and 0
    (invalid) on about 10% of the pixels."""
    dmax = max(2, min(D, W // 3))
    gy, gx = (H + 15) // 16, (W + 47) // 48
    blocks = rng.integers(1, dmax, size=(gy, gx)) if levels is None else np.asarray(levels)[rng.integers(0, len(levels), (gy, gx))]
    gt = np.kron(blocks, np.ones((16, 48), np.int64))[:H, :W]
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


# A raw drive's camera: f B = 384 exactly, and every disparity of RAW_LEVELS gives a depth 384 / d that is exact in fp32 and
# turns back into d exactly, so a scan sampled from the true depth scores 0 against the true disparity.
RAW_F, RAW_B = 768.0, 0.5
RAW_LEVELS = (6, 8, 12, 16, 24, 32, 48)
# velodyne (x forward, y left, z up) to camera 0 (x right, y down, z forward), no offset
RAW_VELO_R = (0.0, -1.0, 0.0, 0.0, 0.0, -1.0, 1.0, 0.0, 0.0)


def raw_calib_text(H, W, f=RAW_F, B=RAW_B, R_rect=(1, 0, 0, 0, 1, 0, 0, 0, 1), R=RAW_VELO_R, T=(0.0, 0.0, 0.0)):
    """(calib_cam_to_cam.txt, calib_velo_to_cam.txt) of a raw drive's date directory, in KITTI's key: value layout"""
    cx, cy = W / 2 - 0.25, H / 2 + 0.5
    num = lambda v: " ".join(repr(float(x)) for x in v)
    P0 = (f, 0, cx, 0, 0, f, cy, 0, 0, 0, 1, 0)
    P1 = (f, 0, cx, -f * B, 0, f, cy, 0, 0, 0, 1, 0)
    cam = ["calib_time: 09-Jan-2012 13:57:47", "corner_dist: 9.950000e-02"]
    for k in ("00", "01", "02", "03"):
        cam += ["S_%s: 1.392000e+03 5.120000e+02" % k, "K_%s: %s" % (k, num((f, 0, cx, 0, f, cy, 0, 0, 1))),
                "S_rect_%s: %d %d" % (k, W, H), "R_rect_%s: %s" % (k, num(R_rect)),
                "P_rect_%s: %s" % (k, num(P1 if k in ("01", "03") else P0))]
    velo = ["calib_time: 15-Mar-2012 11:37:16", "R: %s" % num(R), "T: %s" % num(T),
            "delta_f: 0.000000e+00 0.000000e+00", "delta_c: 0.000000e+00 0.000000e+00"]
    return "\n".join(cam) + "\n", "\n".join(velo) + "\n"


def write_kitti_drive(root, date="2011_09_26", drive=1, n=3, H=40, W=150, seed=0, D=64, levels=RAW_LEVELS, every=3):
    """A seeded KITTI raw drive under ``root/<date>/<date>_drive_<drive>_sync``: grey rectified pairs
    ``image_00/data/%010d.png`` / ``image_01/data/%010d.png`` whose left pixel x matches right pixel x - gt (gt piecewise
    constant over `levels`, 0 on about 10% of the pixels), the date directory's calibration (:func:`raw_calib_text`, written
    once per date) and per frame a velodyne scan ``velodyne_points/data/%010d.bin`` sampled from the same scene: a point at
    the true depth 384 / gt for one pixel in `every` where gt > 0, placed where the projection rule of DESIGN §21 maps it to
    that pixel, plus points hidden behind them on the same pixels, points behind the camera and points outside the image.
    Returns (drive directory, [gt (H, W) float32 per frame])."""
    import os

    from PIL import Image

    rng = np.random.default_rng(seed)
    date_dir = os.path.join(root, date)
    drive_dir = os.path.join(date_dir, "%s_drive_%04d_sync" % (date, drive))
    for sub in ("image_00", "image_01", "velodyne_points"):
        os.makedirs(os.path.join(drive_dir, sub, "data"), exist_ok=True)
    cam, velo = raw_calib_text(H, W)
    for name, text in (("calib_cam_to_cam.txt", cam), ("calib_velo_to_cam.txt", velo)):
        if not os.path.exists(os.path.join(date_dir, name)):
            with open(os.path.join(date_dir, name), "w") as f:
                f.write(text)
    cx, cy = W / 2 - 0.25, H / 2 + 0.5
    fB = np.float32(RAW_F * RAW_B)
    byte = lambda a: np.clip(np.rint(128 + 40 * a), 0, 255).astype(np.uint8)
    gts = []
    for k in range(n):
        views, gt = _scene_views(rng, H, W, D, levels=levels)
        for v, sub in zip(views, ("image_00", "image_01")):
            Image.fromarray(byte(v), "L").save(os.path.join(drive_dir, sub, "data", "%010d.png" % k), format="PNG")
        ys, xs = np.nonzero((gt > 0) & (rng.integers(0, every, gt.shape) == 0))
        z = (fB / gt[ys, xs].astype(np.float32)).astype(np.float32)
        X = (xs + 1 - cx) * z.astype(np.float64) / RAW_F            # the image coordinate u + 1 of pixel u (DESIGN §21)
        Y = (ys + 1 - cy) * z.astype(np.float64) / RAW_F
        pts = [np.stack([z, -X, -Y], 1)]
        m = rng.random(len(z)) < 0.2                                 # hidden: the same ray, further away
        pts.append(np.stack([z[m] * 1.5, -X[m] * 1.5, -Y[m] * 1.5], 1))
        pts.append(np.stack([-rng.uniform(1, 50, 50), rng.uniform(-20, 20, 50), rng.uniform(-2, 2, 50)], 1))
        pts.append(np.stack([rng.uniform(5, 50, 50), rng.uniform(200, 400, 50), rng.uniform(-2, 2, 50)], 1))
        xyz = np.concatenate(pts).astype(np.float32)
        scan = np.concatenate([xyz, rng.uniform(0, 1, (len(xyz), 1)).astype(np.float32)], 1)
        scan[rng.permutation(len(scan))].astype("<f4").tofile(os.path.join(drive_dir, "velodyne_points", "data", "%010d.bin" % k))
        gts.append(gt.astype(np.float32))
    return drive_dir, gts


# An unrectified drive's rigs (DESIGN §22): raw cameras with a moderate 5-coefficient distortion and a small rectifying
# rotation each.  'kitti': the rectified grid lies inside the larger raw image, as KITTI's S_rect_00 does; 'alpha1': P is
# zoomed out, like OpenCV's stereoRectify with alpha = 1, so the rectified grid (the raw size) reaches past the raw image.
# Focal lengths scale with the image: P's f = W 25/24 (200 at W = 192), K's fx, fy = Wraw 35/36, Wraw 26/27 (210, 208 at 216).
EXTRACT_B = 0.5
EXTRACT_D = ((-0.15, 0.04, 0.0006, -0.0004, 0.0), (-0.14, 0.035, -0.0005, 0.0003, 0.0))
EXTRACT_ROT = ((0.004, -0.006, 0.003), (0.002, -0.004, 0.001))
EXTRACT_RIGS = {"kitti": 1.0, "alpha1": 0.68}                   # P's focal length over W 25/24


def _rodrigues(r):
    r = np.asarray(r, np.float64)
    t = np.linalg.norm(r)
    k = r / t
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(t) * Kx + (1 - np.cos(t)) * Kx @ Kx


def extract_cameras(H, W, Hraw, Wraw, rig="kitti"):
    """[(K, D, R, P) float64 per grey camera 00, 01] of an unrectified drive whose rectified grid is H x W and raw images
    Hraw x Wraw; P_rect_01 = P_rect_00 with P[0,3] = -f EXTRACT_B"""
    f = W * 25 / 24 * EXTRACT_RIGS[rig]
    P0 = np.array([[f, 0, W / 2 - 0.25, 0], [0, f, H / 2 + 0.5, 0], [0, 0, 1, 0]])
    P1 = P0.copy()
    P1[0, 3] = -f * EXTRACT_B
    cams = []
    for k, P in enumerate((P0, P1)):
        K = np.array([[Wraw * 35 / 36, 0, Wraw / 2 - 0.5 + 0.3 * (1 - 2 * k)], [0, Wraw * 26 / 27, Hraw / 2 + 0.2], [0, 0, 1]])
        cams.append((K, np.array(EXTRACT_D[k]), _rodrigues(EXTRACT_ROT[k]), P))
    return cams


def extract_calib_text(H, W, Hraw, Wraw, rig="kitti"):
    """(calib_cam_to_cam.txt, calib_velo_to_cam.txt) of an unrectified drive's date directory: K_0i, D_0i, R_rect_0i,
    P_rect_0i, S_0i and S_rect_0i of the grey cameras (:func:`extract_cameras`), and raw_calib_text's velodyne file"""
    num = lambda v: " ".join("%.12e" % float(x) for x in np.asarray(v).reshape(-1))
    cam = ["calib_time: 09-Jan-2012 13:57:47", "corner_dist: 9.950000e-02"]
    for i, (K, D, R, P) in enumerate(extract_cameras(H, W, Hraw, Wraw, rig)):
        k = "0%d" % i
        cam += ["S_%s: %s" % (k, num((Wraw, Hraw))), "K_%s: %s" % (k, num(K)), "D_%s: %s" % (k, num(D)),
                "R_%s: %s" % (k, num(np.eye(3))), "T_%s: %s" % (k, num((-EXTRACT_B * i, 0, 0))),
                "S_rect_%s: %s" % (k, num((W, H))), "R_rect_%s: %s" % (k, num(R)), "P_rect_%s: %s" % (k, num(P))]
    return "\n".join(cam) + "\n", raw_calib_text(H, W)[1]


def unrectify(scene, K, D, R, P, Hraw, Wraw, iters=30):
    """The raw (Hraw, Wraw) float image of a rectified float `scene`: each raw pixel undistorted iteratively in float64,
    rotated by R, projected by P[:, :3] onto the rectified grid, and `scene` sampled there bilinearly (clamped edges)."""
    v, u = np.meshgrid(np.arange(Hraw, dtype=np.float64), np.arange(Wraw, dtype=np.float64), indexing="ij")
    k1, k2, p1, p2, k3 = D
    xd, yd = (u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1]
    x, y = xd.copy(), yd.copy()
    for _ in range(iters):
        r2 = x * x + y * y
        rad = 1 + r2 * (k1 + r2 * (k2 + r2 * k3))
        x = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) / rad
        y = (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) / rad
    q = np.einsum("ij,jhw->ihw", P[:, :3] @ R, np.stack([x, y, np.ones_like(x)]))
    sx, sy = q[0] / q[2], q[1] / q[2]
    H, W = scene.shape
    x0 = np.clip(np.floor(sx), 0, W - 1).astype(np.int64)
    y0 = np.clip(np.floor(sy), 0, H - 1).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    a, b = np.clip(sx - np.floor(sx), 0, 1), np.clip(sy - np.floor(sy), 0, 1)
    a = np.where((sx < 0) | (sx > W - 1), 0, a)
    b = np.where((sy < 0) | (sy > H - 1), 0, b)
    return (1 - b) * ((1 - a) * scene[y0, x0] + a * scene[y0, x1]) + b * ((1 - a) * scene[y1, x0] + a * scene[y1, x1])


def write_kitti_extract_drive(root, date="2011_09_26", drive=1, n=3, H=64, W=192, Hraw=80, Wraw=216, seed=0, D=64,
                              levels=RAW_LEVELS, rig="kitti", sync=False):
    """A seeded unrectified KITTI raw drive under ``root/<date>/<date>_drive_<drive>_extract``: per frame a rectified scene
    of _scene_views (H x W, left pixel x matching right pixel x - gt, gt piecewise constant over `levels`, 0 on about 10% of
    the pixels) made raw by :func:`unrectify` with the cameras of :func:`extract_cameras` (`rig` 'kitti' or 'alpha1') and
    written as grey bytes ``image_00/data/%010d.png`` / ``image_01/data/%010d.png`` (Hraw x Wraw), and the date directory's
    :func:`extract_calib_text` (written once per date).  With `sync`, also ``<date>_drive_<drive>_sync`` holding the same
    scenes' rectified bytes.  Returns (extract drive directory, [gt (H, W) float32 per frame], sync drive directory or
    None)."""
    import os

    from PIL import Image

    rng = np.random.default_rng(seed)
    date_dir = os.path.join(root, date)
    out = os.path.join(date_dir, "%s_drive_%04d_extract" % (date, drive))
    sync_dir = os.path.join(date_dir, "%s_drive_%04d_sync" % (date, drive)) if sync else None
    for d in (out, sync_dir):
        for sub in ("image_00", "image_01"):
            if d is not None:
                os.makedirs(os.path.join(d, sub, "data"), exist_ok=True)
    cam, velo = extract_calib_text(H, W, Hraw, Wraw, rig)
    for name, text in (("calib_cam_to_cam.txt", cam), ("calib_velo_to_cam.txt", velo)):
        if not os.path.exists(os.path.join(date_dir, name)):
            with open(os.path.join(date_dir, name), "w") as f:
                f.write(text)
    cams = extract_cameras(H, W, Hraw, Wraw, rig)
    byte = lambda a: np.clip(np.rint(a), 0, 255).astype(np.uint8)
    gts = []
    for k in range(n):
        views, gt = _scene_views(rng, H, W, D, levels=levels)
        for v, sub, (K, Dk, R, P) in zip(views, ("image_00", "image_01"), cams):
            scene = 128.0 + 40.0 * v.astype(np.float64)
            raw = unrectify(scene, K, Dk, R, P, Hraw, Wraw)
            Image.fromarray(byte(raw), "L").save(os.path.join(out, sub, "data", "%010d.png" % k), format="PNG")
            if sync_dir is not None:
                Image.fromarray(byte(scene), "L").save(os.path.join(sync_dir, sub, "data", "%010d.png" % k), format="PNG")
        gts.append(gt.astype(np.float32))
    return out, gts, sync_dir


def write_kitti_eval_maps(unzip, dataset="kitti", seed=0):
    """The ground truth the devkits' metrics read besides disp_noc, next to a write_kitti_raw tree (`unzip` is what it
    returned): ``training/disp_occ/`` (``disp_occ_0/`` for 'kitti2015') is disp_noc with its invalid pixels filled in
    vertical bands (every third band of 37 columns, with disparities in [1, 64) quantised to 1/256), and for 'kitti2015'
    ``training/obj_map/``, 8-bit, 0 (background) except a few random rectangles numbered 1, 2, ...  Returns the number of
    pairs written."""
    import os

    from PIL import Image

    from . import dataio

    rgb = dataset == "kitti2015"
    sub = os.path.join(unzip, "training")
    noc_dir = os.path.join(sub, "disp_noc_0" if rgb else "disp_noc")
    occ_dir = os.path.join(sub, "disp_occ_0" if rgb else "disp_occ")
    os.makedirs(occ_dir, exist_ok=True)
    if rgb:
        os.makedirs(os.path.join(sub, "obj_map"), exist_ok=True)
    rng = np.random.default_rng(seed)
    names = sorted(os.listdir(noc_dir))
    for name in names:
        noc = dataio.read_png16_raw(os.path.join(noc_dir, name))
        H, W = noc.shape
        band = ((np.arange(W) // 37) % 3 == 0)[None, :] & (noc == 0)
        occ = np.where(band, rng.integers(256, 64 * 256, (H, W)), noc).astype(np.uint16)
        Image.fromarray(occ).save(os.path.join(occ_dir, name), format="PNG")
        if rgb:
            obj = np.zeros((H, W), np.uint8)
            for k in range(1, 5):
                y, x = int(rng.integers(0, H)), int(rng.integers(0, W))
                obj[y:y + int(rng.integers(10, 120)), x:x + int(rng.integers(20, 300))] = k
            Image.fromarray(obj, "L").save(os.path.join(sub, "obj_map", name), format="PNG")
    return len(names)


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


MB_SUBMIT_NAMES = ("Adirondack", "ArtL", "Jadeplant", "Motorcycle", "MotorcycleE", "Piano", "PianoL", "Pipes", "Playroom",
                   "Playtable", "PlaytableP", "Recycle", "Shelves", "Teddy", "Vintage")


def _mb_right_map(rng, d0, p_bad=0.05):
    """a right-view map consistent with d0 where it is finite (d1[y, round(x - d0)] = d0 + small noise), a few entries off
    by more than a pixel, inf elsewhere"""
    H, W = d0.shape
    d1 = np.full((H, W), np.inf, np.float32)
    ys, xs = np.nonzero(np.isfinite(d0))
    x1 = np.floor(xs - d0[ys, xs] + 0.5).astype(np.int64)
    ok = (x1 >= 0) & (x1 < W)
    noise = rng.uniform(-0.4, 0.4, ok.sum()).astype(np.float32)
    noise[rng.random(ok.sum()) < p_bad] += np.float32(3)
    d1[ys[ok], x1[ok]] = d0[ys[ok], xs[ok]] + noise
    return d1


def write_mb_raw(root, n2014=11, full=(80, 192), half_size=(40, 96), D=48, seed=0):
    """A seeded raw Middlebury tree as preprocess_mb.py expects it under ``root/data.mb/unzip``:

    * n2014 2014 scenes ``scenes2014/datasets/Scene<k>-{perfect,imperfect}`` of full x full RGB PNG views (im0, im1, im1E,
      im1L; ``ambient/L<l>/im<c>e<e>.png`` with 1-3 lights and exposure counts cycling through 2, 3, 5, 6, 7, 8, the two
      cameras of some scenes differing), calib.txt (ndisp = D), float PFMs disp0 / disp1 / disp0y (inf holes, a NaN, a
      vertical offset of up to 0.7 px).  Scene 2 carries ``.H.png`` caches for all its views and a ``disp1.pfm.H.pfm``;
      scene 5 caches im0 and im1 only.  Caches are decimated (every other pixel), so they differ from a real halving;
    * 2006 Aloe and Baby1, 2005 Art (and Books, which has no disp1.png and is skipped), ``HalfSize/<s>/Illum<l>/Exp<e>/
      view{1,5}.png`` and 8-bit disp1 / disp5 (value 2 d, 0 invalid);
    * 2003 conesH and teddyH (PPM views, PGM maps of 2 d);
    * 2001 tsukuba (PPM views, truedisp of 16 d, nonocc.png), map (PGM views, maps of 8 d with real 0 disparities) and
      sawtooth (PPM, maps of 8 d);
    * MiddEval3 ``trainingH`` and ``testH``, 15 pairs each.
    Smaller scenes are half_size.  Returns the unzip directory."""
    import os

    from PIL import Image

    from . import dataio

    rng = np.random.default_rng(seed)
    unzip = os.path.join(root, "data.mb", "unzip")
    data = os.path.join(unzip, "vision.middlebury.edu", "stereo", "data")

    def byte(v):
        return np.clip(np.rint(128 + 40 * v), 0, 255).astype(np.uint8)

    def rgb(v):
        return np.stack([byte(v * t) for t in rng.uniform(0.8, 1.2, 3)], axis=2)

    def save(a, *p):
        path = os.path.join(*p)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        Image.fromarray(a).save(path)
        return path

    def pfm(m, *p):
        path = os.path.join(*p)
        dataio.write_pfm(np.flipud(np.asarray(m, np.float32)), path)
        return path

    def calib(ndisp, *p):
        os.makedirs(os.path.join(*p), exist_ok=True)
        with open(os.path.join(*p, "calib.txt"), "w") as f:
            f.write("cam0=[1 0 0; 0 1 0; 0 0 1]\ndoffs=0\nbaseline=100\nwidth=1\nheight=1\nndisp=%d\nisint=0\n" % ndisp)

    exps = (2, 3, 5, 6, 7, 8)
    H, W = full
    for k in range(n2014):
        name = "Scene%02d" % k
        views, gt = _scene_views(rng, H, W, D, n_views=4)
        for kind in ("imperfect", "perfect"):
            base = os.path.join(data, "scenes2014", "datasets", "%s-%s" % (name, kind))
            calib(D, base)
            for v, f in zip(views, ("im0.png", "im1.png", "im1E.png", "im1L.png")):
                p = save(rgb(v), base, f)
                if kind == "imperfect" and (k == 2 or (k == 5 and f in ("im0.png", "im1.png"))):
                    save(np.asarray(Image.open(p))[::2, ::2].copy(), p + ".H.png")
            n_exp = exps[k % len(exps)]
            n_exp_other = n_exp + (1 if k % 3 == 0 else 0)            # the other camera has one more: min(max) wins
            for light in range(1 + k % 3):
                for cam, ne in ((0, n_exp), (1, n_exp_other)):
                    for e in range(ne):
                        v = views[cam] * (0.6 + 0.1 * e) + 0.05 * light
                        p = save(rgb(v), base, "ambient", "L%d" % (light + 1), "im%de%d.png" % (cam, e))
                        if kind == "imperfect" and k == 2:
                            save(np.asarray(Image.open(p))[::2, ::2].copy(), p + ".H.png")
            d0 = np.where(gt > 0, gt + rng.uniform(0, 1, gt.shape), np.inf).astype(np.float32)
            d0[3, 5] = np.nan
            d1 = _mb_right_map(rng, d0)
            dy = rng.uniform(-0.7, 0.7, gt.shape).astype(np.float32)
            pfm(d0, base, "disp0.pfm")
            p1 = pfm(d1, base, "disp1.pfm")
            pfm(dy, base, "disp0y.pfm")
            if kind == "imperfect" and k == 2:
                pfm(np.where(np.isfinite(d1[::2, ::2]), d1[::2, ::2] / 2, np.inf), p1 + ".H.pfm")

    h, w = half_size

    def grey_map(gt, scale, zero_invalid=True):
        return np.clip(np.where(gt > 0, gt * scale, 0) if zero_invalid else gt * scale, 0, 255).astype(np.uint8)

    for year, scenes in ((2006, ("Aloe", "Baby1")), (2005, ("Art", "Books"))):
        for s in scenes:
            base = os.path.join(data, "scenes%d" % year, "HalfSize", s)
            views, gt = _scene_views(rng, h, w, D // 2)
            for light in range(3):
                for e in range(3):
                    for v, f in zip(views, ("view1.png", "view5.png")):
                        save(rgb(v * (0.7 + 0.15 * e) + 0.1 * light), base, "Illum%d" % (light + 1), "Exp%d" % e, f)
            if s != "Books":
                save(grey_map(gt, 2), base, "disp1.png")
            d1 = _mb_right_map(rng, np.where(gt > 0, gt, np.inf).astype(np.float32))
            save(grey_map(np.where(np.isfinite(d1), np.rint(d1 * 2) / 2, 0), 2), base, "disp5.png")

    for s in ("conesH", "teddyH"):
        base = os.path.join(data, "scenes2003", s)
        views, gt = _scene_views(rng, h, w, D // 2)
        save(rgb(views[0]), base, "im2.ppm")
        save(rgb(views[1]), base, "im6.ppm")
        save(grey_map(gt, 2), base, "disp2.pgm")
        d1 = _mb_right_map(rng, np.where(gt > 0, gt, np.inf).astype(np.float32))
        save(grey_map(np.where(np.isfinite(d1), np.rint(d1 * 2) / 2, 0), 2), base, "disp6.pgm")

    base1 = os.path.join(data, "scenes2001", "data")
    views, gt = _scene_views(rng, h, w, 15)
    base = os.path.join(base1, "tsukuba")
    save(rgb(views[0]), base, "scene1.row3.col3.ppm")
    save(rgb(views[1]), base, "scene1.row3.col4.ppm")
    save(grey_map(gt, 16), base, "truedisp.row3.col3.pgm")
    save(np.where(rng.random(gt.shape) < 0.8, 255, 0).astype(np.uint8), base, "nonocc.png")
    for s, names in (("map", ("im0.pgm", "im1.pgm", "disp0.pgm", "disp1.pgm")),
                     ("sawtooth", ("im2.ppm", "im6.ppm", "disp2.pgm", "disp6.pgm"))):
        base = os.path.join(base1, s)
        views, gt = _scene_views(rng, h, w, 24)
        gt[:, : w // 4] = 0                                           # 0 is a real disparity in 2001 maps
        for v, f in zip(views, names[:2]):
            save(byte(v) if s == "map" else rgb(v), base, f)
        save(grey_map(gt, 8, zero_invalid=False), base, names[2])
        d1 = _mb_right_map(rng, gt.astype(np.float32), p_bad=0.1)
        save(grey_map(np.where(np.isfinite(d1), np.rint(d1 * 8) / 8, 0), 8, zero_invalid=False), base, names[3])

    for sub, suffix in (("trainingH", "H"), ("testH", "T")):
        for s in MB_SUBMIT_NAMES:
            base = os.path.join(unzip, "MiddEval3", sub, s + (suffix if sub == "testH" else ""))
            views, _ = _scene_views(rng, h, w, D // 2)
            calib(D // 2, base)
            save(rgb(views[0]), base, "im0.png")
            save(rgb(views[1]), base, "im1.png")
    return unzip


def write_mb_eval_gt(unzip, seed=0):
    """The MiddEval3 training ground truth as the SDK's MiddEval3-GT0-H.zip / -GT0-F.zip unpack it, next to a write_mb_raw
    tree (`unzip` is what it returned): per ``MiddEval3/trainingH/<scene>`` of h x w views, ``disp0GT.pfm`` (rows
    bottom-up; disparities in [0, ndisp) with inf holes) and ``mask0nocc.png`` (8-bit 0 where unknown, else 255 or, on
    about a fifth of the pixels, 128), and the same at exactly 2h x 2w under ``MiddEval3/trainingF/<scene>`` (twice the
    disparities of each half-size pixel's block, jittered by less than a pixel, with holes and masks of their own).
    Returns the number of scenes written."""
    import os
    import re

    from PIL import Image

    from . import dataio

    rng = np.random.default_rng(seed)
    eval3 = os.path.join(unzip, "MiddEval3")
    scenes = sorted(os.listdir(os.path.join(eval3, "trainingH")))

    def write(sub, s, gt, mask):
        base = os.path.join(eval3, sub, s)
        os.makedirs(base, exist_ok=True)
        dataio.write_pfm(np.flipud(gt.astype(np.float32)), os.path.join(base, "disp0GT.pfm"))
        Image.fromarray(mask, "L").save(os.path.join(base, "mask0nocc.png"))

    def holes_and_mask(gt, p_hole):
        gt = np.where(rng.random(gt.shape) < p_hole, np.inf, gt).astype(np.float32)
        mask = np.where(rng.random(gt.shape) < 0.2, 128, 255).astype(np.uint8)
        return gt, np.where(np.isinf(gt), 0, mask).astype(np.uint8)

    for s in scenes:
        base = os.path.join(eval3, "trainingH", s)
        with Image.open(os.path.join(base, "im0.png")) as im:
            w, h = im.size
        with open(os.path.join(base, "calib.txt")) as f:
            ndisp = int(re.search("ndisp=(.*)", f.read()).group(1))
        gt = rng.uniform(0, ndisp, (h, w)).astype(np.float32)
        write("trainingH", s, *holes_and_mask(gt, 0.05))
        full = np.kron(gt, np.ones((2, 2), np.float32)) * 2 + rng.uniform(-0.9, 0.9, (2 * h, 2 * w)).astype(np.float32)
        write("trainingF", s, *holes_and_mask(np.maximum(full, 0), 0.08))
    return len(scenes)


# A posed drive (DESIGN §23): textured planes of one static world, seen from a camera moving forward while it yaws.  The
# world frame is the first frame's rectified left camera (x right, y down, z forward); each plane is (normal, offset):
# n . x = offset.  Ground, a wall ahead and two side walls.
POSED_PLANES = (((0.0, 1.0, 0.0), 1.65), ((0.0, 0.0, 1.0), 14.0), ((1.0, 0.0, 0.0), 3.5), ((1.0, 0.0, 0.0), -4.0))
# A street (DESIGN §26): the ground and the two side walls, no wall ahead.  Every normal lies across the street, so the
# geometry alone cannot fix motion along it.
STREET_PLANES = (POSED_PLANES[0], POSED_PLANES[2], POSED_PLANES[3])
# a plane's in-plane texture axes (indices of x, y, z) by the axis of its normal
_POSED_AXES = {1: (0, 2), 2: (0, 1), 0: (2, 1)}
POSED_B = 0.5
POSED_LATLON = (49.011212804408, 8.4228850417969, 112.83)         # the first frame's GPS position (Karlsruhe)
POSED_RPY = (0.021, -0.013, 0.61)                                 # its roll, pitch, yaw
POSED_IMU_ROT, POSED_IMU_T = (0.012, -0.021, 0.017), (-0.8086759, 0.3195559, -0.7997231)
POSED_R_RECT_ROT = (0.003, -0.002, 0.001)


def _hash01(i, j, k):
    """a value in [0, 1) per integer lattice point (i, j) of texture k"""
    m = np.uint64(0xFFFFFFFF)
    h = (i.astype(np.uint64) * np.uint64(73856093)) ^ (j.astype(np.uint64) * np.uint64(19349663)) ^ np.uint64(k * 83492791 + 1)
    h &= m
    h = ((h ^ (h >> np.uint64(13))) * np.uint64(1274126177)) & m
    h ^= h >> np.uint64(16)
    return h.astype(np.float64) / 4294967296.0


def _value_noise(a, b, cell, k):
    ga, gb = a / cell, b / cell
    i, j = np.floor(ga), np.floor(gb)
    fa, fb = ga - i, gb - j
    i, j = i.astype(np.int64), j.astype(np.int64)
    v = lambda di, dj: _hash01(i + di, j + dj, k)
    return (1 - fb) * ((1 - fa) * v(0, 0) + fa * v(1, 0)) + fb * ((1 - fa) * v(0, 1) + fa * v(1, 1))


def posed_texture(p, plane, planes=POSED_PLANES):
    """the grey level in [0, 255] of world points p (..., 3) on plane number `plane` of `planes`: a function of world
    position only"""
    axes = _POSED_AXES[int(np.argmax(np.abs(planes[plane][0])))]
    a, b = p[..., axes[0]], p[..., axes[1]]
    return 30.0 + 195.0 * (0.6 * _value_noise(a, b, 0.04, 2 * plane) + 0.4 * _value_noise(a, b, 0.15, 2 * plane + 1))


def posed_camera_poses(n, step=0.4, yaw=np.radians(1.5)):
    """[4x4 camera-to-world float64] of n frames: the first is I, each next one `step` metres ahead along its heading and
    turned by `yaw` about the camera's vertical (y) axis; `step` may be a sequence of at least n - 1 steps, step k leading
    from frame k to frame k + 1"""
    steps = [float(step)] * n if np.ndim(step) == 0 else [float(v) for v in step]
    if len(steps) < n - 1:
        raise ValueError("%d frames need at least %d steps, got %d" % (n, n - 1, len(steps)))
    out, R, t = [], np.eye(3), np.zeros(3)
    Ry = np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
    for k in range(n):
        M = np.eye(4)
        M[:3, :3], M[:3, 3] = R, t
        out.append(M)
        if k + 1 == n:
            break
        t = t + R @ np.array([0.0, 0.0, steps[k]])
        R = R @ Ry.T
    return out


def posed_render(pose, H, W, f, cx, cy, shift=0.0, planes=POSED_PLANES):
    """(Z (H, W) camera depth of the nearest plane hit, plane id (H, W) int8, grey float) of the camera at `pose` moved by
    `shift` metres along its own x axis (the right camera: the baseline), in the world of `planes`"""
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    dc = np.stack([(u - cx) / f, (v - cy) / f, np.ones_like(u)], -1)
    R, t = pose[:3, :3], pose[:3, 3] + pose[:3, :3] @ np.array([shift, 0.0, 0.0])
    dw = dc @ R.T
    Z = np.full((H, W), np.inf)
    pid = np.full((H, W), -1, np.int8)
    for k, (nrm, off) in enumerate(planes):
        nrm = np.asarray(nrm)
        den = dw @ nrm
        with np.errstate(divide="ignore", invalid="ignore"):
            s = (off - nrm @ t) / den
        hit = (s > 0) & (s < Z)
        Z = np.where(hit, s, Z)
        pid = np.where(hit, k, pid).astype(np.int8)
    grey = np.zeros((H, W))
    for k in range(len(planes)):
        m = pid == k
        grey[m] = posed_texture(t + dw[m] * Z[m][:, None], k, planes)
    return Z, pid, grey


def _rpy(R):
    """(roll, pitch, yaw) with R = Rz(yaw) Ry(pitch) Rx(roll)"""
    return np.arctan2(R[2, 1], R[2, 2]), np.arctan2(-R[2, 0], np.hypot(R[0, 0], R[1, 0])), np.arctan2(R[1, 0], R[0, 0])


def posed_oxts(imu_poses, lat0):
    """[30 numbers per frame] of IMU poses (4x4, Mercator translation at the scale of latitude lat0): lat, lon, alt, roll,
    pitch, yaw by the inverse Mercator projection, the rest velocities, accelerations and status fields"""
    from . import dataio

    s = np.cos(lat0 * np.pi / 180)
    out = []
    for T in imu_poses:
        mx, my, alt = T[:3, 3]
        lon = mx * 180 / (np.pi * s * dataio.EARTH_RADIUS)
        lat = 360 / np.pi * np.arctan(np.exp(my / (s * dataio.EARTH_RADIUS))) - 90
        out.append([lat, lon, alt, *_rpy(T[:3, :3])] + [0.0] * 17 + [0.05, 0.02, 4, 10, 4, 4, 0])
    return out


def posed_scan(pose, H, W, cal, every=2, planes=POSED_PLANES):
    """(N, 4) float32 velodyne scan of the planes seen from the camera at `pose`: one point per `every`-th pixel in each
    direction, on the plane hit along the ray of image coordinate u + 1 (DESIGN §21's projection puts it on pixel u), taken
    through R_rect_00 and RAW_VELO_R into the velodyne frame; reflectance 0.5"""
    cx, cy = cal.cx - 1.0, cal.cy - 1.0
    Z = posed_render(pose, H, W, cal.f, cx, cy, planes=planes)[0][::every, ::every]
    v, u = np.meshgrid(np.arange(0, H, every, dtype=np.float64), np.arange(0, W, every, dtype=np.float64), indexing="ij")
    ok = np.isfinite(Z)
    z = Z[ok]
    p_rect = np.stack([(u[ok] - cx) * z / cal.f, (v[ok] - cy) * z / cal.f, z], 1)
    p_velo = p_rect @ _rodrigues(POSED_R_RECT_ROT) @ np.asarray(RAW_VELO_R).reshape(3, 3)
    return np.concatenate([p_velo, np.full((len(z), 1), 0.5)], 1).astype(np.float32)


def write_kitti_posed_drive(root, date="2011_09_26", drive=1, n=4, H=48, W=160, step=0.4, yaw=np.radians(1.5), velodyne=False,
                            no_oxts=False, planes=POSED_PLANES):
    """A KITTI raw ``_sync`` drive whose frames view the static world of `planes` (POSED_PLANES; STREET_PLANES is a street
    with no wall ahead) from known poses (:func:`posed_camera_poses`, `step` one length or one per frame): grey pairs ``image_00`` / ``image_01`` rendered by ray casting (nearest plane hit, the
    grey level a function of the world position, so the two views agree), the date directory's calibration (f = W,
    baseline POSED_B, a small R_rect_00, velo-to-cam RAW_VELO_R, and calib_imu_to_velo.txt with a rotation and
    translation), and ``oxts/data/%010d.txt`` records whose poses, through dataio.raw_poses, are the camera poses.  With
    `velodyne`, also ``velodyne_points/data/%010d.bin`` per frame (:func:`posed_scan`).  With `no_oxts`, no ``oxts/``
    directory (a drive only tracking can pose).  Returns (drive directory, [exact disparity fB / Z (H, W) float32], [plane id (H, W) int8], [camera pose 4x4])."""
    import os

    from PIL import Image

    from . import dataio

    date_dir = os.path.join(root, date)
    drive_dir = os.path.join(date_dir, "%s_drive_%04d_sync" % (date, drive))
    for sub in ("image_00", "image_01") + (() if no_oxts else ("oxts",)):
        os.makedirs(os.path.join(drive_dir, sub, "data"), exist_ok=True)
    f = float(W)
    cam, velo = raw_calib_text(H, W, f=f, B=POSED_B, R_rect=_rodrigues(POSED_R_RECT_ROT).ravel())
    num = lambda v: " ".join(repr(float(x)) for x in np.asarray(v).reshape(-1))
    imu = "calib_time: 25-May-2012 16:47:16\nR: %s\nT: %s\n" % (num(_rodrigues(POSED_IMU_ROT)), num(POSED_IMU_T))
    for name, text in ((dataio.RAW_CAM, cam), (dataio.RAW_VELO, velo), (dataio.RAW_IMU, imu)):
        if not os.path.exists(os.path.join(date_dir, name)):
            with open(os.path.join(date_dir, name), "w") as fh:
                fh.write(text)
    cal = dataio.read_calib(date_dir, "kitti_raw")
    c2i = dataio.camera_to_imu(date_dir)
    lat0 = POSED_LATLON[0]
    T0 = dataio.oxts_pose(np.array(POSED_LATLON + POSED_RPY), np.cos(lat0 * np.pi / 180))
    C0 = T0 @ c2i
    poses = posed_camera_poses(n, step, yaw)
    fB = cal.f * cal.baseline
    disps, pids = [], []
    byte = lambda a: np.clip(np.rint(a), 0, 255).astype(np.uint8)
    for k, P in enumerate(poses):
        Z, pid, grey = posed_render(P, H, W, cal.f, cal.cx, cal.cy, planes=planes)
        _, _, grey_r = posed_render(P, H, W, cal.f, cal.cx, cal.cy, shift=cal.baseline, planes=planes)
        Image.fromarray(byte(grey), "L").save(os.path.join(drive_dir, "image_00", "data", "%010d.png" % k), format="PNG")
        Image.fromarray(byte(grey_r), "L").save(os.path.join(drive_dir, "image_01", "data", "%010d.png" % k), format="PNG")
        disps.append((fB / Z).astype(np.float32))
        pids.append(pid)
    for k, rec in enumerate([] if no_oxts else posed_oxts([C0 @ P @ np.linalg.inv(c2i) for P in poses], lat0)):
        with open(os.path.join(drive_dir, "oxts", "data", "%010d.txt" % k), "w") as fh:
            fh.write(" ".join(repr(float(x)) if isinstance(x, float) else str(x) for x in rec) + "\n")
    if velodyne:
        os.makedirs(os.path.join(drive_dir, "velodyne_points", "data"), exist_ok=True)
        for k, P in enumerate(poses):
            posed_scan(P, H, W, cal, planes=planes).astype("<f4").tofile(os.path.join(drive_dir, "velodyne_points", "data", "%010d.bin" % k))
    return drive_dir, disps, pids, poses
