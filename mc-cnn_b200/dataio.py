"""Data formats on either side of the hot path: what `preprocess_*.py/.lua`
write and `main.lua` reads back, the error metric of `-a test_te`, and the submission writers.

* ``fromfile`` / ``tofile``: the ``<name>`` + ``<name>.dim`` + ``<name>.type`` triple
  (main.lua:353-380, preprocess_mb.py:99-106);
* ``read_png16`` / ``write_png16``: KITTI disparity maps, uint16 = disparity * 256, 0 = invalid
  (adcensus.cu:1670-1706);
* ``write_pfm`` / ``read_pfm``: Middlebury disparity maps (adcensus.cu:1708-1722; the reader is
  preprocess_mb.py:13-57 without the down-sampling);
* ``bad_pixel_rate``: share of ground-truth pixels whose error exceeds ``err_at`` (3 px KITTI,
  1 px Middlebury; main.lua:400, 453, 1228-1236);
* ``kitti_submission_image``: the prediction pasted into the bottom rows of the full-size frame
  (main.lua:1203-1205);
* ``read_calib`` / ``write_depth_png16``: the KITTI 2012, KITTI 2015 and MiddEval3 calibration files, and KITTI's depth
  map format (DESIGN §20, an addition beyond the reference);
* ``read_calib(date, 'kitti_raw')`` / ``read_velodyne`` / ``raw_frames``: a KITTI raw drive's calibration, Velodyne scans
  and frame list (DESIGN §21, an addition beyond the reference);
* ``read_rectification``: a raw stereo pair's intrinsics, distortion and rectification, from a KITTI raw date directory or
  OpenCV FileStorage YAML files (DESIGN §22, an addition beyond the reference).

Plain numpy / PIL host code: nothing here touches the GPU.
"""
import os
import re
from collections import namedtuple

import numpy as np

_TYPES = {"float32": np.float32, "int32": np.int32, "int64": np.int64}
ERR_AT = {"kitti": 3.0, "kitti2015": 3.0, "mb": 1.0}


def fromfile(fname):
    """main.lua:353-380: dims from ``fname.dim`` (one per line), dtype from ``fname.type``, raw
    little-endian data from ``fname``.  A ``.dim`` holding the single line ``0`` is an empty tensor."""
    with open(fname + ".dim") as f:
        dim = [int(float(line)) for line in f.read().split()]
    if len(dim) == 1 and dim[0] == 0:
        return np.empty((0,), np.float64)                       # torch.Tensor()
    with open(fname + ".type") as f:
        t = f.read().strip()
    if t not in _TYPES:
        raise ValueError("%s: unsupported type %r (float32, int32, int64)" % (fname, t))
    x = np.fromfile(fname, dtype=np.dtype(_TYPES[t]).newbyteorder("<"))
    n = int(np.prod(dim))
    if x.size != n:
        raise ValueError("%s: %d elements on disk, .dim says %s" % (fname, x.size, dim))
    return x.reshape(dim).astype(_TYPES[t], copy=False)


def tofile(fname, x):
    """preprocess_mb.py:99-106 / preprocess_kitti.lua:118-144: the inverse of :func:`fromfile`"""
    if x is None:
        open(fname + ".dim", "w").write("0\n")
        return
    x = np.ascontiguousarray(x)
    if str(x.dtype) not in _TYPES:
        raise ValueError("unsupported dtype %s" % x.dtype)
    x.astype(x.dtype.newbyteorder("<"), copy=False).tofile(fname)
    open(fname + ".type", "w").write(str(x.dtype))
    open(fname + ".dim", "w").write("\n".join(map(str, x.shape)))


def read_png16_raw(fname):
    """the stored uint16 (H,W) values of a 16-bit grey PNG (disparity * 256, 0 = invalid)"""
    from PIL import Image

    with Image.open(fname) as im:
        if im.mode not in ("I;16", "I;16B", "I"):
            raise ValueError("%s: 16-bit grey PNG expected, got mode %s" % (fname, im.mode))
        return np.asarray(im).astype(np.uint16)


def read_png16(fname):
    """adcensus.cu:1670-1686: 16-bit grey PNG -> float32 (H,W), 0 stays 0 (invalid), else value / 256"""
    v = read_png16_raw(fname)
    return np.where(v == 0, np.float32(0.0), v.astype(np.float32) / np.float32(256.0)).astype(np.float32)


def write_png16(img, fname):
    """adcensus.cu:1688-1706: pixel = (uint16)(val < 1e-5 ? 0 : val * 256), the product in fp32,
    truncated towards zero (values past the uint16 range are clamped instead of wrapping)"""
    from PIL import Image

    img = np.asarray(img, dtype=np.float32)
    assert img.ndim == 2
    v = np.where(img < np.float32(1e-5), np.float32(0.0), img * np.float32(256.0))
    v = np.clip(np.trunc(v), 0, 65535).astype(np.uint16)
    Image.fromarray(v).save(fname, format="PNG")  # uint16 -> mode I;16


def write_pfm(img, fname):
    """adcensus.cu:1708-1722: ``Pf``, width height, scale -0.003922 (little endian), then the rows
    exactly as given (main.lua:1215 passes the vertically flipped map, PFM rows run bottom-up)"""
    img = np.ascontiguousarray(img, dtype="<f4")
    assert img.ndim == 2
    with open(fname, "wb") as f:
        f.write(("Pf\n%d %d\n-0.003922\n" % (img.shape[1], img.shape[0])).encode("ascii"))
        img.tofile(f)


def read_pfm(fname):
    """single-channel PFM -> float32 (H,W) in FILE row order (flip it to get top-down rows)"""
    with open(fname, "rb") as f:
        if f.readline().strip() != b"Pf":
            raise ValueError("%s: not a single-channel PFM" % fname)
        w, h = (int(t) for t in f.readline().split())
        scale = float(f.readline().strip())
        data = np.fromfile(f, dtype="<f4" if scale < 0 else ">f4", count=w * h)
    if data.size != w * h:
        raise ValueError("%s: truncated" % fname)
    return data.reshape(h, w).astype(np.float32)


def bad_pixel_rate(pred, actual, err_at):
    """main.lua:1228-1236: mask = actual != 0; err = #(|actual - pred| > err_at and mask) / #mask"""
    pred = np.asarray(pred, dtype=np.float32)
    actual = np.asarray(actual, dtype=np.float32)
    assert pred.shape == actual.shape
    mask = actual != 0
    n = int(mask.sum())
    if n == 0:
        return float("nan")                                      # 0 / 0 in the reference as well
    bad = (np.abs(actual - pred) > np.float32(err_at)) & mask
    return float(bad.sum()) / n


def kitti_submission_image(pred, img_height, img_width):
    """main.lua:1203-1205: a zero (img_height, img_width) frame whose LAST pred.shape[0] rows are the
    prediction (the networks see the bottom `height` rows of a KITTI frame)"""
    pred = np.asarray(pred, dtype=np.float32)
    h, w = pred.shape
    assert h <= img_height and w == img_width
    out = np.zeros((img_height, img_width), np.float32)
    out[img_height - h:] = pred
    return out


def write_kitti_submission(pred, img_height, img_width, out_dir, idx, dataset="kitti"):
    """main.lua:1203-1212: ``out/%06d_10.png`` (kitti) or ``out/disp_0/%06d_10.png`` (kitti2015)"""
    path = out_dir if dataset == "kitti" else os.path.join(out_dir, "disp_0")
    os.makedirs(path, exist_ok=True)
    fname = os.path.join(path, "%06d_10.png" % idx)
    write_png16(kitti_submission_image(pred, img_height, img_width), fname)
    return fname


# ---- calibration and depth maps (DESIGN §20) ------------------------------------------------------------------------------

Calib = namedtuple("Calib", "f cx cy baseline doffs width height")
Calib.__doc__ = """A rectified stereo pair's camera: focal length f and principal point (cx, cy) in pixels, baseline in metres,
doffs (the x-difference of the two principal points) in pixels, and the image size the file states (None when it states
none)."""

RawCalib = namedtuple("RawCalib", Calib._fields + ("velo",))
RawCalib.__doc__ = """A KITTI raw drive's grey pair (the :data:`Calib` fields) and velo, the 3x4 velodyne-to-image matrix
P_rect_00 R_rect_00 [R|T]_velo_to_cam as a tuple of 12 float64, row-major (DESIGN §21)."""

CALIB_KINDS = ("kitti", "kitti2015", "mb", "kitti_raw")
# the two projection matrices of each KITTI calibration file: the grey pair (2012 and raw drives), the colour pair (2015)
_KITTI_P = {"kitti": ("P0", "P1"), "kitti2015": ("P_rect_02", "P_rect_03"), "kitti_raw": ("P_rect_00", "P_rect_01")}
RAW_CAM, RAW_VELO = "calib_cam_to_cam.txt", "calib_velo_to_cam.txt"


def _calib_entries(path):
    """{key: value text} of a calibration file's ``key: value`` (KITTI) or ``key=value`` (Middlebury) lines"""
    out = {}
    with open(path) as f:
        for line in f:
            m = re.match(r"\s*([A-Za-z_][A-Za-z0-9_]*)\s*[:=]\s*(.*?)\s*$", line)
            if m:
                out[m.group(1)] = m.group(2)
    return out


def _numbers(path, entries, key, n):
    """the n numbers of `key`, refused when the key is missing or does not hold exactly n numbers"""
    if key not in entries:
        raise ValueError("%s: missing key %s" % (path, key))
    try:
        v = [float(t) for t in entries[key].replace("[", " ").replace("]", " ").replace(";", " ").split()]
    except ValueError:
        v = []
    if len(v) != n or not all(np.isfinite(v)):
        raise ValueError("%s: %s must hold %d finite numbers, got %r" % (path, key, n, entries[key]))
    return v


def velo_to_image(P, R_rect, R, T):
    """P (12) . R_rect (9, padded to 4x4) . [R (9) | T (3)] (padded to 4x4), the top 3x4 of the product as 12 float64,
    row-major, in this operation order (DESIGN §21): B[i][j] = (R_rect[i][0] A[0][j] + R_rect[i][1] A[1][j]) +
    R_rect[i][2] A[2][j] with A = [R|T]; M[i][j] = (P[i][0] B[0][j] + P[i][1] B[1][j]) + P[i][2] B[2][j], plus P[i][3]
    when j = 3."""
    A = [[R[3 * i + j] for j in range(3)] + [T[i]] for i in range(3)]
    B = [[(R_rect[3 * i] * A[0][j] + R_rect[3 * i + 1] * A[1][j]) + R_rect[3 * i + 2] * A[2][j] for j in range(4)]
         for i in range(3)]
    M = []
    for i in range(3):
        for j in range(4):
            m = (P[4 * i] * B[0][j] + P[4 * i + 1] * B[1][j]) + P[4 * i + 2] * B[2][j]
            M.append(m + P[4 * i + 3] if j == 3 else m)
    return tuple(M)


def read_calib(path, kind):
    """The :data:`Calib` of a calibration file (DESIGN §20).  kind 'kitti': KITTI 2012's ``calib/%06d.txt``, the grey
    pair P0 / P1; 'kitti2015': ``calib_cam_to_cam/%06d.txt``, the colour pair P_rect_02 / P_rect_03 and the size S_rect_02
    when present; 'mb': a MiddEval3 scene's ``calib.txt`` (cam0, doffs, baseline in millimetres, width, height).  KITTI:
    f = P[0,0], cx = P[0,2], cy = P[1,2] of the left matrix, baseline = (P_left[0,3] - P_right[0,3]) / f, doffs = 0.
    'kitti_raw' (DESIGN §21): `path` is a raw drive's date directory; its ``calib_cam_to_cam.txt`` gives the grey pair
    P_rect_00 / P_rect_01, the size S_rect_00 and R_rect_00, its ``calib_velo_to_cam.txt`` R and T, and the result is a
    :data:`RawCalib` whose velo is :func:`velo_to_image`.
    Refuses a missing key, a malformed matrix, f <= 0 and baseline <= 0, naming the file and the key."""
    if kind not in CALIB_KINDS:
        raise ValueError("calibration kind must be one of %s, got %r" % (", ".join(CALIB_KINDS), kind))
    if kind == "kitti_raw":
        return _read_raw_calib(path)
    e = _calib_entries(path)
    width = height = None
    if kind == "mb":
        cam0 = _numbers(path, e, "cam0", 9)
        f, cx, cy = cam0[0], cam0[2], cam0[5]
        baseline = _numbers(path, e, "baseline", 1)[0] / 1000.0
        doffs = _numbers(path, e, "doffs", 1)[0]
        width, height = (int(_numbers(path, e, k, 1)[0]) for k in ("width", "height"))
        fkey, bkey = "cam0", "baseline"
    else:
        kl, kr = _KITTI_P[kind]
        pl, pr = _numbers(path, e, kl, 12), _numbers(path, e, kr, 12)
        f, cx, cy = pl[0], pl[2], pl[6]
        baseline = (pl[3] - pr[3]) / f if f > 0 else 0.0
        doffs = 0.0
        if kind == "kitti2015" and "S_rect_02" in e:
            width, height = (int(v) for v in _numbers(path, e, "S_rect_02", 2))
        fkey, bkey = kl, "%s / %s" % (kl, kr)
    if not f > 0:
        raise ValueError("%s: %s gives f = %g, must be > 0" % (path, fkey, f))
    if not baseline > 0:
        raise ValueError("%s: %s gives baseline = %g m, must be > 0" % (path, bkey, baseline))
    return Calib(f, cx, cy, baseline, doffs, width, height)


def _read_raw_calib(date_dir):
    cam, velo = os.path.join(date_dir, RAW_CAM), os.path.join(date_dir, RAW_VELO)
    for p in (cam, velo):
        if not os.path.isfile(p):
            raise FileNotFoundError("missing calibration file %s" % p)
    e, ev = _calib_entries(cam), _calib_entries(velo)
    pl, pr = _numbers(cam, e, "P_rect_00", 12), _numbers(cam, e, "P_rect_01", 12)
    width, height = (int(v) for v in _numbers(cam, e, "S_rect_00", 2))
    R_rect = _numbers(cam, e, "R_rect_00", 9)
    R, T = _numbers(velo, ev, "R", 9), _numbers(velo, ev, "T", 3)
    f, cx, cy = pl[0], pl[2], pl[6]
    if not f > 0:
        raise ValueError("%s: P_rect_00 gives f = %g, must be > 0" % (cam, f))
    baseline = (pl[3] - pr[3]) / f
    if not baseline > 0:
        raise ValueError("%s: P_rect_00 / P_rect_01 gives baseline = %g m, must be > 0" % (cam, baseline))
    if not (width > 0 and height > 0):
        raise ValueError("%s: S_rect_00 gives a %dx%d image" % (cam, width, height))
    return RawCalib(f, cx, cy, baseline, 0.0, width, height, velo_to_image(pl, R_rect, R, T))


def read_velodyne(path):
    """a KITTI raw scan ``velodyne_points/data/%010d.bin``: (N, 4) float32 x, y, z, reflectance (little-endian); a file whose
    size is not a multiple of 16 bytes is refused"""
    size = os.path.getsize(path)
    if size % 16:
        raise ValueError("%s: %d bytes, not a whole number of 16-byte points" % (path, size))
    return np.fromfile(path, dtype="<f4").reshape(-1, 4).astype(np.float32, copy=False)


RAW_LEFT, RAW_RIGHT, RAW_SCAN = ("image_00", "data", "%010d.png"), ("image_01", "data", "%010d.png"), \
    ("velodyne_points", "data", "%010d.bin")


def raw_file(drive_dir, what, i):
    """the file of frame i of a raw drive: what is RAW_LEFT, RAW_RIGHT or RAW_SCAN"""
    return os.path.join(drive_dir, what[0], what[1], what[2] % i)


def _raw_indices(drive_dir, what):
    d = os.path.join(drive_dir, what[0], what[1])
    ext = what[2][-4:]
    if not os.path.isdir(d):
        return set()
    return {int(f[:-4]) for f in os.listdir(d) if f.endswith(ext) and len(f) == 14 and f[:10].isdigit()}


def raw_frames(drive_dir, velodyne=False):
    """The ascending frame indices of a KITTI raw drive (``<date>/<date>_drive_<nnnn>_sync``) that have both grey images
    (``image_00/data/%010d.png``, ``image_01/data/%010d.png``) and, with `velodyne`, the scan.  Refuses a drive with no
    frame, or one where some frames lack one of these files, naming the frames."""
    sets = [_raw_indices(drive_dir, RAW_LEFT), _raw_indices(drive_dir, RAW_RIGHT)]
    names = ["image_00", "image_01"]
    if velodyne:
        sets.append(_raw_indices(drive_dir, RAW_SCAN))
        names.append("velodyne_points")
    every = set.union(*sets)
    both = set.intersection(*sets)
    if every != both:
        miss = ["%s lacks %s" % (n, ", ".join("%010d" % i for i in sorted(every - s)[:5]) + (" ..." if len(every - s) > 5 else ""))
                for n, s in zip(names, sets) if every - s]
        raise ValueError("%s: frames missing on one side: %s" % (drive_dir, "; ".join(miss)))
    if not both:
        raise ValueError("%s: no frames (image_00/data/%%010d.png and image_01/data/%%010d.png)" % drive_dir)
    return sorted(both)


# ---- poses of a raw drive (DESIGN §23) ------------------------------------------------------------------------------------

RAW_OXTS = ("oxts", "data", "%010d.txt")
RAW_IMU = "calib_imu_to_velo.txt"
OXTS_FIELDS = 30
EARTH_RADIUS = 6378137.0                 # the KITTI raw devkit's er


def read_oxts(path):
    """One OXTS record ``oxts/data/%010d.txt``: its 30 numbers as float64 (lat, lon, alt, roll, pitch, yaw, ...).  Refuses,
    naming the file, a record that does not hold exactly 30 finite numbers and a latitude with |lat| >= 90."""
    with open(path) as f:
        text = f.read()
    try:
        v = [float(t) for t in text.split()]
    except ValueError:
        raise ValueError("%s: an OXTS record holds %d numbers, got %r" % (path, OXTS_FIELDS, text[:80])) from None
    if len(v) != OXTS_FIELDS or not all(np.isfinite(v)):
        raise ValueError("%s: an OXTS record holds %d finite numbers, got %d" % (path, OXTS_FIELDS, len(v)))
    if not abs(v[0]) < 90:
        raise ValueError("%s: latitude %r is not in (-90, 90)" % (path, v[0]))
    return np.asarray(v, np.float64)


def _rigid(R, T):
    M = np.eye(4)
    M[:3, :3] = np.asarray(R, np.float64).reshape(3, 3)
    M[:3, 3] = T
    return M


def oxts_pose(rec, scale):
    """the 4x4 IMU pose of one OXTS record (the devkit's convertOxtsToPose): Mercator t = (s er lon pi/180,
    s er ln(tan((90 + lat) pi/360)), alt) and R = Rz(yaw) Ry(pitch) Rx(roll), s = `scale`"""
    lat, lon, alt, rx, ry, rz = (float(x) for x in rec[:6])
    t = (scale * EARTH_RADIUS * lon * np.pi / 180, scale * EARTH_RADIUS * np.log(np.tan((90 + lat) * np.pi / 360)), alt)
    c, s = np.cos, np.sin
    Rx = np.array([[1, 0, 0], [0, c(rx), -s(rx)], [0, s(rx), c(rx)]])
    Ry = np.array([[c(ry), 0, s(ry)], [0, 1, 0], [-s(ry), 0, c(ry)]])
    Rz = np.array([[c(rz), -s(rz), 0], [s(rz), c(rz), 0], [0, 0, 1]])
    return _rigid(Rz @ Ry @ Rx, t)


def camera_to_imu(date_dir):
    """inv(T_imu->velo) inv(T_velo->cam) inv(R_rect_00), 4x4 float64: a point of the rectified left camera in the IMU frame.
    Reads R_rect_00 (calib_cam_to_cam.txt), R and T of calib_velo_to_cam.txt and of calib_imu_to_velo.txt; refuses a
    missing file or key, naming it."""
    cam, velo, imu = (os.path.join(date_dir, n) for n in (RAW_CAM, RAW_VELO, RAW_IMU))
    for p in (cam, velo, imu):
        if not os.path.isfile(p):
            raise FileNotFoundError("missing calibration file %s" % p)
    e, ev, ei = _calib_entries(cam), _calib_entries(velo), _calib_entries(imu)
    R_rect = _rigid(_numbers(cam, e, "R_rect_00", 9), (0, 0, 0))
    velo_cam = _rigid(_numbers(velo, ev, "R", 9), _numbers(velo, ev, "T", 3))
    imu_velo = _rigid(_numbers(imu, ei, "R", 9), _numbers(imu, ei, "T", 3))
    return np.linalg.inv(imu_velo) @ np.linalg.inv(velo_cam) @ np.linalg.inv(R_rect)


def raw_poses(drive_dir, frames):
    """[4x4 float64 per frame of `frames`]: each takes a point of that frame's rectified left camera (DESIGN §20's X, Y, Z)
    into the drive's world frame, the rectified left camera of frames[0] (so its pose is I).  C_i = T_i camera_to_imu, T_i
    the frame's :func:`oxts_pose` with the Mercator scale cos(lat0 pi/180) of frames[0]'s latitude; W_i = inv(C_0) C_i
    (DESIGN §23).  Refuses a missing calibration file or key and a frame without its OXTS record, naming them, before
    reading any image."""
    frames = list(frames)
    if not frames:
        raise ValueError("%s: no frames to pose" % drive_dir)
    c2i = camera_to_imu(os.path.dirname(os.path.normpath(drive_dir)))
    recs = []
    for i in frames:
        p = raw_file(drive_dir, RAW_OXTS, i)
        if not os.path.isfile(p):
            raise FileNotFoundError("%s: frame %010d has no OXTS record %s" % (drive_dir, i, p))
        recs.append(read_oxts(p))
    scale = np.cos(recs[0][0] * np.pi / 180)
    T = [oxts_pose(r, scale) for r in recs]
    # inv(C_0) C_i = inv(c2i) (inv(T_0) T_i) c2i, with inv(T_0) T_i = [R_0' R_i | R_0' (t_i - t_0)]: the Mercator
    # translations (~1e6 m) are subtracted before anything else touches them
    R0, t0 = T[0][:3, :3], T[0][:3, 3]
    i2c = np.linalg.inv(c2i)
    out = [np.eye(4)]
    for t in T[1:]:
        rel = _rigid((R0.T @ t[:3, :3]).ravel(), R0.T @ (t[:3, 3] - t0))
        out.append(i2c @ rel @ c2i)
    return out


def check_calib_size(cal, H, W, path):
    """refuses a calibration whose stated image size is not (H, W): nothing is rescaled"""
    if cal.width is not None and (cal.width, cal.height) != (W, H):
        raise ValueError("%s: calibration for %dx%d images, the image is %dx%d" % (path, cal.width, cal.height, W, H))


# ---- rectification of calibrated raw cameras (DESIGN §22) ----------------------------------------------------------------

CameraRect = namedtuple("CameraRect", "K D R P size rect_size")
CameraRect.__doc__ = """One raw camera and its rectification, float64: K the 3x3 intrinsics (9 numbers, row-major), D its 0, 4, 5 or 8
distortion coefficients in OpenCV's order k1 k2 p1 p2 [k3 [k4 k5 k6]], R the 3x3 rectifying rotation (9), P the 3x4
rectified projection (12), size the raw image size (W, H) and rect_size the rectified one (W', H')."""

RECT_KINDS = ("kitti_raw", "opencv")
RAW_EXTRACT = "_extract"                 # a KITTI raw drive of unrectified images: <date>/<date>_drive_<nnnn>_extract


class StereoRect(namedtuple("StereoRect", "left right")):
    """A raw stereo pair's two :data:`CameraRect`; :attr:`calib` is the :data:`Calib` of the rectified pair."""

    __slots__ = ()

    @property
    def calib(self):
        """f = P1[0,0], cx = P1[0,2], cy = P1[1,2], baseline = (P1[0,3] - P2[0,3]) / f, doffs = P2[0,2] - P1[0,2], the size
        rect_size"""
        p1, p2 = self.left.P, self.right.P
        return Calib(p1[0], p1[2], p1[6], (p1[3] - p2[3]) / p1[0], p2[2] - p1[2], *self.left.rect_size)

    def check_size(self, H, W, path):
        """refuses raw images that are not (H, W) = the cameras' size"""
        for side, cam in (("left", self.left), ("right", self.right)):
            if tuple(cam.size) != (W, H):
                raise ValueError("%s: %s camera calibrated for %dx%d images, the image is %dx%d"
                                 % (path, side, cam.size[0], cam.size[1], W, H))


def _all_numbers(path, text, key):
    try:
        v = [float(t) for t in text.replace("[", " ").replace("]", " ").replace(";", " ").replace(",", " ").split()]
    except ValueError:
        raise ValueError("%s: %s must hold numbers, got %r" % (path, key, text)) from None
    if not all(np.isfinite(v)):
        raise ValueError("%s: %s must hold finite numbers, got %r" % (path, key, text))
    return v


def _opencv_entries(paths):
    """{key: (numbers, file)} of the !!opencv-matrix entries (and scalar numbers) of OpenCV FileStorage YAML files, later
    files overriding earlier ones.  A matrix whose data does not hold rows * cols numbers is refused."""
    out = {}
    for path in paths:
        with open(path) as f:
            text = f.read()
        if not text.startswith("%YAML"):
            raise ValueError("%s: not an OpenCV FileStorage YAML file (no %%YAML header)" % path)
        blocks, key = {}, None
        for line in text.splitlines()[1:]:
            m = re.match(r"([A-Za-z_][A-Za-z0-9_]*)\s*:(.*)$", line)
            if m:
                key = m.group(1)
                blocks[key] = [m.group(2)]
            elif key is not None and line[:1].isspace():
                blocks[key].append(line)
            else:
                key = None                       # '---' and anything else at the top level ends an entry
        for key, lines in blocks.items():
            body = "\n".join(lines)
            if "!!opencv-matrix" in body:
                fields = dict(re.findall(r"^\s*(rows|cols|dt)\s*:\s*(\S+)", body, re.M))
                data = re.search(r"data\s*:\s*\[(.*?)\]", body, re.S)
                if "rows" not in fields or "cols" not in fields or data is None:
                    raise ValueError("%s: %s is not an opencv-matrix with rows, cols and data" % (path, key))
                v = _all_numbers(path, data.group(1), key)
                rows, cols = int(fields["rows"]), int(fields["cols"])
                if len(v) != rows * cols:
                    raise ValueError("%s: %s is %dx%d but holds %d numbers" % (path, key, rows, cols, len(v)))
                out[key] = (v, path)
            else:
                try:
                    out[key] = ([float(body.strip())], path)
                except ValueError:
                    pass                         # strings and nested maps are not calibration numbers
    return out


def _camera(src, keys, n_expected, size, rect_size):
    """the :data:`CameraRect` of `keys` (K, D, R, P names) in `src` {key: (numbers, file)}; checks the counts and K"""
    vals = []
    for k, n in zip(keys, n_expected):
        names = k if isinstance(k, tuple) else (k,)
        hit = next((nm for nm in names if nm in src), None)
        if hit is None:
            raise ValueError("%s: missing key %s" % (src["__file__"], " or ".join(names)))
        v, path = src[hit]
        if n is None:
            if len(v) not in (0, 4, 5, 8):
                raise ValueError("%s: %s holds %d distortion coefficients; 0, 4, 5 or 8 are supported" % (path, hit, len(v)))
        elif len(v) != n:
            raise ValueError("%s: %s must hold %d numbers, got %d" % (path, hit, n, len(v)))
        vals.append((tuple(float(x) for x in v), hit, path))
    (K, kname, kpath), (D, _, _), (R, rname, _), (P, pname, ppath) = vals
    if K[1] != 0 or K[3] != 0:
        raise ValueError("%s: %s has skew; a zero-skew camera matrix is expected" % (kpath, kname))
    if K[6:] != (0.0, 0.0, 1.0):
        raise ValueError("%s: %s's last row is %s, not (0, 0, 1)" % (kpath, kname, K[6:]))
    M = np.asarray(P, np.float64).reshape(3, 4)[:, :3] @ np.asarray(R, np.float64).reshape(3, 3)
    if not np.linalg.cond(M) < 1e12:
        raise ValueError("%s: %s[:, :3] . %s is singular" % (ppath, pname, rname))
    return CameraRect(K, D, R, P, tuple(size), tuple(rect_size))


def _check_pair(rect, path, p1name, p2name):
    """the refusals of a rectified pair: f <= 0, baseline <= 0, a vertical rig, rectified sizes that differ"""
    p1, p2 = rect.left.P, rect.right.P
    if not p1[0] > 0:
        raise ValueError("%s: %s gives f = %g, must be > 0" % (path, p1name, p1[0]))
    if p1[4:] != p2[4:] or p2[7] != 0:
        raise ValueError("%s: %s and %s differ in rows 1 and 2 or %s[1,3] != 0: a vertical rig, which is not supported"
                         % (path, p1name, p2name, p2name))
    if not rect.calib.baseline > 0:
        raise ValueError("%s: %s / %s gives baseline = %g, must be > 0" % (path, p1name, p2name, rect.calib.baseline))
    if rect.left.rect_size != rect.right.rect_size:
        raise ValueError("%s: the rectified sizes differ, %s and %s" % (path, rect.left.rect_size, rect.right.rect_size))
    return rect


def _size(path, e, key):
    v = _numbers(path, e, key, 2)
    if not all(x == int(x) and x >= 1 for x in v):
        raise ValueError("%s: %s must hold two positive whole numbers, got %r" % (path, key, e[key]))
    return int(v[0]), int(v[1])


def read_rectification(path, kind, size=None):
    """The :class:`StereoRect` of a raw stereo pair (DESIGN §22).  kind 'kitti_raw': `path` is a KITTI raw date directory;
    its ``calib_cam_to_cam.txt`` gives K_0i, D_0i, R_rect_0i, P_rect_0i, S_0i and S_rect_0i of the grey cameras 00 and 01.
    kind 'opencv': `path` is an OpenCV FileStorage YAML file or a list of them, merged (e.g. stereo_calib's intrinsics.yml
    and extrinsics.yml), holding M1 or K1, D1, M2 or K2, D2, R1, R2, P1, P2; `size` (W, H) is the images' size, and the
    rectified size equals it.  Refuses, naming the file and the key: a missing key or a wrong count of numbers, a distortion
    count other than 0, 4, 5 or 8, a K with skew or whose last row is not (0, 0, 1), a singular P[:, :3] R, f <= 0,
    baseline <= 0, a vertical rig (the two P's rows 1 and 2 differ, or P2[1,3] != 0) and rectified sizes that differ."""
    if kind not in RECT_KINDS:
        raise ValueError("rectification kind must be one of %s, got %r" % (", ".join(RECT_KINDS), kind))
    if kind == "kitti_raw":
        if size is not None:
            raise ValueError("kitti_raw: the raw size comes from S_00 / S_01, not from `size`")
        cam = os.path.join(path, RAW_CAM)
        if not os.path.isfile(cam):
            raise FileNotFoundError("missing calibration file %s" % cam)
        e = _calib_entries(cam)
        src = {k: (_all_numbers(cam, v, k), cam) for k, v in e.items() if k[:2] in ("K_", "D_", "R_", "P_", "S_")}
        src["__file__"] = cam
        cams = []
        for i in ("00", "01"):
            cams.append(_camera(src, ("K_" + i, "D_" + i, "R_rect_" + i, "P_rect_" + i), (9, None, 9, 12),
                                _size(cam, e, "S_" + i), _size(cam, e, "S_rect_" + i)))
        return _check_pair(StereoRect(*cams), cam, "P_rect_00", "P_rect_01")
    paths = [path] if isinstance(path, (str, os.PathLike)) else list(path)
    if not paths:
        raise ValueError("opencv: no calibration file given")
    if size is None or len(size) != 2 or not all(int(s) == s and s >= 1 for s in size):
        raise ValueError("opencv: the images' size (W, H) is needed, got %r" % (size,))
    size = (int(size[0]), int(size[1]))
    src = _opencv_entries(paths)
    src["__file__"] = " + ".join(str(p) for p in paths)
    cams = [_camera(src, (("M%d" % i, "K%d" % i), "D%d" % i, "R%d" % i, "P%d" % i), (9, None, 9, 12), size, size)
            for i in (1, 2)]
    where = src["P1"][1] if src["P1"][1] == src["P2"][1] else src["__file__"]
    return _check_pair(StereoRect(*cams), where, "P1", "P2")


def write_depth_png16(Z, fname):
    """KITTI's depth map format: uint16 = round(Z * 256) (Z in metres, float64 product), 0 where Z has no depth (NaN) or
    rounds to 0; values past the uint16 range are clamped"""
    from PIL import Image

    Z = np.asarray(Z, dtype=np.float32)
    assert Z.ndim == 2
    v = np.rint(np.nan_to_num(Z.astype(np.float64) * 256.0, nan=0.0, posinf=65535.0, neginf=0.0))
    Image.fromarray(np.clip(v, 0, 65535).astype(np.uint16)).save(fname, format="PNG")


def read_depth_png16(fname):
    """:func:`write_depth_png16`'s inverse: float32 (H, W) metres, NaN where the file holds 0"""
    v = read_png16_raw(fname)
    return np.where(v == 0, np.float32(np.nan), v.astype(np.float32) / np.float32(256.0)).astype(np.float32)
