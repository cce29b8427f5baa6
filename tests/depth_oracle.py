"""numpy restatement of depth, the point cloud and the depth metrics (mc-cnn_b200/depth.py, csrc/depth.cu), for
tests/test_depth.py and tests/test_gpu_depth.py.  Written from the definitions in DESIGN §20, whole arrays at a time:
depth32 is the float32 rule the kernels must match bit for bit, depth64 the same quantities in float64, and metrics64 the
depth metrics with every sum, ratio and logarithm in float64 over depth32's depths."""
import math

import numpy as np

NAMES = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3", "n", "coverage")


def fB32(cal):
    return np.float32(float(cal.f) * float(cal.baseline))


def _valid32(d, doffs):
    d = np.asarray(d, np.float32)
    with np.errstate(invalid="ignore"):
        s = d + np.float32(doffs)
        return np.isfinite(d) & (s > 0), s


def depth32(disp, cal, max_depth=None):
    """(Z, X, Y) float32 (H, W) in the kernels' operation order, NaN where there is no depth"""
    d = np.asarray(disp, np.float32)
    ok, s = _valid32(d, cal.doffs)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        z = fB32(cal) / np.where(ok, s, np.float32(1))
    if max_depth is not None:
        ok &= z <= np.float32(max_depth)
    H, W = d.shape
    x = np.arange(W, dtype=np.float32)[None, :]
    y = np.arange(H, dtype=np.float32)[:, None]
    f, cx, cy = np.float32(cal.f), np.float32(cal.cx), np.float32(cal.cy)
    with np.errstate(invalid="ignore", over="ignore"):
        X = ((x - cx) * z) / f
        Y = ((y - cy) * z) / f
    nan = np.float32(np.nan)
    return (np.where(ok, z, nan).astype(np.float32), np.where(ok, X, nan).astype(np.float32),
            np.where(ok, Y, nan).astype(np.float32))


def depth64(disp, cal, max_depth=None):
    """Z float64 (H, W) = f baseline / (d + doffs), NaN where there is no depth (validity from the fp32 add)"""
    d = np.asarray(disp, np.float32)
    ok, _ = _valid32(d, cal.doffs)
    with np.errstate(divide="ignore", invalid="ignore"):
        z = float(cal.f) * float(cal.baseline) / (d.astype(np.float64) + float(cal.doffs))
    if max_depth is not None:
        ok &= z <= max_depth
    return np.where(ok, z, np.nan)


def cloud_records(disp, cal, rgb, max_depth=None):
    """the packed 15-byte PLY records of the valid pixels in row-major order (bytes)"""
    Z, X, Y = depth32(disp, cal, max_depth)
    ok = ~np.isnan(Z)
    rgb = np.asarray(rgb, np.uint8)
    if rgb.ndim == 2:
        rgb = np.repeat(rgb[:, :, None], 3, axis=2)
    rec = np.empty(int(ok.sum()), np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))
    rec["xyz"] = np.stack([X[ok], Y[ok], Z[ok]], axis=1)
    rec["rgb"] = rgb[ok]
    return rec.tobytes()


def metrics64(disp, gt, cal, min_depth=1e-3, max_depth=80.0):
    """{name: value}: S = valid gt depth in [min_depth, max_depth] (fp32 compares), predicted depth clamped in fp32, the
    rest in float64; NaN means when nothing is scored"""
    zg = depth32(gt, cal)[0]
    zp = depth32(disp, cal)[0]
    lo = np.float32(min_depth)
    hi = np.float32(np.inf if max_depth is None else max_depth)
    with np.errstate(invalid="ignore"):
        S = ~np.isnan(zg) & (zg >= lo) & (zg <= hi)
    m = S & ~np.isnan(zp)
    a = np.clip(zp[m], lo, hi).astype(np.float64)
    b = zg[m].astype(np.float64)
    n, nS = int(m.sum()), int(S.sum())
    nan = float("nan")
    if n == 0:
        return dict(abs_rel=nan, sq_rel=nan, rmse=nan, rmse_log=nan, a1=nan, a2=nan, a3=nan, n=0, coverage=nan if nS == 0 else 0.0)
    e = a - b
    r = np.maximum(a / b, b / a)
    return dict(abs_rel=float(np.sum(np.abs(e) / b)) / n, sq_rel=float(np.sum(e * e / b)) / n,
                rmse=math.sqrt(float(np.sum(e * e)) / n), rmse_log=math.sqrt(float(np.sum((np.log(a) - np.log(b)) ** 2)) / n),
                a1=int((r < 1.25).sum()) / n, a2=int((r < 1.25 ** 2).sum()) / n, a3=int((r < 1.25 ** 3).sum()) / n, n=n,
                coverage=n / nS)
