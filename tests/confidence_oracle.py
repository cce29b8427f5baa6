"""numpy restatement of the margin confidence, sparsify and the sparsification counts (mc-cnn_b200/confidence.py,
csrc/confidence.cu), for tests/test_confidence.py and tests/test_gpu_confidence.py.  Written from the definitions in DESIGN
§19, not from the kernels: whole-array scans in ascending d and a stable sort, no top-4 lists and no radix select."""
import numpy as np

POINTS = 20


def margin(vol):
    """(disp, conf) float32 of a (D, H, W) volume: d1 the first strict minimum in ascending d (NaN never taken, start +inf,
    0 when nothing is taken), c2 the same over |d - d1| >= 2, conf = c2 - c1 when both are below +inf, else 0"""
    vol = np.asarray(vol, np.float32)
    D = vol.shape[0]
    inf = np.float32(np.inf)
    c1 = np.full(vol.shape[1:], inf, np.float32)
    d1 = np.zeros(vol.shape[1:], np.int64)
    for d in range(D):
        take = vol[d] < c1
        c1 = np.where(take, vol[d], c1)
        d1 = np.where(take, d, d1)
    c2 = np.full(vol.shape[1:], inf, np.float32)
    for d in range(D):
        take = (np.abs(d - d1) >= 2) & (vol[d] < c2)
        c2 = np.where(take, vol[d], c2)
    ok = (c1 < inf) & (c2 < inf)
    with np.errstate(invalid="ignore", over="ignore"):
        conf = np.where(ok, c2 - c1, np.float32(0)).astype(np.float32)
    return d1.astype(np.float32), conf


def margin_at(curve):
    """margin of one pixel's cost curve by a direct reading of the definition (brute force for the tests)"""
    vals = [float(v) for v in np.asarray(curve, np.float32)]
    best, d1 = np.inf, 0
    for d, v in enumerate(vals):
        if v < best:
            best, d1 = v, d
    c2 = np.inf
    for d, v in enumerate(vals):
        if abs(d - d1) >= 2 and v < c2:
            c2 = v
    conf = np.float32(c2) - np.float32(best) if best < np.inf and c2 < np.inf else np.float32(0)
    return float(d1), np.float32(conf)


def order_key(conf):
    """conf's float32 bits mapped so that they order like the values (NaN above +inf), as uint64"""
    u = np.ascontiguousarray(conf, np.float32).view(np.uint32).astype(np.uint64)
    neg = (u >> np.uint64(31)) == 1
    return np.where(neg, u ^ np.uint64(0xFFFFFFFF), u ^ np.uint64(0x80000000))


def order(conf, pixels=None):
    """flat indices of `pixels` (default: all) by conf descending, then index ascending"""
    flat = np.ravel(conf)
    idx = np.arange(flat.size) if pixels is None else np.flatnonzero(np.ravel(pixels))
    key = order_key(flat[idx]).astype(np.int64)          # < 2^32: the negation is exact
    return idx[np.argsort(-key, kind="stable")]


def sparsify(disp, conf, n_keep, invalid):
    out = np.full(np.shape(disp), np.float32(invalid), np.float32).ravel()
    keep = order(conf)[:n_keep]
    out[keep] = np.ravel(disp)[keep]
    return out.reshape(np.shape(disp))


def counts(pred, conf, gt, err_at):
    """(M, B, [bad among the first ceil(k M / 20), k = 1..20])"""
    pred, gt = np.ravel(np.asarray(pred, np.float32)), np.ravel(np.asarray(gt, np.float32))
    mask = gt != 0
    bad = (np.abs(gt - pred) > np.float32(err_at)) & mask
    ordered = order(conf, mask)
    M, B = int(mask.sum()), int(bad.sum())
    cum = np.concatenate([[0], np.cumsum(bad[ordered])])
    ns = [-(-k * M // POINTS) for k in range(1, POINTS + 1)]
    return M, B, [int(cum[n]) for n in ns]


def curve(M, B, bad):
    """(e_1..e_20, AUC, AUC_opt) in double"""
    if M == 0:
        return [float("nan")] * POINTS, float("nan"), float("nan")
    ns = [-(-k * M // POINTS) for k in range(1, POINTS + 1)]
    e = [b / n for b, n in zip(bad, ns)]
    o = [max(0, n - (M - B)) / n for n in ns]
    area = lambda c: sum(0.05 * (c[k] + c[k + 1]) / 2 for k in range(POINTS - 1))
    return e, area(e), area(o)
