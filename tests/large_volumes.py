"""Sampled references for cost volumes past 2^31 elements (tests/test_gpu_large_volumes.py).

A 2000 x 3002 x 400 volume is 9.6 GB: the kernels run on the whole of it on the device, and the checks compare what they
wrote at chosen places with the CPU oracle run on the few rows or columns that place depends on.  Three index widths can
go wrong in a kernel that addresses such a volume: element indices past 2^31, byte offsets past 2^31 (2^29 floats) and
byte offsets past 2^32 (2^30 floats).  The samples therefore hold, for every layout a kernel reads or writes, the
elements just before and at each of those three flat indices and the last element, plus a few seeded random ones.

Everything here is numpy on host arrays, and `shift` scales the thresholds down (2^29 >> shift, ...), so that
tests/test_large_volume_refs.py proves each helper against the whole-volume oracle at a small shape.
"""
import numpy as np

THRESHOLDS = (1 << 29, 1 << 30, 1 << 31)    # floats: 2^31 bytes, 2^32 bytes, 2^31 elements


def threshold_flats(shape, shift=0):
    """flat indices of `shape` just before and at each threshold (2^k >> shift), and the last element"""
    n = int(np.prod(shape))
    flats = []
    for t in THRESHOLDS:
        t >>= shift
        if t >= n:
            raise ValueError("threshold %d is past the %d elements of %s" % (t, n, shape))
        flats += [t - 1, t]
    return flats + [n - 1]


def positions(shape, shift=0):
    """np.unravel_index of threshold_flats: one index tuple per flat index"""
    return [tuple(int(i) for i in np.unravel_index(f, shape)) for f in threshold_flats(shape, shift)]


def sample_rows(shapes, axis, extent, rng, nrand=2):
    """sorted rows (the index along `axis`) that hold a threshold element of any of `shapes`, shift included as the
    second item of each (shape, shift) pair, plus the first and last row and `nrand` seeded random ones"""
    rows = {0, extent - 1} | {int(r) for r in rng.integers(0, extent, nrand)}
    for shape, shift in shapes:
        rows |= {p[axis] for p in positions(shape, shift)}
    return sorted(rows)


def covered(shape, units, axes):
    """the flat indices of `shape` whose indices along `axes` form one of `units` (tuples): the elements a check on
    those rows / columns / pixels compares"""
    units = set(tuple(u) for u in units)
    idx = np.indices(shape).reshape(len(shape), -1)
    keep = np.array([tuple(int(idx[a, i]) for a in axes) in units for i in range(idx.shape[1])])
    return set(np.flatnonzero(keep).tolist())


def straddles(shape, flats_covered, shift=0):
    """every threshold has the element before it and its own element in `flats_covered`, and so has the last element"""
    n = int(np.prod(shape))
    need = set()
    for t in THRESHOLDS:
        need |= {(t >> shift) - 1, t >> shift}
    need.add(n - 1)
    return need <= set(flats_covered)


# ---------------------------------------------------------------------------------------------- row-local and crops

def stereo_join_row(oracle, fL, fR, D, y):
    """(left, right) rows y, (D, W), of oracle.stereo_join (StereoJoin is row-local); NaN where it writes nothing"""
    L, R = oracle.stereo_join(fL[:, y:y + 1], fR[:, y:y + 1], D)
    return L[:, 0], R[:, 0]


def crop(H, y, halo):
    return max(0, y - halo), min(H, y + halo + 1)


def cost_row(oracle, x0, x1, D, y, direction, kind):
    """row y, (D, W), of oracle.census (kind 'census', x0 / x1 (nch, H, W)) or oracle.ad ('ad', (H, W)) from the image
    rows y - 4 .. y + 4 (the 9 x 9 window)"""
    H = x0.shape[-2]
    a, b = crop(H, y, 4)
    if kind == "census":
        return oracle.census(x0[:, a:b], x1[:, a:b], D, direction)[:, y - a]
    return oracle.ad(x0[a:b], x1[a:b], D, direction)[:, y - a]


def crop_arms(xc, a, b):
    """cross() arms (4, H, W) of rows [a, b) in the coordinates of that crop, vertical end-points clamped to it (as
    rowband.band_arms does: only rows whose outputs are not compared are affected)"""
    q = np.array(xc[:, a:b], np.float32)
    q[2] = np.maximum(q[2] - a, -1)
    q[3] = np.minimum(q[3] - a, b - a)
    return q


def cbca_row(oracle, x0c, x1c, rows, y, halo, direction, cbca_f64=None, planes=None):
    """row y, (D, W), of oracle.cbca from the volume rows [y - halo, y + halo]; rows(a, b) returns vol[:, a:b, :W] as a
    float32 array.  With cbca_f64 (dispatch_cases.cbca_f64), also its row y on `planes` (the other planes NaN)."""
    H = x0c.shape[1]
    a, b = crop(H, y, halo)
    v = np.ascontiguousarray(rows(a, b), np.float32)
    a0, a1 = crop_arms(x0c, a, b), crop_arms(x1c, a, b)
    want = oracle.cbca(a0, a1, v, direction)[:, y - a]
    if cbca_f64 is None:
        return want
    w64 = np.full(want.shape, np.nan)
    w64[planes] = cbca_f64(a0, a1, v, direction, planes=planes)[planes, y - a]
    return want, w64


def sgm_crossings(oracle, x0, x1, row, col, ys, xs, params, direction):
    """{(y, x): (D,)} the sgm2 result (H, W, D) at every crossing of rows ys and columns xs: oracle.sgm2_band with pass
    mask 3 on the 1-row band y gives (0 + right) + left; that goes into row y of the 1-column band at xoff = x, which pass
    mask 12 turns into ((r + l) + down) + up, the reference's order.  row(y) -> (W, D) and col(x) -> (H, D) of the cost
    volume; x0 / x1 the (H, W) images."""
    H, W = x0.shape
    horiz = {}
    for y in ys:
        r = np.ascontiguousarray(row(y), np.float32)[None]
        horiz[y] = oracle.sgm2_band(x0, x1, r, np.zeros_like(r), W, y, 0, *params, direction, 3)[0]
    out = {}
    for x in xs:
        c = np.ascontiguousarray(col(x), np.float32)[:, None]
        acc = np.zeros_like(c)
        for y in ys:
            acc[y, 0] = horiz[y][x]
        oracle.sgm2_band(x0, x1, c, acc, W, 0, x, *params, direction, 12)
        for y in ys:
            out[y, x] = acc[y, 0].copy()
    return out


def argmin_columns(cols):
    """0-based first minimum of each column of (D, n), NaN skipped (strict <, start at +inf: an all-NaN column gives 0)"""
    D, n = cols.shape
    best = np.full(n, np.inf, np.float32)
    arg = np.zeros(n, np.int64)
    for d in range(D):
        lt = cols[d] < best
        best[lt] = cols[d][lt]
        arg[lt] = d
    return arg.astype(np.float32)


def fill_invalid_rows(rows, W, sentinel):
    """mccnn_fill_invalid's rule on rows (D, k, W) of sentinel-filled volumes: (left, right) with NaN where x < d / x >= W - d"""
    D = rows.shape[0]
    d, x = np.arange(D)[:, None, None], np.arange(W)[None, None, :]
    shape = (D, rows.shape[1], W)
    return (np.where(np.broadcast_to(x < d, shape), np.float32(np.nan), np.float32(sentinel)),
            np.where(np.broadcast_to(x >= W - d, shape), np.float32(np.nan), np.float32(sentinel)))
