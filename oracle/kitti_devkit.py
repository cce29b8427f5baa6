"""The KITTI 2012 / 2015 stereo devkits' metrics restated in plain Python and numpy -- TEST INFRASTRUCTURE.

The devkit sources are not part of this tree; this is the specification that csrc/kitti_eval.cu and kitti_eval.py
implement, written loop by loop so that each step can be read against it.  Parity with the devkit binaries is not pinned.

Reading a map
    A stored uint16 value v == 0 is invalid (the devkit stores -1), otherwise d = v / 256 in float32 (exact).  A float map
    is first quantised as dataio.write_png16 writes it: v = d < 1e-5 ? 0 : d * 256 in float32, truncated, clamped to
    [0, 65535] (NaN gives 0).  Ground truth: disp_noc / disp_occ (2012), disp_noc_0 / disp_occ_0 (2015); a pixel has ground
    truth when v > 0.  KITTI 2015's obj_map: 0 is background, anything else foreground.

interpolateBackground, in place on the estimate, in this order
    1. each row, left to right: count a run of invalid pixels; when a valid pixel ends the run [u1, u2], fill it with
       min(d[u1 - 1], d[u2 + 1]) if u1 > 0 and u2 < W - 1 (runs touching either end of the row are left alone);
    2. in the same row, every pixel before the first valid pixel takes its value;
    3. then every pixel after the last valid pixel takes its value;
    4. after all rows: each column, the rows above its first valid row take that row's value, then the rows below its last
       valid row take that one's.
    A fully invalid row between valid rows therefore stays invalid, and a pixel still invalid keeps -1 and is scored with
    that value (an all-invalid estimate is scored against -1 everywhere).

Errors, in float32, over the pixels with ground truth: e = |d_gt - d_ipol|
    2012: Out@tau = #(e > tau) for tau = 2, 3, 4, 5; Avg = sum(e) / #gt.
    2015: D1 bad = e > 3 and e / d_gt > 0.05f (float32 quotient against float32(0.05): whether the devkit compares the
    quotient with a double or a float constant is not pinned; this is the choice), split into background / foreground.
    Each is computed against disp_noc ('noc') and disp_occ ('all').
Density: #(ground truth and the ORIGINAL estimate valid) / #ground truth.
Totals over a set: the sums of the counts and of sum(e) over the pairs, then the same quotients.
"""
import numpy as np

# the count layout of mccnn_kitti_devkit_counts (include/adcensus_b200.h): counts[r, k], r 0 = noc, 1 = all
GT, DENSE, OUT2, OUT3, OUT4, OUT5, D1_BG, D1_FG, GT_BG, GT_FG = range(10)
NCOUNT = 10
OUT = {2: OUT2, 3: OUT3, 4: OUT4, 5: OUT5}


def png16_values(disp):
    """dataio.write_png16's stored values of a float map, NaN -> 0"""
    d = np.asarray(disp, dtype=np.float32)
    v = np.where(d < np.float32(1e-5), np.float32(0), d * np.float32(256))
    v = np.where(np.isnan(v), np.float32(0), v)
    return np.clip(np.trunc(v), 0, 65535).astype(np.uint16)


def read_estimate(v16):
    """the devkit's estimate of stored values: -1 where v == 0, else v / 256 (float32); and the validity mask"""
    v16 = np.asarray(v16, dtype=np.uint16)
    valid = v16 != 0
    return np.where(valid, v16.astype(np.float32) / np.float32(256), np.float32(-1)).astype(np.float32), valid


def interpolate_background(d):
    """interpolateBackground on a copy of the float32 estimate d (H, W), -1 = invalid, step by step as the docstring says"""
    d = np.array(d, dtype=np.float32)
    H, W = d.shape
    ok = lambda v, u: d[v, u] >= 0
    for v in range(H):
        count = 0
        for u in range(W):
            if ok(v, u):
                if count >= 1:
                    u1, u2 = u - count, u - 1
                    if u1 > 0 and u2 < W - 1:
                        fill = min(d[v, u1 - 1], d[v, u2 + 1])
                        for uc in range(u1, u2 + 1):
                            d[v, uc] = fill
                count = 0
            else:
                count += 1
        for u in range(W):                            # extrapolate to the left
            if ok(v, u):
                for u2 in range(u):
                    d[v, u2] = d[v, u]
                break
        for u in range(W - 1, -1, -1):                # extrapolate to the right
            if ok(v, u):
                for u2 in range(u + 1, W):
                    d[v, u2] = d[v, u]
                break
    for u in range(W):
        for v in range(H):                            # extrapolate upwards
            if ok(v, u):
                for v2 in range(v):
                    d[v2, u] = d[v, u]
                break
        for v in range(H - 1, -1, -1):                # extrapolate downwards
            if ok(v, u):
                for v2 in range(v + 1, H):
                    d[v2, u] = d[v, u]
                break
    return d


def devkit_counts(est16, gt_noc16, gt_occ16, obj_map=None):
    """(counts (2, NCOUNT) int64, sums (2,) float64, the interpolated estimate) of one estimate given as stored values"""
    d, valid = read_estimate(est16)
    ipol = interpolate_background(d)
    fg = np.zeros(ipol.shape, bool) if obj_map is None else np.asarray(obj_map) > 0
    counts = np.zeros((2, NCOUNT), np.int64)
    sums = np.zeros(2, np.float64)
    for r, gt16 in enumerate((gt_noc16, gt_occ16)):
        gt16 = np.asarray(gt16, dtype=np.uint16)
        m = gt16 != 0
        dg = gt16[m].astype(np.float32) / np.float32(256)
        e = np.abs(dg - ipol[m]).astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            d1 = (e > np.float32(3)) & ((e / dg).astype(np.float32) > np.float32(0.05))
        counts[r, GT] = m.sum()
        counts[r, DENSE] = valid[m].sum()
        for tau, k in OUT.items():
            counts[r, k] = (e > np.float32(tau)).sum()
        counts[r, D1_BG] = (d1 & ~fg[m]).sum()
        counts[r, D1_FG] = (d1 & fg[m]).sum()
        counts[r, GT_BG] = (~fg[m]).sum()
        counts[r, GT_FG] = fg[m].sum()
        sums[r] = e.astype(np.float64).sum()
    return counts, sums, ipol
