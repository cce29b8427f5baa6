"""The MiddEval3 SDK's evaldisp metrics and the website's A50-A99 error quantiles, restated in numpy -- TEST INFRASTRUCTURE.

The SDK sources are not part of this tree; this is the specification that csrc/mb_eval.cu and mb_eval.py implement, step by
step, so that each step can be read against it.  Parity with the SDK binary and with the website is not pinned.

Inputs
    disp (h, w) float32, the map at the data resolution; gt (Hg, Wg) float32 from disp0GT.pfm, +inf = unknown; mask
    (Hg, Wg) uint8 from mask0nocc.png or None; maxdisp, the ndisp= of the scene's trainingH calib.txt.  Both PFMs are
    stored bottom-up and are flipped to top-down rows before this; the PNG mask is top-down already.
    scale = Wg / w must be 1, 2 or 4 with Hg == scale h and Wg == scale w; the mask must have gt's size.

Per gt pixel (x, y), in fp32 with the SDK's expression order
    1. skip it when gt == +inf;
    2. d = (float)scale * disp[y / scale][x / scale]   (integer division: a nearest-neighbour lookup);
    3. valid = d != +inf;
    4. if valid: maxd = (float)(scale * maxdisp); d = max(0, min(maxd, d)) with min(a, b) = (a < b) ? a : b and
       max(a, b) = (a > b) ? a : b in that argument order, so a NaN d stays NaN and -inf becomes 0;
    5. err = fabsf(d - gt);
    6. region 'all' takes every pixel not skipped, region 'nonocc' those whose mask byte is 255 (every one without a mask,
       as evaldisp scores without one).

Per region
    n counts the pixels; a valid pixel adds err to sum(err), (double)err^2 to sum(err^2) (float64), and 1 to bad_t when
    err > t for t in 0.5, 1, 2, 4 (a NaN err is valid, never bad, and makes the sums NaN); an invalid one adds 1 to
    invalid.  Reported:
        bad_t = (bad_t + invalid) / n      (the SDK's "totbad", the website's column)
        invalid / n
        avgerr = sum(err) / (n - invalid),  rms = sqrt(sum(err^2) / (n - invalid))
        A_q = the k-th smallest err over the valid pixels, k = ceil(q (n - invalid)) 1-based, for q = 0.50, 0.90, 0.95,
              0.99, computed exactly as ceil(P (n - invalid) / 100) in integers (P = 50, 90, 95, 99); errs order by their
              fp32 bits (a NaN err after +inf); NaN when there is no valid pixel
        coverage = n / (Hg Wg)             (evaldisp's first column)
    0 / 0 is NaN.  The sums are float64 where evaldisp accumulates a float: the last digits of avgerr may differ.
A set's summary is the plain mean of each per-scene value (the website's per-scene weights are not applied).
"""
import numpy as np

# the count layout of mccnn_mb_evaldisp (include/adcensus_b200.h): counts[r, k], r 0 = nonocc, 1 = all
N, VALID, BAD05, BAD1, BAD2, BAD4, INVALID = range(7)
NCOUNT = 7
THRESHOLDS = (0.5, 1, 2, 4)
BAD = dict(zip(THRESHOLDS, (BAD05, BAD1, BAD2, BAD4)))
PERCENT = (50, 90, 95, 99)


def scale_of(disp_shape, gt_shape):
    """scale = Wg / w, refused (ValueError) unless it is 1, 2 or 4 and both sizes are scale times the map's"""
    (h, w), (Hg, Wg) = disp_shape, gt_shape
    scale = Wg // w if w else 0
    if scale not in (1, 2, 4) or Wg != scale * w or Hg != scale * h:
        raise ValueError("the ground truth is %dx%d, the map %dx%d: the ratio must be 1, 2 or 4" % (Hg, Wg, h, w))
    return scale


def errors(disp, gt, maxdisp):
    """(known, valid, err) of every gt pixel, steps 1-5"""
    disp = np.asarray(disp, np.float32)
    gt = np.asarray(gt, np.float32)
    scale = scale_of(disp.shape, gt.shape)
    Hg, Wg = gt.shape
    known = gt != np.float32(np.inf)                                      # 1.
    yy, xx = np.meshgrid(np.arange(Hg) // scale, np.arange(Wg) // scale, indexing="ij")
    with np.errstate(over="ignore"):
        d = np.float32(scale) * disp[yy, xx]                              # 2.
    valid = d != np.float32(np.inf)                                       # 3.
    maxd = np.float32(scale * maxdisp)
    with np.errstate(all="ignore"):
        c = np.where(maxd < d, maxd, d)                                   # 4. min(maxd, d)
        c = np.where(np.float32(0) > c, np.float32(0), c)                 #    max(0, ..)
        d = np.where(valid, c, d).astype(np.float32)
        err = np.abs(d - gt).astype(np.float32)                           # 5.
    return known, valid, err


def kth(err, k):
    """the k-th smallest (1-based) of the float32 errs in fp32 bit order"""
    keys = np.sort(np.ascontiguousarray(err, np.float32).view(np.uint32))
    return keys[k - 1:k].view(np.float32)[0]


def evaldisp(disp, gt, mask, maxdisp):
    """(counts (2, NCOUNT) int64, sums (2, 2) float64 [sum(err), sum(err^2)], quantiles (2, 4) float32), r 0 nonocc"""
    known, valid, err = errors(disp, gt, maxdisp)
    if mask is not None:
        mask = np.asarray(mask, np.uint8)
        if mask.shape != known.shape:
            raise ValueError("the mask is %dx%d, the ground truth %dx%d" % (mask.shape + known.shape))
    regions = (known if mask is None else known & (mask == 255), known)  # 6.
    counts = np.zeros((2, NCOUNT), np.int64)
    sums = np.zeros((2, 2), np.float64)
    quantiles = np.full((2, len(PERCENT)), np.nan, np.float32)
    for r, m in enumerate(regions):
        e = err[m & valid]
        counts[r, N] = m.sum()
        counts[r, VALID] = e.size
        counts[r, INVALID] = (m & ~valid).sum()
        with np.errstate(invalid="ignore"):
            for t, k in BAD.items():
                counts[r, k] = (e > np.float32(t)).sum()
        e64 = e.astype(np.float64)
        sums[r] = e64.sum(), (e64 * e64).sum()
        for j, p in enumerate(PERCENT):
            if e.size:
                quantiles[r, j] = kth(e, (p * e.size + 99) // 100)
    return counts, sums, quantiles


def metrics(counts, sums, quantiles, gt_pixels):
    """{region: {name: value}} of the reported values, names bad0.5 bad1 bad2 bad4 invalid avgerr rms A50 A90 A95 A99
    coverage"""
    out = {}
    q = lambda a, b: float(a) / float(b) if b else float("nan")
    for r, reg in enumerate(("nonocc", "all")):
        c = counts[r]
        nv = int(c[N] - c[INVALID])
        v = {}
        for t, k in BAD.items():
            v["bad%g" % t] = q(c[k] + c[INVALID], c[N])
        v["invalid"] = q(c[INVALID], c[N])
        v["avgerr"] = q(sums[r][0], nv)
        v["rms"] = float(np.sqrt(q(sums[r][1], nv)))
        for j, p in enumerate(PERCENT):
            v["A%d" % p] = float(quantiles[r][j])
        v["coverage"] = q(c[N], gt_pixels)
        out[reg] = v
    return out
