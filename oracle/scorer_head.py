"""CPU restatement of the accurate ('slow') architecture's scorer head -- TEST INFRASTRUCTURE ONLY,
prepared for the scorer head kernel (the one dense contraction of mc-cnn); no product code uses it.

What the reference does (main.lua:956-979, 688-695; SpatialConvolution1_fw.lua:12-33): the tower
output `output` (2, fm, H, W) (fm = 112, last layer ReLU, no normalisation) is sliced per disparity d,
    l = output[left ][:, :, d:]      (fm, H, W-d)
    r = output[right][:, :, :W-d]
stacked along channels (2 fm, H, W-d) and pushed through `net_te2`:
    l2 x [ SpatialConvolution1_fw(2 fm | nh2 -> nh2) = per-pixel  W x + b  (cuBLAS addmm) ; ReLU ]
    SpatialConvolution1_fw(nh2 -> 1) ; Sigmoid
(l2 = 4, nh2 = 384 for kitti; l2 = 3 for kitti2015 / mb: main.lua:74-78, 120-124).  The (H, W-d)
result is the matching cost of disparity d: written to vol[d, :, d:] for direction -1 (left volume)
and to vol[d, :, :W-d] for direction +1 (right volume); the rest stays NaN; then fix_border.

Parity: **unpinned**.  The reference holds no golden vectors for the head, the summation order of
cuBLAS sgemm is not defined, and Torch7/cuBLAS cannot run here.  This restatement accumulates in
float64 and rounds once per layer to float32; a GPU implementation is to be compared with it at
the north star's 1e-4 bar.
"""
import numpy as np


def make_weights(rng, fm=112, nh2=384, l2=4, scale=None):
    """random head parameters with the reference's shapes: [(W (out,in), b (out,)), ...]"""
    layers = []
    n_in = 2 * fm
    for _ in range(l2):
        s = scale if scale is not None else 1.0 / np.sqrt(n_in)
        layers.append((rng.standard_normal((nh2, n_in)).astype(np.float32) * np.float32(s),
                       rng.standard_normal(nh2).astype(np.float32) * np.float32(0.1)))
        n_in = nh2
    s = scale if scale is not None else 1.0 / np.sqrt(n_in)
    layers.append((rng.standard_normal((1, n_in)).astype(np.float32) * np.float32(s),
                   rng.standard_normal(1).astype(np.float32) * np.float32(0.1)))
    return layers


def head_pixels(x, layers):
    """x: (2 fm, N) columns = pixels.  Returns (N,) float32: net_te2 on every column."""
    h = np.asarray(x, dtype=np.float32)
    for i, (w, b) in enumerate(layers):
        y = (w.astype(np.float64) @ h.astype(np.float64) + b.astype(np.float64)[:, None]).astype(np.float32)  # addmm + bias
        if i + 1 < len(layers):
            h = np.maximum(y, np.float32(0.0))                                     # cudnn.ReLU
        else:
            h = (1.0 / (1.0 + np.exp(-y.astype(np.float64)))).astype(np.float32)   # cudnn.Sigmoid
    return h[0]


def head_samples(featL, featR, layers, d, y, x):
    """The scores at the entries (d, y, x) of the left volume (x >= d): head_pixels on the gathered columns
    [featL[:, y, x]; featR[:, y, x - d]].  Checks a full-size volume at chosen points without running every disparity."""
    d, y, x = (np.asarray(v, dtype=np.int64) for v in (d, y, x))
    if (x < d).any():
        raise ValueError("head_samples: every entry needs x >= d")
    cols = np.concatenate([np.asarray(featL)[:, y, x], np.asarray(featR)[:, y, x - d]], axis=0)
    return head_pixels(cols, layers)


def head_volume(featL, featR, D, layers, direction):
    """main.lua:963-978 for one direction: (D,H,W) float32, NaN where x - d < 0 (direction -1, left
    volume) / x + d >= W (direction +1, right volume).  fix_border is applied by the caller."""
    featL = np.asarray(featL, dtype=np.float32)
    featR = np.asarray(featR, dtype=np.float32)
    fm, H, W = featL.shape
    vol = np.full((D, H, W), np.nan, np.float32)
    for d in range(min(D, W)):
        l = featL[:, :, d:].reshape(fm, -1)                                      # :967
        r = featR[:, :, :W - d].reshape(fm, -1)                                  # :968
        out = head_pixels(np.concatenate([l, r], axis=0), layers).reshape(H, W - d)   # :969-975
        if direction == -1:
            vol[d, :, d:] = out                                                   # :976
        else:
            vol[d, :, :W - d] = out
    return vol
