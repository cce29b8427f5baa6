"""CPU restatement of the 'fast' architecture's feature tower -- TEST INFRASTRUCTURE ONLY, prepared for
the tower in-library (fused into StereoJoin's producer); no product code uses it.

What the reference does at test time (main.lua:725-745, 907-920; Normalize2.lua:8-13): x_batch
(2,1,H,W) goes through l1 x cudnn.SpatialConvolution(ks x ks, stride 1, pad (ks-1)/2) with a ReLU
after every layer but the last (l1 = 4, fm = 64, ks = 3 for kitti; l1 = 5 for mb: main.lua:212-214,
271-273), then Normalize2 = adcensus.Normalize_forward (x / sqrt(sum_c x^2 + 1e-5),
adcensus.cu:1284-1308).  cuDNN convolutions are cross-correlations (no kernel flip).  The window of
the stack is ws = 1 + l1 (ks - 1) (main.lua:382-391) and fix_border copies n = (ws - 1) / 2 columns.

Parity: **unpinned** -- `cudnn.benchmark = true` (main.lua:330) picks algorithms per run, so the
reference's own outputs are only reproducible to ~1e-6; no trained nets or vectors are in the tree.
This restatement accumulates every layer in float64 and rounds once to float32.
"""
import numpy as np


def make_weights(rng, l1=4, fm=64, ks=3, n_in=1):
    layers = []
    c = n_in
    for _ in range(l1):
        s = 1.0 / np.sqrt(c * ks * ks)
        layers.append((rng.standard_normal((fm, c, ks, ks)).astype(np.float32) * np.float32(s),
                       rng.standard_normal(fm).astype(np.float32) * np.float32(0.1)))
        c = fm
    return layers


def window_size(layers):
    """main.lua:382-391"""
    return 1 + sum(w.shape[-1] - 1 for w, _ in layers)


def conv_same(x, w, b):
    """x (N,C,H,W), w (O,C,k,k), b (O,): zero-padded 'same' cross-correlation, float64 accumulation"""
    import torch

    k = w.shape[-1]
    y = torch.nn.functional.conv2d(torch.from_numpy(np.asarray(x, np.float64)), torch.from_numpy(np.asarray(w, np.float64)),
                                   torch.from_numpy(np.asarray(b, np.float64)), padding=(k - 1) // 2)
    return y.numpy().astype(np.float32)


def tower_forward(x_batch, layers, normalize=True):
    """(N,1,H,W) -> (N,fm,H,W) float32: conv / ReLU stack (no ReLU after the last conv), then Normalize2"""
    h = np.asarray(x_batch, dtype=np.float32)
    for i, (w, b) in enumerate(layers):
        h = conv_same(h, w, b)
        if i + 1 < len(layers):
            h = np.maximum(h, np.float32(0.0))
    if normalize:
        norm = (h.astype(np.float64) ** 2).sum(1, keepdims=True) + 1e-5           # adcensus.cu:1296
        h = (h / np.sqrt(norm)).astype(np.float32)
    return h


def tower_forward_rows(x_batch, layers, y0, y1, normalize=True):
    """Output rows [y0, y1) of tower_forward at full width, from input rows [y0 - l1, y1 + l1) clipped to the image: each
    3x3 layer moves the crop's zero padding one row inwards, so the l1 extra rows keep it out of the kept rows.  Lets a
    full-size image be checked band by band at a fraction of the cost."""
    H = np.shape(x_batch)[2]
    l1 = len(layers)
    a, b = max(0, y0 - l1), min(H, y1 + l1)
    return tower_forward(np.asarray(x_batch)[:, :, a:b], layers, normalize)[:, :, y0 - a:y1 - a]
