"""Seeded inputs of the GPU tests of the feature tower and the scorer head (tests/test_gpu_feature_tower.py,
tests/test_gpu_scorer_head.py).  tests/test_kernel_mistakes.py builds the same inputs on the CPU and checks that common
kernel mistakes move the oracle's output far beyond the bars those tests use, so a pass on the GPU means something."""
import numpy as np

from . import feature_tower as oft
from . import scorer_head as osh


def tower_case(seed, n_in, fm, l1, nimg, H, W, scale=1.0, zero=False):
    """(layers, x): random tower weights of the reference's shapes and an (nimg, n_in, H, W) float32 image batch"""
    rng = np.random.default_rng(seed)
    layers = oft.make_weights(rng, l1=l1, fm=fm, n_in=n_in)
    x = rng.standard_normal((nimg, n_in, H, W)).astype(np.float32) * np.float32(scale)
    return layers, (np.zeros_like(x) if zero else x)


def tower_want(x, layers, arch, rows=None):
    """float64-accumulated tower output for arch 'fast' (Normalize2) or 'slow' (ReLU after every layer); rows = (y0, y1)
    restricts it to a full-width band"""
    fast = arch == "fast"
    out = oft.tower_forward(x, layers, fast) if rows is None else oft.tower_forward_rows(x, layers, rows[0], rows[1], fast)
    return out if fast else np.maximum(out, np.float32(0.0))


def head_case(seed, fm, nh2, l2, H, W, scale=1.0):
    """(layers, featL, featR): random net_te2 weights and ReLU'd (fm, H, W) features times `scale`"""
    rng = np.random.default_rng(seed)
    layers = osh.make_weights(rng, fm, nh2, l2)
    f = [(np.maximum(rng.standard_normal((fm, H, W)), 0) * scale).astype(np.float32) for _ in range(2)]
    return layers, f[0], f[1]


def bf16(a):
    """round to the nearest bfloat16 (ties to even), kept as float32"""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32)


def tower_bf16(x, layers, arch):
    """the tower with plain bf16 operands in the tensor-core layers (nterms = 1: no lo term); layer 1 stays exact fp32"""
    h = np.asarray(x, np.float32)
    for i, (w, b) in enumerate(layers):
        h = oft.conv_same(h if i == 0 else bf16(h), w if i == 0 else bf16(w), b)
        if i + 1 < len(layers) or arch == "slow":
            h = np.maximum(h, np.float32(0.0))
    if arch == "fast":
        h = (h / np.sqrt((h.astype(np.float64) ** 2).sum(1, keepdims=True) + 1e-5)).astype(np.float32)
    return h


def head_volume_bf16(featL, featR, D, layers):
    """the left volume with plain bf16 operands in the hidden layers (nterms = 1: no lo term); the nh2 -> 1 layer stays fp32"""
    L = len(layers)
    rounded = [(bf16(w), b) if i + 1 < L else (w, b) for i, (w, b) in enumerate(layers)]
    fm, H, W = featL.shape
    vol = np.full((D, H, W), np.nan, np.float32)
    for d in range(min(D, W)):
        h = bf16(np.concatenate([featL[:, :, d:].reshape(fm, -1), featR[:, :, :W - d].reshape(fm, -1)], axis=0))
        for i, (w, b) in enumerate(rounded):
            y = (w.astype(np.float64) @ h.astype(np.float64) + b.astype(np.float64)[:, None]).astype(np.float32)
            if i + 1 < L:
                h = np.maximum(y, np.float32(0.0))
                h = bf16(h) if i + 2 < L else h
            else:
                h = (1.0 / (1.0 + np.exp(-y.astype(np.float64)))).astype(np.float32)
        vol[d, :, d:] = h[0].reshape(H, W - d)
    return vol


def right_from_left(volL):
    """the right volume holds the left one's scores shifted by d columns (main.lua:976-978)"""
    volR = np.full_like(volL, np.nan)
    W = volL.shape[2]
    for d in range(min(volL.shape[0], W)):
        volR[d, :, :W - d] = volL[d, :, d:]
    return volR


def head_want(featL, featR, D, layers):
    """(left, right) volumes of the oracle, (D, H, W) each"""
    volL = osh.head_volume(featL, featR, D, layers, -1)
    return volL, right_from_left(volL)


# (seed, n_in, fm, l1, arch, nimg, H, W): one case per kernel variant of csrc/feature_tower.cu.  fm 16 / 32: ring kernel at
# N = 64 with all nine taps in one pass; 48: N = 64, two passes; 64: the resident kernel; 80 / 96 / 112 / 128: ring kernel at
# N = 128 with three to five passes (80, 96, 112 padded planes, 128 none)
TOWER_VARIANTS = [(100 + fm, 1, fm, 3, "fast" if fm in (16, 48, 64, 96, 128) else "slow", 2, 5, 200)
                  for fm in (16, 32, 48, 64, 80, 96, 112, 128)]

# (seed, n_in, fm, l1, arch, nimg, H, W, scale, zero): widths around the 128-pixel tile, one to three rows and images, colour
# input into the resident kernel, the shallowest and deepest towers, an all-zero image (Normalize2 of bias-only features)
# and input scales far from 1
TOWER_EDGES = [
    (301, 1, 64, 4, "fast", 2, 1, 1, 1.0, False),
    (302, 1, 64, 4, "fast", 1, 2, 2, 1.0, False),
    (303, 1, 112, 3, "slow", 3, 3, 127, 1.0, False),
    (304, 1, 64, 4, "fast", 2, 1, 128, 1.0, False),
    (305, 1, 48, 3, "fast", 1, 3, 129, 1.0, False),
    (306, 1, 128, 2, "slow", 2, 2, 257, 1.0, False),
    (307, 1, 16, 2, "slow", 3, 1, 129, 1.0, False),
    (308, 3, 64, 3, "fast", 2, 3, 129, 1.0, False),
    (309, 3, 64, 4, "slow", 1, 2, 257, 1.0, False),
    (310, 1, 32, 1, "slow", 2, 3, 70, 1.0, False),
    (311, 3, 112, 1, "slow", 1, 2, 50, 1.0, False),
    (312, 1, 64, 8, "fast", 1, 3, 130, 1.0, False),
    (313, 1, 16, 8, "slow", 2, 2, 140, 1.0, False),
    (314, 1, 64, 4, "fast", 2, 3, 140, 1.0, True),
    (315, 1, 112, 4, "slow", 1, 3, 140, 1.0, True),
    (316, 1, 64, 4, "fast", 2, 3, 200, 1e-3, False),
    (317, 1, 112, 4, "slow", 2, 3, 200, 1e-3, False),
    (318, 1, 64, 4, "fast", 2, 3, 200, 1e3, False),
    (319, 1, 112, 4, "slow", 2, 3, 200, 1e3, False),
]

# (seed, fm, nh2, l2, H, W, D, scale): a pairwise selection over fm (192 fills layer 1's K = 384; 24 and 120 give an odd
# number of layer-1 K steps), nh2, l2, W and H around the 64-pixel tile, D from 1 to past W, and feature scales (at 30 the
# sigmoid saturates)
HEAD_SWEEP = [
    (201, 8, 128, 1, 1, 1, 1, 1.0),
    (202, 24, 256, 2, 3, 63, 62, 0.01),
    (203, 112, 384, 4, 1, 64, 64, 1.0),
    (204, 120, 128, 3, 3, 65, 70, 30.0),
    (205, 192, 384, 2, 3, 129, 128, 1.0),
    (206, 192, 128, 4, 1, 65, 65, 0.01),
    (207, 24, 384, 3, 1, 129, 134, 1.0),
    (208, 8, 256, 4, 3, 64, 1, 30.0),
    (209, 112, 256, 1, 3, 63, 68, 1.0),
    (210, 120, 384, 1, 1, 1, 6, 1.0),
    (211, 192, 256, 3, 1, 1, 1, 30.0),
    (212, 8, 384, 2, 3, 129, 129, 0.01),
    (213, 24, 128, 4, 3, 65, 64, 1.0),
    (214, 120, 256, 2, 1, 63, 63, 1.0),
]
