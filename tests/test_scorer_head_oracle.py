"""CPU: the restatement of the accurate architecture's scorer head (oracle/scorer_head.py), prepared for the
next hot-path row.  Parity is unpinned (no reference vectors exist); these tests pin the
restatement to the definition in main.lua:963-978 / SpatialConvolution1_fw.lua."""
import numpy as np
import pytest

from oracle import scorer_head as sh


def _feats(rng, fm, H, W):
    return np.maximum(rng.standard_normal((fm, H, W)), 0).astype(np.float32)      # tower ends with ReLU


def test_against_the_per_pixel_definition():
    rng = np.random.default_rng(0)
    fm, nh2, l2, H, W, D = 6, 10, 3, 4, 9, 5
    layers = sh.make_weights(rng, fm, nh2, l2)
    fL, fR = _feats(rng, fm, H, W), _feats(rng, fm, H, W)
    vol = sh.head_volume(fL, fR, D, layers, -1)
    for d in range(D):
        for y in range(H):
            for x in range(W):
                if x - d < 0:
                    assert np.isnan(vol[d, y, x])
                    continue
                h = np.concatenate([fL[:, y, x], fR[:, y, x - d]]).astype(np.float64)
                for i, (w, b) in enumerate(layers):
                    h = w.astype(np.float64) @ h + b
                    h = np.maximum(h, 0) if i + 1 < len(layers) else 1 / (1 + np.exp(-h))
                assert abs(vol[d, y, x] - h[0]) < 1e-5


def test_both_directions_hold_the_same_scores():
    """the (H, W-d) result of disparity d goes to columns d.. of the left and 0..W-d of the right volume"""
    rng = np.random.default_rng(1)
    fm, H, W, D = 5, 3, 12, 7
    layers = sh.make_weights(rng, fm, 8, 2)
    fL, fR = _feats(rng, fm, H, W), _feats(rng, fm, H, W)
    vl, vr = sh.head_volume(fL, fR, D, layers, -1), sh.head_volume(fL, fR, D, layers, 1)
    for d in range(D):
        assert np.array_equal(vl[d, :, d:], vr[d, :, :W - d])
        assert np.isnan(vl[d, :, :d]).all() and np.isnan(vr[d, :, W - d:]).all()
    assert np.nanmin(vl) > 0 and np.nanmax(vl) < 1                                 # sigmoid


def test_first_layer_splits_into_a_left_and_a_right_half():
    """W1 [l; r] = W1[:, :fm] l + W1[:, fm:] r: the per-pixel halves can be computed once per image and only
    added per disparity -- the decomposition the GPU kernel uses"""
    rng = np.random.default_rng(2)
    fm, nh2, H, W = 7, 16, 3, 10
    layers = sh.make_weights(rng, fm, nh2, 4)
    fL, fR = _feats(rng, fm, H, W), _feats(rng, fm, H, W)
    w1, b1 = layers[0]
    a = w1[:, :fm].astype(np.float64) @ fL.reshape(fm, -1).astype(np.float64)     # (nh2, HW), once
    b = w1[:, fm:].astype(np.float64) @ fR.reshape(fm, -1).astype(np.float64)
    d = 3
    idx = np.arange(H * W).reshape(H, W)
    h1 = np.maximum(a[:, idx[:, d:].ravel()] + b[:, idx[:, :W - d].ravel()] + b1.astype(np.float64)[:, None], 0)
    rest = sh.head_pixels(h1.astype(np.float32), [(np.eye(nh2, dtype=np.float32), np.zeros(nh2, np.float32))] + layers[1:])
    want = sh.head_volume(fL, fR, d + 1, layers, -1)[d, :, d:].ravel()
    assert np.abs(rest - want).max() < 1e-5


def test_samples_equal_the_volume():
    """head_samples at chosen (d, y, x) equals head_volume's entries there (to float64 summation order), including x = d
    and x = W - 1"""
    rng = np.random.default_rng(3)
    fm, nh2, l2, H, W, D = 8, 16, 3, 4, 13, 9
    layers = sh.make_weights(rng, fm, nh2, l2)
    fL, fR = _feats(rng, fm, H, W), _feats(rng, fm, H, W)
    vol = sh.head_volume(fL, fR, D, layers, -1)
    d, y, x = np.nonzero(~np.isnan(vol))                            # every valid entry, in one call
    assert np.abs(sh.head_samples(fL, fR, layers, d, y, x) - vol[d, y, x]).max() < 1e-6
    d, y, x = [0, 8, 8, 3], [0, 3, 1, 2], [0, 8, W - 1, 5]           # a few in arbitrary order
    assert np.abs(sh.head_samples(fL, fR, layers, d, y, x) - vol[d, y, x]).max() < 1e-6
    # the right image's pixel is x - d: one column off is far from the volume
    assert np.abs(sh.head_samples(fL, fR, layers, [2, 3], [1, 1], [7, 7]) - vol[[3, 2], [1, 1], [7, 7]]).max() > 1e-4
    with pytest.raises(ValueError):
        sh.head_samples(fL, fR, layers, [4], [0], [3])              # x < d has no score


def test_against_the_pytorch_restatement_fixture():
    """tests/golden/scorer_head.npz: main.lua:962-978 + SpatialConvolution1_fw.lua:11-31 restated in PyTorch (CPU fp32:
    addmm, bias add, relu, sigmoid), generator oracle/make_scorer_head_golden.py.  The float64-accumulating oracle agrees
    with it to fp32 rounding of a 384-term product chain."""
    import os

    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "scorer_head.npz"))
    layers = [(g["w%d" % i], g["b%d" % i]) for i in range(5)]
    D = int(g["D"])
    for direction, key in ((-1, "volL"), (1, "volR")):
        got = sh.head_volume(g["featL"], g["featR"], D, layers, direction)
        want = g[key][0]
        assert np.array_equal(np.isnan(got), np.isnan(want))
        m = ~np.isnan(want)
        assert np.abs(got[m] - want[m]).max() < 2e-6
