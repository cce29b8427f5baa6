"""CPU: the restatement of the fast architecture's feature tower (oracle/feature_tower.py), prepared for
the tower in-library.  Parity unpinned (cudnn.benchmark, no nets in the tree); these tests pin the
restatement to main.lua:725-745 and tie it to the rest of the oracle."""
import numpy as np

import mccnn_b200  # noqa: F401
from mccnn_b200 import pipeline
from oracle import feature_tower as ft


def test_conv_against_the_loop_definition():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 3, 5, 7)).astype(np.float32)
    w = rng.standard_normal((4, 3, 3, 3)).astype(np.float32)
    b = rng.standard_normal(4).astype(np.float32)
    y = ft.conv_same(x, w, b)
    xp = np.pad(x.astype(np.float64), ((0, 0), (0, 0), (1, 1), (1, 1)))
    for n in range(2):
        for o in range(4):
            for i in range(5):
                for j in range(7):
                    want = b[o] + (xp[n, :, i:i + 3, j:j + 3] * w[o]).sum()      # cross-correlation, zero padding
                    assert abs(y[n, o, i, j] - want) < 1e-5


def test_tower_shape_norm_and_border(oracle):
    rng = np.random.default_rng(1)
    layers = ft.make_weights(rng, l1=4, fm=16)
    x = rng.standard_normal((2, 1, 12, 20)).astype(np.float32)
    f = ft.tower_forward(x, layers)
    assert f.shape == (2, 16, 12, 20) and f.dtype == np.float32
    assert np.abs((f.astype(np.float64) ** 2).sum(1) - 1).max() < 1e-3          # unit norm per pixel (up to the 1e-5)
    raw = ft.tower_forward(x, layers, normalize=False)
    assert (raw < 0).any()                                                      # no ReLU after the last conv
    want, _ = oracle.normalize_forward(raw)                                     # Normalize2 = adcensus.Normalize_forward
    assert np.abs(f - want).max() < 1e-6
    # window size 1 + 4 * 2 = 9 -> fix_border copies 4 columns: the presets' `border`
    assert ft.window_size(layers) == 9 and (ft.window_size(layers) - 1) // 2 == pipeline.make_params("kitti", "fast").border
    assert (ft.window_size(ft.make_weights(rng, l1=5, fm=8)) - 1) // 2 == pipeline.make_params("mb", "fast").border


def test_receptive_field_is_the_window():
    """a pixel's features depend exactly on the ws x ws input window around it"""
    rng = np.random.default_rng(2)
    layers = ft.make_weights(rng, l1=4, fm=4)
    x = rng.standard_normal((1, 1, 21, 21)).astype(np.float32)
    base = ft.tower_forward(x, layers, normalize=False)
    x2 = x.copy()
    x2[0, 0, 10 + 5, 10] += 1.0                                                 # 5 rows below the centre: outside 9 x 9
    x3 = x.copy()
    x3[0, 0, 10 + 1, 10 - 1] += 1.0                                             # well inside (ReLUs may gate the far corner)
    assert np.array_equal(ft.tower_forward(x2, layers, normalize=False)[0, :, 10, 10], base[0, :, 10, 10])
    assert not np.array_equal(ft.tower_forward(x3, layers, normalize=False)[0, :, 10, 10], base[0, :, 10, 10])


def test_rows_equal_the_full_tower_in_every_band():
    """tower_forward_rows: a full-width band of output rows from a crop with l1 rows of margin equals those rows of the
    whole image's tower (to float64 summation order), at the top edge, in the middle and at the bottom edge"""
    rng = np.random.default_rng(4)
    for l1, normalize in ((3, True), (5, False)):
        layers = ft.make_weights(rng, l1=l1, fm=8)
        x = rng.standard_normal((2, 1, 23, 17)).astype(np.float32)
        full = ft.tower_forward(x, layers, normalize)
        for y0, y1 in ((0, 3), (0, 1), (9, 14), (20, 23), (22, 23), (0, 23)):
            got = ft.tower_forward_rows(x, layers, y0, y1, normalize)
            assert got.shape == (2, 8, y1 - y0, 17)
            assert np.abs(got - full[:, :, y0:y1]).max() < 1e-6, (l1, y0, y1)
        # one row less of margin lets the crop's zero padding in
        y0, y1 = 9, 14
        short = ft.tower_forward(x[:, :, y0 - l1 + 1:y1 + l1 - 1], layers, normalize)[:, :, l1 - 1:l1 - 1 + y1 - y0]
        assert np.abs(short - full[:, :, y0:y1]).max() > 1e-3


def test_against_the_pytorch_restatement_fixture():
    """tests/golden/feature_tower.npz: the module stack of main.lua:726-749 + Normalize_forward restated in PyTorch (CPU fp32),
    generator oracle/make_feature_tower_golden.py"""
    import os

    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "feature_tower.npz"))
    layers = [(g["w%d" % i], g["b%d" % i]) for i in range(4)]
    got = ft.tower_forward(g["x"], layers)
    assert np.abs(got - g["out"]).max() < 2e-6
