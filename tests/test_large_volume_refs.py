"""CPU: the sampled references of tests/test_gpu_large_volumes.py, with the 2^29 / 2^30 / 2^31 thresholds scaled down by
2^15, at D = 40, H = 37, W = 66 (ld = 68): each helper's rows, crops and crossings equal the whole-volume oracle result,
and every sample set of every layout straddles every threshold."""
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


lv = _load("large_volumes")
dc = _load("dispatch_cases")

SHIFT = 15
D, H, W = 40, 37, 66
LD = dc.sj_ld(W) - 4            # 68: a pitch of W rounded up to 4, as the pitched entry points use it


def _rows(shapes, axis, extent, seed=0):
    return lv.sample_rows([(s, SHIFT) for s in shapes], axis, extent, np.random.default_rng(seed))


def test_thresholds_fit_and_order():
    flats = lv.threshold_flats((D, H, W), SHIFT)
    assert flats == sorted(flats) and len(set(flats)) == 7 and flats[-1] == D * H * W - 1
    with pytest.raises(ValueError):
        lv.threshold_flats((2, 3, 4), SHIFT)


@pytest.mark.parametrize("shape,axes,unit", [
    ((D, H, W), (1,), "row"), ((D, H, LD), (1,), "row"),            # row checks: StereoJoin, CBCA, census / AD, fills
    ((D, H, W), (1, 2), "pixel"), ((D, H, LD), (1, 2), "pixel"),    # D-column checks: arg-min, sub-pixel
    ((H, W, D), (0, 1), "crossing"),                                 # SGM crossings of sampled rows and columns
])
def test_samples_straddle_every_threshold(shape, axes, unit):
    """the units each GPU check compares cover the elements just before and at each threshold and the last element"""
    if unit == "row":
        units = [(y,) for y in _rows([shape], 1, H)]
    elif unit == "pixel":
        units = sorted({(p[1], p[2]) for p in lv.positions(shape, SHIFT)})
    else:
        ys = _rows([shape], 0, H)
        xs = _rows([shape], 1, W)
        units = [(y, x) for y in ys for x in xs]
    assert lv.straddles(shape, lv.covered(shape, units, axes), SHIFT)
    assert not lv.straddles(shape, lv.covered(shape, units[:1], axes), SHIFT), "one unit alone must not pass"


def test_stereo_join_rows(oracle):
    rng = np.random.default_rng(1)
    fL, fR = rng.standard_normal((2, 5, H, W)).astype(np.float32)
    wantL, wantR = oracle.stereo_join(fL, fR, D)
    for y in _rows([(D, H, W), (D, H, LD)], 1, H):
        L, R = lv.stereo_join_row(oracle, fL, fR, D, y)
        assert np.array_equal(L, wantL[:, y], equal_nan=True) and np.array_equal(R, wantR[:, y], equal_nan=True)


@pytest.mark.parametrize("kind,nch", [("census", 1), ("census", 3), ("ad", 1)])
@pytest.mark.parametrize("direction", [-1, 1])
def test_cost_rows(oracle, kind, nch, direction):
    """census / AD rows from a crop of +-4 image rows; rows 0 .. 3 and H - 4 .. H - 1 have the image border in the window"""
    a, b = dc.ad_census_images(dc.AdCensusCase(H, W, D, nch, True))
    if kind == "ad":
        a, b = a[0], b[0]
    whole = oracle.census(a, b, D, direction) if kind == "census" else oracle.ad(a, b, D, direction)
    for y in sorted(set(_rows([(D, H, W)], 1, H)) | {1, 3, 4, H - 5, H - 4, H - 2}):
        got = lv.cost_row(oracle, a, b, D, y, direction, kind)
        assert np.array_equal(got, whole[:, y], equal_nan=True), (kind, y)


@pytest.mark.parametrize("L", [2, 5, 9, 14, 15])
@pytest.mark.parametrize("direction", [-1, 1])
def test_cbca_crop_rows(oracle, L, direction):
    """exact CBCA: row y from the crop [y - halo, y + halo] (arms moved into the crop) equals row y of the whole volume,
    bit for bit; the float64 tap sums of the crop on a few planes agree with the whole volume's"""
    x0c, x1c, _, _ = dc.cbca_arms(dc.CbcaCase(H, W, D, L, direction, "ex", L, None, "cross"))
    vol = dc.cbca_volume("census3", H, W, D, direction)
    want = oracle.cbca(x0c, x1c, vol, direction)
    planes = [0, 17, D - 1]
    w64 = dc.cbca_f64(x0c, x1c, vol, direction, planes=planes)
    halo = L - 1
    for y in sorted(set(_rows([(D, H, W), (D, H, LD)], 1, H)) | {halo, H - 1 - halo}):
        got, g64 = lv.cbca_row(oracle, x0c, x1c, lambda a, b: vol[:, a:b], y, halo, direction, dc.cbca_f64, planes)
        assert np.array_equal(got, want[:, y], equal_nan=True), y
        assert np.allclose(g64[planes], w64[planes, y], rtol=1e-12, atol=1e-9, equal_nan=True), y
        assert np.isnan(g64[1]).all()


def test_cbca_crop_needs_the_halo(oracle):
    """a crop of the row alone changes it (cbca_image's vertical arms are short, its horizontal ones long): the crop's
    rows are what makes the reference right"""
    L, direction = 9, -1
    x0c, x1c, _, _ = dc.cbca_arms(dc.CbcaCase(H, W, D, L, direction, "ex", L, None, "cross"))
    vol = dc.cbca_volume("census3", H, W, D, direction)
    want = oracle.cbca(x0c, x1c, vol, direction)
    differs = [not np.array_equal(lv.cbca_row(oracle, x0c, x1c, lambda a, b: vol[:, a:b], y, 0, direction),
                                  want[:, y], equal_nan=True) for y in range(L, H - L)]
    assert any(differs)


@pytest.mark.parametrize("params", [dc.SGM_TIE, dc.SGM_TEN], ids=["tie", "ten"])
@pytest.mark.parametrize("direction", [-1, 1])
def test_sgm_crossings(oracle, params, direction):
    """the crossings of sampled rows and columns equal oracle.sgm2 (H <= W) there, bit for bit"""
    c = dc.SGMCase(H, W, D, 0, 0, params, dc.sgm_k(D), False)
    x0, x1, vol = dc.sgm_inputs(c, direction)
    want = oracle.sgm2(x0, x1, vol, *params, direction)
    shape = (H, W, D)
    ys, xs = _rows([shape], 0, H), _rows([shape], 1, W)
    got = lv.sgm_crossings(oracle, x0, x1, lambda y: vol[y], lambda x: vol[:, x], ys, xs, params, direction)
    assert len(got) == len(ys) * len(xs)
    for (y, x), v in got.items():
        w = want[y, x]
        assert np.array_equal(v, w, equal_nan=True), (y, x)
        z = w == 0
        assert np.array_equal(np.signbit(v[z]), np.signbit(w[z]))


def test_argmin_columns(oracle):
    rng = np.random.default_rng(2)
    vol = rng.integers(0, 3, (D, H, W)).astype(np.float32)
    vol[rng.random(vol.shape) < 0.3] = np.nan
    vol[:, 0, :4] = np.nan
    want = oracle.spatial_argmin(vol) - 1
    assert np.array_equal(lv.argmin_columns(vol.reshape(D, -1)), want.reshape(-1))


def test_fill_invalid_rows():
    got = np.full((D, H, W), 5.0, np.float32)
    d, x = np.arange(D)[:, None], np.arange(W)[None, :]
    wantL, wantR = lv.fill_invalid_rows(got[:, :3], W, 5.0)
    for y in range(3):
        assert np.array_equal(np.isnan(wantL[:, y]), x < d) and np.array_equal(np.isnan(wantR[:, y]), x >= W - d)
        assert (wantL[:, y][~(x < d)] == 5.0).all() and (wantR[:, y][~(x >= W - d)] == 5.0).all()
