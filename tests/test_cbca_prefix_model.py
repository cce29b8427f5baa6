"""CPU: design study for a tolerance-mode CBCA -- the prefix-sum formulation (constant work per pixel) must
reproduce the reference's tap-by-tap sums within rounding, with the error bounded by the tile size -- and an index-for-index
emulation of the kernel the default mode runs, cbca_ws_kernel, with the mistakes the GPU tests can see."""
import importlib.util
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import synth
from oracle import cbca_prefix_model as model


def _case(oracle, H, W, D, L1, tau1, seed):
    p = synth.make_pair(H, W, 8, D, seed=seed)
    volL, volR = oracle.stereo_join(p["featL"], p["featR"], D)
    return oracle.cross(p["imgL"], L1, tau1), oracle.cross(p["imgR"], L1, tau1), volL, volR


@pytest.mark.parametrize("L1,tau1", [(5, 0.13), (14, 0.02), (0, 0.0)])
@pytest.mark.parametrize("direction", [-1, 1])
def test_prefix_formulation_matches_the_tap_sums(oracle, L1, tau1, direction):
    x0c, x1c, volL, volR = _case(oracle, 40, 150, 12, L1, tau1, seed=L1 + 3)
    vol = volL if direction == -1 else volR
    want = oracle.cbca(x0c, x1c, vol, direction)
    got64 = model.cbca_prefix(x0c, x1c, vol, direction, dtype=np.float64)
    assert np.array_equal(np.isnan(got64), np.isnan(want))
    m = ~np.isnan(want)
    rel = np.abs(got64[m] - want[m]) / np.maximum(1.0, np.abs(want[m]))
    assert rel.max() < 2e-6                                   # same sums up to fp32 rounding of the reference itself
    got32 = model.cbca_prefix(x0c, x1c, vol, direction, dtype=np.float32, tile=(32, 128))
    rel32 = np.abs(got32[m] - want[m]) / np.maximum(1.0, np.abs(want[m]))
    assert rel32.max() < 1e-4 / 4                             # fp32 prefixes on 32x128 tiles: well inside the 1e-4 bar
    # the decision it feeds: arg-min over d (first minimum, NaN skipped) almost never changes
    am_w = np.nanargmin(np.where(np.isnan(want), np.inf, want), axis=0)
    am_g = np.nanargmin(np.where(np.isnan(got32), np.inf, got32), axis=0)
    assert (am_w != am_g).mean() < 5e-3


def test_error_grows_with_prefix_length(oracle):
    """why the kernel must keep prefixes tile-local: whole-row fp32 prefixes lose more digits"""
    x0c, x1c, volL, _ = _case(oracle, 24, 600, 6, 5, 0.13, seed=11)
    want = oracle.cbca(x0c, x1c, volL, -1)
    m = ~np.isnan(want)
    err = {}
    for tile in ((24, 64), (24, 600)):
        got = model.cbca_prefix(x0c, x1c, volL, -1, dtype=np.float32, tile=tile)
        err[tile] = (np.abs(got[m] - want[m]) / np.maximum(1.0, np.abs(want[m]))).max()
    assert err[(24, 64)] <= err[(24, 600)] * 1.5 + 1e-9 and err[(24, 600)] < 1e-4


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("dispatch_cases", os.path.join(ROOT, "tests", "dispatch_cases.py"))
dc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(dc)

# constant-work cases of tests/test_gpu_dispatch_edges.py that cbca_ws_kernel serves, small enough for the emulation
WS_CASES = [c for c in dc.CBCA_FAST_CASES if c.kernel in ("ws1", "ws4") and c.H > 1 and c.W > 1 and c.D * c.H * c.W < 400000]


def _ws_inputs(c):
    x0c, x1c, _, _ = dc.cbca_arms(dc.CbcaCase(c.H, c.W, c.D, c.L, c.direction, "ex", c.max_arm, None, "cross"))
    return x0c, x1c, dc.cbca_volume(c.kind, c.H, c.W, c.D, c.direction)


def _err(got, want):
    """(NaN pattern equal, max relative error over the finite entries of want)"""
    m = ~np.isnan(want)
    with np.errstate(invalid="ignore"):
        e = np.abs(got[m] - want[m]) / np.maximum(1.0, np.abs(want[m]))
    return np.array_equal(np.isnan(got), np.isnan(want)), float(np.nan_to_num(e, nan=np.inf).max()) if m.any() else 0.0


@pytest.mark.parametrize("c", WS_CASES, ids=dc.fast_id)
def test_ws_kernel_indexing_emulated(oracle, c):
    """cbca_ws_kernel's tile, chunk, scan and ring arithmetic, emulated index for index, against the reference's tap
    sums and the float64 tap sums: NaN pattern identical, inside the 1e-4 contract"""
    x0c, x1c, vol = _ws_inputs(c)
    got = model.emulate_ws(x0c, x1c, vol, c.direction, dc.CBCA_R[c.kernel])
    for want in (oracle.cbca(x0c, x1c, vol, c.direction), dc.cbca_f64(x0c, x1c, vol, c.direction)):
        nan_ok, err = _err(got, want)
        assert nan_ok and err <= 1e-4, err


MUTANT_CASES = [c for c in WS_CASES if c.kind in ("stereojoin", "census3", "offset_gradient")]


@pytest.mark.parametrize("c", MUTANT_CASES, ids=dc.fast_id)
def test_ws_kernel_mistakes_exceed_the_bar(c):
    """on the GPU cases' inputs, a run end one column off, U and Dn swapped, or the scrub predicate dropped each move
    the result past the 1e-4 bar (or change its NaN pattern), so the GPU test would see them.  Dropping the centring does
    NOT: on these volumes, the large-offset one included, the uncentred prefixes stay inside the bar too, so the
    centring is a margin the tests do not pin."""
    x0c, x1c, vol = _ws_inputs(c)
    want = dc.cbca_f64(x0c, x1c, vol, c.direction)
    R = dc.CBCA_R[c.kernel]
    for mutation in (dict(run_end=1), dict(swap_ud=True), dict(scrub_rule=False)):
        nan_ok, err = _err(model.emulate_ws(x0c, x1c, vol, c.direction, R, **mutation), want)
        assert not nan_ok or err > 1e-4, mutation
    assert _err(model.emulate_ws(x0c, x1c, vol, c.direction, R, centre=False), want) [1] <= 1e-4
