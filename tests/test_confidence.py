"""CPU: the numpy restatement of the margin confidence, sparsify and the sparsification curve (tests/confidence_oracle.py)
against brute force, the host half of mc-cnn_b200/confidence.py (curve and AUCs from the counts), and the command-line
refusals of -confidence, -density and tools/sparsification.py, which must come before any GPU work and write nothing."""
import importlib.util
import math
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import confidence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


oc = _load("confidence_oracle", "tests", "confidence_oracle.py")


def _brute_margin(vol):
    D, H, W = vol.shape
    disp = np.zeros((H, W), np.float32)
    conf = np.zeros((H, W), np.float32)
    for y in range(H):
        for x in range(W):
            disp[y, x], conf[y, x] = oc.margin_at(vol[:, y, x])
    return disp, conf


def _hard_volume(rng, D, H, W):
    """costs on a coarse grid (many exact ties), NaN triangles as the fill leaves them, all-NaN pixels, +inf entries"""
    vol = rng.integers(0, 6, (D, H, W)).astype(np.float32) / 4
    for d in range(D):
        vol[d, :, :min(d, W)] = np.nan                  # the left volume's x < d
    vol[:, 0, 0] = np.nan                               # nothing taken
    vol[rng.random((D, H, W)) < 0.1] = np.inf
    vol[rng.random((D, H, W)) < 0.05] = np.nan
    return vol


@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 9, 17])
def test_margin_oracle_equals_brute_force(D):
    rng = np.random.default_rng(D)
    vol = _hard_volume(rng, D, 7, 13)
    got, want = oc.margin(vol), _brute_margin(vol)
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(got[1], want[1])
    assert (got[1] >= 0).all()
    if D <= 2:                                          # no d at distance 2 from the winner
        assert (got[1] == 0).all()


def test_margin_band_and_ties():
    inf, nan = np.inf, np.nan
    cases = [  # (curve, d1, conf)
        ([3, 1, 1, 2, 5], 1, 1),          # tie at d1 + 1: first minimum wins, its twin is inside the band
        ([1, 0.5, 0.5, 0.5, 2], 1, 0),    # the tie at d1 + 2 is outside the band: margin 0
        ([nan, nan, nan], 0, 0),          # nothing taken
        ([inf, 2, inf, inf], 1, 0),       # +inf is never taken
        ([2, nan, 1, nan, 4], 2, 1),      # NaN skipped; c2 = d 0
        ([5, 4, 3], 2, 2),                # D = 3: only d 0 is outside the band
        ([7], 0, 0),
    ]
    for curve, d1, conf in cases:
        vol = np.asarray(curve, np.float32)[:, None, None]
        disp, c = oc.margin(vol)
        assert disp[0, 0] == d1 and c[0, 0] == np.float32(conf), curve
        assert oc.margin_at(curve) == (float(d1), np.float32(conf))


def _brute_sparsify(disp, conf, n_keep, invalid):
    flat = conf.ravel()
    idx = sorted(range(flat.size), key=lambda i: (-float(flat[i]), i))[:n_keep]
    out = np.full(flat.size, invalid, np.float32)
    out[idx] = disp.ravel()[idx]
    return out.reshape(disp.shape)


@pytest.mark.parametrize("density", [1e-9, 0.1, 0.5, 0.73, 1.0])
def test_sparsify_oracle_rounding_and_ties(density):
    rng = np.random.default_rng(int(density * 1000))
    H, W = 9, 11
    disp = rng.random((H, W)).astype(np.float32) * 50
    conf = (rng.integers(0, 4, (H, W)) / 2).astype(np.float32)     # many ties
    n = confidence.n_keep(density, H, W)
    assert n == math.ceil(density * H * W) and 1 <= n <= H * W
    for invalid in (0.0, np.inf, np.nan):
        got = oc.sparsify(disp, conf, n, invalid)
        assert np.array_equal(got, _brute_sparsify(disp, conf, n, invalid), equal_nan=True)
        kept = ~np.isnan(got) if np.isnan(invalid) else got != invalid
        assert kept.sum() == n


def test_order_key_orders_like_the_values():
    v = np.array([-np.inf, -2.5, -0.0, 0.0, 1e-30, 1.0, 3.0, np.inf], np.float32)
    k = oc.order_key(v)
    assert (np.diff(k.astype(np.int64)) > 0).all()


def _brute_curve(pred, conf, gt, err_at):
    idx = [i for i in range(gt.size) if gt.ravel()[i] != 0]
    idx.sort(key=lambda i: (-float(conf.ravel()[i]), i))
    bad = [abs(float(np.float32(gt.ravel()[i]) - np.float32(pred.ravel()[i]))) > err_at for i in idx]
    M, B = len(idx), sum(bad)
    if M == 0:
        return None
    e = []
    for k in range(1, 21):
        n = math.ceil(k * M / 20)
        e.append(sum(bad[:n]) / n)
    return M, B, e


@pytest.mark.parametrize("case", ["random", "no_bad", "all_bad", "no_gt", "one_gt"])
def test_curve_auc_and_the_optimum(case):
    rng = np.random.default_rng(len(case))
    H, W = 13, 17
    gt = (rng.random((H, W)) * 40 + 1).astype(np.float32)
    gt[rng.random((H, W)) < 0.3] = 0
    pred = gt + (rng.random((H, W)) * 8 - 4).astype(np.float32)
    conf = (rng.integers(0, 5, (H, W)) / 3).astype(np.float32)
    if case == "no_bad":
        pred = gt.copy()
    elif case == "all_bad":
        pred = gt + 10
    elif case == "no_gt":
        gt[:] = 0
    elif case == "one_gt":
        gt[:] = 0
        gt[3, 4] = 7
    M, B, bad = oc.counts(pred, conf, gt, 3.0)
    curve, auc, auc_opt = confidence.curve_of_counts(M, B, bad)
    assert (curve, auc, auc_opt) == tuple(oc.curve(M, B, bad)) or M == 0
    brute = _brute_curve(pred, conf, gt, 3.0)
    if case == "no_gt":
        assert M == 0 and brute is None
        assert all(math.isnan(v) for v in curve) and math.isnan(auc) and math.isnan(auc_opt)
        return
    assert (M, B) == brute[:2] and curve == brute[2]
    assert curve[-1] == B / M                                          # main.lua's err
    assert auc_opt <= auc + 1e-15
    if case == "no_bad":
        assert B == 0 and auc == 0 and auc_opt == 0
    if case == "all_bad":
        assert B == M and auc == auc_opt == pytest.approx(0.95, abs=1e-12)
    opt = [max(0, math.ceil(k * M / 20) - (M - B)) / math.ceil(k * M / 20) for k in range(1, 21)]
    assert auc_opt == sum(0.05 * (opt[k] + opt[k + 1]) / 2 for k in range(19))


def test_n_points_is_exact_integer_ceil():
    for M in (1, 3, 19, 20, 21, 465750, 2 ** 33 + 7):
        assert confidence.n_points(M) == [-(-k * M // 20) for k in range(1, 21)]
    assert confidence.n_points(20) == list(range(1, 21))


@pytest.mark.parametrize("bad", [0, -0.1, 1.0000001, 2, float("nan"), "0.5", None])
def test_density_outside_the_unit_interval_is_refused(bad):
    with pytest.raises(ValueError, match="density"):
        confidence.n_keep(bad, 10, 10)


# ---- command lines: refused before any GPU work, nothing written ----

def _refused(tmp_path, monkeypatch, mod, argv, match):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(SystemExit) as e:
        mod.main(argv)
    assert match in str(e.value)
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("action", ["test_te", "test_all", "submit", "time"])
def test_run_main_confidence_needs_predict(tmp_path, monkeypatch, action):
    rm = _load("run_main", "tools", "run_main.py")
    _refused(tmp_path, monkeypatch, rm, ["kitti", "census", "-a", action, "-confidence"], "-confidence")


def test_run_main_confidence_parses():
    rm = _load("run_main", "tools", "run_main.py")
    args, _ = rm.parse_args(["kitti", "census", "-a", "predict", "-left", "l", "-right", "r", "-disp_max", "8", "-confidence"])
    assert args.confidence is True
    args, _ = rm.parse_args(["kitti", "census", "-a", "predict"])
    assert args.confidence is False


def test_sparsification_cli(tmp_path, monkeypatch):
    sp = _load("sparsification", "tools", "sparsification.py")
    _refused(tmp_path, monkeypatch, sp, ["mb", "census", "-a", "test_all"], "test_all not supported on Middlebury")
    _refused(tmp_path, monkeypatch, sp, ["kitti", "census", "-gpu", "0"], "1-based")
    _refused(tmp_path, monkeypatch, sp, ["kitti", "census", "-err_at", "-1"], "-err_at")
    with pytest.raises(SystemExit):                                     # argparse: not an action
        sp.parse_args(["kitti", "census", "-a", "submit"])
    with pytest.raises(ValueError, match="cbca1"):                      # a step that does no work in kitti fast
        sp.parse_args(["kitti", "fast", "-sm_terminate", "cbca1"])
    args, over = sp.parse_args(["kitti2015", "census", "-a", "test_all", "-err_at", "2", "-pi1", "3", "-gpu", "2"])
    assert (args.a, args.err_at, args.device, over) == ("test_all", 2.0, 1, {"pi1": 3.0})


@pytest.mark.parametrize("tool,argv,match", [
    ("predict_kitti", ["test", "kitti", "-arch", "census", "-density", "0.5"], "test writes none"),
    ("predict_kitti", ["submit", "kitti", "-arch", "census", "-density", "0"], "(0, 1]"),
    ("predict_kitti", ["submit", "kitti", "-arch", "census", "-density", "1.5"], "(0, 1]"),
    ("kitti_eval", ["predict", "kitti", "-arch", "census", "-density", "-0.5"], "(0, 1]"),
    ("kitti_eval", ["predict", "kitti", "-arch", "census", "-density", "nan"], "(0, 1]"),
    ("mb_eval", ["predict", "census", "-density", "2"], "(0, 1]"),
    ("mb_eval", ["predict", "census", "-density", "0"], "(0, 1]"),
])
def test_density_refusals(tmp_path, monkeypatch, tool, argv, match):
    _refused(tmp_path, monkeypatch, _load(tool + "_tool", "tools", tool + ".py"), argv, match)


def test_density_arguments_reach_the_library():
    import mccnn_b200.predict_kitti as pk

    with pytest.raises(ValueError, match="test writes none"):
        pk.predict_kitti("test", "kitti", arch="census", data_root="/nonexistent", density=0.5)
    for tool, argv in (("predict_kitti", ["submit", "kitti", "-arch", "census", "-density", "1"]),
                       ("kitti_eval", ["predict", "kitti", "-arch", "census", "-density", "0.25"]),
                       ("mb_eval", ["predict", "census", "-density", "0.8"])):
        args = _load(tool + "_tool", "tools", tool + ".py").parse_args(argv)
        assert args.density == float(argv[-1])
