"""CPU: the KITTI devkits' metrics as oracle/kitti_devkit.py states them, on hand-built maps with hand-computed results; the
rates, the printed table and the packing of a pair's counts between ranks (mccnn_b200/kitti_eval.py); the command line of
tools/kitti_eval.py and the refusals that come before any GPU work."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import kitti_eval as ke, synth  # noqa: E402
from oracle import kitti_devkit as kd  # noqa: E402

_ = None                                     # an invalid pixel in the hand-built maps


def v16(rows):
    """stored values of a map given as disparities (multiples of 1/256), None = invalid"""
    return np.array([[0 if d is None else int(round(d * 256)) for d in r] for r in rows], np.uint16)


def ipol(rows):
    d, _valid = kd.read_estimate(v16(rows))
    return kd.interpolate_background(d)


def f32(rows):
    return np.array([[-1 if d is None else d for d in r] for r in rows], np.float32)


# ---- interpolateBackground -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("row,want", [
    ([5, _, _, 3, _, 7], [5, 3, 3, 3, 3, 7]),               # interior runs: min of the two neighbours
    ([_, _, 4, _, 6, _], [4, 4, 4, 4, 6, 6]),               # runs touching either end: extrapolated
    ([_, 2.5, _], [2.5, 2.5, 2.5]),
    ([1, 2, 3], [1, 2, 3]),
    ([_, _, _, _], [-1, -1, -1, -1]),                       # no valid pixel: the row stays -1
    ([9, _, _, _, 1], [9, 1, 1, 1, 1]),
])
def test_rows(row, want):
    assert np.array_equal(ipol([row]), f32([want]))


def test_all_invalid_interior_row_stays_invalid():
    assert np.array_equal(ipol([[1, 2], [_, _], [3, 4]]), f32([[1, 2], [_, _], [3, 4]]))


def test_first_and_last_rows_are_extrapolated():
    assert np.array_equal(ipol([[_, _], [1, 2], [3, 4]]), f32([[1, 2], [1, 2], [3, 4]]))
    assert np.array_equal(ipol([[1, 2], [3, 4], [_, _]]), f32([[1, 2], [3, 4], [3, 4]]))
    # rows first: [1, _] -> [1, 1], [_, 2] -> [2, 2]; then columns: row 0 copies row 1, row 4 copies row 3, row 2 stays
    assert np.array_equal(ipol([[_, _], [1, _], [_, _], [_, 2], [_, _]]),
                          f32([[1, 1], [1, 1], [_, _], [2, 2], [2, 2]]))


def test_all_invalid_image_is_scored_against_minus_one():
    est = v16([[_, _, _], [_, _, _]])
    gt = v16([[1, 4, _], [_, 6.5, 0.5]])
    c, s, ip = kd.devkit_counts(est, gt, gt)
    assert np.array_equal(ip, np.full((2, 3), -1, np.float32))
    # e = 2, 5, 7.5, 1.5
    for r in range(2):
        assert c[r, kd.GT] == 4 and c[r, kd.DENSE] == 0
        assert (c[r, kd.OUT2], c[r, kd.OUT3], c[r, kd.OUT4], c[r, kd.OUT5]) == (2, 2, 2, 1)
        assert c[r, kd.D1_BG] == 2 and c[r, kd.D1_FG] == 0 and c[r, kd.GT_BG] == 4 and c[r, kd.GT_FG] == 0
        assert s[r] == 16.0


# ---- reading and quantising ------------------------------------------------------------------------------------------------

def test_png16_values_of_float_maps():
    d = np.array([[0, 1e-6, 0.003, 1 / 256, 2.5, 300, np.nan, np.inf, -1, 255.999]], np.float32)
    # 0, < 1e-5, below 1/256 (truncated to 0), exactly 1/256, a normal value, past the range (clamped), NaN, inf, < 0
    want = [[0, 0, 0, 1, 640, 65535, 0, 65535, 0, 65535]]
    with np.errstate(invalid="ignore"):
        assert np.array_equal(kd.png16_values(d), np.array(want, np.uint16))


def test_zero_and_sub_1_256_estimates_are_invalid_and_filled():
    with np.errstate(invalid="ignore"):
        est = kd.png16_values(np.array([[4, 0, 0.003, 8]], np.float32))
    gt = v16([[4, 4, 4, 4]])
    c, s, ip = kd.devkit_counts(est, gt, gt)
    assert np.array_equal(ip, f32([[4, 4, 4, 8]]))           # the run [1, 2] takes min(4, 8)
    assert c[0, kd.DENSE] == 2 and c[0, kd.GT] == 4 and s[0] == 4.0 and c[0, kd.OUT3] == 1


# ---- errors ----------------------------------------------------------------------------------------------------------------

def test_errors_exactly_at_the_thresholds_are_not_bad():
    # ground truth 10; e = 2, 3, 4, 5 and 5 + 1/256
    est = v16([[12, 13, 14, 15, 15 + 1 / 256]])
    gt = v16([[10] * 5])
    c, s, _ip = kd.devkit_counts(est, gt, gt)
    assert (c[0, kd.OUT2], c[0, kd.OUT3], c[0, kd.OUT4], c[0, kd.OUT5]) == (4, 3, 2, 1)
    assert c[0, kd.D1_BG] == 3                               # e > 3 and e / 10 > 0.05: e = 4, 5, 5 + 1/256
    assert s[0] == 2 + 3 + 4 + 5 + 5 + 1 / 256


def test_d1_quotient_exactly_0_05f_is_not_bad():
    # ground truth 80: e = 4 gives the fp32 quotient 0.05f exactly, which is not > 0.05f (it is > the double 0.05:
    # this case is the one where a double constant would count the pixel); e = 4 + 1/256 is bad
    assert np.float32(4) / np.float32(80) == np.float32(0.05) and float(np.float32(0.05)) > 0.05
    est = v16([[84, 76, 84 + 1 / 256, 84]])
    gt = v16([[80, 80, 80, 80]])
    obj = np.array([[0, 0, 0, 3]], np.uint8)
    c, _s, _ip = kd.devkit_counts(est, gt, gt, obj)
    assert c[0, kd.D1_BG] == 1 and c[0, kd.D1_FG] == 0
    assert c[0, kd.GT_BG] == 3 and c[0, kd.GT_FG] == 1


def test_d1_needs_both_conditions_and_splits_by_obj_map():
    # gt 100: e = 4 is 4 % (not bad); gt 20: e = 4 is 20 % (bad); gt 2: e = 2 is 100 % but not > 3 (not bad)
    est = v16([[104, 24, 4, 24, 30]])
    occ = v16([[100, 20, 2, 20, 20]])
    noc = v16([[100, 20, 2, _, _]])
    obj = np.array([[1, 1, 0, 0, 2]], np.uint8)
    c, s, _ip = kd.devkit_counts(est, noc, occ, obj)
    assert c[0, kd.GT] == 3 and c[0, kd.D1_FG] == 1 and c[0, kd.D1_BG] == 0
    assert c[1, kd.GT] == 5 and c[1, kd.D1_FG] == 2 and c[1, kd.D1_BG] == 1
    assert c[1, kd.GT_FG] == 3 and c[1, kd.GT_BG] == 2
    assert tuple(s) == (10.0, 24.0)


def test_density_counts_the_original_estimate():
    est = v16([[3, _, _, 3]])
    noc = v16([[3, 3, _, _]])
    occ = v16([[3, 3, 3, 3]])
    c, s, _ip = kd.devkit_counts(est, noc, occ)
    assert (c[0, kd.GT], c[0, kd.DENSE], c[1, kd.GT], c[1, kd.DENSE]) == (2, 1, 4, 2)
    assert tuple(s) == (0.0, 0.0)


# ---- tiny shapes ------------------------------------------------------------------------------------------------------------

def test_tiny_shapes():
    assert np.array_equal(ipol([[_]]), f32([[_]]))
    assert np.array_equal(ipol([[7]]), f32([[7]]))
    assert np.array_equal(ipol([[_, 2, _, _, 5, _]]), f32([[2, 2, 2, 2, 5, 5]]))
    col = ipol([[_], [2], [_], [5], [_]])
    assert np.array_equal(col, f32([[2], [2], [_], [5], [5]]))   # one pixel per row: no row fills, the middle row stays
    c, s, _ip = kd.devkit_counts(v16([[_]]), v16([[3]]), v16([[3]]))
    assert c[1, kd.GT] == 1 and c[1, kd.OUT3] == 1 and c[1, kd.DENSE] == 0 and s[1] == 4.0


# ---- rates, table, packing --------------------------------------------------------------------------------------------------

def test_rates_and_table():
    c = np.zeros((2, ke.NCOUNT), np.int64)
    c[:, ke.GT] = (8, 10)
    c[:, ke.DENSE] = (8, 5)
    c[:, ke.OUT2], c[:, ke.OUT3], c[:, ke.OUT4], c[:, ke.OUT5] = (4, 5), (2, 4), (1, 3), (0, 2)
    c[:, ke.D1_BG], c[:, ke.D1_FG], c[:, ke.GT_BG], c[:, ke.GT_FG] = (1, 2), (1, 1), (6, 6), (2, 4)
    s = np.array([6.0, 12.5])
    r = ke.rates(c, s, "kitti")
    assert list(r) == ke.columns("kitti")
    assert r["out_noc_2"] == 0.5 and r["out_all_5"] == 0.2 and r["avg_noc"] == 0.75 and r["avg_all"] == 1.25
    assert r["density"] == 0.5
    assert ke.table(r, "kitti") == ["Error\tOut-Noc\tOut-All\tAvg-Noc\tAvg-All", "2 px\t0.5\t0.5\t0.75\t1.25",
                                     "3 px\t0.25\t0.4\t0.75\t1.25", "4 px\t0.125\t0.3\t0.75\t1.25",
                                     "5 px\t0\t0.2\t0.75\t1.25", "Density\t0.5"]
    assert ke.pair_line(3, r).split("\t")[:3] == ["3", "0.5", "0.25"]
    r = ke.rates(c, s, "kitti2015")
    assert list(r) == ke.columns("kitti2015")
    assert ke.table(r, "kitti2015") == ["Error\tD1-bg\tD1-fg\tD1-all", "noc\t%.14g\t0.5\t0.25" % (1 / 6),
                                        "all\t%.14g\t0.25\t0.3" % (2 / 6), "Density\t0.5"]
    c[:] = 0
    assert all(np.isnan(v) for v in ke.rates(c, np.zeros(2), "kitti").values())


def test_pack_round_trip_keeps_every_bit():
    import torch

    rng = np.random.default_rng(1)
    counts = torch.from_numpy(rng.integers(0, 1 << 24, (2, ke.NCOUNT)))
    sums = torch.from_numpy(np.array([rng.random() * 1e6, np.pi], np.float64))
    t = ke._pack(ke.Counts(counts, sums))
    assert t.dtype == torch.float32
    c, s = ke._unpack(t.clone())
    assert np.array_equal(c, counts.numpy()) and s.tobytes() == sums.numpy().tobytes()


# ---- the command line and the refusals ------------------------------------------------------------------------------------

def _tool():
    import importlib

    return importlib.import_module("kitti_eval")


def test_parse_args(tmp_path):
    t = _tool()
    a = t.parse_args(["predict", "kitti2015", "-net_fname", "n.t7", "-data_root", "/d", "-gpu", "2", "-out", "o"])
    assert (a.action, a.dataset, a.net_fname, a.arch, a.data_root, a.disp_max, a.gpu, a.out) == \
        ("predict", "kitti2015", "n.t7", "fast", "/d", 228, 2, "o")
    a = t.parse_args(["predict", "kitti", "-arch", "census", "-disp_max", "96"])
    assert (a.arch, a.disp_max, a.out) == ("census", 96, None)
    a = t.parse_args(["score", "kitti", str(tmp_path), "-data_root", "/d"])
    assert (a.action, a.dataset, a.pred_dir, a.data_root, a.gpu) == ("score", "kitti", str(tmp_path), "/d", 1)


@pytest.mark.parametrize("argv,msg", [
    (["predict", "kitti"], "needs -net_fname"),
    (["predict", "kitti", "-arch", "slow"], "needs -net_fname"),
    (["predict", "kitti", "-arch", "census", "-disp_max", "0"], "-disp_max"),
    (["predict", "kitti", "-arch", "ad", "-gpu", "0"], "1-based"),
    (["score", "kitti", "/nonexistent/dir"], "not a directory"),
])
def test_parse_args_refusals(argv, msg):
    with pytest.raises(SystemExit, match=msg):
        _tool().parse_args(argv)


@pytest.mark.parametrize("argv", [["predict", "kitti2012", "-arch", "ad"], ["score", "kitti"], ["test", "kitti"], []])
def test_parse_args_usage_errors(argv, capsys):
    with pytest.raises(SystemExit) as e:
        _tool().parse_args(argv)
    assert e.value.code == 2
    capsys.readouterr()


@pytest.fixture
def raw(tmp_path):
    root = str(tmp_path / "data")
    for k, ds in enumerate(("kitti", "kitti2015")):
        unzip = synth.write_kitti_raw(root, ds, n_tr=2, n_te=1, H=20, widths=(90, 88), seed=k, D=16)
        assert synth.write_kitti_eval_maps(unzip, ds, seed=k) == 2
    return root


def _unzip(root, ds):
    return os.path.join(root, "data.kitti" if ds == "kitti" else "data.kitti2015", "unzip", "training")


def test_synthetic_eval_maps(raw):
    from mccnn_b200 import dataio

    for ds, noc, occ in (("kitti", "disp_noc", "disp_occ"), ("kitti2015", "disp_noc_0", "disp_occ_0")):
        files = ke.training_files(raw, ds)
        assert len(files) == 2 and (files[0][4] is None) == (ds == "kitti")
        for f in files:
            n, o = dataio.read_png16_raw(f[2]), dataio.read_png16_raw(f[3])
            assert f[3].endswith(os.path.join(occ, os.path.basename(f[2])))
            assert np.array_equal(o[n != 0], n[n != 0]) and (o != 0).sum() > (n != 0).sum()
        ke.check_maps([(None,) + f[2:] for f in files], [(20, 90), (20, 88)])


@pytest.mark.parametrize("ds,victim", [("kitti", "disp_occ"), ("kitti2015", "disp_occ_0"), ("kitti2015", "obj_map")])
def test_missing_ground_truth_is_refused(raw, ds, victim):
    os.remove(os.path.join(_unzip(raw, ds), victim, "000001_10.png"))
    with pytest.raises(FileNotFoundError, match=victim):
        ke.evaluate_training(ds, None, "census", data_root=raw)
    os.makedirs(str(raw) + "_pred")
    with pytest.raises(FileNotFoundError, match=victim):
        ke.score_dir(ds, str(raw) + "_pred", data_root=raw)


@pytest.mark.parametrize("ds,victim,kind", [("kitti", "disp_occ", "16"), ("kitti2015", "disp_occ_0", "16"),
                                            ("kitti2015", "obj_map", "8")])
def test_wrong_size_or_kind_is_refused(raw, ds, victim, kind):
    from PIL import Image

    p = os.path.join(_unzip(raw, ds), victim, "000001_10.png")
    a = np.zeros((20, 89), np.uint16 if kind == "16" else np.uint8)
    Image.fromarray(a).save(p)
    with pytest.raises(ValueError, match="is 20x89, the pair is 20x88"):
        ke.evaluate_training(ds, None, "census", data_root=raw)
    Image.fromarray(np.zeros((20, 88), np.uint8 if kind == "16" else np.uint16)).save(p)
    with pytest.raises(ValueError, match="8-bit PNG expected" if kind == "8" else "16-bit grey PNG expected"):
        ke.evaluate_training(ds, None, "census", data_root=raw)


def test_score_refuses_missing_and_mis_sized_estimates(raw, tmp_path):
    from mccnn_b200 import dataio

    pred = str(tmp_path / "pred")
    for i, W in enumerate((90, 88)):
        dataio.write_kitti_submission(np.ones((20, W), np.float32), 20, W, pred, i, "kitti2015")
    with pytest.raises(FileNotFoundError, match="missing estimate .*000000_10.png"):
        ke.score_dir("kitti", pred, data_root=raw)            # 2012 maps are not under disp_0/
    dataio.write_kitti_submission(np.ones((20, 91), np.float32), 20, 91, pred, 1, "kitti2015")
    with pytest.raises(ValueError, match="is 20x91, the pair is 20x88"):
        ke.score_dir("kitti2015", pred, data_root=raw)
    from PIL import Image

    Image.fromarray(np.ones((20, 88), np.uint8)).save(ke.submission_file(pred, "kitti2015", 1))
    with pytest.raises(ValueError, match="16-bit grey PNG expected"):
        ke.score_dir("kitti2015", pred, data_root=raw)


def test_predict_refuses_a_non_empty_out_and_bad_arguments(raw, tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    (out / "x").write_text("")
    with pytest.raises(ValueError, match="not empty"):
        ke.evaluate_training("kitti", None, "census", data_root=raw, out=str(out))
    with pytest.raises(ValueError, match="disp_max"):
        ke.evaluate_training("kitti", None, "census", data_root=raw, disp_max=0)
    with pytest.raises(ValueError, match="dataset"):
        ke.evaluate_training("mb", None, "census", data_root=raw)
    with pytest.raises(ValueError, match="dataset"):
        ke.score_dir("middlebury", str(out), data_root=raw)
