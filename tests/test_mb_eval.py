"""CPU: the MiddEval3 SDK's evaldisp metrics as oracle/mb_evaldisp.py states them, on hand-built maps with hand-computed
results; the reported values and lines of mccnn_b200/mb_eval.py; the PFM orientation of the files; the command line of
tools/mb_eval.py, the refusals that come before any GPU work, -alg and the -res paths."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, mb_eval as me, preprocess, synth  # noqa: E402
from oracle import mb_evaldisp as od  # noqa: E402

INF, NAN = np.inf, np.nan


def f32(rows):
    return np.array(rows, np.float32)


def run(disp, gt, mask=None, maxdisp=100):
    c, s, q = od.evaldisp(f32(disp), f32(gt), None if mask is None else np.array(mask, np.uint8), maxdisp)
    return c, s, q, od.metrics(c, s, q, np.asarray(gt).size)


def test_errors_exactly_on_the_thresholds_are_not_bad():
    # err = 0.5, 1, 2, 4 and 4.5
    c, s, q, m = run([[10.5, 11, 12, 14, 14.5]], [[10] * 5])
    for r in range(2):
        assert list(c[r]) == [5, 5, 4, 3, 2, 1, 0]
        assert tuple(s[r]) == (12.0, 41.5)
        assert list(q[r]) == [2, 4.5, 4.5, 4.5]                   # ranks 3, 5, 5, 5 of 5
    assert m["all"]["bad0.5"] == 0.8 and m["all"]["bad4"] == 0.2 and m["all"]["avgerr"] == 2.4
    assert m["all"]["rms"] == math.sqrt(41.5 / 5) and m["all"]["coverage"] == 1.0


def test_infinite_maps_invalid_and_minus_inf_clamped_to_0():
    # +inf: invalid; -inf: clamped to 0, err 2; 3: err 1
    c, s, q, m = run([[INF, -INF, 3]], [[2, 2, 2]])
    assert list(c[1]) == [3, 2, 2, 1, 0, 0, 1]
    assert tuple(s[1]) == (3.0, 5.0)
    assert list(q[1]) == [1, 2, 2, 2]                              # ranks 1, 2, 2, 2 of 2
    r = m["all"]
    assert (r["bad0.5"], r["bad1"], r["bad2"], r["bad4"], r["invalid"]) == (1.0, 2 / 3, 1 / 3, 1 / 3, 1 / 3)
    assert r["avgerr"] == 1.5 and r["rms"] == math.sqrt(2.5)


def test_nan_is_valid_never_bad_and_makes_the_sums_nan():
    c, s, q, m = run([[NAN, 1, 7]], [[1, 1, 1]])
    assert list(c[1]) == [3, 3, 1, 1, 1, 1, 0]                     # only err 6 is bad
    assert np.isnan(s[1]).all()
    assert q[1, 0] == 6 and np.isnan(q[1, 1:]).all()              # rank 2 of [0, 6, NaN] is 6; ranks 3 are NaN
    assert np.isnan(m["all"]["avgerr"]) and m["all"]["bad0.5"] == 1 / 3


def test_values_above_maxd_are_clamped():
    # maxdisp 5: d 7 -> 5 (err 0), 5 (err 0), 4 (err 1); a gt of 9 with d 20 -> 5 (err 4, not > 4)
    c, s, q, m = run([[7, 5, 4, 20]], [[5, 5, 5, 9]], maxdisp=5)
    assert list(c[1]) == [4, 4, 2, 1, 1, 0, 0]
    assert tuple(s[1]) == (5.0, 17.0)


def test_scale_2_lookup():
    # d = 2 * disp[y / 2][x / 2]: columns 0-1 give 2, columns 2-3 give 6; one unknown pixel
    gt = [[2, 2.5, 6, 9], [INF, 1, 6, 6]]
    c, s, q, m = run([[1, 3]], gt, maxdisp=10)
    # errs 0, 0.5, 0, 3 / -, 1, 0, 0
    assert list(c[1]) == [7, 7, 2, 1, 1, 0, 0]
    assert tuple(s[1]) == (4.5, 10.25)
    assert m["all"]["coverage"] == 7 / 8
    assert list(q[1]) == [0, 3, 3, 3]                             # ranks 4, 7, 7, 7 of 7: [0, 0, 0, 0, .5, 1, 3]


def test_scale_4_lookup_and_clamp():
    gt = np.full((4, 4), 10, np.float32)
    gt[3, 3] = 7
    c, s, q, m = run([[2.5]], gt, maxdisp=3)                     # d = 10 everywhere, maxd 12
    assert list(c[1]) == [16, 16, 1, 1, 1, 0, 0] and s[1, 0] == 3.0
    c, s, q, m = run([[2.5]], gt, maxdisp=2)                     # maxd 8: d = 8, errs 2 (15 pixels) and 1
    assert list(c[1]) == [16, 16, 16, 15, 0, 0, 0] and tuple(s[1]) == (31.0, 61.0)


def test_mask_bytes_0_128_255():
    # only 255 is non-occluded; 0 and 128 count in 'all' only
    c, s, q, m = run([[1, 3, 6]], [[1, 1, 1]], mask=[[0, 128, 255]])
    assert list(c[0]) == [1, 1, 1, 1, 1, 1, 0] and tuple(s[0]) == (5.0, 25.0) and list(q[0]) == [5] * 4
    assert list(c[1]) == [3, 3, 2, 2, 1, 1, 0] and tuple(s[1]) == (7.0, 29.0)
    assert m["nonocc"]["coverage"] == 1 / 3 and m["all"]["coverage"] == 1.0
    # an unknown pixel is in no region whatever its mask byte
    c, _s, _q, _m = run([[1, 3]], [[INF, 1]], mask=[[255, 255]])
    assert c[0, od.N] == 1 and c[1, od.N] == 1


def test_all_unknown_ground_truth_gives_nan_quotients():
    c, s, q, m = run([[1, 2], [3, 4]], [[INF, INF], [INF, INF]], mask=[[255, 255], [255, 255]])
    assert not c.any() and not s.any() and np.isnan(q).all()
    for r in ("nonocc", "all"):
        assert m[r]["coverage"] == 0.0
        assert all(np.isnan(v) for k, v in m[r].items() if k != "coverage")


def test_all_invalid_map():
    c, s, q, m = run([[INF, INF]], [[1, 2]])
    assert list(c[1]) == [2, 0, 0, 0, 0, 0, 2] and np.isnan(q).all()
    assert m["all"]["bad0.5"] == 1.0 and m["all"]["invalid"] == 1.0 and np.isnan(m["all"]["avgerr"])


@pytest.mark.parametrize("errs,want", [
    ([3.0], [3, 3, 3, 3]),                                      # n_valid 1: every rank is 1
    ([2.0, 1.0], [1, 2, 2, 2]),                                 # 2: ranks 1, 2, 2, 2
    ([3.0, 0.25, 2.0, 1.0], [1, 3, 3, 3]),                      # 4: ranks 2, 4, 4, 4
    ([4.0, 0.0, 3.0, 1.0, 2.0], [2, 4, 4, 4]),                  # 5: ranks 3, 5, 5, 5
    ([1.0] * 3 + [2.0] * 17, [2, 2, 2, 2]),                     # 20: ranks 10, 18, 19, 20 fall in a run of ties
])
def test_quantile_ranks(errs, want):
    n = len(errs)
    c, s, q, m = run([[10 + e for e in errs]], [[10] * n])
    assert list(q[1]) == want
    assert [m["all"]["A%d" % p] for p in od.PERCENT] == want


def test_size_rules():
    for disp, gt in (((2, 3), (6, 9)), ((2, 3), (4, 7)), ((2, 3), (3, 6)), ((2, 3), (16, 24))):
        with pytest.raises(ValueError, match="ratio must be 1, 2 or 4"):
            od.evaldisp(np.ones(disp, np.float32), np.ones(gt, np.float32), None, 10)
    with pytest.raises(ValueError, match="mask is"):
        od.evaldisp(np.ones((2, 3), np.float32), np.ones((2, 3), np.float32), np.ones((2, 4), np.uint8), 10)


def test_product_metrics_and_lines_equal_the_oracle():
    rng = np.random.default_rng(3)
    disp = rng.uniform(-2, 30, (6, 9)).astype(np.float32)
    disp[0, :3] = INF
    gt = rng.uniform(0, 60, (12, 18)).astype(np.float32)
    gt[rng.random(gt.shape) < 0.2] = INF
    mask = rng.choice(np.array([0, 128, 255], np.uint8), gt.shape)
    c, s, q = od.evaldisp(disp, gt, mask, 25)
    want = od.metrics(c, s, q, gt.size)
    got = me.metrics(c, s, q, gt.size)
    assert list(got) == me.columns() and len(got) == 24
    assert list(got.values()) == [want[r][n] for r in ("nonocc", "all") for n in me.NAMES]
    assert me.line("Adirondack", got) == "\t".join(["Adirondack"] + ["%.14g" % v for v in got.values()])
    mean = me.mean_row([got, me.metrics(c * 2, s * 2, q, gt.size)])
    assert mean["all_coverage"] == (want["all"]["coverage"] * 3) / 2
    assert (me.N, me.VALID, me.BAD05, me.BAD4, me.INVALID, me.NCOUNT) == (od.N, od.VALID, od.BAD05, od.BAD4, od.INVALID,
                                                                           od.NCOUNT)


def test_scratch_bytes_from_the_header():
    assert me.scratch_bytes() == 49152


# ---- PFM orientation ---------------------------------------------------------------------------------------------------------

def test_pfms_are_flipped_to_top_down_rows(tmp_path):
    """The map and the ground truth are stored bottom-up, the mask top-down: the score is right only with both PFMs
    flipped."""
    rng = np.random.default_rng(5)
    disp = (np.arange(4)[:, None] * 5 + rng.uniform(0, 2, (4, 6))).astype(np.float32)       # rows differ
    gt = (np.kron(disp, np.ones((2, 2), np.float32)) * 2).astype(np.float32)
    gt[:2] += 0.75                                                                              # the top rows are off
    mask = np.full(gt.shape, 255, np.uint8)
    mask[-3:] = 128                                                                             # the bottom rows occluded
    dataio.write_pfm(np.flipud(disp), str(tmp_path / "map.pfm"))
    dataio.write_pfm(np.flipud(gt), str(tmp_path / "gt.pfm"))
    from PIL import Image

    Image.fromarray(mask, "L").save(str(tmp_path / "mask.png"))
    assert np.array_equal(dataio.read_pfm(str(tmp_path / "gt.pfm"))[0], gt[-1])               # the file's first row
    want = od.evaldisp(disp, gt, mask, 64)
    assert want[0][1, od.BAD05] == 24 and want[0][0, od.N] == 5 * 12
    d, g = me._read_topdown(str(tmp_path / "map.pfm")), me._read_topdown(str(tmp_path / "gt.pfm"))
    m = preprocess._read_grey(str(tmp_path / "mask.png"))
    got = od.evaldisp(d, g, m, 64)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    for dd, gg in ((np.flipud(d), g), (d, np.flipud(g)), (np.flipud(d), np.flipud(g))):
        other = od.evaldisp(dd, gg, m, 64)
        assert not np.array_equal(other[0], want[0])


# ---- the command line ---------------------------------------------------------------------------------------------------------

def _tool():
    import importlib

    return importlib.import_module("mb_eval")


def test_parse_args(tmp_path):
    t = _tool()
    a = t.parse_args(["predict", "fast", "-net_fname", "n.t7", "-data_root", "/d", "-gpu", "2", "-out", "o"])
    assert (a.action, a.arch, a.net_fname, a.data_root, a.res, a.out, a.gpu) == ("predict", "fast", "n.t7", "/d", "F", "o", 2)
    a = t.parse_args(["predict", "census", "-res", "H"])
    assert (a.arch, a.res, a.out, a.gpu) == ("census", "H", None, 1)
    a = t.parse_args(["score", str(tmp_path), "-data_root", "/d", "-alg", "MC-CNN-fst", "-res", "H"])
    assert (a.action, a.out, a.data_root, a.alg, a.res, a.gpu) == ("score", str(tmp_path), "/d", "MC-CNN-fst", "H", 1)


@pytest.mark.parametrize("argv,msg", [
    (["predict", "fast"], "needs -net_fname"),
    (["predict", "slow", "-data_root", "/d"], "needs -net_fname"),
    (["predict", "ad", "-gpu", "0"], "1-based"),
    (["score", "/nonexistent/dir"], "not a directory"),
])
def test_parse_args_refusals(argv, msg):
    with pytest.raises(SystemExit, match=msg):
        _tool().parse_args(argv)


@pytest.mark.parametrize("argv", [["predict", "accurate"], ["predict", "census", "-res", "Q"], ["score"], ["test"], []])
def test_parse_args_usage_errors(argv, capsys):
    with pytest.raises(SystemExit) as e:
        _tool().parse_args(argv)
    assert e.value.code == 2
    capsys.readouterr()


# ---- files and refusals -----------------------------------------------------------------------------------------------------

@pytest.fixture
def raw(tmp_path):
    root = str(tmp_path / "data")
    unzip = synth.write_mb_raw(root, n2014=0, half_size=(12, 20), D=16)
    assert synth.write_mb_eval_gt(unzip, seed=1) == 15
    return root


def _scene(root, sub, s="Adirondack"):
    return os.path.join(root, preprocess.MB_EVAL, sub, s)


def _submit_layout(root, out, names=("disp0MC-CNN-fst.pfm",), size=(12, 20)):
    for s in me.training_scenes(root):
        os.makedirs(os.path.join(out, "trainingH", s), exist_ok=True)
        for n in names:
            dataio.write_pfm(np.ones(size, np.float32), os.path.join(out, "trainingH", s, n))


def test_synthetic_ground_truth(raw):
    scenes = me.training_scenes(raw)
    assert scenes == sorted(synth.MB_SUBMIT_NAMES)
    for s in scenes:
        for sub, size in (("trainingH", (12, 20)), ("trainingF", (24, 40))):
            gt = me._read_topdown(os.path.join(_scene(raw, sub, s), "disp0GT.pfm"))
            mask = preprocess._read_grey(os.path.join(_scene(raw, sub, s), "mask0nocc.png"))
            assert gt.shape == mask.shape == size
            assert np.isinf(gt).any() and np.isfinite(gt).any()
            assert set(np.unique(mask).tolist()) == {0, 128, 255}
            assert np.array_equal(mask == 0, np.isinf(gt))
            assert me.check_scene((12, 20), *me.gt_files(raw, s, sub[-1])) == size


def test_res_paths(raw):
    gt, mask = me.gt_files(raw, "Piano", "H")
    assert gt == os.path.join(_scene(raw, "trainingH", "Piano"), "disp0GT.pfm")
    assert mask == os.path.join(_scene(raw, "trainingH", "Piano"), "mask0nocc.png")
    gt, mask = me.gt_files(raw, "Piano", "F")
    assert gt == os.path.join(_scene(raw, "trainingF", "Piano"), "disp0GT.pfm")
    assert mask == os.path.join(_scene(raw, "trainingF", "Piano"), "mask0nocc.png")
    with pytest.raises(ValueError, match="res must be"):
        me.gt_files(raw, "Piano", "Q")
    with pytest.raises(ValueError, match="res must be"):
        me.score_dir(raw, data_root=raw, res="Q")


def test_alg_selection(raw, tmp_path):
    out = str(tmp_path / "out")
    _submit_layout(raw, out)
    d = os.path.join(out, "trainingH", "Piano")
    assert me.find_map(out, "Piano") == os.path.join(d, "disp0MC-CNN-fst.pfm")
    dataio.write_pfm(np.ones((12, 20), np.float32), os.path.join(d, "disp0MC-CNN-acrt.pfm"))
    with pytest.raises(ValueError, match="disp0MC-CNN-acrt.pfm, disp0MC-CNN-fst.pfm: name the method with -alg"):
        me.find_map(out, "Piano")
    with pytest.raises(ValueError, match="name the method with -alg"):
        me.score_dir(out, data_root=raw)
    assert me.find_map(out, "Piano", "MC-CNN-acrt") == os.path.join(d, "disp0MC-CNN-acrt.pfm")
    with pytest.raises(FileNotFoundError, match="missing map .*disp0SGM.pfm"):
        me.find_map(out, "Piano", "SGM")


@pytest.mark.parametrize("victim", ["disp0GT.pfm", "mask0nocc.png"])
@pytest.mark.parametrize("res", ["F", "H"])
def test_missing_ground_truth_is_refused(raw, tmp_path, victim, res):
    os.remove(os.path.join(_scene(raw, "training" + res), victim))
    with pytest.raises(FileNotFoundError, match=victim):
        me.evaluate_training("census", data_root=raw, res=res)
    out = str(tmp_path / "out")
    _submit_layout(raw, out)
    with pytest.raises(FileNotFoundError, match=victim):
        me.score_dir(out, data_root=raw, res=res)


def test_missing_calib_and_map_are_refused(raw, tmp_path):
    out = str(tmp_path / "out")
    _submit_layout(raw, out)
    os.remove(os.path.join(out, "trainingH", "Pipes", "disp0MC-CNN-fst.pfm"))
    with pytest.raises(FileNotFoundError, match="missing map .*Pipes"):
        me.score_dir(out, data_root=raw)
    os.remove(os.path.join(_scene(raw, "trainingH", "Jadeplant"), "calib.txt"))
    with pytest.raises(FileNotFoundError, match="Jadeplant.*calib.txt"):
        me.evaluate_training("census", data_root=raw)
    with pytest.raises(FileNotFoundError, match="Jadeplant.*calib.txt"):
        me.score_dir(out, data_root=raw)


def test_files_of_the_wrong_kind_are_refused(raw, tmp_path):
    from PIL import Image

    out = str(tmp_path / "out")
    _submit_layout(raw, out)
    p = os.path.join(out, "trainingH", "Teddy", "disp0MC-CNN-fst.pfm")
    with open(p, "wb") as f:                                     # a three-channel PFM
        f.write(b"PF\n20 12\n-1\n" + np.zeros(12 * 20 * 3, "<f4").tobytes())
    with pytest.raises(ValueError, match="Teddy.*single-channel PFM"):
        me.score_dir(out, data_root=raw)
    gt = os.path.join(_scene(raw, "trainingF", "Teddy"), "disp0GT.pfm")
    with open(gt, "wb") as f:
        f.write(b"PF\n40 24\n-1\n" + np.zeros(24 * 40 * 3, "<f4").tobytes())
    with pytest.raises(ValueError, match="Teddy.*disp0GT.pfm.*single-channel PFM"):
        me.evaluate_training("census", data_root=raw)
    mask = os.path.join(_scene(raw, "trainingH", "Vintage"), "mask0nocc.png")
    Image.fromarray(np.zeros((12, 20, 3), np.uint8)).save(mask)
    with pytest.raises(ValueError, match="Vintage.*mask0nocc.png.*8-bit grey"):
        me.evaluate_training("census", data_root=raw, res="H")
    Image.fromarray(np.zeros((12, 20), np.uint16)).save(mask)
    with pytest.raises(ValueError, match="Vintage.*mask0nocc.png.*8-bit grey"):
        me.evaluate_training("census", data_root=raw, res="H")


@pytest.mark.parametrize("size,msg", [((36, 60), "ratio must be 1, 2 or 4"), ((24, 41), "ratio must be 1, 2 or 4"),
                                      ((25, 40), "ratio must be 1, 2 or 4"), ((96, 160), "ratio must be 1, 2 or 4")])
def test_size_ratios_are_refused(raw, tmp_path, size, msg):
    from PIL import Image

    d = _scene(raw, "trainingF", "Shelves")
    dataio.write_pfm(np.ones(size, np.float32), os.path.join(d, "disp0GT.pfm"))
    Image.fromarray(np.full(size, 255, np.uint8), "L").save(os.path.join(d, "mask0nocc.png"))
    with pytest.raises(ValueError, match="Shelves.*" + msg):
        me.evaluate_training("census", data_root=raw)
    out = str(tmp_path / "out")
    _submit_layout(raw, out)
    with pytest.raises(ValueError, match="Shelves.*" + msg):
        me.score_dir(out, data_root=raw)


def test_scale_4_is_accepted_and_a_mask_of_another_size_refused(raw):
    from PIL import Image

    d = _scene(raw, "trainingF", "Shelves")
    dataio.write_pfm(np.ones((48, 80), np.float32), os.path.join(d, "disp0GT.pfm"))
    Image.fromarray(np.full((48, 80), 255, np.uint8), "L").save(os.path.join(d, "mask0nocc.png"))
    assert me.check_scene((12, 20), *me.gt_files(raw, "Shelves")) == (48, 80)
    Image.fromarray(np.full((24, 40), 255, np.uint8), "L").save(os.path.join(d, "mask0nocc.png"))
    with pytest.raises(ValueError, match="mask0nocc.png is 24x40, the ground truth 48x80"):
        me.evaluate_training("census", data_root=raw)


def test_predict_refuses_a_non_empty_out(raw, tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    (out / "x").write_text("")
    with pytest.raises(ValueError, match="not empty"):
        me.evaluate_training("census", data_root=raw, out=str(out))
