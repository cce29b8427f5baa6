"""CPU: Middlebury training (dataset mb) without a GPU -- the mb presets, the light / exposure draws against the
one-draw-at-a-time restatement (oracle/train_mb.py), chunked building, the loader's and the command line's refusals, and
the names and lines of main.lua for mb fast / slow."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, preprocess, train  # noqa: E402
from oracle import train as ot  # noqa: E402
from oracle import train_mb as otm  # noqa: E402


def test_mb_presets():
    f = train.options("mb", "fast")
    assert (f["m"], f["pow"], f["l1"], f["fm"], f["ks"], f["lr"], f["bs"], f["mom"]) == (0.2, 1, 5, 64, 3, 0.002, 128, 0.9)
    assert (f["true1"], f["false1"], f["false2"]) == (0.5, 1.5, 6.0)
    s = train.options("mb", "slow")
    assert (s["l1"], s["fm"], s["ks"], s["l2"], s["nh2"], s["lr"], s["bs"], s["mom"]) == (5, 112, 3, 3, 384, 0.003, 128, 0.9)
    assert (s["true1"], s["false1"], s["false2"]) == (0.5, 1.5, 18.0)
    assert "m" not in s and "pow" not in s and "at" not in s and "at" not in f
    for o in (f, s):                                                              # main.lua:50-66
        assert (o["rotate"], o["hscale"], o["scale"], o["trans"], o["hshear"], o["brightness"], o["contrast"]) == \
            (28, 0.8, 0.8, 0, 0.1, 1.3, 1.1)
        assert (o["d_vtrans"], o["d_rotate"], o["d_hscale"], o["d_hshear"], o["d_brightness"], o["d_contrast"]) == \
            (1, 3, 0.9, 0.3, 0.7, 1.1)
        assert (o["hflip"], o["vflip"], o["ds"], o["d_exp"], o["d_light"]) == (0, 0, 2001, 0.2, 0.2)
    assert train.options("mb", "fast", ds=2014, d_exp=0.5)["ds"] == 2014
    with pytest.raises(ValueError, match="-m is not a training option"):
        train.options("mb", "slow", m=0.3)
    with pytest.raises(ValueError, match="-d_exp is not a training option"):
        train.options("kitti", "fast", d_exp=0.3)
    k = train.options("kitti", "fast")                                            # KITTI unchanged
    assert (k["rotate"], k["l1"], k["fm"], k["false2"], k["at"]) == (7, 4, 64, 10, 0) and "ds" not in k


# per image (1-based): (light groups j >= 2, exposures in each) -- 1 and 3 lights, 1, 2 and 3 exposures
COUNTS = {1: (1, 1), 2: (3, 3), 3: (1, 2), 4: (3, 1), 5: (2, 3), 6: (3, 2)}


def _oracle_stream(g, o, imgs):
    return [otm.sample_params_mb(g, o, *COUNTS[int(i)]) for i in imgs]


def _assert_same(got, want):
    p, light, exp, light_, exp_ = got
    for i, (wp, wl, we, wl_, we_) in enumerate(want):
        assert (light[i], exp[i], light_[i], exp_[i]) == (wl, we, wl_, we_), i
        for k, v in wp.items():
            g = p[k]
            if isinstance(v, list):
                assert [g[0][i], g[1][i]] == v, (i, k)
            else:
                assert g[i] == v, (i, k)


@pytest.mark.parametrize("d_exp", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("d_light", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("flips", [0, 1])
def test_draws_equal_oracle(d_exp, d_light, flips):
    o = train.options("mb", "fast", d_exp=d_exp, d_light=d_light, hflip=flips, vflip=flips)
    rng = np.random.default_rng(int(10 * d_exp + 100 * d_light + flips))
    imgs = rng.integers(1, len(COUNTS) + 1, 300)
    nl = np.array([COUNTS[i][0] for i in imgs])
    ne = np.array([COUNTS[i][1] for i in imgs])
    s, g = train.Stream(11), preprocess.MT19937(11)
    got = train.draw_params_mb(s, o, nl, ne)
    want = _oracle_stream(g, o, imgs)
    _assert_same(got, want)
    assert s.raw(5).tolist() == [g.random() for _ in range(5)]              # the carried words come first
    light, exp, light_, exp_ = got[1:]
    assert (light >= 2).all() and (light <= nl + 1).all() and (exp >= 1).all() and (exp <= ne).all()
    assert (light_ >= 2).all() and (exp_ <= ne).all()
    if d_exp == 0:
        assert (exp_ == exp).all()
    if d_light == 0:
        assert (light_ == light).all()
    if d_light == 1:
        assert (light_ == np.maximum(2, light - 1)).all()


def test_chunked_equals_all_at_once():
    o = train.options("mb", "slow", hflip=1)
    rng = np.random.default_rng(4)
    imgs = rng.integers(1, len(COUNTS) + 1, 500)
    nl = np.array([COUNTS[i][0] for i in imgs])
    ne = np.array([COUNTS[i][1] for i in imgs])
    s = train.Stream(3)
    whole = train.draw_params_mb(s, o, nl, ne)
    after = s.raw(4)
    s = train.Stream(3)
    parts, a = [], 0
    for n in (1, 7, 64, 0, 128, 300):
        parts.append(train.draw_params_mb(s, o, nl[a:a + n], ne[a:a + n]))
        a += n
    assert a == 500
    for j in range(1, 5):
        assert np.array_equal(np.concatenate([p[j] for p in parts]), whole[j])
    for k, v in whole[0].items():
        cat = (lambda x: np.concatenate(x))
        if isinstance(v, tuple):
            assert np.array_equal(cat([p[0][k][0] for p in parts]), v[0]) and \
                np.array_equal(cat([p[0][k][1] for p in parts]), v[1])
        else:
            assert np.array_equal(cat([p[0][k] for p in parts]), v), k
    assert s.raw(4).tolist() == after.tolist()


def test_sample_starts_walk():
    base = 3
    raw = np.array([0, 0, 0, 1, 1, 0xFFFFFFFF, 1,               # test fails (d_exp 0.5): 7 words
                    0, 0, 0, 1, 1, 0, 9, 1,                     # test passes: 8 words
                    0, 0, 0, 1, 1, 0], np.uint32)              # incomplete: the test passes, 2 words missing
    starts, used = train.mb_sample_starts(raw, base, 0.5, 10)
    assert starts.tolist() == [0, 7] and used == 15
    starts, used = train.mb_sample_starts(raw, base, 0.5, 1)
    assert starts.tolist() == [0] and used == 7
    starts, used = train.mb_sample_starts(raw[:6], base, 0.5, 10)
    assert starts.tolist() == [] and used == 0


def _write_set(root, groups, rows_tr, rows_te=(), rect="imperfect", n_img=None):
    """a data.mb.<rect>_gray directory: groups {image: [(n_exp, H, W) per light j >= 2]}, nnz rows (img, y, x, d)"""
    d = os.path.join(str(root), "data.mb.%s_gray" % rect)
    os.makedirs(d)
    rng = np.random.default_rng(0)
    n_img = n_img or max(groups)
    meta = []
    for i in range(1, n_img + 1):
        shapes = groups.get(i, [(1, 12, 20)])
        H, W = shapes[0][1:]
        dataio.tofile(os.path.join(d, "x_%d_1.bin" % i), rng.standard_normal((2, 1, H, W)).astype(np.float32))
        for j, (ne, h, w) in enumerate(groups.get(i, []), 2):
            dataio.tofile(os.path.join(d, "x_%d_%d.bin" % (i, j)), rng.standard_normal((ne, 2, 1, h, w)).astype(np.float32))
        meta.append((H, W, 8))
    dataio.tofile(os.path.join(d, "meta.bin"), np.array(meta, np.int32))
    dataio.tofile(os.path.join(d, "nnz_tr.bin"), np.array(rows_tr, np.float32).reshape(-1, 4))
    dataio.tofile(os.path.join(d, "nnz_te.bin"), np.array(rows_te, np.float32).reshape(-1, 4))
    dataio.tofile(os.path.join(d, "te.bin"), np.array([1], np.int64))
    with open(os.path.join(d, "fname_submit.txt"), "w") as f:
        f.write("trainingH/Adirondack")
    return d


def _listing(root):
    return sorted(os.path.relpath(os.path.join(a, f), root) for a, _, fs in os.walk(root) for f in fs)


def test_loader_pairs_and_warps(tmp_path):
    groups = {1: [(3, 10, 17), (3, 10, 17)], 2: [(1, 6, 9)], 3: [(2, 8, 30), (2, 8, 30), (2, 8, 30)]}
    _write_set(tmp_path, groups, [(1, 2, 3, 1.5), (3, 1, 20, 4), (3, 5, 7, 2)], [(2, 1, 2, 1)], n_img=4)
    ts = train.MbTrainSet(str(tmp_path), "imperfect", "train_tr")
    assert len(ts.nnz) == 3 and ts.n_pairs == 2 * 3 + 3 * 2
    assert ts.nbytes == 4 * (2 * 3 * 2 * 10 * 17 + 3 * 2 * 2 * 8 * 30)
    assert (ts.n_light[1], ts.n_exp[1], ts.n_light[3], ts.n_exp[3]) == (2, 3, 3, 2)
    assert ts.pair_index(1, 2, 1) == 0 and ts.pair_index(1, 3, 3) == 5 and ts.pair_index(3, 2, 1) == 6
    assert ts.pair_index(3, 4, 2) == 11
    ta = train.MbTrainSet(str(tmp_path), "imperfect", "train_all")
    assert len(ta.nnz) == 4 and ta.n_pairs == ts.n_pairs + 1 and ta.pair_index(2, 2, 1) == 6
    ts.check_fits(ts.nbytes)
    # the warp records: the left patches name (img, light, exp) with view 0, the right (img, light_, exp_) with view 1
    o = train.options("mb", "fast", d_exp=0.5, d_light=0.5)
    rows = ts.nnz[[0, 1, 2, 1, 0, 2]]
    s, g = train.Stream(8), preprocess.MT19937(8)
    w = ts.warps(s, o, rows, 11).reshape(-1, 4)
    for i, r in enumerate(rows):
        img = int(r[0])
        p, light, exp, light_, exp_ = otm.sample_params_mb(g, o, int(ts.n_light[img]), int(ts.n_exp[img]))
        assert w["image"][i].tolist() == [ts.pair_index(img, light, exp), ts.pair_index(img, light_, exp_)] * 2
        assert w["view"][i].tolist() == [0, 1, 0, 1]
        want = ot.patch_matrix(11, float(r[1]), float(r[2]) - float(r[3]) + p["d_neg"], p["scale_"], p["phi_"],
                               p["trans_"], p["hshear_"])
        assert np.array_equal(w["m"][i, 3].view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("case,msg", [
    ("no_light", "no light group x_2_2.bin"),
    ("unequal", "unequal exposure counts"),
    ("missing_nnz", "missing data file"),
    ("missing_group_data", "missing data file"),
    ("outside", "outside 1 .. 2"),
    ("bad_group", "(n_exp, 2, 1, H, W)"),
])
def test_loader_refusals(case, msg, tmp_path):
    groups = {1: [(2, 10, 17)], 2: [(1, 6, 9)]}
    rows = [(1, 2, 3, 1.5), (2, 1, 2, 1)]
    if case == "no_light":
        groups = {1: [(2, 10, 17)]}
    elif case == "unequal":
        groups = {1: [(2, 10, 17), (3, 10, 17)], 2: [(1, 6, 9)]}
    elif case == "outside":
        rows = rows + [(3, 1, 1, 1)]
    d = _write_set(tmp_path, groups, rows, n_img=2)
    if case == "missing_nnz":
        os.remove(os.path.join(d, "nnz_tr.bin"))
    elif case == "missing_group_data":
        os.remove(os.path.join(d, "x_2_2.bin"))
    elif case == "bad_group":
        dataio.tofile(os.path.join(d, "x_2_2.bin"), np.zeros((1, 1, 6, 9), np.float32))
    before = _listing(tmp_path)
    with pytest.raises((ValueError, OSError), match=msg.replace("(", r"\(").replace(")", r"\)").replace(".", r"\.")):
        train.MbTrainSet(str(tmp_path), "imperfect", "train_tr")
    assert _listing(tmp_path) == before


def test_loader_refuses_a_set_that_does_not_fit(tmp_path):
    _write_set(tmp_path, {1: [(2, 10, 17)]}, [(1, 2, 3, 1.5)])
    ts = train.MbTrainSet(str(tmp_path), "imperfect", "train_tr")
    with pytest.raises(MemoryError, match="need %d bytes" % ts.nbytes):
        ts.check_fits(ts.nbytes - 1)


def test_train_all_needs_nnz_te(tmp_path):
    d = _write_set(tmp_path, {1: [(2, 10, 17)]}, [(1, 2, 3, 1.5)])
    os.remove(os.path.join(d, "nnz_te.bin"))
    train.MbTrainSet(str(tmp_path), "imperfect", "train_tr")
    with pytest.raises(FileNotFoundError, match="nnz_te"):
        train.MbTrainSet(str(tmp_path), "imperfect", "train_all")


def test_names_and_lines():
    f, s = train.options("mb", "fast"), train.options("mb", "slow")
    assert train.cmd_str("mb", ["-a", "train_tr"], "fast") == "mb_fast_-a_train_tr"
    assert train.net_path("R", "mb", ["-a", "train_all", "-rect", "perfect"], "slow") == \
        os.path.join("R", "net", "net_mb_slow_-a_train_all_-rect_perfect.t7")
    assert train.net_lines(f) == ["conv(in=1, out=64, k=3)", "cudnn.ReLU"] + \
        ["conv(in=64, out=64, k=3)", "cudnn.ReLU"] * 3 + ["conv(in=64, out=64, k=3)", "nn.Normalize2", "nn.StereoJoin1"]
    want = ["conv(in=1, out=112, k=3)", "cudnn.ReLU"] + ["conv(in=112, out=112, k=3)", "cudnn.ReLU"] * 4 + \
        ["nn.Reshape(128x224)", "nn.Linear(224 -> 384)", "cudnn.ReLU", "nn.Linear(384 -> 384)", "cudnn.ReLU",
         "nn.Linear(384 -> 384)", "cudnn.ReLU", "nn.Linear(384 -> 1)", "cudnn.Sigmoid"]
    assert train.net_lines(s) == want


def test_cli_parsing():
    import train_mb as tool

    args, o, stereo = tool.parse_args(["mb", "fast", "-a", "train_tr", "-rect", "perfect", "-d_exp", "0.5", "-ds", "2014",
                                       "-L1", "3", "-data_root", "R"])
    assert (args.dataset, args.arch, args.a, args.rect, args.data_root) == ("mb", "fast", "train_tr", "perfect", "R")
    assert o["d_exp"] == 0.5 and o["ds"] == 2014 and o["l1"] == 5 and o["fm"] == 64 and o["rotate"] == 28
    assert stereo == {"L1": 3}
    import train as ktool
    assert ktool.main_args(args.argv) == ["-a", "train_tr", "-rect", "perfect", "-d_exp", "0.5", "-ds", "2014", "-L1", "3"]
    args, o, _ = tool.parse_args(["mb", "slow", "-a", "train_all", "-l2", "2"])
    assert (args.rect, o["l2"], o["fm"], o["false2"]) == ("imperfect", 2, 112, 18.0)


@pytest.mark.parametrize("argv,msg", [
    (["kitti", "fast", "-a", "train_tr"], "Middlebury"),
    (["kitti2015", "slow", "-a", "train_tr"], "train_slow.py"),
    (["mb", "census", "-a", "train_tr"], "fast and slow"),
    (["mb", "fast", "-a", "train_tr", "-color", "rgb"], "3-plane first layer"),
    (["mb", "fast", "-a", "train_tr", "-subset", "0.5"], "-subset"),
    (["mb", "slow", "-a", "train_tr", "-debug"], "-debug"),
    (["mb", "slow", "-a", "train_tr", "-m", "0.3"], "-m is not a training option of arch slow"),
    (["mb", "slow", "-a", "train_tr", "-pow", "2"], "-pow is not a training option of arch slow"),
    (["mb", "fast", "-a", "train_tr", "-l2", "2"], "-l2 is not a training option of arch fast"),
    (["mb", "fast", "-a", "train_tr", "-nh2", "128"], "-nh2 is not a training option of arch fast"),
    (["mb", "fast", "-a", "test_te"], "not a training action"),
    (["mb", "fast", "-a", "train_tr", "-fm", "40"], "-fm 40"),
    (["mb", "fast", "-a", "train_tr", "-gpu", "0"], "1-based"),
    (["mb", "fast", "-a", "train_tr"], "missing data file"),
])
def test_cli_refusals_write_nothing(argv, msg, tmp_path):
    import train_mb as tool

    with pytest.raises(SystemExit) as e:
        tool.main(argv + ["-data_root", str(tmp_path)])
    assert msg in str(e.value)
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("case", ["no_light", "unequal"])
def test_cli_refuses_a_bad_set_writing_nothing(case, tmp_path, capsys):
    import train_mb as tool

    groups = {1: [(2, 10, 17)]} if case == "no_light" else {1: [(2, 10, 17), (1, 10, 17)], 2: [(1, 6, 9)]}
    _write_set(tmp_path, groups, [(1, 2, 3, 1.5), (2, 1, 2, 1)], n_img=2)
    before = _listing(tmp_path)
    with pytest.raises(SystemExit, match="no light group" if case == "no_light" else "unequal exposure"):
        tool.main(["mb", "fast", "-a", "train_tr", "-data_root", str(tmp_path)])
    assert _listing(tmp_path) == before
    assert capsys.readouterr().out == ""


def test_kitti_tools_still_refuse_mb(tmp_path):
    import train as tool
    import train_slow as tool_slow

    for t, arch in ((tool, "fast"), (tool_slow, "slow")):
        with pytest.raises(SystemExit) as e:
            t.main(["mb", arch, "-a", "train_tr", "-data_root", str(tmp_path)])
        assert "Middlebury" in str(e.value) and "train_mb.py" in str(e.value)
    assert os.listdir(tmp_path) == []
