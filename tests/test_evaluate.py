"""CPU: the data side of main.lua's -a test_te / test_all / submit / time (mccnn_b200/evaluate.py) on sets written by
synth.write_*_set -- loading, example lists, refusals, the net-derived fix_border width, the zip -- and the command line
of tools/run_main.py.  The GPU side is tests/test_gpu_evaluate.py."""
import importlib.util
import os
import zipfile

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, evaluate, frontend, synth, t7
from oracle import feature_tower as oft

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_main():
    spec = importlib.util.spec_from_file_location("run_main", os.path.join(ROOT, "tools", "run_main.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("data"))
    synth.write_kitti_set(root, "kitti", n_tr=5, n_te=3, H=24, width=70, widths=(70, 61, 66), seed=1)
    synth.write_kitti_set(root, "kitti2015", n_tr=4, n_te=2, H=20, width=50, widths=(50, 47), seed=2)
    synth.write_mb_set(root, n=6, shapes=((20, 40, 12), (24, 50, 16)), seed=3)
    return root


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015"])
def test_kitti_layout_and_examples(sets, dataset):
    d = evaluate.load_data(dataset, sets)
    n = len(d.X0)
    assert d.n_te == n - len(d.dispnoc) and d.n_te > 0
    te, tr = dataio.fromfile(os.path.join(sets, "data." + ("kitti" if dataset == "kitti" else "kitti2015"), "te.bin")), d.tr
    assert te.dtype == np.int64 and d.metadata.dtype == np.int32 and d.metadata.shape == (n, 3)
    assert d.examples("test_te") == [int(i) - 1 for i in te]                                   # 1-based on disk
    assert d.examples("test_all") == [int(i) - 1 for i in tr] + [int(i) - 1 for i in te]       # tr, then te
    assert sorted(d.examples("test_all")) == list(range(len(d.dispnoc)))
    assert d.examples("submit") == list(range(n - d.n_te, n))                                  # the last n_te rows
    for i in range(n):
        x, disp_max, id_, img_height, img_width = d.example(i)
        assert disp_max == 228 and img_width == d.metadata[i, 1] and id_ == d.metadata[i, 2]
        assert x.shape == (2, 1, d.height, img_width) and x.flags.c_contiguous
        assert np.array_equal(x[0, 0], d.X0[i, 0, :, :img_width]) and np.array_equal(x[1, 0], d.X1[i, 0, :, :img_width])
        if i < len(d.dispnoc):
            gt = d.ground_truth(i, img_width)
            assert gt.shape == (d.height, img_width) and (gt == 0).any() and (gt > 0).any()


def test_kitti_widths_include_an_odd_one(sets):
    d = evaluate.load_data("kitti", sets)
    ws = set(int(w) for w in d.metadata[:, 1])
    assert ws == {70, 61, 66} and any(w % 2 for w in ws)
    assert d.shape_of(1) == (24, 61, 228)


def test_mb_layout_and_examples(sets):
    d = evaluate.load_data("mb", sets)
    te = [int(i) for i in d.te]
    assert d.examples("test_te") == [(i - 1, 2) for i in te] + [(4, 3), (4, 4)]
    assert d.examples("submit") == [(i, 2) for i in range(6)]                                  # fewer than 30 images
    x, disp_max, id_, H, W = d.example((4, 4))
    assert id_ == "5_4" and disp_max == d.metadata[4, 2] and x.shape == (2, 1, H, W)
    assert np.array_equal(x[1], d.X[4][3]) and d.X[4].shape[0] >= 4
    x, disp_max, id_, H, W = d.example((1, 2))
    assert (H, W, disp_max) == (24, 50, 16) and id_ == "2_2"
    assert d.ground_truth((1, 2)).shape == (24, 50)
    assert len(d.fname_submit) == 6


def test_mb_submit_takes_the_last_30(tmp_path):
    synth.write_mb_set(str(tmp_path), n=33, shapes=((8, 16, 4),), seed=0)
    d = evaluate.load_data("mb", str(tmp_path))
    assert d.examples("submit") == [(i, 2) for i in range(3, 33)]
    assert len(d.fname_submit) == 30


def test_refusals(sets, tmp_path):
    d = evaluate.load_data("mb", sets)
    with pytest.raises(ValueError, match="test_all not supported on Middlebury"):
        d.examples("test_all")
    with pytest.raises(ValueError, match="-at 1"):
        evaluate.check_options("kitti", at=1)
    with pytest.raises(ValueError, match="-color rgb"):
        evaluate.load_data("mb", sets, color="rgb")
    for opt in ("debug", "use_cache", "make_cache"):
        with pytest.raises(ValueError, match="-" + opt):
            evaluate.check_options("kitti", **{opt: True})
    with pytest.raises(ValueError, match="-sm_skip"):
        evaluate.check_options("kitti", sm_skip="sgm")
    # a missing file: the error names the path
    with pytest.raises(FileNotFoundError, match=os.path.join(str(tmp_path), "data.kitti", "x0.bin")):
        evaluate.load_data("kitti", str(tmp_path))
    # disp_max < 1 names the example
    root = str(tmp_path / "neg")
    dd = synth.write_mb_set(root, n=5, shapes=((8, 16, 4),), seed=0)
    meta = dataio.fromfile(os.path.join(dd, "meta.bin"))
    meta[2, 2] = -1
    dataio.tofile(os.path.join(dd, "meta.bin"), meta)
    m = evaluate.load_data("mb", root)
    with pytest.raises(ValueError, match="example 3_2: disp_max -1"):
        m.example((2, 2))
    with pytest.raises(ValueError, match="example 3_2"):
        m.shape_of((2, 2))


def test_submit_refuses_a_non_empty_directory(tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    (out / "old.png").write_bytes(b"x")
    ev = evaluate.Evaluator.__new__(evaluate.Evaluator)               # the check comes before any GPU work
    with pytest.raises(ValueError, match="not empty"):
        ev.submit(data_root=str(tmp_path), out=str(out))


def test_border_comes_from_the_net(tmp_path):
    rng = np.random.default_rng(0)
    net = str(tmp_path / "net.t7")
    t7.save_net(net, oft.make_weights(rng, l1=3, fm=16))
    loaded = frontend.load_net(net, "fast")
    assert frontend.net_border(loaded) == 3                            # not the preset's 4
    assert frontend.net_border(t7.load_net(net)) == (oft.window_size(oft.make_weights(rng, l1=3, fm=16)) - 1) // 2
    with pytest.raises(ValueError, match="'fast' network"):
        frontend.load_net(net, "slow")


def test_zip_members(tmp_path):
    out = tmp_path / "out"
    (out / "disp_0").mkdir(parents=True)
    (out / ".empty").write_bytes(b"")
    (out / "disp_0" / "000000_10.png").write_bytes(b"a")
    (out / "top.txt").write_bytes(b"b")
    with zipfile.ZipFile(evaluate.write_zip(str(out))) as z:
        assert sorted(z.namelist()) == ["disp_0/", "disp_0/000000_10.png", "top.txt"]
        assert z.read("top.txt") == b"b"


def test_lua_number_format():
    assert evaluate.lua_num(0.1) == "0.1" and evaluate.lua_num(1 / 3) == "0.33333333333333"
    assert evaluate.lua_num(2.0) == "2" and evaluate.lua_num(1e-20) == "1e-20"


def test_cli_parsing():
    rm = _run_main()
    args, ov = rm.parse_args(["kitti", "fast", "-a", "test_te", "-net_fname", "n.t7", "-gpu", "2", "-pi1", "3.5",
                              "-sgm_i", "2", "-data_root", "/d"])
    assert args.device == 1 and args.a == "test_te" and args.net_fname == "n.t7" and args.data_root == "/d"
    assert ov == {"pi1": 3.5, "sgm_i": 2} and isinstance(ov["sgm_i"], int)
    args, ov = rm.parse_args(["mb", "census", "-a", "time", "-tiny"])
    assert args.tiny is True and args.device == 0 and ov == {} and args.rect == "imperfect" and args.color == "gray"
    args, _ = rm.parse_args(["kitti", "census", "-a", "predict", "-left", "l.png", "-right", "r.png", "-disp_max", "70"])
    assert (args.left, args.right, args.disp_max) == ("l.png", "r.png", 70)
    for bad, msg in ((["kitti", "fast", "-a", "train_tr"], "training"), (["kitti", "fast", "-a", "nope"], "unknown action"),
                     (["kitti", "fast", "-gpu", "0"], "1-based")):
        with pytest.raises(SystemExit, match=msg):
            rm.parse_args(bad)
    for bad, msg in ((["kitti", "slow", "-at", "1"], "-at 1"), (["mb", "fast", "-color", "rgb"], "-color rgb"),
                     (["kitti", "fast", "-debug"], "-debug"), (["kitti", "fast", "-sm_terminate", "cbca1"], "-sm_terminate")):
        with pytest.raises(ValueError, match=msg):
            rm.parse_args(bad)
