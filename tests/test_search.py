"""CPU: the test_te parameter search (mccnn_b200/search.py, tools/hs.py) -- hs.py's grids, valid(), log lines and proposal
methods restated, the command line's refusals, and the argument checks of mccnn_pipeline_set_params / _run_volumes that need
no device.  The GPU side is tests/test_gpu_search.py."""
import ctypes
import importlib.util
import os
import random

import pytest

import mccnn_b200
from mccnn_b200 import adcensus, pipeline, search

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_grids():
    for ds in ("kitti", "kitti2015"):
        for arch in ("slow", "ad", "census"):
            assert search.grid(ds, arch) is search.KITTI_TE
        assert search.grid(ds, "fast") is search.KITTI_FAST
    for arch in search.ARCHS:
        assert search.grid("mb", arch) is search.MB_TE
    assert [n for n, _ in search.KITTI_TE] == ["L1", "cbca_i1", "cbca_i2", "tau1", "pi1", "pi2", "sgm_q1", "sgm_q2",
                                              "alpha1", "tau_so", "blur_sigma", "blur_t"]
    assert [n for n, _ in search.KITTI_FAST] == [n for n, _ in search.KITTI_TE][4:]
    assert [n for n, _ in search.MB_TE] == [n for n, _ in search.KITTI_FAST]
    assert dict(search.MB_TE)["blur_t"] == [1, 2, 3, 4, 5] and dict(search.KITTI_TE)["blur_t"] == list(range(1, 8))
    # every name is a stereo-method option of the pipeline
    fields = {n for n, _ in pipeline.Params._fields_}
    assert all(n in fields for g in (search.KITTI_TE, search.KITTI_FAST, search.MB_TE) for n, _ in g)
    with pytest.raises(search.SearchError):
        search.grid("middlebury", "fast")


def test_valid():
    assert search.valid({"pi1": 4.0, "pi2": 8.0}) and search.valid({"pi1": 4.0, "pi2": 4.0})
    assert not search.valid({"pi1": 4.0, "pi2": 2.0})


def test_line_format_round_trips_and_prints_literals_as_hs_py():
    params = search.KITTI_TE
    x = [3, 1, 2, 5, 6, 10, 1, 0, 4, 4, 9, 5]
    ps = search.point(params, x)
    line = search.format_line(0.0421, "kitti", "slow", ps)
    assert line == ("0.0421 kitti slow test_te -L1 3 -cbca_i1 2 -cbca_i2 4 -tau1 0.13 -pi1 1.32 -pi2 128.0 -sgm_q1 3.5 "
                    "-sgm_q2 2 -alpha1 2.0 -tau_so 0.08 -blur_sigma 10.0 -blur_t 6 -use_cache")
    res = search.parse_log([line], "kitti", "slow", params)
    assert res == [(0.0421, line.split(" ", 4)[4])]
    assert search.recover(params, res[0][1]) == x
    fast = search.format_line(0.5, "kitti", "fast", search.point(search.KITTI_FAST, [0] * 8), "net/n.t7")
    assert fast.endswith("-blur_sigma 1.0 -blur_t 1 -net_fname net/n.t7") and " -pi2 8.0 -sgm_q1 3 " in fast
    assert search.recover(search.KITTI_FAST, fast.split(" ", 4)[4]) == [0] * 8
    assert search.format_line(1.0, "mb", "census", search.point(search.MB_TE, [0] * 8)).endswith(" -net_fname -")


def test_recover_takes_the_nearest_grid_value_ties_low():
    params = [("pi1", [1.0, 2.0, 4.0]), ("blur_t", [1, 2, 3])]
    assert search.recover(params, "-pi1 1.5 -blur_t 2.6") == [0, 2]
    assert search.recover(params, "-pi1 3.0 -blur_t 0 -use_cache") == [1, 0]
    assert search.recover(params, "-pi1 9 -blur_t 3 -net_fname x") == [2, 2]


LOG = """\
0.30 kitti fast test_te -pi1 0.25 -pi2 8.0 -sgm_q1 3 -sgm_q2 2 -alpha1 1.0 -tau_so 0.01 -blur_sigma 1.0 -blur_t 1 -net_fname a
0.10 kitti slow test_te -L1 0 -cbca_i1 0 -cbca_i2 0 -tau1 0.01 -pi1 0.25 -pi2 8.0 -sgm_q1 3 -sgm_q2 2 -alpha1 1.0 -tau_so 0.01 -blur_sigma 1.0 -blur_t 1 -use_cache
0.20 kitti fast test_te -pi1 2.3 -pi2 32.0 -sgm_q1 4 -sgm_q2 3 -alpha1 1.5 -tau_so 0.08 -blur_sigma 5.99 -blur_t 5 -net_fname a
0.05 kitti2015 fast test_te -pi1 0.25 -pi2 8.0 -sgm_q1 3 -sgm_q2 2 -alpha1 1.0 -tau_so 0.01 -blur_sigma 1.0 -blur_t 1 -net_fname a
not-a-number kitti fast test_te -pi1 0.25
0.01 kitti fast
garbage
0.25 kitti fast test_te -pi1 4.0 -pi2 128.0 -sgm_q1 5 -sgm_q2 4.5 -alpha1 2.75 -tau_so 1.0 -blur_sigma 10.0 -blur_t 7 -net_fname a
"""
BEST = [8, 5, 2, 2, 2, 4, 7, 4]           # the 0.20 line's indices in KITTI_FAST


def test_parse_log_takes_matching_lines_only():
    res = search.parse_log(LOG.splitlines(), "kitti", "fast", search.KITTI_FAST)
    assert sorted(s for s, _ in res) == [0.2, 0.25, 0.3]
    assert search.recover(search.KITTI_FAST, min(res)[1]) == BEST


@pytest.mark.parametrize("method", ["hillclimb_fast", "hillclimb_slow", "hillclimb_dim"])
def test_hillclimb_starts_from_the_minimum_and_stays_on_the_grid(method):
    params = search.KITTI_FAST
    res = search.parse_log(LOG.splitlines(), "kitti", "fast", params)
    rng = random.Random(5)
    seen = set()
    for _ in range(300):
        x = search.propose(method, params, rng, res)
        assert all(0 <= v < len(params[i][1]) for i, v in enumerate(x))
        diff = [i for i in range(len(x)) if x[i] != BEST[i]]
        if method == "hillclimb_fast":
            assert all(abs(x[i] - BEST[i]) == 1 for i in diff)
        elif method == "hillclimb_slow":
            assert len(diff) <= 1 and all(abs(x[i] - BEST[i]) == 1 for i in diff)
        else:
            assert len(diff) <= 1
        seen.add(tuple(x))
    assert len(seen) > 5
    # reproducible with a seed, and hs.py's order of draws
    a = [search.propose(method, params, random.Random(9), res) for _ in range(3)]
    assert a == [search.propose(method, params, random.Random(9), res) for _ in range(3)]


def test_hillclimb_dim_changes_exactly_one_coordinate_when_it_moves():
    params = search.KITTI_FAST
    res = [(0.1, search.format_params(search.point(params, BEST)))]
    rng = random.Random(1)
    moved = 0
    for _ in range(200):
        x = search.propose("hillclimb_dim", params, rng, res)
        d = sum(a != b for a, b in zip(x, BEST))
        assert d <= 1
        moved += d
    assert moved > 150


def test_random_is_uniform_over_the_grid_and_seeded():
    params = search.KITTI_TE
    x = search.propose("random", params, random.Random(3))
    assert x == search.propose("random", params, random.Random(3))
    r = random.Random(3)
    assert x == [r.randint(0, len(v) - 1) for _, v in params]


def test_misordered_line_is_refused():
    bad = ("0.1 kitti fast test_te -pi2 8.0 -pi1 0.25 -sgm_q1 3 -sgm_q2 2 -alpha1 1.0 -tau_so 0.01 -blur_sigma 1.0 "
           "-blur_t 1 -net_fname a")
    with pytest.raises(search.SearchError, match="not -pi1"):
        search.parse_log([bad], "kitti", "fast", search.KITTI_FAST)
    short = "0.1 kitti fast test_te -pi1 0.25 -pi2 8.0"
    with pytest.raises(search.SearchError):
        search.parse_log([short], "kitti", "fast", search.KITTI_FAST)
    # a line for another dataset / arch is not looked at
    assert search.parse_log([bad], "kitti", "slow", search.KITTI_TE) == []
    with pytest.raises(search.SearchError, match="no line"):
        search.propose("hillclimb_fast", search.KITTI_FAST, random.Random(0), [])


def test_hs_refusals_and_arguments(tmp_path):
    hs = _tool("hs")
    net = tmp_path / "n.t7"
    net.write_text("x")
    log = tmp_path / "log"
    for argv, msg in [
        (["random", "kitti", "fast", "train_tr", str(net)], "training"),
        (["random", "kitti", "slow", "da", str(net)], "training"),
        (["random", "kitti", "fast", "test_te", "-"], "needs a net"),
        (["random", "kitti", "slow", "test_te", str(tmp_path / "missing.t7")], "does not exist"),
        (["hillclimb_fast", "kitti", "census", "test_te", "-", "-log", str(log)], "no line"),
        (["random", "kitti", "census", "test_te", "-", "-gpu", "0"], "1-based"),
        (["random", "mb", "census", "test_te", "-", "-color", "rgb"], "color"),
    ]:
        with pytest.raises(SystemExit, match=msg):
            hs.parse_args(argv)
    log.write_text(LOG)
    with pytest.raises(SystemExit, match="no line"):
        hs.parse_args(["hillclimb_slow", "mb", "census", "test_te", "-", "-log", str(log)])
    a = hs.parse_args(["hillclimb_dim", "kitti", "fast", "test_te", str(net), "-log", str(log), "-n", "4", "-seed", "7",
                       "-gpu", "2", "-data_root", "/d", "-rect", "perfect"])
    assert (a.method, a.dataset, a.arch, a.n, a.seed, a.device, a.data_root, a.rect) == \
        ("hillclimb_dim", "kitti", "fast", 4, 7, 1, "/d", "perfect")
    assert a.params is search.KITTI_FAST
    a = hs.parse_args(["random", "kitti2015", "ad", "test_te", "-"])
    assert a.n == 0 and a.log == "hs.log" and a.params is search.KITTI_TE
    with pytest.raises(SystemExit):
        hs.parse_args(["random", "kitti", "sgm", "test_te", "-"])
    log.write_text(LOG + "0.01 kitti fast test_te -pi2 8.0 -pi1 0.25\n")
    with pytest.raises(SystemExit, match="not -pi1"):
        hs.parse_args(["hillclimb_fast", "kitti", "fast", "test_te", str(net), "-log", str(log)])


def test_hs_appends_one_line_per_write(tmp_path):
    hs = _tool("hs")
    p = str(tmp_path / "log")
    hs.append_line(p, "a b")
    hs.append_line(p, "c")
    assert open(p).read() == "a b\nc\n"


def test_time_search_arguments():
    ts = _tool("time_search")
    a = ts.parse_args([])
    assert (a.n_te, a.archs, a.evals) == (40, ["fast", "slow", "census"], 3)
    assert ts.parse_args(["-archs", "slow", "-n_te", "5"]).archs == ["slow"]
    with pytest.raises(SystemExit):
        ts.parse_args(["-archs", "sgm"])
    assert ts.SLOW_IMAGE_BYTES == 2 * 228 * 350 * 1242 * 4


@pytest.fixture(scope="module")
def lib():
    mccnn_b200.build()
    return adcensus.lib()


def test_set_params_and_run_volumes_reject_bad_arguments_without_a_gpu(lib):
    prm = pipeline.make_params("kitti", "slow")
    one = ctypes.c_void_p(16)
    lib.mccnn_pipeline_set_params.restype = lib.mccnn_pipeline_run_volumes.restype = ctypes.c_int
    assert lib.mccnn_pipeline_set_params(None, ctypes.byref(prm)) == -1
    assert lib.mccnn_pipeline_run_volumes(None, 4, 8, 4, one, one, one, one, one, None, None, None) == -1
    sp = pipeline.StereoPipeline.__new__(pipeline.StereoPipeline)    # no device: a handle-less mirror for the type checks
    sp._h, sp.params, sp.D = ctypes.c_void_p(), prm, 4
    with pytest.raises(adcensus.AdcensusError, match="Params expected"):
        sp.set_params(prm.as_dict())
    import torch

    with pytest.raises(adcensus.AdcensusError, match="imgL must be"):
        sp.run_volumes(torch.zeros(4, 8, 8), None, torch.zeros(1, 8, 8), torch.zeros(8, 8))
    with pytest.raises(adcensus.AdcensusError, match="volL must be"):
        sp.run_volumes(torch.zeros(3, 8, 8), None, torch.zeros(8, 8), torch.zeros(8, 8))
    with pytest.raises(adcensus.AdcensusError, match="volR is needed"):
        sp.run_volumes(torch.zeros(1, 4, 8, 8), None, torch.zeros(8, 8), torch.zeros(8, 8))
    with pytest.raises(adcensus.AdcensusError, match="torch.CudaTensor expected"):
        sp.run_volumes(torch.zeros(1, 4, 8, 8), torch.zeros(1, 4, 8, 8), torch.zeros(8, 8), torch.zeros(8, 8))
