"""CPU: training of the slow architecture without a GPU -- presets, printed lines and names, the init's stream order
(including net_te's discarded draws) against oracle/train_slow.py, the float64 step against finite differences, and the
command line tools/train_slow.py with its refusals."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import preprocess, train  # noqa: E402
from oracle import train as ot  # noqa: E402
from oracle import train_slow as ots  # noqa: E402


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015"])
def test_presets(dataset):
    o = train.options(dataset, "slow")
    want = dict(at=0, l1=4, fm=112, ks=3, l2=4, nh2=384, lr=0.003, bs=128, mom=0.9, true1=1.0, false1=4.0, false2=10.0)
    assert {k: o[k] for k in want} == want
    assert "m" not in o and "pow" not in o
    assert {k: o[k] for k in train.AUGMENT} == train.AUGMENT
    assert train.options(dataset) == dict(train.AUGMENT, **train.NET)                # fast unchanged


def test_net_lines_and_names():
    o = train.options("kitti", "slow")
    assert train.net_lines(o) == (["conv(in=1, out=112, k=3)", "cudnn.ReLU"] + ["conv(in=112, out=112, k=3)", "cudnn.ReLU"] * 3
                                  + ["nn.Reshape(128x224)", "nn.Linear(224 -> 384)", "cudnn.ReLU"]
                                  + ["nn.Linear(384 -> 384)", "cudnn.ReLU"] * 3 + ["nn.Linear(384 -> 1)", "cudnn.Sigmoid"])
    assert train.cmd_str("kitti", ["-a", "train_tr"], "slow") == "kitti_slow_-a_train_tr"
    assert train.net_path("R", "kitti2015", ["-a", "train_all"], "slow") == \
        os.path.join("R", "net", "net_kitti2015_slow_-a_train_all.t7")


@pytest.mark.parametrize("shape", [(2, 16, 1, 128), (4, 112, 4, 384)])
def test_init_and_stream_order(shape):
    """randperm, net_tr's convolutions and Linears, net_te's discarded convolutions, then the per-sample draws"""
    l1, fm, l2, nh2 = shape
    o = train.options("kitti", "slow", l1=l1, fm=fm, l2=l2, nh2=nh2)
    s, g = train.Stream(11), preprocess.MT19937(11)
    n = 30
    perm = train.randperm(s, n)
    assert perm.tolist() == preprocess.randperm(n, 11).tolist()
    for _ in range(n - 1):
        g.random()
    tower, head = train.init_slow(s, o)
    want_t, want_h = ots.init_weights_slow(g, l1, fm, l2, nh2)
    for (a, b), (c, d) in zip(tower + head, want_t + want_h):
        assert a.dtype == np.float32 and np.array_equal(a, c) and np.array_equal(b, d)
    assert [w.shape for w, _ in head] == [(nh2, 2 * fm)] + [(nh2, nh2)] * (l2 - 1) + [(1, nh2)]
    # the first per-sample draw comes after the discarded net_te draws
    skipped = 2 * sum(fm * (1 if i == 0 else fm) * 9 + fm for i in range(l1)) + \
        sum(w.size + b.size for w, b in head)
    g2 = preprocess.MT19937(11)
    for _ in range(n - 1 + skipped):
        g2.random()
    p = train.draw_params(s, o, 1)
    want = ot.sample_params(g2, o)
    assert p["d_pos"][0] == want["d_pos"] and p["phi"][0] == want["phi"]


def _layers(rng, l1, fm, l2, nh2):
    tower = [(rng.standard_normal((fm, 1 if i == 0 else fm, 3, 3)) * 0.4, rng.standard_normal(fm) * 0.1) for i in range(l1)]
    head = [(rng.standard_normal((nh2, 2 * fm if j == 0 else nh2)) * 0.3, rng.standard_normal(nh2) * 0.1)
            for j in range(l2)]
    return tower, head + [(rng.standard_normal((1, nh2)) * 0.3, rng.standard_normal(1) * 0.1)]


def test_step64_slow_finite_differences():
    rng = np.random.default_rng(2)
    tower, head = _layers(rng, 2, 3, 2, 5)
    patches = rng.standard_normal((8, 1, 5, 5))
    loss, gt, gh, y = ots.step64_slow(patches, tower, head)
    assert loss > 0 and y.shape == (4,)
    eps = 1e-6
    for layers, grads in ((tower, gt), (head, gh)):
        for li, (w, b) in enumerate(layers):
            for arr, g in ((w, grads[li][0]), (b, grads[li][1])):
                for idx in list(np.ndindex(arr.shape))[:10]:
                    old = arr[idx]
                    arr[idx] = old + eps
                    lp = ots.step64_slow(patches, tower, head)[0]
                    arr[idx] = old - eps
                    lm = ots.step64_slow(patches, tower, head)[0]
                    arr[idx] = old
                    assert abs((lp - lm) / (2 * eps) - g[idx]) <= 1e-6 + 1e-5 * abs(g[idx]), (li, idx)


def test_flatten_roundtrip_with_head():
    rng = np.random.default_rng(3)
    tower, head = _layers(rng, 3, 16, 2, 128)
    v = train.flatten(tower + head)
    assert v.size == sum(w.size + b.size for w, b in tower + head)
    for (a, b), (c, d) in zip(train.unflatten(v, 3, 16) + train.unflatten_head(v, 3, 16, 2, 128), tower + head):
        assert np.array_equal(a, np.float32(c)) and np.array_equal(b, np.float32(d))


def test_cli_parsing():
    import train_slow as tool

    args, o, stereo = tool.parse_args(["kitti2015", "slow", "-a", "train_all", "-l2", "2", "-nh2", "256", "-lr", "0.01",
                                       "-pi1", "3", "-gpu", "2"])
    assert (args.dataset, args.arch, args.a, args.device) == ("kitti2015", "slow", "train_all", 1)
    assert (o["l2"], o["nh2"], o["lr"], o["fm"], o["l1"]) == (2, 256, 0.01, 112, 4)
    assert stereo == {"pi1": 3.0}
    assert tool.parse_args(["kitti", "slow"])[1] == train.options("kitti", "slow")


@pytest.mark.parametrize("argv,msg", [
    (["kitti", "fast", "-a", "train_tr"], "slow architecture"),
    (["kitti", "ad", "-a", "train_tr"], "slow architecture"),
    (["kitti", "census", "-a", "train_tr"], "slow architecture"),
    (["mb", "slow", "-a", "train_tr"], "Middlebury"),
    (["kitti", "slow", "-a", "test_te"], "not a training action"),
    (["kitti", "slow", "-a", "train_tr", "-at", "1"], "-at 1"),
    (["kitti", "slow", "-a", "train_tr", "-subset", "0.5"], "-subset"),
    (["kitti", "slow", "-a", "train_tr", "-debug"], "-debug"),
    (["kitti", "slow", "-a", "train_tr", "-m", "0.3"], "-m is not a training option of arch slow"),
    (["kitti", "slow", "-a", "train_tr", "-pow", "2"], "-pow is not a training option of arch slow"),
    (["kitti", "slow", "-a", "train_tr", "-l2", "0"], "-l2 0"),
    (["kitti", "slow", "-a", "train_tr", "-l2", "5"], "-l2 5"),
    (["kitti", "slow", "-a", "train_tr", "-nh2", "200"], "-nh2 200"),
    (["kitti", "slow", "-a", "train_tr", "-nh2", "512"], "-nh2 512"),
    (["kitti", "slow", "-a", "train_tr", "-fm", "120"], "-fm 120"),
    (["kitti", "slow", "-a", "train_tr", "-fm", "144"], "-fm 144"),
    (["kitti", "slow", "-a", "train_tr", "-l1", "9"], "-l1 9"),
    (["kitti", "slow", "-a", "train_tr", "-l1", "0"], "-l1 0"),
    (["kitti", "slow", "-a", "train_tr", "-ks", "5"], "-ks 5"),
    (["kitti", "slow", "-a", "train_tr", "-bs", "127"], "-bs 127"),
    (["kitti", "slow", "-a", "train_tr", "-hscale", "1.1"], "main.lua:797"),
    (["kitti", "slow", "-a", "train_tr", "-contrast", "0.9"], "main.lua:810"),
    (["kitti", "slow", "-a", "train_tr", "-gpu", "0"], "1-based"),
])
def test_cli_refusals_write_nothing(argv, msg, tmp_path):
    import train_slow as tool

    with pytest.raises(SystemExit) as e:
        tool.main(argv + ["-data_root", str(tmp_path)])
    assert msg in str(e.value)
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("opt", ["-l2", "-nh2"])
def test_fast_tool_refuses_slow_options(opt, tmp_path):
    import train as tool

    with pytest.raises(SystemExit) as e:
        tool.main(["kitti", "fast", "-a", "train_tr", opt, "2", "-data_root", str(tmp_path)])
    assert "%s is not a training option of arch fast" % opt in str(e.value)
    with pytest.raises(SystemExit, match="fast architecture"):
        tool.main(["kitti", "slow", "-a", "train_tr", "-data_root", str(tmp_path)])
    assert os.listdir(tmp_path) == []


def test_existing_slow_net_refused(tmp_path):
    import train_slow as tool

    p = train.net_path(str(tmp_path), "kitti", ["-a", "train_tr"], "slow")
    os.makedirs(os.path.dirname(p))
    open(p, "w").close()
    with pytest.raises(SystemExit, match="already exists"):
        tool.main(["kitti", "slow", "-a", "train_tr", "-data_root", str(tmp_path)])
    assert os.listdir(os.path.dirname(p)) == [os.path.basename(p)]
