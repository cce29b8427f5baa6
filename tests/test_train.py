"""CPU: the training driver of main.lua (mccnn_b200/train.py, tools/train.py) without a GPU -- the random stream against
preprocess.MT19937 and the line-by-line oracle, the cubic warp against OpenCV, the float64 step against finite differences,
the command line and its refusals, names, schedule and line formats."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import preprocess, train  # noqa: E402
from oracle import train as ot  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "train", "warp.npz")


def test_stream_is_torch_generator():
    s, g = train.Stream(42), preprocess.MT19937(42)
    assert s.raw(2000).tolist() == [g.random() for _ in range(2000)]
    s, g = train.Stream(7), preprocess.MT19937(7)
    u = s.uniform(50, -0.3, 0.7)
    assert u.tolist() == [ot.uniform(g, -0.3, 0.7) for _ in range(50)]


@pytest.mark.parametrize("n,seed", [(1, 1), (2, 42), (97, 42), (1000, 3)])
def test_randperm(n, seed):
    assert train.randperm(train.Stream(seed), n).tolist() == preprocess.randperm(n, seed).tolist()


def _opts(**kw):
    return train.options("kitti", **kw)


@pytest.mark.parametrize("kw", [{}, dict(hflip=1, vflip=1, trans=1.5, d_vtrans=0.5, d_rotate=2.0, d_hscale=0.8,
                                         d_hshear=0.2, d_contrast=1.2, scale=0.8)])
def test_stream_order_weights_then_samples(kw):
    """randperm, the reset() draws, then per sample the uniform calls of :791-818 -- the warp records of the first samples
    equal the pure-Python restatement"""
    o = _opts(l1=2, fm=16, **kw)
    rng = np.random.default_rng(0)
    nnz = np.stack([rng.integers(1, 4, 40), rng.integers(0, 30, 40), rng.integers(0, 90, 40),
                    rng.uniform(0, 40, 40)], 1).astype(np.float32)
    s, g = train.Stream(5), preprocess.MT19937(5)
    perm = train.randperm(s, len(nnz))
    assert perm.tolist() == preprocess.randperm(len(nnz), 5).tolist()
    for _ in range(len(nnz) - 1):
        g.random()
    got_w = train.init_weights(s, o["l1"], o["fm"])
    want_w = ot.init_weights(g, o["l1"], o["fm"])
    for (a, b), (c, d) in zip(got_w, want_w):
        assert np.array_equal(a, c) and np.array_equal(b, d)
    n = 12
    rows = nnz[perm[:n] - 1]
    got = train.make_warps(train.draw_params(s, o, n), rows, 5)
    for i in range(n):
        p = ot.sample_params(g, o)
        _, dim3, dim4, d = (float(v) for v in rows[i])
        want = [ot.patch_matrix(5, dim3, dim4, p["scale"], p["phi"], p["trans"], p["hshear"]),
                ot.patch_matrix(5, dim3, dim4 - d + p["d_pos"], p["scale_"], p["phi_"], p["trans_"], p["hshear_"]),
                ot.patch_matrix(5, dim3, dim4, p["scale"], p["phi"], p["trans"], p["hshear"]),
                ot.patch_matrix(5, dim3, dim4 - d + p["d_neg"], p["scale_"], p["phi_"], p["trans_"], p["hshear_"])]
        for j in range(4):
            r = got[4 * i + j]
            assert np.array_equal(r["m"].view(np.int32), want[j].view(np.int32)), (i, j)
            c, b = (p["contrast"], p["brightness"]) if j % 2 == 0 else (p["contrast_"], p["brightness_"])
            assert r["contrast"] == np.float32(c) and r["brightness"] == np.float32(b)
            assert r["image"] == int(rows[i, 0]) - 1 and r["view"] == j % 2
    assert s.raw(3).tolist() == [g.random() for _ in range(3)]


def test_warp_equals_opencv_fixture():
    """bit for bit: the fixture holds cv2.warpAffine's own output (OpenCV 4.x)"""
    g = np.load(GOLDEN)
    for i in range(len(g["ws"])):
        w = int(g["ws"][i])
        got = ot.warp_affine(g["src"], g["m"][i], w)
        assert np.array_equal(got.view(np.int32), g["out"][i, :w, :w].view(np.int32)), i


def test_warp_equals_live_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    src = rng.standard_normal((20, 33)).astype(np.float32)
    for k in range(300):
        m = ot.patch_matrix(9, rng.uniform(-10, 30), rng.uniform(-10, 43), [rng.uniform(-1, 1), rng.uniform(-1, 1)],
                            rng.uniform(-0.5, 0.5), [rng.uniform(-2, 2), 0], rng.uniform(-0.4, 0.4))
        want = cv2.warpAffine(src, m.reshape(2, 3), (9, 9), flags=cv2.INTER_CUBIC, borderMode=cv2.BORDER_CONSTANT,
                              borderValue=0)
        assert np.array_equal(ot.warp_affine(src, m, 9).view(np.int32), want.view(np.int32)), k


@pytest.mark.parametrize("pow_", [1, 2])
def test_step64_finite_differences(pow_):
    rng = np.random.default_rng(pow_)
    layers = [(rng.standard_normal((4, 1, 3, 3)) * 0.5, rng.standard_normal(4) * 0.1),
              (rng.standard_normal((4, 4, 3, 3)) * 0.5, rng.standard_normal(4) * 0.1)]
    patches = rng.standard_normal((8, 1, 5, 5))
    margin = 0.9
    loss, grads = ot.step64(patches, layers, margin, pow_)
    assert loss > 0
    eps = 1e-6
    for li, (w, b) in enumerate(layers):
        for arr, g in ((w, grads[li][0]), (b, grads[li][1])):
            for idx in list(np.ndindex(arr.shape))[:12]:
                old = arr[idx]
                arr[idx] = old + eps
                lp = ot.step64(patches, layers, margin, pow_)[0]
                arr[idx] = old - eps
                lm = ot.step64(patches, layers, margin, pow_)[0]
                arr[idx] = old
                assert abs((lp - lm) / (2 * eps) - g[idx]) <= 1e-6 + 1e-5 * abs(g[idx]), (li, idx)


def test_update32_order():
    p, v = ot.update32(np.float32([1.0]), np.float32([0.5]), np.float32([3.0]), 0.9, 0.002)
    f = np.float32
    vv = f(f(f(0.5) * f(0.9)) + f(f(-0.002) * f(3.0)))
    assert v[0] == vv and p[0] == f(f(1.0) + vv)


def test_schedule_and_names():
    assert train.steps_per_epoch(64 * 10 + 1, 128) == 10
    assert train.steps_per_epoch(64 * 10, 128) == 9
    assert train.steps_per_epoch(64, 128) == 0
    n = 12345
    assert train.steps_per_epoch(n, 128) == len(range(1, n - 64 + 1, 64))
    assert [train.lr_at(0.002, e) for e in (1, 11, 12, 14)] == [0.002, 0.002, 0.002 / 10, 0.002 / 10]
    assert train.cmd_str("kitti", ["-a", "train_tr"]) == "kitti_fast_-a_train_tr"
    assert train.net_path("R", "kitti2015", ["-a", "train_all", "-lr", "0.01"]) == \
        os.path.join("R", "net", "net_kitti2015_fast_-a_train_all_-lr_0.01.t7")
    assert train.net_lines(_opts()) == ["conv(in=1, out=64, k=3)", "cudnn.ReLU", "conv(in=64, out=64, k=3)", "cudnn.ReLU",
                                        "conv(in=64, out=64, k=3)", "cudnn.ReLU", "conv(in=64, out=64, k=3)",
                                        "nn.Normalize2", "nn.StereoJoin1"]
    assert train.epoch_line(1, 0.125, 0.002, 12.5) == "1\t0.125\t0.002\t12.5"
    assert train.epoch_line(12, 1 / 3, 0.002 / 10, 3) == "12\t0.33333333333333\t0.0002\t3"


def test_cli_parsing():
    import train as tool

    args, o, stereo = tool.parse_args(["kitti", "fast", "-a", "train_tr", "-data_root", "R", "-lr", "0.01", "-pi1", "3",
                                       "-hflip", "1", "-gpu", "2"])
    assert (args.dataset, args.a, args.device, args.data_root) == ("kitti", "train_tr", 1, "R")
    assert o["lr"] == 0.01 and o["hflip"] == 1 and o["bs"] == 128 and o["l1"] == 4 and o["m"] == 0.2
    assert stereo == {"pi1": 3.0}
    assert tool.main_args(args.argv) == ["-a", "train_tr", "-lr", "0.01", "-pi1", "3", "-hflip", "1", "-gpu", "2"]


@pytest.mark.parametrize("argv,msg", [
    (["kitti", "slow", "-a", "train_tr"], "fast architecture"),
    (["kitti", "census", "-a", "train_tr"], "fast architecture"),
    (["kitti", "ad", "-a", "train_tr"], "fast architecture"),
    (["mb", "fast", "-a", "train_tr"], "Middlebury"),
    (["kitti", "fast", "-a", "test_te"], "not a training action"),
    (["kitti", "fast", "-a", "train_tr", "-at", "1"], "-at 1"),
    (["kitti", "fast", "-a", "train_tr", "-subset", "0.5"], "-subset"),
    (["kitti", "fast", "-a", "train_tr", "-debug"], "-debug"),
    (["kitti", "fast", "-a", "train_tr", "-ks", "5"], "-ks 5"),
    (["kitti", "fast", "-a", "train_tr", "-fm", "40"], "-fm 40"),
    (["kitti", "fast", "-a", "train_tr", "-fm", "256"], "-fm 256"),
    (["kitti", "fast", "-a", "train_tr", "-l1", "9"], "-l1 9"),
    (["kitti", "fast", "-a", "train_tr", "-bs", "127"], "-bs 127"),
    (["kitti", "fast", "-a", "train_tr", "-bs", "0"], "-bs 0"),
    (["kitti", "fast", "-a", "train_tr", "-pow", "3"], "pow"),
    (["kitti", "fast", "-a", "train_tr", "-hscale", "1.1"], "main.lua:797"),
    (["kitti", "fast", "-a", "train_tr", "-scale", "1.5"], "main.lua:797"),
    (["kitti", "fast", "-a", "train_tr", "-contrast", "0.9"], "main.lua:810"),
    (["kitti", "fast", "-a", "train_tr", "-d_contrast", "0.5"], "main.lua:810"),
    (["kitti", "fast", "-a", "train_tr", "-gpu", "0"], "1-based"),
])
def test_cli_refusals_write_nothing(argv, msg, tmp_path, capsys):
    import train as tool

    with pytest.raises(SystemExit) as e:
        tool.main(argv + ["-data_root", str(tmp_path)])
    assert msg in str(e.value)
    assert os.listdir(tmp_path) == []


def test_existing_net_refused(tmp_path):
    import train as tool

    p = train.net_path(str(tmp_path), "kitti", ["-a", "train_tr"])
    os.makedirs(os.path.dirname(p))
    open(p, "w").close()
    with pytest.raises(SystemExit, match="already exists"):
        tool.main(["kitti", "fast", "-a", "train_tr", "-data_root", str(tmp_path)])
    assert os.listdir(os.path.dirname(p)) == [os.path.basename(p)]


def test_run_main_still_refuses_training():
    import run_main

    with pytest.raises(SystemExit, match="training"):
        run_main.parse_args(["kitti", "fast", "-a", "train_tr"])


def test_patch_matrix_vectorised_equals_scalar():
    rng = np.random.default_rng(9)
    n = 50
    dim3, dim4 = rng.uniform(0, 300, n), rng.uniform(0, 1200, n)
    sc = (rng.uniform(-1, 1, n), rng.uniform(0.5, 1, n))
    phi, hs = rng.uniform(-0.2, 0.2, n), rng.uniform(-0.1, 0.1, n)
    tr = (rng.uniform(-1, 1, n), rng.uniform(-1, 1, n))
    got = train.patch_matrices(9, dim3, dim4, sc, phi, tr, hs)
    for i in range(n):
        want = ot.patch_matrix(9, dim3[i], dim4[i], [sc[0][i], sc[1][i]], phi[i], [tr[0][i], tr[1][i]], hs[i])
        assert np.array_equal(got[i].view(np.int32), want.view(np.int32))
