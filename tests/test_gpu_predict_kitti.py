"""GPU: the image front end on the device (frontend.make_batch_cuda, csrc/frontend.cu) against frontend.make_batch bit for bit,
the device error counts against dataio.bad_pixel_rate, and predict_kitti.lua's loop (mccnn_b200/predict_kitti.py) against
frontend.predict run on the same files pair by pair, with the parameters Evaluator uses."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, evaluate, frontend, predict_kitti as pk, synth, t7  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _host_batch(left, right):
    f = lambda b: b.astype(np.float32) if b.ndim == 2 else np.ascontiguousarray(b.transpose(2, 0, 1).astype(np.float32))
    return frontend.make_batch(f(left), f(right))


# n < 8, 8..128, 129, around 8192, the KITTI sizes, odd widths
SIZES = [(1, 2), (1, 7), (2, 3), (4, 10), (3, 43), (1, 129), (5, 31), (64, 128), (91, 90), (1, 8193), (2, 4097), (7, 1171),
         (375, 1242), (375, 1241), (370, 1224), (376, 1241)]


@pytest.mark.parametrize("nch", [1, 3])
@pytest.mark.parametrize("H,W", SIZES)
def test_make_batch_cuda_equals_make_batch(H, W, nch):
    rng = np.random.default_rng(H * 10007 + W + nch)
    shape = (H, W) if nch == 1 else (H, W, 3)
    for lo, hi in ((0, 256), (118, 123)):               # full range, and a low-contrast pair (long runs of equal terms)
        left = rng.integers(lo, hi, shape, dtype=np.uint8)
        right = rng.integers(lo, hi, shape, dtype=np.uint8)
        left.reshape(-1)[0], right.reshape(-1)[-1] = lo, hi - 1  # never constant
        got = frontend.make_batch_cuda(left, right, 0).cpu().numpy()
        want = _host_batch(left, right)
        assert got.shape == want.shape == (2, 1, H, W)
        assert np.array_equal(_bits(got), _bits(want)), "%dx%d nch %d range %d..%d" % (H, W, nch, lo, hi)


def test_make_batch_cuda_from_files_grey_rgb_and_16_bit(tmp_path):
    from PIL import Image

    rng = np.random.default_rng(5)
    files = {}
    files["grey"] = [rng.integers(0, 256, (37, 53), dtype=np.uint8) for _ in range(2)]
    files["rgb"] = [rng.integers(0, 256, (37, 53, 3), dtype=np.uint8) for _ in range(2)]
    for kind, views in files.items():
        paths = [str(tmp_path / ("%s%d.png" % (kind, k))) for k in range(2)]
        for v, p in zip(views, paths):
            Image.fromarray(v).save(p)
        got = frontend.make_batch_cuda(frontend.load_bytes(paths[0]), frontend.load_bytes(paths[1]), 0).cpu().numpy()
        assert np.array_equal(_bits(got), _bits(frontend.make_batch(paths[0], paths[1]))), kind
    paths = [str(tmp_path / ("w%d.png" % k)) for k in range(2)]
    for k, p in enumerate(paths):                        # 16-bit grey: the high byte is the image
        Image.fromarray(rng.integers(0, 65536, (29, 61), dtype=np.uint16)).save(p)
    with Image.open(paths[0]) as im:
        assert im.mode.startswith("I")
    got = frontend.make_batch_cuda(frontend.load_bytes(paths[0]), frontend.load_bytes(paths[1]), 0).cpu().numpy()
    assert np.array_equal(_bits(got), _bits(frontend.make_batch(paths[0], paths[1])))


def test_make_batch_cuda_from_device_tensors():
    rng = np.random.default_rng(6)
    v = [rng.integers(0, 256, (30, 41, 3), dtype=np.uint8) for _ in range(2)]
    got = frontend.make_batch_cuda(torch.from_numpy(v[0]).cuda(), torch.from_numpy(v[1]).cuda(), torch.device("cuda", 0))
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(_host_batch(*v)))


def test_make_batch_cuda_refusals():
    rng = np.random.default_rng(7)
    ok = rng.integers(0, 256, (6, 9), dtype=np.uint8)
    with pytest.raises(ValueError, match="right view: constant"):
        frontend.make_batch_cuda(ok, np.full((6, 9), 17, np.uint8), 0)
    with pytest.raises(ValueError, match="left view: constant"):
        frontend.make_batch_cuda(np.zeros((6, 9, 3), np.uint8), np.zeros((6, 9, 3), np.uint8), 0)
    with pytest.raises(ValueError, match="same size"):
        frontend.make_batch_cuda(ok, ok[:, :8], 0)
    with pytest.raises(ValueError, match="same size"):
        frontend.make_batch_cuda(ok, np.stack([ok] * 3, 2), 0)
    with pytest.raises(ValueError, match="uint8"):
        frontend.make_batch_cuda(ok.astype(np.float32), ok, 0)
    from mccnn_b200.adcensus import AdcensusError

    with pytest.raises(AdcensusError, match="invalid argument"):         # one pixel: no standard deviation
        frontend.make_batch_cuda(ok[:1, :1], ok[:1, :1], 0)


@pytest.mark.parametrize("H,W", [(1, 1), (5, 33), (375, 1242), (370, 1224)])
def test_error_counts_equal_bad_pixel_rate(H, W):
    rng = np.random.default_rng(H + W)
    gt16 = rng.integers(0, 256 * 80, (H, W)).astype(np.uint16)
    gt16[rng.random((H, W)) < 0.3] = 0
    disp = (gt16 / np.float32(256) + rng.normal(0, 3, (H, W))).astype(np.float32)
    disp[rng.random((H, W)) < 0.05] = np.nan
    flat = disp.reshape(-1)
    flat[: min(8, flat.size)] = gt16.reshape(-1)[: min(8, flat.size)] / np.float32(256) + np.float32(3)   # exactly 3 off: not bad
    bad, valid = (int(v) for v in pk.error_counts(torch.from_numpy(disp).cuda(), gt16).cpu())
    want = dataio.bad_pixel_rate(disp, np.where(gt16 == 0, 0, gt16.astype(np.float32) / np.float32(256)), 3)
    assert valid == int((gt16 != 0).sum())
    assert pk.error_rate(bad, valid) == want or (np.isnan(want) and valid == 0)


# ---- predict_kitti against frontend.predict --------------------------------------------------------------------------------

DATASETS = ("kitti", "kitti2015")


@pytest.fixture(scope="module")
def world(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("pk"))
    other = str(tmp_path_factory.mktemp("pk370"))
    for k, ds in enumerate(DATASETS):
        synth.write_kitti_raw(root, ds, n_tr=2, n_te=1, seed=20 + k)
        # one hand-written pair of another height (370 rows, as real KITTI has) appended to each directory
        src = synth.write_kitti_raw(other, ds, n_tr=1, n_te=1, H=370, widths=(1226,), seed=30 + k)
        dst = os.path.join(root, "data.kitti" if ds == "kitti" else "data.kitti2015", "unzip")
        for sub, idx in (("training", 2), ("testing", 1)):
            for d in os.listdir(os.path.join(src, sub)):
                shutil.copy(os.path.join(src, sub, d, "000000_10.png"), os.path.join(dst, sub, d, "%06d_10.png" % idx))
    rng = np.random.default_rng(40)
    nets = {"fast": os.path.join(root, "fast.t7"), "slow": os.path.join(root, "slow.t7")}
    t7.save_net(nets["fast"], oft.make_weights(rng, l1=4, fm=64))                         # the published KITTI fast shape
    t7.save_net(nets["slow"], oft.make_weights(rng, l1=3, fm=16), osh.make_weights(rng, 16, 128, 2))
    return dict(root=root, nets=nets)


def _run_capturing_maps(monkeypatch, *args, **kw):
    maps = []
    orig = evaluate.Evaluator.stereo_predict

    def spy(self, x_batch, disp_max):
        d = orig(self, x_batch, disp_max)
        maps.append(d.cpu().numpy().copy())
        return d

    monkeypatch.setattr(evaluate.Evaluator, "stereo_predict", spy)
    res = pk.predict_kitti(*args, **kw)
    monkeypatch.undo()
    return res, maps


def _frontend_map(world, files, dataset, arch, disp_max):
    return frontend.predict(files[0], files[1], dataset=dataset, arch=arch, disp_max=disp_max, net_fname=world["nets"].get(arch))


@pytest.mark.parametrize("dataset,arch,disp_max", [("kitti", "fast", 228), ("kitti2015", "fast", 228), ("kitti", "census", 228),
                                                   ("kitti2015", "census", 96), ("kitti", "slow", 64),
                                                   ("kitti2015", "slow", 64)])
def test_test_equals_frontend_predict(world, monkeypatch, capsys, dataset, arch, disp_max):
    res, maps = _run_capturing_maps(monkeypatch, "test", dataset, net_fname=world["nets"].get(arch), arch=arch,
                                    data_root=world["root"], disp_max=disp_max)
    lines = capsys.readouterr().out.splitlines()
    files = pk.pair_files(world["root"], dataset, "test")
    assert len(maps) == len(files) == len(res.errors) == 3 and len(lines) == 4
    assert {m.shape for m in maps} == {(375, 1242), (375, 1241), (370, 1226)}
    s = 0.0
    for i, (f, m, err) in enumerate(zip(files, maps, res.errors)):
        want = _frontend_map(world, f, dataset, arch, disp_max)
        assert np.array_equal(m, want, equal_nan=True), "%s %s pair %d: map differs from frontend.predict" % (dataset, arch, i)
        rate = dataio.bad_pixel_rate(m, dataio.read_png16(f[2]), 3)
        assert err == rate
        assert lines[i] == "%d\t%.14g" % (i, rate)
        s = s + rate
    assert res.mean == s / 3 and lines[3] == "%.14g" % res.mean


@pytest.mark.parametrize("dataset,arch", [("kitti", "fast"), ("kitti2015", "census")])
def test_submit_files_equal_write_png16_of_frontend_predict(world, monkeypatch, tmp_path, capsys, dataset, arch):
    out = str(tmp_path / "out")
    files, maps = _run_capturing_maps(monkeypatch, "submit", dataset, net_fname=world["nets"].get(arch), arch=arch,
                                      data_root=world["root"], out=out)
    assert capsys.readouterr().out.splitlines() == ["0", "1"]
    sub = out if dataset == "kitti" else os.path.join(out, "disp_0")
    assert files == [os.path.join(sub, "%06d_10.png" % i) for i in range(2)]
    assert sorted(os.listdir(sub)) == ["000000_10.png", "000001_10.png"]
    for i, (pair, m) in enumerate(zip(pk.pair_files(world["root"], dataset, "submit"), maps)):
        want = _frontend_map(world, pair, dataset, arch, 228)
        assert np.array_equal(m, want, equal_nan=True)
        p = str(tmp_path / ("want%d.png" % i))
        dataio.write_png16(want, p)
        assert open(files[i], "rb").read() == open(p, "rb").read()


def test_prefetch_off_and_the_tool_give_the_same_lines(world, capsys):
    pk.predict_kitti("test", "kitti", net_fname=world["nets"]["fast"], data_root=world["root"])
    with_prefetch = capsys.readouterr().out
    pk.predict_kitti("test", "kitti", net_fname=world["nets"]["fast"], data_root=world["root"], prefetch=False)
    assert capsys.readouterr().out == with_prefetch
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "predict_kitti.py"), "test", "kitti", "-net_fname",
                        world["nets"]["fast"], "-data_root", world["root"]], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout == with_prefetch
