"""CPU: the image front end of `-a predict` (main.lua:1084-1100): PNG loading, grey conversion,
standardisation, and the host phase of the stereo method's resolver.  (The GPU part of predict() is covered in
tests/test_gpu_parity.py.)"""
import os
import subprocess
import sys

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import frontend

PIL = pytest.importorskip("PIL.Image")


def _png(tmp_path, name, arr, mode):
    p = tmp_path / name
    PIL.fromarray(arr).save(p)  # mode follows dtype / shape (L, RGB, RGBA)
    return str(p)


def test_load_grey_and_rgb(tmp_path):
    rng = np.random.default_rng(0)
    g = rng.integers(0, 256, (7, 11), dtype=np.uint8)
    c = rng.integers(0, 256, (7, 11, 3), dtype=np.uint8)
    a = frontend.load_image(_png(tmp_path, "g.png", g, "L"))
    assert a.shape == (1, 7, 11) and a.dtype == np.float32 and np.array_equal(a[0], g.astype(np.float32))
    b = frontend.load_image(_png(tmp_path, "c.png", c, "RGB"))
    assert b.shape == (3, 7, 11) and np.array_equal(b, c.transpose(2, 0, 1).astype(np.float32))
    rgba = np.concatenate([c, np.full((7, 11, 1), 200, np.uint8)], axis=2)
    assert np.array_equal(frontend.load_image(_png(tmp_path, "a.png", rgba, "RGBA")), b)   # alpha dropped


def test_rgb2y_is_the_fp32_weighted_sum():
    rng = np.random.default_rng(1)
    x = rng.integers(0, 256, (3, 5, 9)).astype(np.float32)
    y = frontend.rgb2y(x)
    assert y.shape == (1, 5, 9) and y.dtype == np.float32
    want = 0.299 * x[0].astype(np.float64) + 0.587 * x[1] + 0.114 * x[2]
    assert np.abs(y[0] - want).max() < 1e-4
    grey = np.stack([x[0]] * 3)
    assert np.abs(frontend.rgb2y(grey)[0] - x[0]).max() < 1e-4                 # weights sum to 1


def test_standardise_zero_mean_unit_unbiased_std():
    rng = np.random.default_rng(2)
    x = rng.integers(0, 256, (1, 37, 53)).astype(np.float32)
    s = frontend.standardise(x)
    assert s.dtype == np.float32 and s.shape == x.shape
    assert abs(float(s.astype(np.float64).mean())) < 1e-6
    assert abs(float(s.astype(np.float64).std(ddof=1)) - 1.0) < 1e-6
    # an affine change of the input does not change the result beyond rounding
    s2 = frontend.standardise(2.0 * x + 10.0)
    assert np.abs(s - s2).max() < 1e-5
    with pytest.raises(AssertionError):
        frontend.standardise(np.full((1, 4, 4), 3.0, np.float32))


def test_make_batch_from_files_and_arrays(tmp_path):
    rng = np.random.default_rng(3)
    l = rng.integers(0, 256, (6, 10, 3), dtype=np.uint8)
    r = rng.integers(0, 256, (6, 10), dtype=np.uint8)
    b = frontend.make_batch(_png(tmp_path, "l.png", l, "RGB"), _png(tmp_path, "r.png", r, "L"))
    assert b.shape == (2, 1, 6, 10) and b.dtype == np.float32 and b.flags["C_CONTIGUOUS"]
    b2 = frontend.make_batch(l.transpose(2, 0, 1).astype(np.float32), r.astype(np.float32))
    assert np.array_equal(b, b2)
    with pytest.raises(AssertionError):
        frontend.make_batch(r.astype(np.float32), r[:, :5].astype(np.float32))


def test_write_bin_roundtrip(tmp_path):
    t = np.arange(24, dtype=np.float32).reshape(1, 2, 3, 4)
    p = tmp_path / "x.bin"
    frontend.write_bin(str(p), t)
    assert p.stat().st_size == 96 and np.array_equal(np.fromfile(str(p), "<f4"), t.ravel())


def test_predict_refuses_bad_net_arguments_before_any_gpu_work(tmp_path):
    """main.lua:893-901: 'fast' / 'slow' load opt.net_fname; a missing file name, a net of the other architecture or an
    unknown arch are errors -- raised on the host, before images are read or the device is touched"""
    from mccnn_b200 import t7

    rng = np.random.default_rng(0)
    fast = str(tmp_path / "fast.t7")
    t7.save_net(fast, [(rng.standard_normal((16, 1, 3, 3)).astype(np.float32), np.zeros(16, np.float32)),
                       (rng.standard_normal((16, 16, 3, 3)).astype(np.float32), np.zeros(16, np.float32))])
    with pytest.raises(ValueError, match="net_fname"):
        frontend.predict("no-such-left.png", "no-such-right.png", "kitti", "fast", disp_max=8)
    with pytest.raises(ValueError, match="'fast' network"):
        frontend.predict("no-such-left.png", "no-such-right.png", "kitti", "slow", disp_max=8, net_fname=fast)
    with pytest.raises(ValueError, match="needs -net_fname"):
        frontend.predict("no-such-left.png", "no-such-right.png", "kitti", "slow", disp_max=8,
                         features=np.zeros((2, 16, 4, 4), np.float32))
    with pytest.raises(ValueError, match="arch must be"):
        frontend.predict("no-such-left.png", "no-such-right.png", "kitti", "sad", disp_max=8)
    with pytest.raises(t7.T7Error):
        frontend.predict("no-such-left.png", "no-such-right.png", "kitti", "fast", disp_max=8,
                         net_fname=str(_png(tmp_path, "x.png", np.zeros((4, 4), np.uint8), "L")))


DEPTHS = (2, 4, 5)


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    """{(arch, depth): .t7 file} of random networks with `depth` 3x3 layers, a scorer head for 'slow'"""
    from mccnn_b200 import t7
    from oracle import feature_tower as oft
    from oracle import scorer_head as osh

    tmp = tmp_path_factory.mktemp("nets")
    rng = np.random.default_rng(0)
    out = {}
    for arch in ("fast", "slow"):
        for depth in DEPTHS:
            out[arch, depth] = str(tmp / ("%s_%d.t7" % (arch, depth)))
            t7.save_net(out[arch, depth], oft.make_weights(rng, l1=depth, fm=8),
                        osh.make_weights(rng, 8, 16, 2) if arch == "slow" else None)
    return out


@pytest.mark.parametrize("border", [None, 7])
@pytest.mark.parametrize("depth", (None,) + DEPTHS)
@pytest.mark.parametrize("arch", ["fast", "slow", "ad", "census"])
@pytest.mark.parametrize("dataset", ["kitti", "kitti2015", "mb"])
def test_stereo_method_parameters(nets, dataset, arch, depth, border):
    """the preset of (dataset, arch) -- kitti's for kitti2015 ad / census (main.lua:146-204) -- with fix_border's width from
    the net for 'fast' / 'slow' (main.lua:382-391, 923: one per 3x3 layer), the preset's without a net, an explicit border
    over both; 'ad' / 'census' take no net"""
    from mccnn_b200 import pipeline

    net_fname = nets["slow" if arch == "slow" else "fast", depth] if depth else None
    takes_net = arch in ("fast", "slow") and depth is not None
    over = {} if border is None else {"border": border}
    method = frontend.StereoMethod(dataset, arch, net_fname, **over)
    preset = "kitti" if dataset == "kitti2015" and arch in ("ad", "census") else dataset
    want = border if border is not None else depth if takes_net else pipeline.PRESETS[preset, arch]["border"]
    assert method.opt.as_dict() == pipeline.make_params(preset, arch, border=want).as_dict()
    assert method.needs_net == (arch in ("fast", "slow") and not takes_net)
    assert method.tower is None and method.head is None


def test_kitti2015_shares_the_kitti_ad_and_census_presets():
    from mccnn_b200 import pipeline

    for arch in ("ad", "census"):
        assert pipeline.make_params("kitti2015", arch).as_dict() == pipeline.make_params("kitti", arch).as_dict()
    assert pipeline.make_params("kitti2015", "census", L1=2).as_dict() == pipeline.make_params("kitti", "census", L1=2).as_dict()


def test_stereo_method_host_phase_makes_no_cuda_call(nets):
    """in a fresh process, so that no other test has initialised CUDA before"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys, torch\nsys.path.insert(0, %r)\nimport mccnn_b200\nfrom mccnn_b200 import frontend\n"
            "for arch, f in %r:\n    frontend.StereoMethod('kitti', arch, f, L1=3)\n"
            "print(torch.cuda.is_initialized())\n" % (root, [(a, f) for (a, _), f in sorted(nets.items())]))
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["False"]


def test_stereo_method_refusals(nets):
    with pytest.raises(ValueError, match="arch must be 'fast', 'slow', 'ad' or 'census'"):
        frontend.StereoMethod("kitti", "sad")
    with pytest.raises(ValueError, match="'fast' network"):
        frontend.StereoMethod("kitti", "slow", nets["fast", 4])
    with pytest.raises(ValueError, match="arch 'slow' needs -net_fname"):
        frontend.StereoMethod("kitti", "slow").stages(0)             # refused before the device is touched
