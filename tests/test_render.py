"""The result images without a GPU: the numpy restatement (oracle/render.py) against the reference's own grey2jet and the
reference's sample PNGs, grey2jet's refusals, and what tools/bin2png.py, tools/debug_images.py and run_main.py -debug refuse
before any GPU work."""
import importlib.util
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import adcensus, render
from oracle import refdriver
from oracle import render as orr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLES = ("left", "right", "left_cnn", "right_cnn")


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "render.npz"))


def test_oracle_colours_equal_the_reference_fixture(golden):
    assert np.array_equal(orr.jet_colours(golden["grey"]), golden["rgb"])
    val = golden["grey"] * 4
    for b in (-0.1, 0.5, 1.5, 2.5, 3.5, 4.1):            # every band edge is in the fixture, hit exactly
        assert (val == b).any()
    for disp_max in (70, 228):
        assert np.isin((np.arange(disp_max) + 1) / disp_max, golden["grey"]).all()


@pytest.mark.skipif(not os.path.exists(refdriver.REF_LIB), reason="the reference's shim build (oracle/_ref) is not built")
def test_oracle_colours_equal_the_live_reference(golden):
    from oracle import make_render_golden

    got = make_render_golden.reference_grey2jet(golden["grey"])
    assert np.array_equal(got, golden["rgb"])
    rng = np.random.default_rng(5)
    grey = rng.uniform(-0.025, 1.025, (7, 13))
    assert np.array_equal(make_render_golden.reference_grey2jet(grey), orr.jet_colours(grey))


def test_quantiser_gives_the_sample_pngs_level_sets(golden_dir):
    from PIL import Image

    levels = set(orr.quantise(np.arange(1, 71, dtype=np.float32) / np.float32(70)).tolist())
    assert levels == {255 * k // 70 for k in range(1, 71)}
    assert {3, 10, 14, 21, 25} <= levels                                  # truncated; rounding would give 4, 11, 15, 22, 26
    for name in SAMPLES + ("disp",):
        with Image.open(os.path.join(golden_dir, "render", name + ".png")) as im:
            assert im.mode == "L" and im.size == (1226, 370), name
            a = np.asarray(im)
        if name != "disp":
            assert set(np.unique(a).tolist()) == levels, name


def test_quantiser_clamps_and_truncates():
    x = np.array([-np.inf, -1, -0.0, 0, 0.5, 1 / 255, 254.999 / 255, 1, 2, np.inf, np.nan])
    assert orr.quantise(x).tolist() == [0, 0, 0, 0, 127, 1, 254, 255, 255, 255, 0]


def test_volume_and_map_grey_restate_bin2png():
    inf, nan = np.inf, np.nan
    cols = [[3, 3, 1], [nan, nan, nan], [1e38, nan, 2e38], [2e38, nan, inf], [2, 2, 5], [-inf, 0, -inf]]
    vol = np.array(cols, np.float32).T[:, None, :]
    # all-NaN -> index 1; NaN ties with f32(1e38) and beats 2e38 and inf; the first minimum on ties
    assert orr.volume_grey(vol).tolist() == [[255, 85, 85, 170, 85, 85]]
    x = np.array([[0, 35, 70, 80, -1, np.nan]], np.float32)
    assert orr.map_grey(x, 70).tolist() == [[0, 127, 255, 255, 0, 255]]


@pytest.mark.parametrize("x", [np.nan, -1 - 0.026 * 70, 1.026 * 70 - 1, np.inf])
def test_grey2jet_refuses_nan_and_out_of_range(x):
    m = np.array([[0, 5, x]], np.float32)
    with pytest.raises(orr.RangeError):
        orr.grey2jet(m, 70)


def test_error_image_tints():
    x0 = np.zeros((1, 4), np.float32)
    gt = np.array([[0, 10, 10, 10]], np.float32)
    pred = np.array([[50, 13, 13.5, 7]], np.float32)
    img = orr.error_image(x0, pred, gt, 3.0)
    g = int(np.trunc(np.float64((np.float32(150) * (np.float32(1) / np.float32(255)))) * 255))
    assert img[0, 0].tolist() == [g] * 3                                  # no ground truth: grey only
    assert img[0, 1].tolist() == img[0, 3].tolist() and img[0, 1, 1] > img[0, 1, 0]   # |err| <= 3: green
    assert img[0, 2, 0] > img[0, 2, 1] and img[0, 2, 1] == img[0, 2, 2]  # |err| > 3: red


def test_c_abi_refuses_bad_arguments_before_any_gpu_work(tmp_path):
    l = adcensus.lib()
    assert l.mccnn_render_volume_file(os.fsencode(str(tmp_path / "none.bin")), 2, 2, 2, 16, None) == -4
    short = tmp_path / "short.bin"
    short.write_bytes(b"\0" * (2 * 2 * 2 * 4 - 1))
    assert l.mccnn_render_volume_file(os.fsencode(str(short)), 2, 2, 2, 16, None) == -4
    assert l.mccnn_render_volume_file(os.fsencode(str(short)), 0, 2, 2, 16, None) == -1
    assert l.mccnn_render_map(16, 2, 2, 0, 16, None) == -1
    assert l.mccnn_render_jet(None, 2, 2, 70, 0, 16, None) == -1
    assert l.mccnn_render_jet(16, 2, 2, 0, 0, 16, None) == -1
    assert l.mccnn_render_error(16, 16, 16, 2, 2, float("nan"), 16, None) == -1


def _bins(d, D, H, W, sizes=None):
    sizes = sizes or {}
    for name in render.BIN2PNG:
        n = sizes.get(name, (1 if name == "disp" else D) * H * W * 4)
        (d / (name + ".bin")).write_bytes(b"\0" * n)


def test_bin2png_tool_parses_and_refuses(tmp_path):
    tool = _tool("bin2png")
    _bins(tmp_path, 3, 2, 5)
    args = tool.parse_args([str(tmp_path), "-disp_max", "3", "-height", "2", "-width", "5"])
    assert (args.dir, args.disp_max, args.height, args.width) == (str(tmp_path), 3, 2, 5)
    with pytest.raises(SystemExit, match="left.bin holds 120 bytes, a 70x370x1226"):
        tool.parse_args([str(tmp_path)])                                  # the script's constants are the defaults
    with pytest.raises(SystemExit, match="disp.bin holds 39 bytes"):
        _bins(tmp_path, 3, 2, 5, {"disp": 39})
        tool.parse_args([str(tmp_path), "-disp_max", "3", "-height", "2", "-width", "5"])
    os.remove(tmp_path / "right.bin")
    with pytest.raises(SystemExit, match="right.bin not found"):
        tool.parse_args([str(tmp_path), "-disp_max", "3", "-height", "2", "-width", "5"])
    with pytest.raises(SystemExit, match="positive"):
        tool.parse_args([str(tmp_path), "-disp_max", "0"])
    with pytest.raises(ValueError, match="not found"):
        render.bin2png(str(tmp_path / "nowhere"))


def test_debug_images_tool_parses_and_refuses():
    tool = _tool("debug_images")
    args = tool.parse_args(["kitti", "fast", "-a", "test_all", "-net_fname", "n.t7", "-data_root", "d", "-out", "o",
                            "-gpu", "2"])
    assert (args.a, args.net_fname, args.data_root, args.out, args.device) == ("test_all", "n.t7", "d", "o", 1)
    assert tool.parse_args(["mb", "census"]).out == "tmp"
    for argv, msg in ((["kitti", "census", "-a", "submit"], "test_te and test_all"),
                      (["kitti", "census", "-gpu", "0"], "1-based"), (["kitti", "slow"], "needs -net_fname"),
                      (["mb", "census", "-a", "test_all"], "Middlebury")):
        with pytest.raises(SystemExit, match=msg):
            tool.parse_args(argv)


def test_run_main_keeps_refusing_debug():
    rm = _tool("run_main")
    for argv in (["kitti", "fast", "-debug"], ["mb", "census", "-a", "test_te", "-debug", "true"]):
        with pytest.raises(ValueError, match=r"-debug is not supported: write its images with tools/debug_images.py.*"
                                             r"main.lua:877"):
            rm.parse_args(argv)
    assert not rm.parse_args(["kitti", "fast", "-debug", "false"])[0].debug


def test_debug_names_follow_main_lua():
    assert render.debug_names("kitti", "fast", 3) == ("kitti_3_gt.png", "kitti_fast_3_pred.png", "kitti_fast_3_err.png")
    assert render.debug_names("mb", "slow", "5_2") == ("mb_5_2_gt.png", "mb_slow_5_2_pred.png", "mb_slow_5_2_err.png")
