"""CPU: calibration parsing (KITTI 2012, KITTI 2015, MiddEval3) and its refusals, the PLY layout, the depth PNG format, the
numpy depth / metrics oracle (tests/depth_oracle.py) on hand cases, and the command-line refusals of the depth flags
(DESIGN §20)."""
import importlib.util
import math
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, depth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


do = _load("depth_oracle", "tests", "depth_oracle.py")

KITTI_2012 = """P0: 7.215377000000e+02 0.000000000000e+00 6.095593000000e+02 0.000000000000e+00 0.000000000000e+00 7.215377000000e+02 1.728540000000e+02 0.000000000000e+00 0.000000000000e+00 0.000000000000e+00 1.000000000000e+00 0.000000000000e+00
P1: 7.215377000000e+02 0.000000000000e+00 6.095593000000e+02 -3.875744000000e+02 0.000000000000e+00 7.215377000000e+02 1.728540000000e+02 0.000000000000e+00 0.000000000000e+00 0.000000000000e+00 1.000000000000e+00 0.000000000000e+00
P2: 7.215377000000e+02 0.000000000000e+00 6.095593000000e+02 4.485728000000e+01 0.000000000000e+00 7.215377000000e+02 1.728540000000e+02 2.163791000000e-01 0.000000000000e+00 0.000000000000e+00 1.000000000000e+00 2.745884000000e-03
P3: 7.215377000000e+02 0.000000000000e+00 6.095593000000e+02 -3.395242000000e+02 0.000000000000e+00 7.215377000000e+02 1.728540000000e+02 2.199936000000e+00 0.000000000000e+00 0.000000000000e+00 1.000000000000e+00 2.729905000000e-03
"""
KITTI_2015 = """calib_time: 09-Jan-2012 13:57:47
corner_dist: 9.950000e-02
S_00: 1.392000e+03 5.120000e+02
K_00: 9.842439e+02 0.000000e+00 6.900000e+02 0.000000e+00 9.808141e+02 2.331966e+02 0.000000e+00 0.000000e+00 1.000000e+00
S_rect_02: 1.242000e+03 3.750000e+02
R_rect_02: 9.998817e-01 1.511453e-02 -2.841595e-03 -1.511724e-02 9.998853e-01 -9.338510e-04 2.827154e-03 9.766976e-04 9.999955e-01
P_rect_02: 7.215377e+02 0.000000e+00 6.095593e+02 4.485728e+01 0.000000e+00 7.215377e+02 1.728540e+02 2.163791e-01 0.000000e+00 0.000000e+00 1.000000e+00 2.745884e-03
S_rect_03: 1.242000e+03 3.750000e+02
P_rect_03: 7.215377e+02 0.000000e+00 6.095593e+02 -3.395242e+02 0.000000e+00 7.215377e+02 1.728540e+02 2.199936e+00 0.000000e+00 0.000000e+00 1.000000e+00 2.729905e-03
"""
MIDDLEBURY = """cam0=[1758.23 0 829.15; 0 1758.23 552.78; 0 0 1]
cam1=[1758.23 0 976.39; 0 1758.23 552.78; 0 0 1]
doffs=147.24
baseline=178.089
width=1482
height=994
ndisp=135
isint=0
vmin=35
vmax=128
dyavg=0
dymax=0
"""


def _write(tmp_path, text, name="calib.txt"):
    p = str(tmp_path / name)
    with open(p, "w") as f:
        f.write(text)
    return p


def test_kitti_2012_calib(tmp_path):
    c = dataio.read_calib(_write(tmp_path, KITTI_2012), "kitti")
    assert (c.f, c.cx, c.cy, c.doffs) == (721.5377, 609.5593, 172.854, 0.0)
    assert c.baseline == (0.0 - -387.5744) / 721.5377 and 0.53 < c.baseline < 0.54     # metres, left minus right
    assert c.width is None and c.height is None


def test_kitti_2015_calib(tmp_path):
    c = dataio.read_calib(_write(tmp_path, KITTI_2015), "kitti2015")
    assert (c.f, c.cx, c.cy, c.doffs, c.width, c.height) == (721.5377, 609.5593, 172.854, 0.0, 1242, 375)
    assert c.baseline == (44.85728 - -339.5242) / 721.5377 and 0.53 < c.baseline < 0.54
    dataio.check_calib_size(c, 375, 1242, "x")
    with pytest.raises(ValueError, match="calibration for 1242x375 images, the image is 1240x375"):
        dataio.check_calib_size(c, 375, 1240, "x")
    # without S_rect_02 there is no size to hold the image to
    c2 = dataio.read_calib(_write(tmp_path, KITTI_2015.replace("S_rect_02", "X_rect_02")), "kitti2015")
    assert c2.width is None


def test_middlebury_calib(tmp_path):
    c = dataio.read_calib(_write(tmp_path, MIDDLEBURY), "mb")
    assert (c.f, c.cx, c.cy, c.doffs, c.width, c.height) == (1758.23, 829.15, 552.78, 147.24, 1482, 994)
    assert c.baseline == 178.089 / 1000                                                  # millimetres in the file
    with pytest.raises(ValueError, match="the image is 1482x993"):
        dataio.check_calib_size(c, 993, 1482, "calib.txt")


@pytest.mark.parametrize("kind, text, key", [
    ("kitti", KITTI_2012.replace("P1:", "Q1:"), "missing key P1"),
    ("kitti2015", KITTI_2015.replace("P_rect_03", "P_rect_13"), "missing key P_rect_03"),
    ("mb", MIDDLEBURY.replace("doffs", "dofs"), "missing key doffs"),
    ("mb", MIDDLEBURY.replace("cam0=[1758.23 0 829.15; 0 1758.23 552.78; 0 0 1]", "cam0=[1758.23 0 829.15; 0 1758.23]"),
     "cam0 must hold 9 finite numbers"),
    ("kitti", KITTI_2012.replace("P0: 7.215377000000e+02", "P0: abc"), "P0 must hold 12 finite numbers"),
    ("kitti", KITTI_2012.replace("P0: 7.215377000000e+02", "P0: -7.215377000000e+02"), "P0 gives f = -721.538, must be > 0"),
    ("mb", MIDDLEBURY.replace("cam0=[1758.23", "cam0=[0"), "cam0 gives f = 0, must be > 0"),
    ("mb", MIDDLEBURY.replace("baseline=178.089", "baseline=-178.089"), "baseline gives baseline"),
    ("kitti", KITTI_2012.replace("-3.875744000000e+02", "3.875744000000e+02"), "P0 / P1 gives baseline"),
])
def test_calib_refusals_name_the_file_and_key(tmp_path, kind, text, key):
    p = _write(tmp_path, text)
    with pytest.raises(ValueError) as e:
        dataio.read_calib(p, kind)
    assert p in str(e.value) and key in str(e.value)


def test_calib_kind_refused(tmp_path):
    with pytest.raises(ValueError, match="calibration kind"):
        dataio.read_calib(_write(tmp_path, MIDDLEBURY), "eth3d")


def test_ply_layout(tmp_path):
    xyz = np.array([[1.5, -2.25, 10.0], [0.0, 0.5, 80.0], [-1e-3, 3e4, 0.125]], np.float32)
    rgb = np.array([[255, 0, 7], [1, 2, 3], [128, 129, 130]], np.uint8)
    body = b"".join(x.astype("<f4").tobytes() + c.tobytes() for x, c in zip(xyz, rgb))
    p = str(tmp_path / "c.ply")
    depth.write_ply(p, depth.Cloud(np.frombuffer(body, np.uint8), 3))
    raw = open(p, "rb").read()
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex 3\nproperty float x\nproperty float y\n"
              b"property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    assert raw == header + body and len(body) == 3 * 15
    got = np.frombuffer(raw[len(header):], np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))
    assert np.array_equal(got["xyz"], xyz) and np.array_equal(got["rgb"], rgb)
    gx, gc = depth.read_ply(p)
    assert np.array_equal(gx, xyz) and np.array_equal(gc, rgb)
    depth.write_ply(p, depth.Cloud(np.zeros(0, np.uint8), 0))
    assert open(p, "rb").read() == header.replace(b"vertex 3", b"vertex 0")


def test_depth_png16(tmp_path):
    Z = np.array([[1.0, np.nan, 0.001], [255.99, 300.0, 1 / 512]], np.float32)
    p = str(tmp_path / "z.png")
    dataio.write_depth_png16(Z, p)
    v = dataio.read_png16_raw(p)
    assert v.tolist() == [[256, 0, 0], [65533, 65535, 0]]         # round(Z * 256); 0.256 -> 0, 0.5 -> 0 (half to even)
    back = dataio.read_depth_png16(p)
    assert back[0, 0] == 1.0 and np.isnan(back[0, 1])


CAL = dataio.Calib(700.0, 600.5, 170.25, 0.54, 0.0, None, None)
MB = dataio.Calib(1758.23, 829.15, 552.78, 0.178089, 147.24, None, None)


def test_oracle_depth_hand_cases():
    d = np.array([[0.0, 1.0, np.nan, np.inf], [-np.inf, 54.0, 3.78, -1.0]], np.float32)
    Z64 = do.depth64(d, CAL)
    fb = 700.0 * 0.54
    assert np.isnan(Z64[0, 0]) and np.isnan(Z64[0, 2]) and np.isnan(Z64[0, 3]) and np.isnan(Z64[1, 0]) and np.isnan(Z64[1, 3])
    assert Z64[0, 1] == fb and Z64[1, 1] == fb / 54.0 and Z64[1, 2] == fb / np.float64(np.float32(3.78))
    Z, X, Y = do.depth32(d, CAL)
    assert np.array_equal(np.isnan(Z), np.isnan(Z64)) and np.array_equal(np.isnan(X), np.isnan(Z))
    ok = ~np.isnan(Z)
    assert np.allclose(Z[ok], Z64[ok], rtol=1e-6, atol=0)
    assert X[1, 1] == np.float32((np.float32(1) - np.float32(600.5)) * Z[1, 1]) / np.float32(700.0)
    assert Y[1, 1] == np.float32((np.float32(1) - np.float32(170.25)) * Z[1, 1]) / np.float32(700.0)
    # max_depth: Z = 378 / 3.78 = 100 m is dropped at 80 m, kept at 100
    assert np.isnan(do.depth32(d, CAL, 80.0)[0][1, 2]) and not np.isnan(do.depth32(d, CAL, 101.0)[0][1, 2])
    # Middlebury: d = -doffs has no depth, d slightly above it does
    m = np.array([[-147.24, -147.0, 0.0]], np.float32)
    Zm = do.depth64(m, MB)
    assert np.isnan(Zm[0, 0]) and Zm[0, 1] > 0 and Zm[0, 2] == 1758.23 * 0.178089 / 147.24


def test_oracle_metrics_hand_cases():
    fb = float(np.float32(700.0 * 0.54))
    zg = np.array([10.0, 20.0, 40.0, 5.0, 1.0, 100.0, 30.0], np.float64)       # 100 m: outside [1e-3, 80]
    gt = (fb / zg).astype(np.float32)
    gt = np.append(gt, [0.0, np.nan]).reshape(1, -1).astype(np.float32)          # no ground truth
    zp = np.array([11.0, 20.0, 60.0, 5.0, 1.0, 100.0, 0.0])
    pred = np.where(zp > 0, fb / np.where(zp > 0, zp, 1), 0.0).astype(np.float32)  # last pixel: d = 0, no prediction
    pred = np.append(pred, [5.0, 5.0]).reshape(1, -1).astype(np.float32)
    pred[0, 4] = np.inf                                                          # invalid prediction
    m = do.metrics64(pred, gt, CAL)
    Zg = do.depth32(gt, CAL)[0][0, :4].astype(np.float64)
    Zp = do.depth32(pred, CAL)[0][0, :4].astype(np.float64)
    assert m["n"] == 4 and m["coverage"] == 4 / 6
    assert m["abs_rel"] == pytest.approx(np.mean(np.abs(Zp - Zg) / Zg), rel=1e-15)
    assert m["rmse"] == pytest.approx(math.sqrt(np.mean((Zp - Zg) ** 2)), rel=1e-15)
    assert m["rmse_log"] == pytest.approx(math.sqrt(np.mean((np.log(Zp) - np.log(Zg)) ** 2)), rel=1e-15)
    assert (m["a1"], m["a2"], m["a3"]) == (3 / 4, 4 / 4, 4 / 4)                    # 60 / 40 = 1.5 < 1.5625
    # the predicted depth is clamped: 100 m becomes 80 m against a ground truth of 80 m
    g1 = np.array([[fb / 80.0]], np.float32)
    p1 = np.array([[fb / 100.0]], np.float32)
    m1 = do.metrics64(p1, g1, CAL)
    assert m1["n"] == 1 and m1["abs_rel"] == abs(80.0 - float(do.depth32(g1, CAL)[0][0, 0])) / float(do.depth32(g1, CAL)[0][0, 0])
    # nothing scored: every mean is NaN
    e = do.metrics64(np.zeros((2, 2), np.float32), np.zeros((2, 2), np.float32), CAL)
    assert e["n"] == 0 and all(math.isnan(e[k]) for k in ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "coverage"))


def test_metrics_of_counts():
    m = depth.metrics_of([10, 4, 3, 4, 4], [0.4, 0.8, 16.0, 0.04])
    assert m == depth.DepthMetrics(0.1, 0.2, 2.0, 0.1, 0.75, 1.0, 1.0, 4, 0.4)
    e = depth.metrics_of([0, 0, 0, 0, 0], [0.0] * 4)
    assert e.n == 0 and all(math.isnan(v) for v in (e.abs_rel, e.rmse, e.a1, e.coverage))


@pytest.mark.parametrize("argv, msg", [
    (["-a", "test_te", "-calib", "c.txt"], "-calib writes depth.bin"),
    (["-a", "predict", "-ply"], "need -calib"),
    (["-a", "predict", "-max_depth", "80"], "need -calib"),
    (["-a", "predict", "-calib", "c.txt", "-density", "0.5"], "it needs -confidence"),
    (["-a", "predict", "-calib", "c.txt", "-confidence", "-density", "1.5"], "-density must be in (0, 1]"),
    (["-a", "predict", "-calib", "c.txt", "-max_depth", "0"], "-max_depth must be > 0"),
])
def test_run_main_depth_refusals(argv, msg):
    rm = _load("run_main", "tools", "run_main.py")
    with pytest.raises(SystemExit) as e:
        rm.parse_args(["kitti", "census"] + argv)
    assert msg in str(e.value)


def test_tool_refusals(tmp_path):
    pk = _load("predict_kitti_tool", "tools", "predict_kitti.py")
    with pytest.raises(SystemExit, match="-ply .* needs -depth"):
        pk.parse_args(["submit", "kitti", "-arch", "census", "-ply"])
    de = _load("depth_eval_tool", "tools", "depth_eval.py")
    with pytest.raises(SystemExit, match="needs -net_fname"):
        de.parse_args(["predict", "kitti"])
    with pytest.raises(SystemExit, match="disparity PFMs only"):
        de.parse_args(["score", "mb", str(tmp_path), "-source", "depth"])
    with pytest.raises(SystemExit, match="not a directory"):
        de.parse_args(["score", "kitti", str(tmp_path / "nope")])
