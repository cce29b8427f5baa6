"""CPU: rectification of calibrated raw cameras (DESIGN §22) -- the numpy restatement (tests/rectify_oracle.py) against
OpenCV's initUndistortRectifyMap and remap (golden fixture tests/golden/rectify.npz, written by
oracle/make_rectify_golden.py), both calibration readers and every refusal, mccnn_rectify_pair's argument checks, the
synthetic unrectified drive, and the command-line refusals before any GPU work."""
import importlib.util
import os
import shutil

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import adcensus, dataio, depth_eval, predict_raw, rectify, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
INTR, EXTR = os.path.join(GOLDEN, "rectify_intrinsics.yml"), os.path.join(GOLDEN, "rectify_extrinsics.yml")
CAMS = ("kitti", "rational", "alpha1")


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ro = _load("rectify_oracle", "tests", "rectify_oracle.py")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "rectify.npz"))


def _cam(g, name):
    t = lambda k: tuple(float(v) for v in g[name + "_" + k])
    return dataio.CameraRect(t("K"), t("D"), t("R"), t("P"), tuple(int(v) for v in g[name + "_size"]),
                             tuple(int(v) for v in g[name + "_rect_size"]))


# ---- the oracle against OpenCV ----

@pytest.mark.parametrize("name", CAMS)
def test_oracle_coordinates_are_opencvs_within_1e_3_px(golden, name):
    cam = _cam(golden, name)
    assert len(cam.D) == {"kitti": 5, "rational": 8, "alpha1": 4}[name]
    Wo, Ho = cam.rect_size
    sx, sy, front = ro.source_map(rectify.params(cam), Ho, Wo)
    assert front.all()
    r, c = golden[name + "_rows"], golden[name + "_cols"]
    assert np.abs(sx[np.ix_(r, c)] - golden[name + "_mapx"]).max() <= 1e-3
    assert np.abs(sy[np.ix_(r, c)] - golden[name + "_mapy"]).max() <= 1e-3


def test_oracle_bytes_agree_with_opencv_remap(golden):
    # cv2.remap quantises the coordinates to 1/32 px: up to 1/64 px off on each axis, about 4 levels per axis across a full
    # 0..255 edge of this high-contrast texture, so up to 8 levels where both axes cross one; the mean stays small.
    cam = _cam(golden, "alpha1")
    out, valid = ro.rectify(golden["alpha1_tex"], rectify.params(cam), *cam.rect_size[::-1])
    d = np.abs(out.astype(np.int64) - golden["alpha1_remap"].astype(np.int64))
    assert d.max() <= 8 and d.mean() <= 0.75
    assert 0.5 < valid.mean() < 1                              # alpha = 1: part of the grid lies outside the raw image


def test_oracle_invalid_rules():
    img = np.arange(12, dtype=np.uint8).reshape(3, 4) * 20
    sx = np.array([[-0.5, -0.51, 3.49, 3.5, np.nan, np.inf]], np.float32)
    sy = np.array([[0.0, 0.0, 2.49, 0.0, 0.0, 0.0]], np.float32)
    out, valid = ro.sample(img, sx, sy)
    assert valid.tolist() == [[True, False, True, False, False, False]]
    assert out[0, 4] == 0 and out[0, 5] == 0
    assert out[0, 1] == img[0, 0] and out[0, 3] == img[0, 3]          # the border is replicated


# ---- readers ----

def test_opencv_reader_reads_the_fixture_pair(golden):
    rect = dataio.read_rectification([INTR, EXTR], "opencv", size=(160, 120))
    want = _cam(golden, "alpha1")
    assert rect.left == want
    assert rect.left.size == rect.left.rect_size == rect.right.rect_size == (160, 120)
    c = rect.calib
    P1, P2 = rect.left.P, rect.right.P
    assert (c.f, c.cx, c.cy, c.width, c.height) == (P1[0], P1[2], P1[6], 160, 120)
    assert c.baseline == (P1[3] - P2[3]) / P1[0] and c.baseline > 0 and c.doffs == P2[2] - P1[2]


def test_opencv_reader_against_cv2_filestorage(tmp_path):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    K1 = np.array([[700.0, 0, 330.5], [0, 702.25, 241.0], [0, 0, 1]])
    K2 = np.array([[705.0, 0, 318.0], [0, 703.0, 239.5], [0, 0, 1]])
    D1, D2 = rng.normal(0, 0.05, (1, 8)), rng.normal(0, 0.05, (1, 5))
    R1, R2 = cv2.Rodrigues(np.array([0.01, -0.02, 0.003]))[0], cv2.Rodrigues(np.array([0.012, -0.018, 0.002]))[0]
    P1 = np.array([[690.0, 0, 320.0, 0], [0, 690.0, 240.0, 0], [0, 0, 1, 0]])
    P2 = P1.copy()
    P2[0, 3] = -690.0 * 0.54
    f = str(tmp_path / "rig.yml")
    fs = cv2.FileStorage(f, cv2.FILE_STORAGE_WRITE)
    for k, v in dict(K1=K1, D1=D1, K2=K2, D2=D2, R1=R1, R2=R2, P1=P1, P2=P2).items():
        fs.write(k, v)
    fs.write("width", 640)
    fs.release()
    rect = dataio.read_rectification(f, "opencv", size=(640, 480))
    for got, want in ((rect.left.K, K1), (rect.left.D, D1), (rect.left.R, R1), (rect.left.P, P1), (rect.right.K, K2),
                      (rect.right.D, D2), (rect.right.R, R2), (rect.right.P, P2)):
        assert got == tuple(want.reshape(-1))
    assert rect.calib.baseline == pytest.approx(0.54, rel=1e-15)


def test_kitti_raw_reader_and_calib_equal_read_calib(tmp_path):
    d, _, _ = synth.write_kitti_extract_drive(str(tmp_path), n=1, H=24, W=40, Hraw=30, Wraw=48)
    date = os.path.dirname(d)
    rect = dataio.read_rectification(date, "kitti_raw")
    cal = dataio.read_calib(date, "kitti_raw")
    c = rect.calib
    assert (c.f, c.cx, c.cy, c.baseline, c.doffs, c.width, c.height) == tuple(cal[:7])
    for cam, (K, D, R, P) in zip(rect, synth.extract_cameras(24, 40, 30, 48)):
        assert cam.size == (48, 30) and cam.rect_size == (40, 24)
        for got, want in ((cam.K, K), (cam.D, D), (cam.R, R), (cam.P, P)):
            np.testing.assert_allclose(got, np.reshape(want, -1), rtol=1e-12, atol=1e-15)
    rect.check_size(30, 48, "x")
    with pytest.raises(ValueError, match="calibrated for 48x30 images, the image is 49x30"):
        rect.check_size(30, 49, "x")


def test_params_pad_the_distortion_and_invert_in_float64(golden):
    cam = _cam(golden, "alpha1")
    p = rectify.params(cam)
    assert p.dtype == np.float32 and p.shape == (rectify.NPARAM,)
    M = np.reshape(cam.P, (3, 4))[:, :3] @ np.reshape(cam.R, (3, 3))
    assert np.array_equal(p[:9], np.linalg.inv(M).reshape(-1).astype(np.float32))
    assert p[9:13].tolist() == [np.float32(v) for v in (cam.K[0], cam.K[4], cam.K[2], cam.K[5])]
    assert p[13:17].tolist() == [np.float32(v) for v in cam.D] and p[17:].tolist() == [0, 0, 0, 0]


# ---- refusals ----

def _edit_yml(tmp_path, key, new_body):
    """a copy of the fixture pair with `key`'s entry replaced by new_body (None drops it)"""
    out = []
    for src in (INTR, EXTR):
        lines, skip = [], False
        for line in open(src).read().splitlines():
            if line.startswith(key + ":"):
                skip = True
                if new_body is not None:
                    lines.append(new_body)
                continue
            if skip and line[:1].isspace():
                continue
            skip = False
            lines.append(line)
        p = str(tmp_path / os.path.basename(src))
        with open(p, "w") as f:
            f.write("\n".join(lines) + "\n")
        out.append(p)
    return out


def _mat(key, rows, cols, data):
    return "%s: !!opencv-matrix\n   rows: %d\n   cols: %d\n   dt: d\n   data: [ %s ]" % (key, rows, cols,
                                                                                     ", ".join(repr(float(v)) for v in data))


@pytest.mark.parametrize("key, body, msg", [
    ("M1", None, "missing key M1 or K1"),
    ("P2", None, "missing key P2"),
    ("R1", _mat("R1", 3, 2, [1, 0, 0, 1, 0, 0]), "R1 must hold 9 numbers, got 6"),
    ("R1", _mat("R1", 3, 3, [1, 0, 0, 0, 1]), r"R1 is 3x3 but holds 5 numbers"),
    ("D1", _mat("D1", 1, 6, [0.1] * 6), "D1 holds 6 distortion coefficients; 0, 4, 5 or 8"),
    ("M1", _mat("M1", 3, 3, [150, 0.5, 81, 0, 149, 58.5, 0, 0, 1]), "M1 has skew"),
    ("M1", _mat("M1", 3, 3, [150, 0, 81, 0, 149, 58.5, 0, 0.1, 1]), r"M1's last row"),
    ("R1", _mat("R1", 3, 3, [1, 0, 0, 0, 1, 0, 0, 0, 0]), r"P1\[:, :3\] \. R1 is singular"),
    ("P1", "f", "f = -"),
    ("P2", "baseline", "baseline = -"),
    ("P2", "row", "vertical rig"),
    ("P2", "ty", "vertical rig"),
    ("P1", "inf", "P1 must hold finite numbers"),
])
def test_opencv_refusals_name_the_file_and_key(tmp_path, golden, key, body, msg):
    P = [float(v) for v in golden["alpha1_P"]]                 # the fixture's P1, edited
    edits = {"f": {0: -P[0]}, "baseline": {3: 20.0}, "row": {3: -20.0, 6: P[6] + 1}, "ty": {3: -20.0, 7: 5.0},
             "inf": {11: float("inf")}}
    if body in edits:
        body = _mat(key, 3, 4, [edits[body].get(i, v) for i, v in enumerate(P)])
    files = _edit_yml(tmp_path, key, body)
    with pytest.raises(ValueError, match=msg) as e:
        dataio.read_rectification(files, "opencv", size=(160, 120))
    assert "rectify_" in str(e.value)                          # the file is named


def test_opencv_reader_refuses_bad_files_and_sizes(tmp_path):
    p = tmp_path / "a.yml"
    p.write_text("M1: 1\n")
    with pytest.raises(ValueError, match="no %YAML header"):
        dataio.read_rectification(str(p), "opencv", size=(4, 4))
    with pytest.raises(ValueError, match=r"the images' size \(W, H\) is needed"):
        dataio.read_rectification([INTR, EXTR], "opencv")
    with pytest.raises(ValueError, match="kind must be one of"):
        dataio.read_rectification(INTR, "eth3d")


def _kitti_date(tmp_path, edit):
    d, _, _ = synth.write_kitti_extract_drive(str(tmp_path), n=1, H=24, W=40, Hraw=30, Wraw=48)
    cam = os.path.join(os.path.dirname(d), dataio.RAW_CAM)
    lines = [edit(line) for line in open(cam).read().splitlines()]
    with open(cam, "w") as f:
        f.write("\n".join(l for l in lines if l is not None) + "\n")
    return os.path.dirname(d)


@pytest.mark.parametrize("key, value, msg", [
    ("K_01", None, "missing key K_01"),
    ("D_00", "1 2 3", "D_00 holds 3 distortion coefficients"),
    ("P_rect_00", "1 2 3", "P_rect_00 must hold 12 numbers, got 3"),
    ("S_00", "48.5 30", "S_00 must hold two positive whole numbers"),
    ("S_rect_01", "41 24", "the rectified sizes differ"),
    ("R_rect_00", "x 0 0 0 1 0 0 0 1", "R_rect_00 must hold numbers"),
])
def test_kitti_raw_refusals_name_the_file_and_key(tmp_path, key, value, msg):
    date = _kitti_date(tmp_path, lambda l: l if not l.startswith(key + ":") else (None if value is None else key + ": " + value))
    with pytest.raises(ValueError, match=msg) as e:
        dataio.read_rectification(date, "kitti_raw")
    assert dataio.RAW_CAM in str(e.value)
    with pytest.raises(FileNotFoundError, match="missing calibration file"):
        dataio.read_rectification(str(tmp_path / "nowhere"), "kitti_raw")


# ---- mccnn_rectify_pair's argument checks (nothing is launched) ----

def test_rectify_pair_refuses_before_any_launch():
    lib = adcensus.lib()
    ok = np.zeros(rectify.NPARAM, np.float32)
    ok[8] = ok[0] = ok[4] = 1
    bad = ok.copy()
    bad[15] = np.inf
    A, B, C, E, F = 1 << 20, 1 << 24, 1 << 28, 1 << 32, 1 << 36          # disjoint fake device addresses

    def call(left=A, right=B, nch=1, H=4, W=5, pl=ok, pr=ok, Ho=3, Wo=2, ol=C, orr=E, valid=F):
        return lib.mccnn_rectify_pair(left, right, nch, H, W, None if pl is None else pl.ctypes.data,
                                      None if pr is None else pr.ctypes.data, Ho, Wo, ol, orr, valid, None)

    assert call(left=None) == call(right=None) == call(ol=None) == call(orr=None) == call(pl=None) == -1
    assert call(nch=2) == call(nch=0) == call(H=0) == call(W=0) == call(Ho=0) == call(Wo=0) == -1
    assert call(pl=bad) == call(pr=bad) == -1
    assert call(ol=A) == call(orr=C) == call(valid=C + 5) == call(ol=B + 19) == -1       # overlaps
    assert call(H=1 << 16, W=1 << 15) == -2
    assert call(Ho=1 << 15, Wo=1 << 15, nch=3) == -2


# ---- the synthetic unrectified drive ----

@pytest.mark.parametrize("rig", ["kitti", "alpha1"])
def test_extract_drive_rectifies_back_to_its_scene(tmp_path, rig):
    from mccnn_b200 import frontend

    d, gts, s = synth.write_kitti_extract_drive(str(tmp_path), n=1, rig=rig, sync=True)
    assert d.endswith("_extract") and predict_raw.is_extract(d) and not predict_raw.is_extract(s)
    rect = dataio.read_rectification(os.path.dirname(d), "kitti_raw")
    for cam, sub in zip(rect, ("image_00", "image_01")):
        raw = frontend.load_bytes(os.path.join(d, sub, "data", "0000000000.png"))
        assert raw.shape == (80, 216)
        out, valid = ro.rectify(raw, rectify.params(cam), 64, 192)
        ref = frontend.load_bytes(os.path.join(s, sub, "data", "0000000000.png"))
        err = np.abs(out.astype(np.int64) - ref.astype(np.int64))[valid]
        assert err.mean() < 1.5                                  # two bilinear resamplings of a textured scene
        assert (valid.mean() == 1) if rig == "kitti" else (0.5 < valid.mean() < 0.8)


# ---- command lines ----

def test_run_main_rectify_refusals(tmp_path):
    tool = _load("run_main_tool_rect", "tools", "run_main.py")
    base = ["kitti", "census", "-a", "predict", "-left", "l.png", "-right", "r.png", "-disp_max", "8"]
    for argv, msg in [(base + ["-rectify", INTR, "-calib", "c.txt"], "not both"),
                      (["kitti", "census", "-a", "test_te", "-rectify", INTR], "reads no raw pair"),
                      (base + ["-rectify", INTR, "-rectify", EXTR, "-rectify", INTR], "one or two files"),
                      (base + ["-rectify", str(tmp_path / "none.yml")], "is not a file"),
                      (base + ["-ply"], "need -calib or -rectify")]:
        with pytest.raises(SystemExit, match=msg):
            tool.parse_args(argv)
    args, _ = tool.parse_args(base + ["-rectify", INTR, "-rectify", EXTR, "-ply"])
    assert args.rectify == [INTR, EXTR] and args.ply


def test_rectify_tool_refusals(tmp_path):
    tool = _load("rectify_tool", "tools", "rectify.py")
    d, _, s = synth.write_kitti_extract_drive(str(tmp_path), n=1, H=24, W=40, Hraw=30, Wraw=48, sync=True)
    full = tmp_path / "full"
    full.mkdir()
    (full / "x").write_text("")
    for argv, msg in [(["-out", "o"], "or -drive"),
                      (["-left", INTR, "-drive", d, "-out", "o"], "or -drive"),
                      (["-left", INTR, "-right", INTR, "-out", "o"], "needs -left, -right and -rectify"),
                      (["-drive", s, "-out", "o"], "not an unrectified"),
                      (["-drive", d, "-out", str(full)], "not empty"),
                      (["-drive", d, "-out", "o", "-every", "0"], "-every")]:
        with pytest.raises(SystemExit, match=msg):
            tool.parse_args(argv)
    assert tool.parse_args(["-drive", d, "-out", str(tmp_path / "o")]).drive == d


def test_extract_drives_are_refused_where_scans_are_scored(tmp_path):
    d, _, _ = synth.write_kitti_extract_drive(str(tmp_path), n=1, H=24, W=40, Hraw=30, Wraw=48)
    tool = _load("depth_eval_tool_rect", "tools", "depth_eval.py")
    with pytest.raises(SystemExit, match="unrectified .*not synchronised with the cameras"):
        tool.parse_args(["raw", "predict", "kitti", "census", "-drive", d])
    lst = tmp_path / "split.txt"
    lst.write_text("%s/%s 0\n" % (os.path.basename(os.path.dirname(d)), os.path.basename(d)))
    with pytest.raises(ValueError, match="unrectified"):
        predict_raw.read_list(str(lst), str(tmp_path))
    with pytest.raises(ValueError, match="unrectified"):
        depth_eval.evaluate_raw("kitti", "census", [predict_raw.Frame(d, 0)])


def test_predict_raw_refuses_a_bad_extract_drive_before_any_gpu_work(tmp_path):
    d, _, _ = synth.write_kitti_extract_drive(str(tmp_path), n=1, H=24, W=40, Hraw=30, Wraw=48)
    cam = os.path.join(os.path.dirname(d), dataio.RAW_CAM)
    shutil.copy(cam, cam + ".bak")
    with open(cam, "w") as f:
        f.write("".join(l for l in open(cam + ".bak") if not l.startswith("D_01")))
    with pytest.raises(ValueError, match="missing key D_01"):
        predict_raw.predict_raw("kitti", "census", [d], out=str(tmp_path / "o"), disp=True, device=99)
    shutil.copy(cam + ".bak", cam)
    with open(cam, "w") as f:
        f.write(open(cam + ".bak").read().replace("S_00: 4.8", "S_00: 5.0"))
    with pytest.raises(ValueError, match="calibrated for 50x30 images, the image is 48x30"):
        predict_raw.predict_raw("kitti", "census", [d], out=str(tmp_path / "o"), disp=True, device=99)
