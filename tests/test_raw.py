"""CPU: KITTI raw drives (DESIGN §21) -- the 'kitti_raw' calibration against a float64 restatement and its refusals, the
scan and frame readers, the projection oracle (tests/raw_oracle.py) against a brute-force per-pixel minimum, the synthetic
drive against the rule, and the refusals of tools/predict_raw.py and depth_eval.py raw before any GPU work."""
import importlib.util
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, depth_eval, predict_raw, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ro = _load("raw_oracle", "tests", "raw_oracle.py")


def _rotation(rng):
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    return q * np.sign(np.linalg.det(q))


def _write_date(d, H=40, W=150, **kw):
    os.makedirs(d, exist_ok=True)
    cam, velo = synth.raw_calib_text(H, W, **kw)
    with open(os.path.join(d, dataio.RAW_CAM), "w") as f:
        f.write(cam)
    with open(os.path.join(d, dataio.RAW_VELO), "w") as f:
        f.write(velo)
    return d


# ---- calibration ----

def test_kitti_raw_calib_matches_a_float64_restatement(tmp_path):
    rng = np.random.default_rng(1)
    R_rect = _rotation(rng) * 0.01 + np.eye(3)
    R, T = _rotation(rng), rng.uniform(-0.5, 0.5, 3)
    d = _write_date(str(tmp_path / "2011_09_26"), 375, 1242, f=721.5377, B=0.5327, R_rect=R_rect.ravel(), R=R.ravel(), T=T)
    cal = dataio.read_calib(d, "kitti_raw")
    cx, cy = 1242 / 2 - 0.25, 375 / 2 + 0.5
    assert (cal.f, cal.cx, cal.cy, cal.doffs, cal.width, cal.height) == (721.5377, cx, cy, 0.0, 1242, 375)
    assert cal.baseline == (0.0 - (-721.5377 * 0.5327)) / 721.5377
    P = np.array([[721.5377, 0, cx, 0], [0, 721.5377, cy, 0], [0, 0, 1, 0]])
    Rr4, Tr4 = np.eye(4), np.eye(4)
    Rr4[:3, :3] = R_rect
    Tr4[:3, :3], Tr4[:3, 3] = R, T
    want = P @ Rr4 @ Tr4
    got = np.array(cal.velo).reshape(3, 4)
    assert np.allclose(got, want, rtol=1e-13, atol=1e-10)
    # the stated operation order, exactly
    B = [[sum_ordered(R_rect[i, k] * np.append(R[k], T[k])[j] for k in range(3)) for j in range(4)] for i in range(3)]
    for i in range(3):
        for j in range(4):
            m = sum_ordered(P[i, k] * B[k][j] for k in range(3))
            assert got[i, j] == (m + P[i, 3] if j == 3 else m)
    # a RawCalib is a Calib where one is expected
    assert isinstance(cal, tuple) and cal[:7] == tuple(dataio.Calib(*cal[:7]))


def sum_ordered(terms):
    terms = [float(t) for t in terms]
    return (terms[0] + terms[1]) + terms[2]


@pytest.mark.parametrize("fname, key, text", [
    (dataio.RAW_CAM, "P_rect_00", None), (dataio.RAW_CAM, "P_rect_01", None), (dataio.RAW_CAM, "S_rect_00", None),
    (dataio.RAW_CAM, "R_rect_00", None), (dataio.RAW_VELO, "R", None), (dataio.RAW_VELO, "T", None),
    (dataio.RAW_CAM, "P_rect_00", "1 2 3"), (dataio.RAW_CAM, "R_rect_00", "1 0 0 0 1 0 0 0 x"),
    (dataio.RAW_VELO, "T", "0 0 nan"), (dataio.RAW_VELO, "R", "1 0 0 0 1 0 0 0 1 0")])
def test_kitti_raw_calib_refusals_name_the_file_and_key(tmp_path, fname, key, text):
    d = _write_date(str(tmp_path / "date"))
    p = os.path.join(d, fname)
    lines = [ln for ln in open(p).read().splitlines() if not ln.startswith(key + ":")]
    if text is not None:
        lines.append("%s: %s" % (key, text))
    open(p, "w").write("\n".join(lines) + "\n")
    with pytest.raises(ValueError, match=r"%s: .*\b%s\b" % (fname.replace(".", r"\."), key)):
        dataio.read_calib(d, "kitti_raw")


def test_kitti_raw_calib_refuses_f_baseline_and_missing_files(tmp_path):
    d = _write_date(str(tmp_path / "f"), f=-700.0)
    with pytest.raises(ValueError, match=r"calib_cam_to_cam\.txt: P_rect_00 gives f = -700"):
        dataio.read_calib(d, "kitti_raw")
    d = _write_date(str(tmp_path / "b"), B=-0.5)
    with pytest.raises(ValueError, match=r"calib_cam_to_cam\.txt: P_rect_00 / P_rect_01 gives baseline = -0.5"):
        dataio.read_calib(d, "kitti_raw")
    d = _write_date(str(tmp_path / "v"))
    os.remove(os.path.join(d, dataio.RAW_VELO))
    with pytest.raises(FileNotFoundError, match="calib_velo_to_cam.txt"):
        dataio.read_calib(d, "kitti_raw")
    with pytest.raises(ValueError, match="calibration kind must be one of kitti, kitti2015, mb, kitti_raw, got 'eth3d'"):
        dataio.read_calib(d, "eth3d")


# ---- readers ----

def test_read_velodyne_round_trips_and_refuses_ragged_files(tmp_path):
    rng = np.random.default_rng(2)
    pts = rng.standard_normal((1000, 4)).astype(np.float32)
    p = str(tmp_path / "0000000000.bin")
    pts.astype("<f4").tofile(p)
    got = dataio.read_velodyne(p)
    assert got.dtype == np.float32 and got.shape == (1000, 4) and np.array_equal(got.view(np.uint32), pts.view(np.uint32))
    open(p, "wb").close()
    assert dataio.read_velodyne(p).shape == (0, 4)
    for nbytes in (4, 15, 17, 16 * 5 + 8):
        with open(p, "wb") as f:
            f.write(b"\0" * nbytes)
        with pytest.raises(ValueError, match="%d bytes, not a whole number of 16-byte points" % nbytes):
            dataio.read_velodyne(p)


def _touch(*p):
    os.makedirs(os.path.dirname(os.path.join(*p)), exist_ok=True)
    open(os.path.join(*p), "wb").close()


def test_raw_frames_ascending_and_one_sided_frames_reported(tmp_path):
    d = str(tmp_path / "2011_09_26" / "2011_09_26_drive_0001_sync")
    for i in (7, 0, 3, 12):
        for what in (dataio.RAW_LEFT, dataio.RAW_RIGHT, dataio.RAW_SCAN):
            _touch(dataio.raw_file(d, what, i))
    _touch(d, "image_00", "data", "notes.txt")
    assert dataio.raw_frames(d) == [0, 3, 7, 12]
    assert dataio.raw_frames(d, velodyne=True) == [0, 3, 7, 12]
    os.remove(dataio.raw_file(d, dataio.RAW_SCAN, 3))
    assert dataio.raw_frames(d) == [0, 3, 7, 12]
    with pytest.raises(ValueError, match="velodyne_points lacks 0000000003"):
        dataio.raw_frames(d, velodyne=True)
    _touch(dataio.raw_file(d, dataio.RAW_LEFT, 20))
    os.remove(dataio.raw_file(d, dataio.RAW_RIGHT, 7))
    with pytest.raises(ValueError, match="frames missing on one side: image_01 lacks 0000000007, 0000000020"):
        dataio.raw_frames(d)
    with pytest.raises(ValueError, match="no frames"):
        dataio.raw_frames(str(tmp_path / "empty"))


# ---- the projection rule ----

def _scan(rng, n, H, W, dup):
    """random points in front of and behind the camera, in and around the image, with `dup` of them copied onto the
    rays of others (same pixel) at the same or a different depth"""
    P = np.array([[700.0, 0, W / 2, 0], [0, 700.0, H / 2, 0], [0, 0, 1, 0]])
    z = rng.uniform(-5, 60, n)
    u = rng.uniform(-3, W + 3, n)
    v = rng.uniform(-3, H + 3, n)
    pts = np.stack([(u - W / 2) * z / 700.0, (v - H / 2) * z / 700.0, z, rng.uniform(0, 1, n)], 1).astype(np.float32)
    src = rng.integers(0, n, dup)
    copy = pts[src].copy()
    scale = np.where(rng.random(dup) < 0.5, 1.0, rng.uniform(0.5, 2.0, dup)).astype(np.float32)
    copy[:, :3] *= scale[:, None]
    return np.concatenate([pts, copy]), P


@pytest.mark.parametrize("seed", range(4))
def test_oracle_equals_the_brute_force_minimum(seed):
    rng = np.random.default_rng(seed)
    H, W = 9, 13
    pts, P = _scan(rng, 300, H, W, 200)
    for min_depth in (0.0, 1e-3, 10.0):
        a = ro.velo_depth_map(pts, P, H, W, min_depth)
        b = ro.brute_force(pts, P, H, W, min_depth)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        assert (a == 0).any() and (a > min_depth).any()


def test_oracle_hand_cases():
    P = np.array([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, 1.0, 0]])
    # y / z = 1 -> v 0; x / z = 1.5 rounds to 2 (ties to even) -> u 1; 2.5 -> 2 -> u 1; 0.4 -> 0 -> u -1 (outside);
    # 3 -> u 2 = W (outside); (2, 2, 1) lands on (u 1, v 1) at z 1; z = 0 is dropped
    pts = np.array([[3, 2, 2, 0], [5, 2, 2, 0], [0.8, 2, 2, 0], [6, 2, 2, 0], [2, 2, 1, 0], [1, 1, 0, 0]], np.float32)
    m = ro.velo_depth_map(pts, P, 2, 2, 0.0)
    assert m.tolist() == [[0, 2], [0, 1]]


def test_synthetic_drive_follows_the_rule(tmp_path):
    drive, gts = synth.write_kitti_drive(str(tmp_path), n=2, H=40, W=150, seed=3)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    assert cal.f * cal.baseline == 384.0 and cal.velo[8:] == (1.0, 0.0, 0.0, 0.0)
    assert dataio.raw_frames(drive, velodyne=True) == [0, 1]
    for k, gt in enumerate(gts):
        scan = dataio.read_velodyne(dataio.raw_file(drive, dataio.RAW_SCAN, k))
        Z = ro.velo_depth_map(scan, cal.velo, 40, 150, 1e-3)
        hit = Z > 0
        assert hit.sum() > 100 and (gt[hit] > 0).all()
        assert np.array_equal(Z[hit], np.float32(384) / gt[hit])            # the true depth, the nearest point
        assert np.array_equal(np.float32(384) / Z[hit], gt[hit])            # and back to the disparity exactly


# ---- command-line refusals, before any GPU work ----

@pytest.fixture()
def drive(tmp_path):
    return synth.write_kitti_drive(str(tmp_path / "raw"), n=3, seed=4)[0]


def test_predict_raw_tool_refusals(drive, tmp_path):
    tool = _load("predict_raw_tool", "tools", "predict_raw.py")
    base = ["kitti", "census", "-drive", drive, "-out", str(tmp_path / "o")]
    for argv, msg in ((["kitti", "fast", "-drive", drive, "-disp"], "arch 'fast' needs -net_fname"),
                      (["kitti", "census", "-disp"], "at least one -drive"),
                      (base, "nothing to write"),
                      (base + ["-disp", "-density", "0.5"], "needs -confidence"),
                      (base + ["-confidence", "-density", "1.5"], r"-density must be in \(0, 1\]"),
                      (base + ["-disp", "-every", "0"], "-every must be at least 1"),
                      (base + ["-disp", "-disp_max", "0"], "-disp_max must be at least 1"),
                      (base + ["-disp", "-gpu", "0"], "-gpu is 1-based"),
                      (["kitti", "census", "-drive", str(tmp_path / "nope"), "-disp"], "is not a directory")):
        with pytest.raises(SystemExit, match=msg):
            tool.parse_args(argv)
    with pytest.raises(SystemExit):
        tool.parse_args(["eth3d", "census", "-drive", drive, "-disp"])
    assert tool.parse_args(base + ["-disp", "-depth", "-ply", "-confidence", "-density", "0.3", "-every", "2"]).every == 2


def test_predict_raw_refuses_before_any_gpu_work(drive, tmp_path):
    import torch

    from mccnn_b200 import predict_raw as pr

    out = tmp_path / "o"
    (out / os.path.basename(drive)).mkdir(parents=True)
    (out / os.path.basename(drive) / "x").write_text("")
    with pytest.raises(ValueError, match="output directory .* is not empty"):
        pr.predict_raw("kitti", "census", [drive], out=str(out), disp=True)
    with pytest.raises(ValueError, match="named twice"):
        pr.predict_raw("kitti", "census", [drive, drive], out=str(tmp_path / "p"), disp=True)
    with pytest.raises(ValueError, match="nothing to write"):
        pr.predict_raw("kitti", "census", [drive], out=str(tmp_path / "p"))
    with pytest.raises(ValueError, match="needs confidence"):
        pr.predict_raw("kitti", "census", [drive], out=str(tmp_path / "p"), disp=True, density=0.5)
    os.remove(dataio.raw_file(drive, dataio.RAW_RIGHT, 1))
    with pytest.raises(ValueError, match="image_01 lacks 0000000001"):
        pr.predict_raw("kitti", "census", [drive], out=str(tmp_path / "p"), disp=True)
    assert not torch.cuda.is_initialized()


def test_drive_frames_every_and_list_files(drive, tmp_path):
    frames = predict_raw.drive_frames([drive], every=2)
    assert [f.index for f in frames] == [0, 2]
    date = os.path.basename(os.path.dirname(drive))
    assert predict_raw.frame_name(frames[1]) == "%s/%s 0000000002" % (date, os.path.basename(drive))
    root = os.path.dirname(os.path.dirname(drive))
    lst = tmp_path / "split.txt"
    lst.write_text("%s/%s 2\n\n%s/%s 0000000000\n" % (date, os.path.basename(drive), date, os.path.basename(drive)))
    got = predict_raw.read_list(str(lst), root)
    assert [(os.path.normpath(f.drive), f.index) for f in got] == [(os.path.normpath(drive), 2), (os.path.normpath(drive), 0)]
    for text, msg in (("%s/%s\n" % (date, os.path.basename(drive)), "expected"), ("a/b/c 1\n", "expected"),
                      ("%s/%s 9\n" % (date, os.path.basename(drive)), "missing .*0000000009.png")):
        lst.write_text(text)
        with pytest.raises((ValueError, FileNotFoundError), match=msg):
            predict_raw.read_list(str(lst), root)


def test_depth_eval_raw_refusals(drive, tmp_path):
    tool = _load("depth_eval_tool_raw", "tools", "depth_eval.py")
    lst = tmp_path / "split.txt"
    lst.write_text("x 1\n")
    p = ["raw", "predict", "kitti", "census"]
    for argv, msg in ((p, "-drive .* or -list, not both"), (p + ["-drive", drive, "-list", str(lst)], "not both"),
                      (p + ["-list", str(tmp_path / "nope")], "is not a file"),
                      (p + ["-drive", drive, "-every", "0"], "-every must be at least 1"),
                      (p + ["-list", str(lst), "-every", "2"], "-every applies to -drive"),
                      (p + ["-drive", drive, "-min_depth", "0"], "0 < -min_depth <= -max_depth"),
                      (p + ["-drive", drive, "-min_depth", "90"], "0 < -min_depth <= -max_depth"),
                      (["raw", "predict", "kitti", "fast", "-drive", drive], "arch 'fast' needs -net_fname"),
                      (p + ["-drive", drive, "-disp_max", "0"], "-disp_max must be at least 1"),
                      (p + ["-drive", drive, "-gpu", "0"], "-gpu is 1-based"),
                      (["raw", "score", str(tmp_path / "nope"), "-drive", drive], "is not a directory")):
        with pytest.raises(SystemExit, match=msg):
            tool.parse_args(argv)
    with pytest.raises(SystemExit):
        tool.parse_args(p + ["-drive", drive, "-crop", "kitti"])
    a = tool.parse_args(p + ["-drive", drive, "-crop", "garg", "-max_depth", "50"])
    assert (a.crop, a.max_depth, a.min_depth) == ("garg", 50.0, 1e-3)
    with pytest.raises(FileNotFoundError, match="missing map"):
        depth_eval.score_raw(predict_raw.drive_frames([drive], velodyne=True), str(tmp_path))


def test_crop_boxes():
    assert depth_eval.crop_box("garg", 375, 1242) == (153, 371, 44, 1197)
    assert depth_eval.crop_box("eigen", 375, 1242) == (124, 342, 44, 1197)
    with pytest.raises(ValueError, match="crop must be"):
        depth_eval.crop_box("full", 375, 1242)
