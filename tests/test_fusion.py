"""CPU: world-frame fusion of raw drives (DESIGN §23) -- the OXTS reader and dataio.raw_poses against an independent
restatement of the KITTI raw devkit's formulas, a pure yaw and known latitude / longitude steps, the synthetic posed drive's
poses read back from its OXTS files, the fusion oracle (tests/fusion_oracle.py) against a brute-force per-voxel loop, and
every refusal of fusion.fuse_drive and tools/fuse_raw.py before any GPU work."""
import importlib.util
import math
import os
import shutil

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, fusion, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


fo = _load("fusion_oracle", "tests", "fusion_oracle.py")
fuse_tool = _load("fuse_raw_tool", "tools", "fuse_raw.py")


def _oxts_line(lat, lon, alt=100.0, roll=0.0, pitch=0.0, yaw=0.0):
    return " ".join(repr(float(v)) for v in [lat, lon, alt, roll, pitch, yaw] + [0.0] * 17) + " 0.05 0.02 4 10 4 4 0\n"


def _date(d, R_rect=(1, 0, 0, 0, 1, 0, 0, 0, 1), R=synth.RAW_VELO_R, T=(0.0, 0.0, 0.0), R_imu=(1, 0, 0, 0, 1, 0, 0, 0, 1),
          T_imu=(0.0, 0.0, 0.0)):
    os.makedirs(d, exist_ok=True)
    cam, velo = synth.raw_calib_text(40, 150, R_rect=R_rect, R=R, T=T)
    num = lambda v: " ".join(repr(float(x)) for x in np.asarray(v).reshape(-1))
    for name, text in ((dataio.RAW_CAM, cam), (dataio.RAW_VELO, velo),
                       (dataio.RAW_IMU, "R: %s\nT: %s\n" % (num(R_imu), num(T_imu)))):
        with open(os.path.join(d, name), "w") as f:
            f.write(text)
    return d


def _drive(tmp_path, records, date="2011_09_26", **calib):
    d = _date(str(tmp_path / date), **calib)
    drive = os.path.join(d, "%s_drive_0001_sync" % date)
    os.makedirs(os.path.join(drive, "oxts", "data"), exist_ok=True)
    for i, rec in enumerate(records):
        with open(dataio.raw_file(drive, dataio.RAW_OXTS, i), "w") as f:
            f.write(_oxts_line(*rec))
    return drive


def _rotation(rng, scale=1.0):
    return synth._rodrigues(rng.uniform(-1, 1, 3) * scale)


# ---- poses ----

def _devkit_poses(recs, R_rect, R, T, R_imu, T_imu):
    """convertOxtsToPose, then the camera chain, written out independently: every matrix inverted with np.linalg.inv"""
    er = 6378137.0
    scale = math.cos(recs[0][0] * math.pi / 180.0)
    pad = lambda R3, t: np.vstack([np.hstack([np.reshape(R3, (3, 3)), np.reshape(t, (3, 1))]), [[0, 0, 0, 1]]])
    C = []
    for lat, lon, alt, roll, pitch, yaw in recs:
        tx = scale * lon * math.pi * er / 180
        ty = scale * er * math.log(math.tan((90 + lat) * math.pi / 360))
        Rx = np.array([[1, 0, 0], [0, math.cos(roll), -math.sin(roll)], [0, math.sin(roll), math.cos(roll)]])
        Ry = np.array([[math.cos(pitch), 0, math.sin(pitch)], [0, 1, 0], [-math.sin(pitch), 0, math.cos(pitch)]])
        Rz = np.array([[math.cos(yaw), -math.sin(yaw), 0], [math.sin(yaw), math.cos(yaw), 0], [0, 0, 1]])
        Ti = pad(Rz.dot(Ry).dot(Rx), [tx, ty, alt])
        C.append(Ti.dot(np.linalg.inv(pad(R_imu, T_imu))).dot(np.linalg.inv(pad(R, T))).dot(np.linalg.inv(pad(R_rect, [0, 0, 0]))))
    return [np.linalg.inv(C[0]).dot(c) for c in C]


def test_raw_poses_match_the_devkit_restatement(tmp_path):
    rng = np.random.default_rng(3)
    R_rect = (_rotation(rng, 0.01)).ravel()
    R, T = _rotation(rng).ravel(), rng.uniform(-1, 1, 3)
    R_imu, T_imu = _rotation(rng, 0.05).ravel(), rng.uniform(-1, 1, 3)
    recs = [(49.01 + 1e-4 * k, 8.42 + 2e-4 * k, 110 + 0.3 * k, rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05),
             rng.uniform(-3, 3)) for k in range(6)]
    drive = _drive(tmp_path, recs, R_rect=R_rect, R=R, T=T, R_imu=R_imu, T_imu=T_imu)
    got = dataio.raw_poses(drive, range(6))
    want = _devkit_poses(recs, R_rect, R, T, R_imu, T_imu)
    assert np.array_equal(got[0], np.eye(4))
    for g, w in zip(got, want):
        assert g.shape == (4, 4) and g.dtype == np.float64
        assert np.abs(g - w).max() < 1e-9
    # a later first frame: the world and the Mercator scale follow it
    got = dataio.raw_poses(drive, [2, 4, 5])
    want = _devkit_poses([recs[i] for i in (2, 4, 5)], R_rect, R, T, R_imu, T_imu)
    assert np.array_equal(got[0], np.eye(4))
    assert max(np.abs(g - w).max() for g, w in zip(got, want)) < 1e-9


def test_pure_yaw_and_known_steps(tmp_path):
    """with R_rect = I, no velodyne or IMU offsets, the camera (x right, y down, z forward) sits on the IMU (x forward, y
    left, z up): a yaw theta turns the camera left, Ry(-theta); a step east moves it forward, a step north to its left"""
    lat0, lon0, th = 49.0, 8.4, 0.3
    s = math.cos(lat0 * math.pi / 180)
    east = s * 6378137.0 * 1e-3 * math.pi / 180                                  # lon + 1e-3 degrees
    north = s * 6378137.0 * (math.log(math.tan((90 + lat0 + 1e-3) * math.pi / 360)) - math.log(math.tan((90 + lat0) * math.pi / 360)))
    drive = _drive(tmp_path, [(lat0, lon0), (lat0, lon0, 100.0, 0.0, 0.0, th), (lat0, lon0 + 1e-3), (lat0 + 1e-3, lon0),
                              (lat0, lon0, 102.5)])
    W = dataio.raw_poses(drive, range(5))
    Ry = np.array([[math.cos(-th), 0, math.sin(-th)], [0, 1, 0], [-math.sin(-th), 0, math.cos(-th)]])
    assert np.abs(W[1][:3, :3] - Ry).max() < 1e-12 and np.abs(W[1][:3, 3]).max() < 1e-9
    assert np.abs(W[2][:3, 3] - [0, 0, east]).max() < 1e-6 and np.abs(W[2][:3, :3] - np.eye(3)).max() < 1e-12
    assert np.abs(W[3][:3, 3] - [-north, 0, 0]).max() < 1e-6
    assert np.abs(W[4][:3, 3] - [0, -2.5, 0]).max() < 1e-9                       # up is -y
    assert 72.5 < east < 73.5 and 111 < north < 112              # 1e-3 degree: 111.3 m cos(49 deg) east, 111.3 m north


def test_synthetic_drive_poses_read_back(tmp_path):
    drive, disps, pids, poses = synth.write_kitti_posed_drive(str(tmp_path), n=5)
    got = dataio.raw_poses(drive, range(5))
    for g, p in zip(got, poses):
        assert np.abs(g[:3, 3] - p[:3, 3]).max() < 1e-6
        assert np.abs(g[:3, :3] - p[:3, :3]).max() < 1e-9
    assert len(disps) == len(pids) == 5 and disps[0].dtype == np.float32
    assert all(np.isfinite(d).all() for d in disps) and all((p >= 0).all() for p in pids)
    # the calibration is not trivial: R_rect_00 and the IMU's R, T are not identities
    c2i = dataio.camera_to_imu(os.path.dirname(drive))
    assert np.abs(c2i[:3, 3]).max() > 0.1


def test_read_oxts_refusals(tmp_path):
    p = str(tmp_path / "0000000000.txt")
    for text, msg in (("1 2 3\n", "30 finite numbers, got 3"), (_oxts_line(49, 8).replace("0.05", "nan"), "30 finite"),
                      (_oxts_line(49, 8) + " 1", "got 31"), (_oxts_line(49, 8).replace("0.05", "x"), "30 numbers"),
                      (_oxts_line(90.0, 8), "latitude 90.0"), (_oxts_line(-91.0, 8), "latitude -91.0")):
        with open(p, "w") as f:
            f.write(text)
        with pytest.raises(ValueError, match=msg) as e:
            dataio.read_oxts(p)
        assert p in str(e.value)
    with open(p, "w") as f:
        f.write(_oxts_line(49, 8))
    assert dataio.read_oxts(p).shape == (30,)


def test_raw_poses_refusals(tmp_path):
    drive = _drive(tmp_path, [(49.0, 8.4), (49.0, 8.4)])
    with pytest.raises(FileNotFoundError, match="frame 0000000002 has no OXTS record"):
        dataio.raw_poses(drive, [0, 1, 2])
    date = os.path.dirname(drive)
    for name in (dataio.RAW_IMU, dataio.RAW_VELO, dataio.RAW_CAM):
        keep = open(os.path.join(date, name)).read()
        os.remove(os.path.join(date, name))
        with pytest.raises(FileNotFoundError, match="missing calibration file .*%s" % name):
            dataio.raw_poses(drive, [0, 1])
        with open(os.path.join(date, name), "w") as f:
            f.write(keep.replace("R_rect_00", "R_rect_xx").replace("T:", "T_:"))
        with pytest.raises(ValueError, match="%s: missing key (R_rect_00|T)" % name):
            dataio.raw_poses(drive, [0, 1])
        with open(os.path.join(date, name), "w") as f:
            f.write(keep)
    with pytest.raises(ValueError, match="no frames"):
        dataio.raw_poses(drive, [])


# ---- the oracle against a brute-force loop ----

def _brute(frames, voxel, max_depth=None):
    """{key: [n_pix, n_frames, [sx, sy, sz], [cr, cg, cb]]} and (pixels, outside), one pixel at a time in Python floats"""
    table, kept, outside = {}, 0, 0
    for disp, cal, rgb, pose in frames:
        Z, X, Y = fo.depth_oracle.depth32(disp, cal, max_depth)
        P = np.asarray(pose, np.float64)
        part = {}
        H, W = disp.shape
        for y in range(H):
            for x in range(W):
                if np.isnan(Z[y, x]):
                    continue
                p = (float(X[y, x]), float(Y[y, x]), float(Z[y, x]))
                w = [((P[k, 0] * p[0] + P[k, 1] * p[1]) + P[k, 2] * p[2]) + P[k, 3] for k in range(3)]
                q = [math.floor(v / voxel) for v in w]
                if not all(-2 ** 20 <= v < 2 ** 20 for v in q):
                    outside += 1
                    continue
                kept += 1
                key = ((q[0] + 2 ** 20) << 42) | ((q[1] + 2 ** 20) << 21) | (q[2] + 2 ** 20)
                e = part.setdefault(key, [0, [0.0, 0.0, 0.0], [0, 0, 0]])
                e[0] += 1
                c = rgb[y, x] if rgb.ndim == 3 else [rgb[y, x]] * 3
                for a in range(3):
                    e[1][a] = e[1][a] + w[a]
                    e[2][a] += int(c[a])
        for key, (n, s, c) in part.items():
            t = table.setdefault(key, [0, 0, [0.0, 0.0, 0.0], [0, 0, 0]])
            t[0] += n
            t[1] += 1
            t[2] = [t[2][a] + s[a] for a in range(3)]
            t[3] = [t[3][a] + c[a] for a in range(3)]
    return table, (kept, outside)


def _frames(rng, n, H, W, rgb=False):
    cal = dataio.Calib(20.0, W / 2 - 0.5, H / 2 + 0.25, 0.5, 0.0, None, None)
    out = []
    for k in range(n):
        d = rng.uniform(0.5, 6, (H, W)).astype(np.float32)
        d[rng.random((H, W)) < 0.15] = np.nan
        d[rng.random((H, W)) < 0.05] = -1.0
        img = rng.integers(0, 256, (H, W, 3) if rgb else (H, W), dtype=np.uint8)
        pose = np.eye(4)
        pose[:3, :3] = _rotation(rng, 0.1)
        pose[:3, 3] = rng.uniform(-0.3, 0.3, 3)
        out.append((d, cal, img, pose))
    return out


@pytest.mark.parametrize("rgb", [False, True])
def test_oracle_matches_a_brute_force_loop(rgb):
    rng = np.random.default_rng(7 + rgb)
    frames = _frames(rng, 3, 9, 13, rgb)
    # a frame whose points straddle the +2^20 edge of x: some land outside
    d, cal, img, pose = frames[-1]
    pose = pose.copy()
    pose[0, 3] = 2 ** 20 * 0.5 - 1.0
    frames[-1] = (d, cal, img, pose)
    for voxel, max_depth in ((0.5, None), (0.5, 6.0), (2.0, None)):
        want, (kept, outside) = _brute(frames, voxel, max_depth)
        t = fo.Table(voxel)
        for d, cal, img, pose in frames:
            t.add(d, cal, img, pose, max_depth)
        assert (t.pixels, t.outside) == (kept, outside)
        if voxel == 0.5:
            assert outside > 0
        assert list(t.keys) == sorted(want)
        for i, k in enumerate(t.keys):
            n, nf, s, c = want[int(k)]
            assert (t.n_pix[i], t.n_frames[i]) == (n, nf)
            assert [float(v) for v in t.sums[i]] == s                    # bit for bit: the same additions in order
            assert list(t.colours[i]) == c
        assert t.n_frames.max() > 1
        for m in (1, 2, 3):
            xyz, col = t.vertices(m)
            sel = t.n_frames >= m
            assert len(xyz) == int(sel.sum())
            n = t.n_pix[sel]
            assert np.array_equal(col, ((t.colours[sel] + n[:, None] // 2) // n[:, None]).astype(np.uint8))
            assert len(t.records(m)) == 15 * len(xyz)


def test_oracle_long_runs_sum_in_order():
    """every pixel in one voxel: the partial is the left-to-right sum, not a pairwise one"""
    H, W = 30, 40
    cal = dataio.Calib(1000.0, 0.0, 0.0, 0.1, 0.0, None, None)
    d = np.full((H, W), 1.0, np.float32)
    d += np.random.default_rng(1).uniform(0, 1e-3, (H, W)).astype(np.float32)
    t = fo.Table(1000.0)
    t.add(d, cal, np.zeros((H, W), np.uint8), np.eye(4))
    assert len(t.keys) == 1 and t.n_pix[0] == H * W
    Z, X, Y = fo.depth_oracle.depth32(d, cal)
    s = 0.0
    for v in Z.reshape(-1).astype(np.float64):
        s = s + v
    assert t.sums[0, 2] == s


def test_key_index_inverts_the_key():
    i = np.array([[-2 ** 20, 0, 2 ** 20 - 1], [5, -7, 11]])
    keys = fo.voxel_keys(i.astype(np.float64) + 0.5, 1.0)[0]
    assert [list(v) for v in fusion.key_index(keys)] == [list(i[:, 0]), list(i[:, 1]), list(i[:, 2])]


# ---- refusals before any GPU work ----

def test_fuse_drive_refusals(tmp_path):
    root = str(tmp_path / "raw")
    drive, _, _, _ = synth.write_kitti_posed_drive(root, n=3, H=16, W=40)
    out = str(tmp_path / "out")
    run = lambda **kw: fusion.fuse_drive("kitti", "census", kw.pop("drives", [drive]), out=out, **kw)
    for kw, msg in (({"voxel": 0.0}, "voxel must be"), ({"voxel": float("nan")}, "voxel must be"),
                    ({"voxel": float("inf")}, "voxel must be"), ({"min_frames": 0}, "min_frames must be"),
                    ({"density": 0.5}, "needs confidence"), ({"max_depth": -1.0}, "max_depth must be"),
                    ({"disp_max": 0}, "disp_max must be")):
        with pytest.raises(ValueError, match=msg):
            run(**kw)
    ext = drive.replace("_sync", "_extract")
    shutil.copytree(drive, ext)
    with pytest.raises(ValueError, match="_extract.*OXTS records run at their own rate"):
        run(drives=[ext])
    os.remove(dataio.raw_file(drive, dataio.RAW_OXTS, 1))
    with pytest.raises(FileNotFoundError, match="frame 0000000001 has no OXTS record"):
        run()
    # -every 2 skips frame 1: its record is not needed
    os.remove(os.path.join(os.path.dirname(drive), dataio.RAW_IMU))
    with pytest.raises(FileNotFoundError, match="missing calibration file .*calib_imu_to_velo.txt"):
        run(every=2)
    os.makedirs(os.path.join(out, os.path.basename(drive)))
    open(os.path.join(out, os.path.basename(drive), "fused.ply"), "w").close()
    with pytest.raises(ValueError, match="fused.ply exists"):
        run()


def test_fuse_drive_refuses_several_processes(monkeypatch):
    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda: 2)
    with pytest.raises(ValueError, match="in order on one device"):
        fusion.fuse_drive("kitti", "census", ["nowhere"], voxel=0.1)


def test_fusion_argument_checks():
    for bad in (0, -1.0, float("nan"), float("inf"), "0.1", None):
        with pytest.raises(ValueError, match="voxel must be"):
            fusion.check_voxel(bad)
    for bad in (0, -2, 1.5):
        with pytest.raises(ValueError, match="min_frames must be"):
            fusion.check_min_frames(bad)
    P = fusion.pose12(np.eye(4))
    assert P.dtype == np.float64 and list(P) == [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]
    assert list(fusion.pose12(np.arange(12.0).reshape(3, 4))) == list(range(12))
    bad = np.eye(4)
    bad[3, 0] = 1
    for p, msg in ((bad, "last row"), (np.eye(3), "4x4 or 3x4"), (np.full((3, 4), np.nan), "finite")):
        with pytest.raises(ValueError, match=msg):
            fusion.pose12(p)


def _tool(tmp_path, *extra):
    return ["kitti", "census", "-drive", str(tmp_path), "-out", str(tmp_path / "o"), *extra]


def test_tool_refusals(tmp_path, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    args = fuse_tool.parse_args(_tool(tmp_path, "-voxel", "0.2", "-min_frames", "2"))
    assert (args.voxel, args.min_frames, args.density, args.every) == (0.2, 2, None, 1)
    for extra, msg in ((("-voxel", "0"), "-voxel must be a finite length > 0"),
                       (("-voxel", "-1"), "-voxel must be a finite length > 0"),
                       (("-voxel", "nan"), "-voxel must be a finite length > 0"),
                       (("-voxel", "inf"), "-voxel must be a finite length > 0"),
                       (("-voxel", "0.1", "-min_frames", "0"), "-min_frames must be at least 1"),
                       (("-voxel", "0.1", "-density", "0.5"), "-density ranks pixels by their confidence"),
                       (("-voxel", "0.1", "-confidence", "-density", "1.5"), r"-density must be in \(0, 1\]"),
                       (("-voxel", "0.1", "-max_depth", "0"), "-max_depth must be > 0"),
                       (("-voxel", "0.1", "-every", "0"), "-every must be at least 1"),
                       (("-voxel", "0.1", "-gpu", "0"), "-gpu is 1-based")):
        with pytest.raises(SystemExit, match=msg):
            fuse_tool.parse_args(_tool(tmp_path, *extra))
    with pytest.raises(SystemExit, match="needs -net_fname"):
        fuse_tool.parse_args(["kitti", "fast", "-drive", str(tmp_path), "-voxel", "0.1"])
    with pytest.raises(SystemExit, match="is not a directory"):
        fuse_tool.parse_args(["kitti", "census", "-drive", str(tmp_path / "missing"), "-voxel", "0.1"])
    with pytest.raises(SystemExit):
        fuse_tool.parse_args(["kitti", "census", "-drive", str(tmp_path)])           # -voxel is required
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(SystemExit, match="run it as one process, not under torchrun"):
        fuse_tool.parse_args(_tool(tmp_path, "-voxel", "0.1"))


def test_tool_refuses_missing_files_before_the_gpu(tmp_path, monkeypatch, capsys):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=2, H=16, W=40)
    os.remove(dataio.raw_file(drive, dataio.RAW_OXTS, 0))
    with pytest.raises(FileNotFoundError, match="frame 0000000000 has no OXTS record"):
        fuse_tool.main(["kitti", "census", "-drive", drive, "-out", str(tmp_path / "o"), "-voxel", "0.1"])
    assert not os.path.exists(str(tmp_path / "o"))
