"""CPU: frame-to-model tracking (DESIGN §25) -- the numpy restatement (tests/track_oracle.py) against a brute-force loop,
its ICP alone converging on exact plane depths, the trajectory metrics on cases worked out by hand, the poses.txt round
trip, and every refusal of Tracker, fuse_drive and tools/fuse_raw.py before any GPU work."""
import importlib.util
import math
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, fusion, synth, track

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


to = _load("track_oracle", "tests", "track_oracle.py")
fuse_tool = _load("fuse_raw_tool_track", "tools", "fuse_raw.py")
traj_tool = _load("traj_eval_tool", "tools", "traj_eval.py")


def _offset(deg, metres, axis=(0.0, 1.0, 0.3), direction=(0.5, 0.2, 0.8)):
    T = np.eye(4)
    ax, dr = np.asarray(axis), np.asarray(direction)
    T[:3, :3] = track.rodrigues(math.radians(deg) * ax / np.linalg.norm(ax))
    T[:3, 3] = metres * dr / np.linalg.norm(dr)
    return T


def _plane_frame(H=96, W=320, k=2):
    """(cal, disparity, fp32 depth) of the exact planes seen from posed frame k"""
    cal = dataio.Calib(float(W), W / 2 - 0.25, H / 2 + 0.5, synth.POSED_B, 0.0, None, None)
    P = synth.posed_camera_poses(k + 1)[k]
    Z = synth.posed_render(P, H, W, cal.f, cal.cx, cal.cy)[0]
    disp = (np.float32(cal.f * cal.baseline) / Z).astype(np.float32)
    Zm = Z.astype(np.float32)
    Zm[~np.isfinite(Zm)] = np.nan
    return cal, disp, Zm, P


def test_terms_and_tree_are_a_brute_force_loop():
    """every pixel's 28 terms, recomputed with Python floats one operation at a time, and their sums through the tree"""
    rng = np.random.default_rng(0)
    cal, disp, Zm, _ = _plane_frame(H=37, W=71)
    disp = disp * (1 + 0.02 * rng.standard_normal(disp.shape)).astype(np.float32)
    disp[rng.random(disp.shape) < 0.1] = np.nan
    Zm[rng.random(Zm.shape) < 0.1] = np.nan
    src, mod = to.source_pyramid(disp, cal, 30.0), to.model_pyramid(Zm, cal)
    T = _offset(1.0, 0.05)
    p12 = T[:3].reshape(12)
    f, cx, cy = (float(np.float32(v)) for v in (cal.f, cal.cx, cal.cy))
    for level in range(3):
        delta, cos_t = 0.3 * (level + 1), math.cos(math.radians(30))
        t, ok = to.terms(src, mod, cal, level, p12, delta, cos_t)
        V, N = src[level]
        Vm, Nm = mod[level]
        _, hl, wl = V.shape
        want = np.zeros((hl * wl, 28))
        for i in range(hl * wl):
            y, x = divmod(i, wl)
            p, n = [float(V[a, y, x]) for a in range(3)], [float(N[a, y, x]) for a in range(3)]
            if math.isnan(n[0]):
                continue
            q = [((p12[4 * a] * p[0] + p12[4 * a + 1] * p[1]) + p12[4 * a + 2] * p[2]) + p12[4 * a + 3] for a in range(3)]
            nr = [(p12[4 * a] * n[0] + p12[4 * a + 1] * n[1]) + p12[4 * a + 2] * n[2] for a in range(3)]
            if not q[2] > 0:
                continue
            u = math.floor((((q[0] / q[2]) * f + cx) * 2.0 ** -level) + 0.5)
            v = math.floor((((q[1] / q[2]) * f + cy) * 2.0 ** -level) + 0.5)
            if not (0 <= u < wl and 0 <= v < hl) or math.isnan(Nm[0, v, u]):
                continue
            m, nm = [float(Vm[a, v, u]) for a in range(3)], [float(Nm[a, v, u]) for a in range(3)]
            d = [q[a] - m[a] for a in range(3)]
            if not ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] <= delta * delta and
                    (nr[0] * nm[0] + nr[1] * nm[1]) + nr[2] * nm[2] >= cos_t):
                continue
            J = [q[1] * nm[2] - q[2] * nm[1], q[2] * nm[0] - q[0] * nm[2], q[0] * nm[1] - q[1] * nm[0], nm[0], nm[1], nm[2],
                 (nm[0] * d[0] + nm[1] * d[1]) + nm[2] * d[2]]
            want[i] = [J[a] * J[b] for a in range(6) for b in range(a, 6)] + [J[a] * J[6] for a in range(6)] + [J[6] * J[6]]
        assert ok.sum() > 50
        assert np.array_equal(t.view(np.uint64), want.view(np.uint64)), "level %d terms" % level
        # the tree, element by element: chunks of 1024 by stride halving, then the chunk sums padded to 2^k
        n = len(want)
        chunks = []
        for c in range(0, max(n, 1), 1024):
            a = [list(want[c + i]) if c + i < n else [0.0] * 28 for i in range(1024)]
            s = 512
            while s:
                a = [[a[i][k] + a[i + s][k] for k in range(28)] for i in range(s)]
                s //= 2
            chunks.append(a[0])
        P = 1
        while P < len(chunks):
            P *= 2
        a = chunks + [[0.0] * 28] * (P - len(chunks))
        while len(a) > 1:
            h = len(a) // 2
            a = [[a[i][k] + a[i + h][k] for k in range(28)] for i in range(h)]
        assert np.array_equal(to.tree_sum(t).view(np.uint64), np.array(a[0]).view(np.uint64)), "level %d sums" % level


def test_tree_spans_several_chunks():
    rng = np.random.default_rng(1)
    t = rng.standard_normal((3 * 1024 + 5, 28))
    ref = np.zeros((4 * 1024, 28))
    ref[:len(t)] = t
    a = ref.reshape(4, 1024, 28)
    for s in (512, 256, 128, 64, 32, 16, 8, 4, 2, 1):
        a = a[:, :s] + a[:, s:2 * s]
    a = a[:, 0]
    a = (a[:2] + a[2:])
    assert np.array_equal(to.tree_sum(t), a[0] + a[1])


def test_icp_converges_on_exact_planes():
    """the three plane families seen from posed frame 2, the estimate started 0.2 m and 2 degrees off"""
    cal, disp, Zm, P = _plane_frame()
    T0 = _offset(2.0, 0.2)
    pose, inliers, lost = to.track(track, disp, cal, Zm, P, P @ T0)
    E = track.rigid_inv(P) @ pose
    assert not lost and inliers > 0.9 * np.isfinite(disp).sum()
    assert np.linalg.norm(E[:3, 3]) < 1e-4 and math.degrees(track.rotation_angle(E[:3, :3])) < 1e-3


def test_lost_when_the_model_is_empty():
    cal, disp, Zm, P = _plane_frame(H=24, W=80)
    pred = P @ _offset(1.0, 0.1)
    pose, inliers, lost = to.track(track, disp, cal, np.full_like(Zm, np.nan), P, pred)
    assert lost and inliers == 0 and np.array_equal(pose, pred)


def test_solve_refuses_degenerate_sums():
    s = np.zeros(28)
    k = 0
    for a in range(6):
        for b in range(a, 6):
            s[k] = 1.0 if a == b else 0.0
            k += 1
    s[21:27] = [0.1, 0, 0, 0, 0, -0.2]
    assert np.allclose(track.solve(s, 6), [-0.1, 0, 0, 0, 0, 0.2])
    assert track.solve(s, 5) is None
    bad = s.copy()
    bad[3] = np.inf
    assert track.solve(bad, 100) is None
    flat = s.copy()
    flat[20] = 0.0                              # A[5, 5] = 0: one direction unconstrained
    assert track.solve(flat, 100) is None


def _line(n, scale=1.0, yaw=0.0):
    out = []
    for k in range(n):
        P = np.eye(4)
        P[:3, :3] = track.rodrigues([0.0, yaw * k, 0.0])
        P[2, 3] = scale * k
        out.append(P)
    return out


def test_identical_trajectories_score_zero():
    gt = _line(901)
    m = track.trajectory_metrics(gt, gt)
    assert (m.ate, m.rpe_t, m.rpe_r, m.t_err, m.r_err) == (0.0, 0.0, 0.0, 0.0, 0.0) and m.segments > 0


def test_scaled_straight_path():
    """900 m in 1 m steps, the estimate's translations 1.01 times the truth's: a segment of length L spans L + 1 m of
    path (its last frame is the first one beyond L), so its error is 0.01 (L + 1) m and t_err 1 % (L + 1) / L"""
    gt, est = _line(901), _line(901, 1.01)
    m = track.trajectory_metrics(est, gt)
    want = []
    for first in range(0, 901, 10):
        for L in range(100, 900, 100):
            if first + L + 1 <= 900:
                want.append((L + 1) / L)
    assert m.segments == len(want)
    assert m.t_err == pytest.approx(sum(want) / len(want), rel=1e-9)
    assert m.r_err == 0.0 and m.rpe_r == 0.0
    assert m.rpe_t == pytest.approx(0.01, rel=1e-9)
    assert m.ate == pytest.approx(0.01 * math.sqrt(sum(k * k for k in range(901)) / 901), rel=1e-9)


def test_extra_yaw_gives_its_rpe_angle():
    gt, est = _line(30), _line(30, yaw=math.radians(0.3))
    for P in est:
        P[2, 3] = 0.0
    for P in gt:
        P[2, 3] = 0.0
    m = track.trajectory_metrics(est, gt)
    assert m.rpe_r == pytest.approx(0.3, rel=1e-9) and m.rpe_t == pytest.approx(0.0, abs=1e-12)


def test_short_drive_has_no_segment():
    m = track.trajectory_metrics(_line(51, 1.02), _line(51))
    assert m.segments == 0 and math.isnan(m.t_err) and math.isnan(m.r_err) and m.ate > 0


def test_poses_round_trip_bit_for_bit(tmp_path):
    rng = np.random.default_rng(3)
    poses = []
    for _ in range(7):
        P = np.eye(4)
        P[:3, :3] = track.rodrigues(rng.standard_normal(3))
        P[:3, 3] = rng.standard_normal(3) * 1e3
        poses.append(P)
    p = str(tmp_path / "poses.txt")
    track.write_poses(p, poses)
    back = track.read_poses(p)
    assert all(np.array_equal(a.view(np.uint64), b.view(np.uint64)) for a, b in zip(poses, back))
    with open(str(tmp_path / "bad.txt"), "w") as f:
        f.write("1 0 0 0 0 1 0 0 0 0 1\n")
    with pytest.raises(ValueError, match="bad.txt line 1: a pose is 12 finite numbers"):
        track.read_poses(str(tmp_path / "bad.txt"))
    with open(str(tmp_path / "nan.txt"), "w") as f:
        f.write("1 0 0 0 0 1 0 0 0 0 1 nan\n")
    with pytest.raises(ValueError, match="12 finite"):
        track.read_poses(str(tmp_path / "nan.txt"))


def test_traj_eval_tool(tmp_path, capsys):
    gt, est = _line(40, 1.0), _line(40, 1.01)
    track.write_poses(str(tmp_path / "gt.txt"), gt)
    track.write_poses(str(tmp_path / "est.txt"), est)
    assert traj_tool.main([str(tmp_path / "est.txt"), str(tmp_path / "gt.txt")]) == 0
    assert capsys.readouterr().out.strip() == track.metrics_line("est.txt", track.trajectory_metrics(est, gt))
    with pytest.raises(SystemExit, match="equally long"):
        track.write_poses(str(tmp_path / "short.txt"), gt[:3])
        traj_tool.main([str(tmp_path / "est.txt"), str(tmp_path / "short.txt")])


def test_tracker_refusals():
    """each refused before a CUDA handle is made"""
    for kw, msg in ((dict(iters=(10, 5)), "iters"), (dict(iters=(10, 5, 0)), "iters"), (dict(delta=(1.0, 0.5, -1.0)), "delta"),
                    (dict(delta=(1.0, math.inf, 0.2)), "delta"), (dict(theta=0.0), "theta"), (dict(theta=120.0), "theta")):
        with pytest.raises(ValueError, match=msg):
            track.Tracker(8, 8, **kw)
    with pytest.raises(ValueError, match="H and W"):
        track.Tracker(0, 8)
    with pytest.raises(ValueError, match="4x4 or 3x4"):
        track.as4(np.eye(3))
    with pytest.raises(ValueError, match="trajectories of 2 and 3"):
        track.trajectory_metrics(_line(2), _line(3))


def _base(drive, out):
    return ["kitti", "census", "-drive", drive, "-out", out, "-voxel", "0.1"]


def test_fuse_raw_tracking_refusals(tmp_path, monkeypatch):
    """each before any GPU work, with its own message"""
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=2, H=16, W=48, no_oxts=True)
    out = str(tmp_path / "out")
    b = _base(drive, out)
    with pytest.raises(SystemExit, match="-poses track tracks each frame against the distance field; it needs -mesh"):
        fuse_tool.main(b + ["-poses", "track"])
    with pytest.raises(SystemExit, match="-poses refine .* it needs -mesh"):
        fuse_tool.main(b + ["-poses", "refine"])
    with pytest.raises(SystemExit, match="-traj compares tracked poses with OXTS; it needs -poses track or refine"):
        fuse_tool.main(b + ["-mesh", "-traj"])
    with pytest.raises(ValueError, match="it needs mesh"):
        fusion.fuse_drive("kitti", "census", [drive], out=out, poses="track")
    with pytest.raises(ValueError, match="poses must be"):
        fusion.fuse_drive("kitti", "census", [drive], out=out, mesh=True, poses="gps")
    with pytest.raises(ValueError, match="traj compares"):
        fusion.fuse_drive("kitti", "census", [drive], out=out, mesh=True, traj=True)
    # a drive without oxts/: refine and -traj need it (refused naming the record), oxts too
    for extra in (["-poses", "refine"], ["-poses", "track", "-traj"], []):
        with pytest.raises(FileNotFoundError, match="has no OXTS record"):
            fuse_tool.main(b + ["-mesh"] + extra)
    os.makedirs(os.path.join(out, os.path.basename(drive)))
    with open(fusion.poses_file(out, drive), "w") as f:
        f.write("")
    with pytest.raises(ValueError, match="poses.txt exists; tracking does not overwrite a trajectory"):
        fuse_tool.main(b + ["-mesh", "-poses", "track"])
    extract = str(tmp_path / "2011_09_26" / "2011_09_26_drive_0001_extract")
    os.makedirs(extract)
    with pytest.raises(ValueError, match="_extract"):
        fuse_tool.main(_base(extract, out) + ["-mesh", "-poses", "track"])


def test_no_oxts_drive_keeps_the_other_files(tmp_path):
    a, da, _, pa = synth.write_kitti_posed_drive(str(tmp_path / "a"), n=2, H=16, W=48)
    b, db, _, pb = synth.write_kitti_posed_drive(str(tmp_path / "b"), n=2, H=16, W=48, no_oxts=True)
    assert os.path.isdir(os.path.join(a, "oxts")) and not os.path.exists(os.path.join(b, "oxts"))
    for what in (dataio.RAW_LEFT, dataio.RAW_RIGHT):
        for k in range(2):
            fa, fb = (dataio.raw_file(d, what, k) for d in (a, b))
            assert open(fa, "rb").read() == open(fb, "rb").read()
    assert all(np.array_equal(x, y) for x, y in zip(da, db)) and all(np.array_equal(x, y) for x, y in zip(pa, pb))
