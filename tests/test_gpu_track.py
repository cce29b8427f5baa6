"""GPU: frame-to-model tracking (DESIGN §25) -- mccnn_track_* bit for bit against the numpy restatement
(tests/track_oracle.py): both pyramids, the 28 sums and the counts at every level, and a whole tracked drive's poses and
field, twice; the accuracy of 'track' and 'refine' on the synthetic posed drive's exact disparities, with a lost frame; and
tools/fuse_raw.py -mesh -poses track -traj -score with census against the oracle loop on the same predicted maps."""
import ctypes
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, depth, depth_eval, fusion, predict_kitti, predict_raw, synth, track  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


to = _load("track_oracle", "tests", "track_oracle.py")
fuse_tool = _load("fuse_raw_tool_gpu_track", "tools", "fuse_raw.py")
COS30 = math.cos(math.radians(30.0))


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def png(path):
    from PIL import Image

    with Image.open(path) as im:
        return np.array(im)


def same_bits(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, what
    assert np.array_equal(np.isnan(a), np.isnan(b)), "%s: NaN patterns differ" % what
    assert np.array_equal(a.view(np.uint64)[~np.isnan(a)], b.view(np.uint64)[~np.isnan(b)]), "%s: values differ" % what


def _offset(rng, deg, metres):
    T = np.eye(4)
    ax, dr = rng.standard_normal(3), rng.standard_normal(3)
    T[:3, :3] = track.rodrigues(math.radians(deg) * ax / np.linalg.norm(ax))
    T[:3, 3] = metres * dr / np.linalg.norm(dr)
    return T


def _frame(H, W, k=2, seed=0):
    """(cal, noisy disparity with holes, rendered-like depth with NaN holes) of the planes seen from posed frame k"""
    rng = np.random.default_rng(seed)
    cal = dataio.Calib(float(W), W / 2 - 0.25, H / 2 + 0.5, synth.POSED_B, 0.0, None, None)
    P = synth.posed_camera_poses(k + 1)[k]
    Z = synth.posed_render(P, H, W, cal.f, cal.cx, cal.cy)[0]
    disp = (np.float32(cal.f * cal.baseline) / Z * (1 + 1e-4 * rng.standard_normal(Z.shape))).astype(np.float32)
    disp[rng.random(disp.shape) < 0.08] = np.nan
    disp[rng.random(disp.shape) < 0.02] = -1.0
    Zm = (Z * (1 + 1e-4 * rng.standard_normal(Z.shape))).astype(np.float32)
    Zm[rng.random(Zm.shape) < 0.08] = np.nan
    Zm[~np.isfinite(Zm)] = np.nan
    return cal, disp, Zm


@pytest.mark.parametrize("H,W", [(53, 91), (96, 320), (7, 5)])
def test_pyramids_are_the_oracle(H, W):
    cal, disp, Zm = _frame(H, W, seed=H)
    for max_depth in (None, 12.0):
        with track.Tracker(H, W) as tr:
            tr.source(cu(disp), cal, max_depth)
            tr.model(cu(Zm), cal)
            src, mod = to.source_pyramid(disp, cal, max_depth), to.model_pyramid(Zm, cal)
            for level in range(3):
                for which, ref in (("source", src), ("model", mod)):
                    V, N = tr.maps(which, level)
                    same_bits(V, ref[level][0], "%dx%d %s level %d vertices" % (H, W, which, level))
                    same_bits(N, ref[level][1], "%dx%d %s level %d normals" % (H, W, which, level))
            if H * W > 1000 and max_depth is None:
                assert (~np.isnan(src[0][1][0])).sum() > H * W // 2


def test_sums_and_counts_are_the_oracle():
    rng = np.random.default_rng(5)
    H, W = 150, 331                               # several chunks at level 0, a partial last chunk at every level
    cal, disp, Zm = _frame(H, W, seed=9)
    src, mod = to.source_pyramid(disp, cal), to.model_pyramid(Zm, cal)
    empty = to.model_pyramid(np.full_like(Zm, np.nan), cal)
    with track.Tracker(H, W) as tr:
        tr.source(cu(disp), cal)
        cases = [(np.eye(4), 0.5, COS30)] + [(_offset(rng, 2.0 * k, 0.1 * k), 0.25 * k, COS30) for k in range(1, 5)]
        shift, behind = np.eye(4), np.eye(4)
        shift[0, 3], behind[2, 3] = 0.05, -100.0
        cases += [(shift, 1e-9, COS30), (behind, 1.0, COS30)]     # every pixel rejected: no pair that near; q_z < 0
        for model, ref in (("rendered", mod), ("empty", empty)):
            tr.model(cu(Zm if model == "rendered" else np.full_like(Zm, np.nan)), cal)
            for k, (T, delta, cos_t) in enumerate(cases):
                for level in range(3):
                    got = tr.step(level, T, delta, cos_t)
                    want = to.step(src, ref, cal, level, T[:3].reshape(12), delta, cos_t)
                    what = "%s model case %d level %d" % (model, k, level)
                    assert got[1:] == want[1:], "%s: counts %s vs %s" % (what, got[1:], want[1:])
                    assert np.array_equal(got[0].view(np.uint64), want[0].view(np.uint64)), what
                    if model == "rendered" and k == 0:
                        assert got[1] > 0.3 * got[3], what
                    if model == "empty" or k >= 5:
                        assert got[1] == 0 and not got[0].any(), what


def test_abi_refusals():
    lib = adcensus.lib()
    h = ctypes.c_void_p()
    for H, W, dev in ((0, 5, 0), (5, 0, 0), (5, 5, -1), (5, 5, 1 << 20)):
        assert lib.mccnn_track_create(ctypes.byref(h), H, W, dev) == -1
    assert lib.mccnn_track_create(ctypes.byref(h), 1 << 16, 1 << 15, 0) == -2
    assert lib.mccnn_track_create(ctypes.byref(h), 4, 5, 0) == 0
    s = torch.cuda.current_stream().cuda_stream
    sums, counts = np.zeros(28), np.zeros(3, np.int64)
    pose = np.eye(4)[:3].reshape(-1).copy()
    step = (h, 0, pose.ctypes.data, 0.5, 0.5, None, sums.ctypes.data, counts.ctypes.data, s)
    assert lib.mccnn_track_step(*step) == -1                      # no pyramids yet
    d = torch.ones((4, 5), device="cuda")
    V = torch.empty(3 * 20, dtype=torch.float64, device="cuda")
    assert lib.mccnn_track_maps(h, 0, 0, V.data_ptr(), V.data_ptr(), s) == -1
    src = (h, d.data_ptr(), 2.0, 2.0, 2.0, 1.0, 0.0, float("inf"), s)
    for k, v in ((0, None), (1, None), (2, 0.0), (3, float("nan")), (5, -1.0), (6, float("inf")), (7, 0.0)):
        args = list(src)
        args[k] = v
        assert lib.mccnn_track_source(*args) == -1, "source argument %d = %r" % (k, v)
    assert lib.mccnn_track_source(*src) == 0
    assert lib.mccnn_track_step(*step) == -1                      # no model yet
    for k, v in ((0, None), (1, None), (2, -1.0), (4, float("inf"))):
        args = list((h, d.data_ptr(), 2.0, 2.0, 2.0, s))
        args[k] = v
        assert lib.mccnn_track_model(*args) == -1, "model argument %d = %r" % (k, v)
    assert lib.mccnn_track_model(h, d.data_ptr(), 2.0, 2.0, 2.0, s) == 0
    bad_pose = pose.copy()
    bad_pose[3] = np.nan
    for k, v in ((0, None), (1, -1), (1, 3), (2, None), (2, bad_pose.ctypes.data), (3, 0.0), (3, float("inf")), (4, 1.5),
                 (4, float("nan")), (6, None), (7, None)):
        args = list(step)
        args[k] = v
        assert lib.mccnn_track_step(*args) == -1, "step argument %d = %r" % (k, v)
    assert lib.mccnn_track_step(*step) == 0
    for which, level in ((2, 0), (-1, 0), (0, 3)):
        assert lib.mccnn_track_maps(h, which, level, V.data_ptr(), V.data_ptr(), s) == -1
    assert lib.mccnn_track_maps(h, 1, 0, None, V.data_ptr(), s) == -1
    lib.mccnn_track_destroy(h)
    with track.Tracker(4, 5) as tr:
        with pytest.raises(ValueError, match="is 3x5"):
            tr.source(torch.ones((3, 5), device="cuda"), dataio.Calib(2.0, 2.0, 2.0, 0.5, 0.0, None, None))
    with pytest.raises(ValueError, match="closed"):
        tr.step(0, np.eye(4), 0.5, 0.5)


def gpu_track_drive(disps, imgs, cal, voxel, trunc=None, mode="track", oxts=None, max_depth=None):
    """fuse_drive's tracked loop over maps already on hand, on the GPU: (poses, lost frame indices, the TSDF)"""
    H, W = disps[0].shape
    ts, tr = fusion.TSDF(voxel, trunc), track.Tracker(H, W)
    poses, lost = [], []
    for k, (d, img) in enumerate(zip(disps, imgs)):
        if k == 0:
            pose = np.eye(4)
        else:
            Z = ts.render(cal, poses[-1], H, W, 1, max_depth)
            pose, _, is_lost = tr.track(cu(d), cal, Z, poses[-1], track.predict(mode, poses, oxts), max_depth)
            if is_lost:
                lost.append(k)
                poses.append(pose)
                continue
        ts.add(cu(d), cal, img, pose, max_depth=max_depth)
        poses.append(pose)
    tr.close()
    return poses, lost, ts


def same_table(ts, ref, what):
    t = ts.table()
    assert np.array_equal(t.keys, ref.keys), what
    assert np.array_equal(t.S.reshape(-1, 512).view(np.uint64), ref.S.view(np.uint64)), what
    assert np.array_equal(t.n.reshape(-1, 512), ref.n) and np.array_equal(t.nc.reshape(-1, 512), ref.nc), what
    assert np.array_equal(t.colours.reshape(-1, 512, 3), ref.col), what


def _posed(tmp_path, n, H, W):
    drive, disps, _, truth = synth.write_kitti_posed_drive(str(tmp_path), n=n, H=H, W=W)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    imgs = [png(dataio.raw_file(drive, dataio.RAW_LEFT, k)) for k in range(n)]
    return drive, disps, imgs, truth, cal


def test_tracked_drive_is_the_oracle(tmp_path):
    """5 frames at 96 x 320: every pose and the field bit for bit, and a second run with the same bits"""
    _, disps, imgs, truth, cal = _posed(tmp_path, 5, 96, 320)
    want, wlost, ref = to.track_drive(track, disps, imgs, cal, 0.05, 0.2)
    runs = []
    for r in range(2):
        poses, lost, ts = gpu_track_drive(disps, imgs, cal, 0.05, 0.2)
        assert lost == wlost == []
        for k, (a, b) in enumerate(zip(poses, want)):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), "run %d pose %d" % (r, k)
        same_table(ts, ref, "run %d" % r)
        t = ts.table()
        runs.append((np.stack(poses).tobytes(), t.keys.tobytes(), t.S.tobytes()))
        ts.close()
    assert runs[0] == runs[1]


def _errors(poses, truth):
    out = []
    for P, G in zip(poses, truth):
        E = track.rigid_inv(G) @ P
        out.append((float(np.linalg.norm(E[:3, 3])), math.degrees(track.rotation_angle(E[:3, :3]))))
    return np.array(out)


# v = 0.05 m: every pose within v / 5 and 0.05 degrees of the truth.  160 x 320 with f = 320 gives a vertical half field of
# view of 14 degrees, KITTI's (375 rows at f 721 give 14.6), so the ground, the only plane fixing the height, spans rows
BOUND_T, BOUND_R = 0.01, 0.05
ACC_H, ACC_W = 160, 320


def test_track_accuracy(tmp_path):
    _, disps, imgs, truth, cal = _posed(tmp_path, 5, ACC_H, ACC_W)
    poses, lost, ts = gpu_track_drive(disps, imgs, cal, 0.05, 0.2)
    e = _errors(poses, truth)
    print("track: max %.5f m, %.5f deg; per frame %s" % (e[:, 0].max(), e[:, 1].max(), e.round(5).tolist()))
    assert lost == [] and e[:, 0].max() < BOUND_T and e[:, 1].max() < BOUND_R
    ts.close()


def test_refine_accuracy_and_a_lost_frame(tmp_path):
    """refine from OXTS poses off by 0.1 m and 1 degree; then a drive whose frame 2 has no disparity: lost, nothing
    integrated, and the later frames still within the bounds"""
    drive, disps, imgs, truth, cal = _posed(tmp_path, 5, ACC_H, ACC_W)
    rng = np.random.default_rng(11)
    oxts = dataio.raw_poses(drive, range(5))
    noisy = [oxts[0]] + [O @ _offset(rng, 1.0, 0.1) for O in oxts[1:]]
    poses, lost, ts = gpu_track_drive(disps, imgs, cal, 0.05, 0.2, "refine", noisy)
    e = _errors(poses, truth)
    print("refine: max %.5f m, %.5f deg; per frame %s" % (e[:, 0].max(), e[:, 1].max(), e.round(5).tolist()))
    assert lost == [] and e[:, 0].max() < BOUND_T and e[:, 1].max() < BOUND_R
    ts.close()
    holed = list(disps)
    holed[2] = np.full_like(disps[2], np.nan)
    ts_a, tr = fusion.TSDF(0.05, 0.2), track.Tracker(ACC_H, ACC_W)
    for k in range(2):
        ts_a.add(cu(disps[k]), cal, imgs[k], poses[k])
    before = ts_a.table()
    pose, inliers, is_lost = tr.track(cu(holed[2]), cal, ts_a.render(cal, poses[1], ACC_H, ACC_W), poses[1], poses[1])
    assert is_lost and inliers == 0 and np.array_equal(pose, poses[1])
    ts_a.close()
    tr.close()
    poses, lost, ts = gpu_track_drive(holed, imgs, cal, 0.05, 0.2)
    assert lost == [2]
    e = _errors(poses, truth)
    print("track with frame 2 lost: per frame %s" % e.round(5).tolist())
    assert e[3:, 0].max() < BOUND_T and e[3:, 1].max() < BOUND_R
    ref = fusion.TSDF(0.05, 0.2)
    for k in (0, 1, 3, 4):
        ref.add(cu(disps[k]), cal, imgs[k], poses[k])
    a, b = ts.table(), ref.table()
    assert np.array_equal(a.keys, b.keys) and np.array_equal(a.S.view(np.uint64), b.S.view(np.uint64))
    assert len(before.keys) <= len(a.keys)
    ts.close()
    ref.close()


def test_fuse_raw_tracked_is_the_oracle(tmp_path, capsys, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    n, H, W, voxel = 4, 96, 192, 0.08
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=n, H=H, W=W, velodyne=True)
    out = str(tmp_path / "out")
    argv = ["kitti", "census", "-drive", drive, "-out", out, "-voxel", str(voxel), "-disp_max", "64", "-mesh", "-poses",
            "track", "-traj", "-score"]
    assert fuse_tool.main(argv) == 0
    lines = capsys.readouterr().out.splitlines()
    name = "2011_09_26/%s" % predict_raw.drive_name(drive)
    frames = predict_raw.drive_frames([drive])
    files = predict_raw.pair_files(frames)
    shapes = predict_kitti.scan(files)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    run = predict_kitti.PairRunner(files, shapes, "kitti", "census", None, 64, 0, 0, 1)
    preds, lefts = [], []
    try:
        run.prepare()
        for i in range(n):
            left, _, _, pred, _ = run.predict(i)
            preds.append(pred.clone())
            lefts.append(left)
    finally:
        run.close()
    want, wlost, ref = to.track_drive(track, [p.cpu().numpy() for p in preds], lefts, cal, voxel)
    assert lines[:n] == ["%s %010d" % (name, k) + (" lost" if k in wlost else "") for k in range(n)]
    d = os.path.join(out, predict_raw.drive_name(drive))
    track.write_poses(str(tmp_path / "want.txt"), want)
    assert open(os.path.join(d, "poses.txt"), "rb").read() == open(str(tmp_path / "want.txt"), "rb").read()
    assert open(os.path.join(d, "mesh.ply"), "rb").read() == ref.mesh_ply(1)
    xyz, _, faces = ref.mesh(1)
    assert lines[n] == "%s: frames %d pixels %d outside 0 bricks %d vertices %d faces %d" % (
        name, n - len(wlost), ref.pixels, len(ref.keys), len(xyz), len(faces))
    m = track.trajectory_metrics(want, dataio.raw_poses(drive, range(n)))
    assert lines[n + 1] == track.metrics_line(name, m)
    print("census -poses track: %s (voxel %g m)" % (lines[n + 1], voxel))
    assert math.isfinite(m.ate) and wlost == []
    rows = []
    for i in range(n):
        gt = depth_eval.lidar_gt(dataio.read_velodyne(dataio.raw_file(drive, dataio.RAW_SCAN, i)), cal, H, W,
                                 torch.device("cuda", 0), depth.MIN_DEPTH, "none")
        Z = cu(ref.render(cal, want[i], H, W))
        rows.append(list(depth.metrics(preds[i], gt, cal)) + list(depth.metrics(Z, gt, cal, is_depth=True)))
        assert lines[n + 2 + i] == depth_eval.line("%s %010d" % (name, i), rows[-1])
    mean = [sum(r[j] for r in rows) / n for j in range(18)]
    assert lines[2 * n + 2] == depth_eval.line("mean", mean)
    with pytest.raises(ValueError, match="mesh.ply exists"):
        fuse_tool.main(argv)


def test_track_runs_without_oxts(tmp_path, capsys, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=3, H=48, W=160, no_oxts=True)
    out = str(tmp_path / "out")
    assert fuse_tool.main(["kitti", "census", "-drive", drive, "-out", out, "-voxel", "0.1", "-disp_max", "64", "-mesh",
                           "-poses", "track"]) == 0
    poses = track.read_poses(os.path.join(out, predict_raw.drive_name(drive), "poses.txt"))
    assert len(poses) == 3 and np.array_equal(poses[0], np.eye(4))
