"""GPU: the truncated signed distance field (DESIGN §24) -- mccnn_tsdf_* bit for bit against the numpy restatement
(tests/tsdf_oracle.py): the table, the mesh PLY bytes and the rendered maps, grey and RGB, an empty frame, the ±2^20
brick-key edges and points beyond them, key and pool growth across reallocations, each min_frames and a second run; the
synthetic drive's planes fused from their exact disparities (vertices on their planes, renders at each pose against the
exact depth); free-space carving of a spurious block that §23's Fusion keeps; and tools/fuse_raw.py -mesh -score with census
against the oracle fused and rendered from the same predicted maps and poses."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, depth, depth_eval, fusion, predict_kitti, predict_raw, synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


to = _load("tsdf_oracle", "tests", "tsdf_oracle.py")
fuse_tool = _load("fuse_raw_tool", "tools", "fuse_raw.py")
CAL = dataio.Calib(160.0, 79.75, 24.5, 0.5, 0.0, None, None)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def png(path):
    from PIL import Image

    with Image.open(path) as im:
        return np.array(im)


def same_table(ts, ref, what):
    t = ts.table()
    assert np.array_equal(t.keys, ref.keys), "%s: keys differ (%d vs %d bricks)" % (what, len(t.keys), len(ref.keys))
    bad = t.S.reshape(-1, 512).view(np.uint64) != ref.S.view(np.uint64)
    assert not bad.any(), "%s: %d float64 S differ" % (what, int(bad.sum()))
    assert np.array_equal(t.n.reshape(-1, 512), ref.n), "%s: n" % what
    assert np.array_equal(t.nc.reshape(-1, 512), ref.nc), "%s: nc" % what
    assert np.array_equal(t.colours.reshape(-1, 512, 3), ref.col), "%s: colour sums" % what
    st = ts.stats
    assert (st.pixels, st.outside, st.bricks) == (ref.pixels, ref.outside, len(ref.keys)), what
    assert st.pool_bytes >= st.bricks * 14336


def same_mesh(ts, ref, tmp_path, what, frames=(1, 2, 3)):
    for m in frames:
        p = str(tmp_path / ("m%d.ply" % m))
        depth.write_mesh_ply(p, ts.mesh(m))
        assert open(p, "rb").read() == ref.mesh_ply(m), "%s: mesh PLY bytes differ at min_frames %d" % (what, m)


def same_render(ts, ref, cal, pose, H, W, what, min_frames=1, max_depth=None):
    got = ts.render(cal, pose, H, W, min_frames, max_depth).cpu().numpy()
    want = ref.render(cal, pose, H, W, min_frames, max_depth)
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: hit pixels differ" % what
    assert np.array_equal(got.view(np.uint32)[~np.isnan(got)], want.view(np.uint32)[~np.isnan(want)]), "%s: depths differ" % what
    return want


def run_both(frames, voxel, trunc=None, max_depth=None):
    ts, ref = fusion.TSDF(voxel, trunc), to.Field(voxel, trunc)
    for d, cal, img, pose in frames:
        ts.add(cu(d), cal, img, pose, max_depth=max_depth)
        ref.add(d, cal, img, pose, max_depth)
    return ts, ref


def posed_frames(tmp_path, n=4, H=48, W=160, rgb=False, seed=0):
    drive, disps, _, poses = synth.write_kitti_posed_drive(str(tmp_path / ("raw%d" % seed)), n=n, H=H, W=W)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    rng = np.random.default_rng(seed)
    out = []
    for k, (d, P) in enumerate(zip(disps, poses)):
        img = png(dataio.raw_file(drive, dataio.RAW_LEFT, k))
        if rgb:
            img = np.stack([img, rng.integers(0, 256, img.shape, dtype=np.uint8), 255 - img], -1)
        d = d.copy()
        d[rng.random(d.shape) < 0.05] = np.nan
        out.append((d, cal, img, P))
    return out, cal


@pytest.mark.parametrize("rgb", [False, True])
def test_field_mesh_and_renders_are_the_oracle(rgb, tmp_path):
    frames, cal = posed_frames(tmp_path, rgb=rgb, seed=int(rgb))
    H, W = frames[0][0].shape
    frames.insert(2, (np.full((H, W), np.nan, np.float32), cal, frames[0][2], frames[1][3]))   # an empty frame
    for voxel, trunc, max_depth in ((0.1, None, None), (0.08, 0.5, 12.0)):
        ts, ref = run_both(frames, voxel, trunc, max_depth)
        what = "rgb %s voxel %g" % (rgb, voxel)
        assert ref.n.max() >= 3 and len(ref.keys) > 50
        same_table(ts, ref, what)
        same_mesh(ts, ref, tmp_path, what, (1, 2, 3, 6))
        assert ts.mesh(6).n == 0
        for k, (_, _, _, P) in enumerate(frames):
            Z = same_render(ts, ref, cal, P, H, W, "%s pose %d" % (what, k), 1)
            same_render(ts, ref, cal, P, H, W, "%s pose %d min_frames 3" % (what, k), 3)
            assert np.isfinite(Z).sum() > H * W // 4
        same_render(ts, ref, cal, frames[0][3], H, W, what + " max_depth", 1, 9.0)
        ts.close()


def test_empty_field():
    with fusion.TSDF(0.1) as ts:
        ts.add(cu(np.full((7, 9), np.nan, np.float32)), CAL, np.zeros((7, 9), np.uint8), np.eye(4))
        assert ts.stats[:3] == (0, 0, 0)
        m = ts.mesh()
        assert m.n == 0 and m.faces.shape == (0, 3)
        assert torch.isnan(ts.render(CAL, np.eye(4), 5, 6)).all()
        assert len(ts.table().keys) == 0


def test_key_range_edges(tmp_path):
    """w_x = Z + t0 and w_y = Y + t1 with exact depths near brick indices 2^20 - 1 and -2^20, and points beyond them"""
    cal = dataio.Calib(1.0, 0.0, 0.0, 1.0, 0.0, None, None)                  # fB = 1: Z = 1 / d exactly
    levels = np.array([4.0, 2.0, 1.0, 0.5, 0.25], np.float32)
    rng = np.random.default_rng(2)
    d = levels[rng.integers(0, len(levels), (9, 11))]
    img = rng.integers(0, 256, (9, 11), dtype=np.uint8)
    for voxel in (1.0, 0.5):
        e = 8.0 * 2 ** 20 * voxel
        frames = []
        for t0, t1 in ((e - 6 * voxel, 0.25), (0.25, -e + 3 * voxel), (-e - 2 * voxel, 0.0), (0.0, e - 9 * voxel)):
            P = np.zeros((4, 4))
            P[0, 2], P[1, 1], P[2, 0], P[3, 3] = 1.0, 1.0, 1.0, 1.0
            P[0, 3], P[1, 3], P[2, 3] = t0, t1, 0.5
            frames.append((d, cal, img, P))
        ts, ref = run_both(frames, voxel)
        b = to.brick_index(ref.keys)
        assert ref.outside > 0 and b[:, 0].max() == 2 ** 20 - 1 and b[:, 1].min() == -2 ** 20
        same_table(ts, ref, "edges voxel %g" % voxel)
        same_mesh(ts, ref, tmp_path, "edges voxel %g" % voxel, (1, 2))
        for k, (_, _, _, P) in enumerate(frames):
            same_render(ts, ref, cal, P, 9, 11, "edges voxel %g pose %d" % (voxel, k), max_depth=16.0)
        ts.close()


def test_growth_across_reallocations(tmp_path):
    """fine voxels and frames 20 m apart: each frame brings thousands of new bricks, so the keys and the pool are
    reallocated several times"""
    frames, cal = posed_frames(tmp_path, n=5, H=96, W=320, seed=7)
    ts, ref = fusion.TSDF(0.03), to.Field(0.03)
    sizes, pools = [], []
    for k, (d, c, img, P) in enumerate(frames):
        P = P.copy()
        P[0, 3] += 20.0 * k
        frames[k] = (d, c, img, P)
        ts.add(cu(d), c, img, P)
        ref.add(d, c, img, P)
        st = ts.stats
        sizes.append(st.bricks)
        pools.append(st.pool_bytes)
        assert st.bricks == len(ref.keys)
    print("bricks per frame %s, pool bytes %s" % (sizes, pools))
    assert sizes[-1] > 4 * sizes[0] and len(set(pools)) >= 3, (sizes, pools)
    same_table(ts, ref, "growth")
    H, W = frames[0][0].shape
    same_render(ts, ref, cal, frames[-1][3], H, W, "growth", max_depth=30.0)
    ts.close()


def test_runs_repeat_bit_for_bit(tmp_path):
    frames, cal = posed_frames(tmp_path, seed=3)
    out = []
    for k in range(2):
        ts = fusion.TSDF(0.1)
        for d, c, img, P in frames:
            ts.add(cu(d), c, img, P)
        p = str(tmp_path / ("run%d.ply" % k))
        depth.write_mesh_ply(p, ts.mesh(2))
        t = ts.table()
        Z = ts.render(cal, frames[1][3], *frames[0][0].shape).cpu().numpy()
        out.append((open(p, "rb").read(), t.keys.tobytes(), t.S.tobytes(), t.colours.tobytes(), Z.tobytes()))
        ts.close()
    assert out[0] == out[1]


def test_abi_refusals():
    lib = adcensus.lib()
    h = ctypes.c_void_p()
    for voxel, trunc, dev in ((0.0, 0.4, 0), (float("nan"), 0.4, 0), (0.1, 0.05, 0), (0.1, float("inf"), 0),
                              (0.1, float("nan"), 0), (0.1, 0.4, -1), (0.1, 0.4, 1 << 20)):
        assert lib.mccnn_tsdf_create(ctypes.byref(h), voxel, trunc, dev) == -1
    assert lib.mccnn_tsdf_create(ctypes.byref(h), 0.1, 100.0, 0) == -2
    assert lib.mccnn_tsdf_create(ctypes.byref(h), 0.1, 0.4, 0) == 0
    d = torch.ones((4, 5), device="cuda")
    img = torch.zeros((4, 5), dtype=torch.uint8, device="cuda")
    st = torch.zeros(2, dtype=torch.int64, device="cuda")
    pose = np.eye(4)[:3].reshape(-1).copy()
    s = torch.cuda.current_stream().cuda_stream
    ok = (h, d.data_ptr(), img.data_ptr(), 1, 4, 5, 1.0, 2.0, 2.0, 1.0, 0.0, float("inf"), pose.ctypes.data, st.data_ptr(), s)
    bad_pose = pose.copy()
    bad_pose[5] = np.inf
    for k, v in ((0, None), (1, None), (2, None), (3, 2), (4, 0), (5, 0), (6, 0.0), (7, float("nan")), (9, -1.0),
                 (11, 0.0), (12, bad_pose.ctypes.data), (12, None), (13, None)):
        args = list(ok)
        args[k] = v
        assert lib.mccnn_tsdf_add(*args) == -1, "argument %d = %r" % (k, v)
    assert lib.mccnn_tsdf_add(*ok) == 0
    torch.cuda.synchronize()
    assert st.tolist() == [20, 0] and lib.mccnn_tsdf_bricks(h) > 0
    cnt = torch.zeros(2, dtype=torch.int64, device="cuda")
    Z = torch.zeros((3, 3), device="cuda")
    assert lib.mccnn_tsdf_mesh_count(h, 0, cnt.data_ptr(), s) == -1
    assert lib.mccnn_tsdf_mesh_count(h, 1, None, s) == -1
    assert lib.mccnn_tsdf_mesh_fill(h, 0, None, 0, None, 0, s) == -1
    assert lib.mccnn_tsdf_mesh_fill(h, 1, None, 5, None, 0, s) == -1
    assert lib.mccnn_tsdf_mesh_fill(h, 1, None, 0, None, 5, s) == -1
    assert lib.mccnn_tsdf_mesh_fill(h, 1, Z.data_ptr(), 1 << 31, None, 0, s) == -2
    r = (h, 1, 3, 3, 1.0, 1.0, 1.0, float("inf"), pose.ctypes.data, Z.data_ptr(), s)
    for k, v in ((0, None), (1, 0), (2, 0), (3, 0), (4, 0.0), (5, float("nan")), (7, 0.0), (8, None), (9, None)):
        args = list(r)
        args[k] = v
        assert lib.mccnn_tsdf_render(*args) == -1, "render argument %d = %r" % (k, v)
    singular = np.zeros(12)
    assert lib.mccnn_tsdf_render(h, 1, 3, 3, 1.0, 1.0, 1.0, float("inf"), singular.ctypes.data, Z.data_ptr(), s) == -1
    assert lib.mccnn_tsdf_render(h, 1, 3, 3, 1.0, 1.0, 1.0, 10.0, singular.ctypes.data, Z.data_ptr(), s) == 0
    assert lib.mccnn_tsdf_table(h, None, None, None, None, None, s) == -1
    assert lib.mccnn_tsdf_bricks(None) == -1 and lib.mccnn_tsdf_pool_bytes(None) == -1
    lib.mccnn_tsdf_destroy(h)
    with fusion.TSDF(0.1) as ts:
        with pytest.raises(ValueError, match="conf and density go together"):
            ts.add(d, CAL, img, np.eye(4), conf=d)
        with pytest.raises(ValueError, match="min_frames"):
            ts.mesh(0)
    with pytest.raises(ValueError, match="closed"):
        ts.add(d, CAL, img, np.eye(4))


def _nearest_plane(w):
    return np.stack([np.abs(w @ np.asarray(n) - off) for n, off in synth.POSED_PLANES], 1)


def test_posed_planes(tmp_path):
    """exact disparities at the drive's OXTS poses: vertices whose neighbourhood (within 2 trunc) holds one plane lie within
    v/2 of it, and each pose's render is within v/2 of the exact depth in median"""
    n, H, W, voxel = 5, 96, 320, 0.05
    drive, disps, _, truth = synth.write_kitti_posed_drive(str(tmp_path), n=n, H=H, W=W)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    poses = dataio.raw_poses(drive, range(n))
    ts = fusion.TSDF(voxel)
    for k in range(n):
        ts.add(cu(disps[k]), cal, png(dataio.raw_file(drive, dataio.RAW_LEFT, k)), poses[k])
    m = ts.mesh()
    p = str(tmp_path / "planes.ply")
    depth.write_mesh_ply(p, m)
    xyz, _, faces = depth.read_mesh_ply(p)
    dist = _nearest_plane(xyz.astype(np.float64))
    one = (dist < 2 * ts.trunc).sum(1) == 1
    err = dist.min(1)[one]
    assert one.sum() > 2000 and len(faces) > 2000
    print("vertex-to-plane: max %.4f p99 %.4f m over %d vertices (bound v/2 = %.3f)" % (err.max(), np.percentile(err, 99),
                                                                                          len(err), voxel / 2))
    assert err.max() < voxel / 2
    for k in range(n):
        Z = ts.render(cal, poses[k], H, W).cpu().numpy().astype(np.float64)
        Zt = synth.posed_render(truth[k], H, W, cal.f, cal.cx, cal.cy)[0]
        both = np.isfinite(Z) & np.isfinite(Zt)
        dz = np.abs(Z[both] - Zt[both])
        print("pose %d: render |dZ| median %.4f p99 %.4f max %.4f m over %d pixels" % (k, np.median(dz), np.percentile(dz, 99),
                                                                                     dz.max(), both.sum()))
        assert both.sum() > H * W // 2 and np.median(dz) < voxel / 2
    ts.close()


def test_free_space_carves_a_spurious_block(tmp_path):
    """frame 0 sees a wall at 10 m with a block of spurious depths at 5 m; three more frames see the wall through it.  The
    block's voxels end with phi > 0 and no face lies near them; §23's Fusion with min_frames 1 keeps them"""
    H, W = 60, 80
    cal = dataio.Calib(100.0, 39.5, 29.5, 0.5, 0.0, None, None)
    fB = np.float32(50.0)
    wall = np.full((H, W), fB / np.float32(10.0), np.float32)
    first = wall.copy()
    first[20:40, 30:50] = fB / np.float32(5.0)
    img = np.full((H, W), 128, np.uint8)
    poses = []
    for k in range(4):
        P = np.eye(4)
        P[0, 3] = 0.05 * k
        poses.append(P)
    ts, fu = fusion.TSDF(0.1), fusion.Fusion(0.1)
    for k in range(4):
        for m in (ts, fu):
            m.add(cu(first if k == 0 else wall), cal, img, poses[k])
    t = ts.table()
    c = to.centres(t.keys, 0.1).reshape(-1, 3)
    n, S = t.n.reshape(-1), t.S.reshape(-1)
    block = (np.abs(c[:, 2] - 5.0) < 0.3) & (np.abs(c[:, 0]) < 0.5) & (np.abs(c[:, 1]) < 0.5)
    assert block.sum() > 100 and (n[block] == 4).all()
    assert (S[block] / n[block] > 0).all()
    p = str(tmp_path / "carved.ply")
    depth.write_mesh_ply(p, ts.mesh())
    xyz, _, _ = depth.read_mesh_ply(p)
    assert (xyz[:, 2] < 8.0).sum() == 0 and (np.abs(xyz[:, 2] - 10.0) < 0.2).sum() > 1000
    pts = fu.cloud(1)
    cloud = pts.data.cpu().numpy().view(np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))["xyz"]
    assert (cloud[:, 2] < 8.0).sum() > 50
    ts.close()
    fu.close()


def test_fuse_raw_mesh_and_score_are_the_oracle(tmp_path, capsys, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=4, H=64, W=192, velodyne=True)
    out = str(tmp_path / "out")
    argv = ["kitti", "census", "-drive", drive, "-out", out, "-voxel", "0.08", "-disp_max", "64", "-mesh", "-score",
            "-crop", "garg"]
    assert fuse_tool.main(argv) == 0
    lines = capsys.readouterr().out.splitlines()
    name = "2011_09_26/%s" % predict_raw.drive_name(drive)
    assert lines[:4] == ["%s %010d" % (name, k) for k in range(4)]
    frames = predict_raw.drive_frames([drive])
    files = predict_raw.pair_files(frames)
    shapes = predict_kitti.scan(files)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    poses = dataio.raw_poses(drive, range(4))
    run = predict_kitti.PairRunner(files, shapes, "kitti", "census", None, 64, 0, 0, 1)
    ref = to.Field(0.08)
    preds = []
    try:
        run.prepare()
        for i in range(4):
            left, _, _, pred, _ = run.predict(i)
            preds.append(pred.clone())
            ref.add(pred.cpu().numpy(), cal, left, poses[i])
    finally:
        run.close()
    assert open(os.path.join(out, predict_raw.drive_name(drive), "mesh.ply"), "rb").read() == ref.mesh_ply(1)
    xyz, _, faces = ref.mesh(1)
    assert lines[4] == "%s: frames 4 pixels %d outside 0 bricks %d vertices %d faces %d" % (name, ref.pixels, len(ref.keys),
                                                                                             len(xyz), len(faces))
    assert len(faces) > 1000
    rows = []
    for i in range(4):
        gt = depth_eval.lidar_gt(dataio.read_velodyne(dataio.raw_file(drive, dataio.RAW_SCAN, i)), cal, 64, 192,
                                 torch.device("cuda", 0), depth.MIN_DEPTH, "garg")
        Z = cu(ref.render(cal, poses[i], 64, 192))
        rows.append(list(depth.metrics(preds[i], gt, cal)) + list(depth.metrics(Z, gt, cal, is_depth=True)))
        assert lines[5 + i] == depth_eval.line("%s %010d" % (name, i), rows[-1])
        assert rows[-1][7] > 1000 and rows[-1][16] > 1000
    mean = [sum(r[j] for r in rows) / 4 for j in range(18)]
    assert lines[9] == depth_eval.line("mean", mean)
    print("\n".join(lines[5:10]))
    with pytest.raises(ValueError, match="mesh.ply exists"):
        fuse_tool.main(argv)
