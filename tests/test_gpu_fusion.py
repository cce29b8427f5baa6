"""GPU: world-frame fusion (DESIGN §23) -- mccnn_fusion_* bit for bit against the numpy restatement (tests/fusion_oracle.py):
the table's keys, counts, float64 and colour sums and the PLY bytes, grey and RGB, several frames, an empty frame, one long
run, the ±2^20 key edges, table growth across reallocations and each min_frames; run to run; posed planes of the
synthetic drive fused from their exact disparities at their OXTS poses lie on their planes; and tools/fuse_raw.py with
census equals the oracle fused from the same predicted maps and poses."""
import ctypes
import importlib.util
import os
import shutil

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, confidence, dataio, depth, fusion, predict_kitti, predict_raw, synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


fo = _load("fusion_oracle", "tests", "fusion_oracle.py")
fuse_tool = _load("fuse_raw_tool", "tools", "fuse_raw.py")
KITTI = dataio.Calib(721.5377, 609.5593, 172.854, 0.5372, 0.0, None, None)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pose(rng, rot=0.2, trans=1.0):
    P = np.eye(4)
    P[:3, :3] = synth._rodrigues(rng.uniform(-1, 1, 3) * rot)
    P[:3, 3] = rng.uniform(-trans, trans, 3)
    return P


def _disp(rng, H, W, lo=5.0, hi=120.0, holes=0.1):
    d = rng.uniform(lo, hi, (H, W)).astype(np.float32)
    d[rng.random((H, W)) < holes] = np.nan
    d[rng.random((H, W)) < holes / 4] = -3.0
    return d


def same_table(fu, ref, what):
    t = fu.table()
    assert np.array_equal(t.keys, ref.keys), "%s: keys differ (%d vs %d voxels)" % (what, len(t.keys), len(ref.keys))
    assert np.array_equal(t.n_pix, ref.n_pix), "%s: n_pix" % what
    assert np.array_equal(t.n_frames, ref.n_frames), "%s: n_frames" % what
    bad = t.sums.view(np.uint64) != ref.sums.view(np.uint64)
    assert not bad.any(), "%s: %d float64 sums differ" % (what, int(bad.sum()))
    assert np.array_equal(t.colours, ref.colours), "%s: colour sums" % what
    st = fu.stats
    assert (st.pixels, st.outside, st.voxels) == (ref.pixels, ref.outside, len(ref.keys)), what


def same_cloud(fu, ref, tmp_path, what, frames=(1, 2, 3)):
    for m in frames:
        pts = fu.cloud(m)
        p = str(tmp_path / ("m%d.ply" % m))
        depth.write_ply(p, pts)
        want = depth.ply_bytes(int((ref.n_frames >= m).sum())) + ref.records(m)
        assert open(p, "rb").read() == want, "%s: PLY bytes differ at min_frames %d" % (what, m)


def run_both(frames, voxel, max_depth=None):
    fu, ref = fusion.Fusion(voxel), fo.Table(voxel)
    for d, cal, img, pose in frames:
        fu.add(cu(d), cal, img, pose, max_depth=max_depth)
        ref.add(d, cal, img, pose, max_depth)
    return fu, ref


@pytest.mark.parametrize("rgb", [False, True])
def test_frames_are_the_oracle(rgb, tmp_path):
    rng = np.random.default_rng(11 + rgb)
    H, W = 375, 1242
    frames = []
    for k in range(4):
        img = rng.integers(0, 256, (H, W, 3) if rgb else (H, W), dtype=np.uint8)
        frames.append((_disp(rng, H, W), KITTI, img, _pose(rng)))
    # a frame with no valid pixel, then one more real frame
    frames.insert(2, (np.full((H, W), np.nan, np.float32), KITTI, frames[0][2], _pose(rng)))
    for voxel, max_depth in ((0.2, None), (0.05, 30.0)):
        fu, ref = run_both(frames, voxel, max_depth)
        assert ref.n_frames.max() >= 3 and len(ref.keys) > 10000
        same_table(fu, ref, "rgb %s voxel %g" % (rgb, voxel))
        same_cloud(fu, ref, tmp_path, "rgb %s voxel %g" % (rgb, voxel), (1, 2, 3, 5, 6))
        assert fu.cloud(6).n == 0
        fu.close()


def test_empty_table_and_empty_frame(tmp_path):
    fu, ref = run_both([(np.full((7, 9), np.nan, np.float32), KITTI, np.zeros((7, 9), np.uint8), np.eye(4))], 0.1)
    assert fu.stats == fusion.FusionStats(0, 0, 0)
    same_table(fu, ref, "empty")
    pts = fu.cloud()
    assert pts.n == 0 and pts.data.numel() == 0
    fu.close()
    with fusion.Fusion(0.1) as fu:
        assert fu.cloud().n == 0 and len(fu.table().keys) == 0


def test_one_long_run():
    """every pixel of a full-size map in one voxel: one partial summed over 465750 pixels in row-major order"""
    rng = np.random.default_rng(5)
    H, W = 375, 1242
    d = rng.uniform(20, 21, (H, W)).astype(np.float32)
    P = np.eye(4)
    P[:3, 3] = 500.0                                                         # X and Y change sign: keep w in [0, 1000)
    frames = [(d, KITTI, rng.integers(0, 256, (H, W), dtype=np.uint8), P),
              (d[::-1].copy(), KITTI, rng.integers(0, 256, (H, W), dtype=np.uint8), P @ _pose(rng, 0.01, 0.1))]
    fu, ref = run_both(frames, 1000.0)
    assert len(ref.keys) == 1 and ref.n_pix[0] == 2 * H * W
    same_table(fu, ref, "one voxel")
    fu.close()


def test_key_range_edges(tmp_path):
    """w_x = Z + t0 and w_y = -Z + t1 with exact depths: indices at 2^20 - 1, 2^20, -2^20 and -2^20 - 1"""
    cal = dataio.Calib(1.0, 0.0, 0.0, 1.0, 0.0, None, None)                  # fB = 1: Z = 1 / d exactly
    levels = np.array([4.0, 2.0, 1.0, 0.5, 0.25, 1.0 / 3], np.float32)     # Z = 0.25 .. 4 and 3.0000002
    rng = np.random.default_rng(2)
    d = levels[rng.integers(0, len(levels), (33, 47))]
    img = rng.integers(0, 256, (33, 47), dtype=np.uint8)
    frames = []
    for voxel in (1.0, 0.5):
        e = 2.0 ** 20 * voxel
        for t0, t1 in ((e - 2 * voxel, 0.25), (0.25, -e + voxel), (-e - voxel / 2, 0.0), (0.0, e - 4 * voxel)):
            P = np.zeros((4, 4))
            P[0, 2], P[1, 2], P[3, 3] = 1.0, -1.0, 1.0
            P[0, 3], P[1, 3], P[2, 3] = t0, t1, 0.5
            frames.append((d, cal, img, P))
        fu, ref = run_both(frames[-4:], voxel)
        assert ref.outside > 0 and ref.pixels > 0
        ix, iy, _ = fusion.key_index(ref.keys)
        assert ix.max() == 2 ** 20 - 1 and iy.min() == -2 ** 20
        same_table(fu, ref, "edges voxel %g" % voxel)
        same_cloud(fu, ref, tmp_path, "edges voxel %g" % voxel)
        fu.close()


def test_table_growth_across_reallocations(tmp_path):
    """fine voxels: each frame brings hundreds of thousands of new ones, so the table is reallocated several times"""
    rng = np.random.default_rng(9)
    H, W = 375, 1242
    base = _disp(rng, H, W, 10, 90, 0.02)
    frames = [(base + np.float32(0.05 * k), KITTI, rng.integers(0, 256, (H, W), dtype=np.uint8), _pose(rng, 0.02, 0.05))
              for k in range(5)]
    fu, ref = fusion.Fusion(0.004), fo.Table(0.004)
    sizes = []
    for d, cal, img, pose in frames:
        fu.add(cu(d), cal, img, pose)
        ref.add(d, cal, img, pose)
        sizes.append(fu.stats.voxels)
        assert sizes[-1] == len(ref.keys)
    assert sizes[-1] > 4 * sizes[0] / 2 and sizes[0] > 100000
    same_table(fu, ref, "growth")
    same_cloud(fu, ref, tmp_path, "growth", (1, 2, 4))
    fu.close()


def test_confidence_density_and_device_left():
    rng = np.random.default_rng(4)
    H, W = 64, 96
    d = _disp(rng, H, W)
    conf = rng.uniform(0, 10, (H, W)).astype(np.float32)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    with fusion.Fusion(0.1) as fu:
        fu.add(cu(d), KITTI, cu(img), np.eye(4)[:3], conf=cu(conf), density=0.3)
        ref = fo.Table(0.1)
        ref.add(confidence.sparsify(cu(d), cu(conf), 0.3).cpu().numpy(), KITTI, img, np.eye(4))
        same_table(fu, ref, "density")


def test_runs_repeat_bit_for_bit(tmp_path):
    rng = np.random.default_rng(8)
    H, W = 375, 1242
    frames = [(_disp(rng, H, W), KITTI, rng.integers(0, 256, (H, W), dtype=np.uint8), _pose(rng)) for _ in range(3)]
    out = []
    for k in range(2):
        fu = fusion.Fusion(0.1)
        for d, cal, img, pose in frames:
            fu.add(cu(d), cal, img, pose)
        p = str(tmp_path / ("run%d.ply" % k))
        depth.write_ply(p, fu.cloud(2))
        t = fu.table()
        out.append((open(p, "rb").read(), t.keys.tobytes(), t.sums.tobytes(), t.colours.tobytes()))
        fu.close()
    assert out[0] == out[1]


def test_abi_refusals():
    lib = adcensus.lib()
    h = ctypes.c_void_p()
    for voxel, dev in ((0.0, 0), (-1.0, 0), (float("nan"), 0), (float("inf"), 0), (0.1, -1), (0.1, 1 << 20)):
        assert lib.mccnn_fusion_create(ctypes.byref(h), voxel, dev) == -1
    assert lib.mccnn_fusion_create(ctypes.byref(h), 0.1, 0) == 0
    d = torch.zeros((4, 5), device="cuda")
    img = torch.zeros((4, 5), dtype=torch.uint8, device="cuda")
    st = torch.zeros(3, dtype=torch.int64, device="cuda")
    d += 1.0
    pose = np.zeros(12)
    pose[3] = pose[7] = pose[11] = 0.05                                  # every point at (0.05, 0.05, 0.05): one voxel
    s = torch.cuda.current_stream().cuda_stream
    ok = (h, d.data_ptr(), img.data_ptr(), 1, 4, 5, 1.0, 2.0, 2.0, 1.0, 0.0, float("inf"), pose.ctypes.data, st.data_ptr(), s)
    bad_pose = pose.copy()
    bad_pose[5] = np.nan
    for k, v in ((0, None), (1, None), (2, None), (3, 2), (4, 0), (5, 0), (6, 0.0), (7, float("nan")), (9, -1.0),
                 (11, 0.0), (12, bad_pose.ctypes.data), (12, None), (13, None)):
        args = list(ok)
        args[k] = v
        assert lib.mccnn_fusion_add(*args) == -1, "argument %d = %r" % (k, v)
    assert lib.mccnn_fusion_add(*ok) == 0
    torch.cuda.synchronize()
    assert st.tolist() == [20, 0, 1] and lib.mccnn_fusion_size(h) == 1
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.mccnn_fusion_count(h, 0, cnt.data_ptr(), s) == -1
    assert lib.mccnn_fusion_fill(h, 0, None, 0, s) == -1
    assert lib.mccnn_fusion_fill(h, 1, None, 5, s) == -1
    assert lib.mccnn_fusion_table(h, None, None, None, None, None, s) == -1
    assert lib.mccnn_fusion_size(None) == -1
    lib.mccnn_fusion_destroy(h)
    with pytest.raises(ValueError, match="voxel must be"):
        fusion.Fusion(0.0)
    with fusion.Fusion(0.1) as fu:
        with pytest.raises(ValueError, match="conf and density go together"):
            fu.add(d, KITTI, img, np.eye(4), conf=d)
        with pytest.raises(ValueError, match="4x4 or 3x4"):
            fu.add(d, KITTI, img, np.eye(3))
    with pytest.raises(ValueError, match="closed"):
        fu.add(d, KITTI, img, np.eye(4))


def _plane_of(pts, k):
    n, off = synth.POSED_PLANES[k]
    return np.abs(pts @ np.asarray(n) - off)


def test_posed_planes_lie_on_their_planes(tmp_path):
    """the synthetic drive's exact disparities at the poses read from its OXTS files: every vertex whose voxel holds points
    of one plane only lies on that plane within 1e-4 m; the same maps at poses missing the IMU-to-velodyne extrinsics do not"""
    drive, disps, pids, poses = synth.write_kitti_posed_drive(str(tmp_path), n=5, H=96, W=320)
    date = os.path.dirname(drive)
    cal = dataio.read_calib(date, "kitti_raw")
    got = dataio.raw_poses(drive, range(5))
    lefts = [np.asarray(synth_png(dataio.raw_file(drive, dataio.RAW_LEFT, k))) for k in range(5)]
    voxel = 0.05

    def fuse(ps):
        fu, ref = fusion.Fusion(voxel), fo.Table(voxel)
        plane_sets = {}
        for d, img, P, pid in zip(disps, lefts, ps, pids):
            fu.add(cu(d), cal, img, P)
            ref.add(d, cal, img, P)
            w, idx = fo.world_points(d, cal, P)
            keys, keep, _ = fo.voxel_keys(w, voxel)
            for key, pl in zip(keys, pid.reshape(-1)[idx[keep]]):
                plane_sets.setdefault(int(key), set()).add(int(pl))
        return fu, ref, plane_sets

    fu, ref, plane_sets = fuse(got)
    same_table(fu, ref, "posed planes")
    xyz, _ = depth.read_ply(_write(fu.cloud(), tmp_path / "planes.ply"))
    single = np.array([len(plane_sets[int(k)]) == 1 for k in ref.keys])
    plane = np.array([min(plane_sets[int(k)]) for k in ref.keys])
    assert single.sum() > 5000 and (ref.n_frames[single] >= 3).sum() > 1000
    err = np.zeros(len(xyz))
    for k in range(len(synth.POSED_PLANES)):
        m = single & (plane == k)
        err[m] = _plane_of(xyz[m].astype(np.float64), k)
    assert err[single].max() < 1e-4, err[single].max()
    # the chain without the IMU-to-velodyne extrinsics (an identity calib_imu_to_velo.txt) puts the later frames elsewhere
    wrong_drive = os.path.join(str(tmp_path / "wrong"), os.path.basename(date), os.path.basename(drive))
    shutil.copytree(os.path.join(drive, "oxts"), os.path.join(wrong_drive, "oxts"))
    for name in (dataio.RAW_CAM, dataio.RAW_VELO):
        shutil.copy(os.path.join(date, name), os.path.dirname(wrong_drive))
    with open(os.path.join(os.path.dirname(wrong_drive), dataio.RAW_IMU), "w") as f:
        f.write("R: 1 0 0 0 1 0 0 0 1\nT: 0 0 0\n")
    wrong = dataio.raw_poses(wrong_drive, range(5))
    assert not np.allclose(wrong[-1], got[-1], atol=1e-3)
    t = fo.Table(voxel)
    sets_w = {}
    for d, img, P, pid in zip(disps, lefts, wrong, pids):
        t.add(d, cal, img, P)
        w, idx = fo.world_points(d, cal, P)
        keys, keep, _ = fo.voxel_keys(w, voxel)
        for key, pl in zip(keys, pid.reshape(-1)[idx[keep]]):
            sets_w.setdefault(int(key), set()).add(int(pl))
    xyz_w, _ = t.vertices()
    errs = [_plane_of(xyz_w[i:i + 1].astype(np.float64), min(sets_w[int(k)]))[0]
            for i, k in enumerate(t.keys) if len(sets_w[int(k)]) == 1]
    assert max(errs) > 1e-3
    fu.close()


def synth_png(path):
    from PIL import Image

    with Image.open(path) as im:
        return np.array(im)


def _write(pts, path):
    depth.write_ply(str(path), pts)
    return str(path)


def test_fuse_raw_is_the_oracle_of_its_maps(tmp_path, capsys, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=4, H=64, W=192)
    out = str(tmp_path / "out")
    argv = ["kitti", "census", "-drive", drive, "-out", out, "-voxel", "0.08", "-min_frames", "2", "-disp_max", "64"]
    assert fuse_tool.main(argv) == 0
    lines = capsys.readouterr().out.splitlines()
    name = "2011_09_26/%s" % predict_raw.drive_name(drive)
    assert lines[:4] == ["%s %010d" % (name, k) for k in range(4)]
    # the oracle over the same maps: the stereo method run again through the same runner
    frames = predict_raw.drive_frames([drive])
    files = predict_raw.pair_files(frames)
    shapes = predict_kitti.scan(files)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    poses = dataio.raw_poses(drive, range(4))
    run = predict_kitti.PairRunner(files, shapes, "kitti", "census", None, 64, 0, 0, 1)
    ref = fo.Table(0.08)
    try:
        run.prepare()
        for i in range(4):
            left, _, _, pred, _ = run.predict(i)
            ref.add(pred.cpu().numpy(), cal, left, poses[i])
    finally:
        run.close()
    assert lines[4] == "%s: frames 4 pixels %d outside 0 voxels %d vertices %d" % (name, ref.pixels, len(ref.keys),
                                                                                    int((ref.n_frames >= 2).sum()))
    want = depth.ply_bytes(int((ref.n_frames >= 2).sum())) + ref.records(2)
    assert open(os.path.join(out, predict_raw.drive_name(drive), "fused.ply"), "rb").read() == want
    assert (ref.n_frames >= 2).sum() > 1000
    with pytest.raises(ValueError, match="fused.ply exists"):
        fuse_tool.main(argv)
