"""GPU: the photometric term of tracking (DESIGN §26) -- mccnn_track_intensity / mccnn_track_step with gates bit for bit
against the numpy restatement (tests/track_photometric_oracle.py): intensity pyramids and gradients, the 56 sums and 3
counts at every level, the geometric half against the gate-less step, a whole tracked street drive twice; tools/fuse_raw.py
-photometric with census against the oracle loop, and -photometric 0 against no flag; the accuracy on a street, where
geometry alone cannot fix motion along it, and on the default drive."""
import ctypes
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, fusion, predict_kitti, predict_raw, synth, track  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


po = _load("track_photometric_oracle", "tests", "track_photometric_oracle.py")
to = po.track_oracle
fuse_tool = _load("fuse_raw_tool_gpu_track_photometric", "tools", "fuse_raw.py")
COS30 = math.cos(math.radians(30.0))
LAMBDA = 0.01
STREET_STEPS = (0.4, 0.55, 0.45, 0.6, 0.5)


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


def _frames(H, W, seed=0):
    """(cal, noisy disparity of frame 2 with holes, frame 1's depth with NaN holes, frame 2's and frame 1's grey images)"""
    rng = np.random.default_rng(seed)
    cal = dataio.Calib(float(W), W / 2 - 0.25, H / 2 + 0.5, synth.POSED_B, 0.0, None, None)
    poses = synth.posed_camera_poses(3)
    Z2, _, g2 = synth.posed_render(poses[2], H, W, cal.f, cal.cx, cal.cy)
    Z1, _, g1 = synth.posed_render(poses[1], H, W, cal.f, cal.cx, cal.cy)
    disp = (np.float32(cal.f * cal.baseline) / Z2 * (1 + 1e-4 * rng.standard_normal(Z2.shape))).astype(np.float32)
    disp[rng.random(disp.shape) < 0.08] = np.nan
    Zm = (Z1 * (1 + 1e-4 * rng.standard_normal(Z1.shape))).astype(np.float32)
    Zm[rng.random(Zm.shape) < 0.08] = np.nan
    Zm[~np.isfinite(Zm)] = np.nan
    byte = lambda g: np.clip(np.rint(g), 0, 255).astype(np.uint8)
    return cal, disp, Zm, byte(g2), byte(g1), poses


@pytest.mark.parametrize("H,W", [(53, 91), (96, 320), (7, 5)])
@pytest.mark.parametrize("nch", [1, 3])
def test_intensity_pyramids_are_the_oracle(H, W, nch):
    rng = np.random.default_rng(H * W + nch)
    shape = (H, W) if nch == 1 else (H, W, 3)
    imgs = [rng.integers(0, 256, shape, dtype=np.uint8) for _ in range(2)]
    with track.Tracker(H, W) as tr:
        tr.intensity("source", imgs[0])
        tr.intensity("reference", cu(imgs[1]))
        for which, img in (("source", imgs[0]), ("reference", imgs[1])):
            ref = po.pyramid(img)
            for level in range(3):
                I, gx, gy = tr.intensity_maps(which, level)
                same_bits(I, ref[level][0], "%dx%dx%d %s level %d I" % (H, W, nch, which, level))
                if which == "reference":
                    same_bits(gx, ref[level][1], "%s level %d g_x" % (which, level))
                    same_bits(gy, ref[level][2], "%s level %d g_y" % (which, level))
                else:
                    assert gx is None and gy is None


def test_sums_and_counts_are_the_oracle():
    rng = np.random.default_rng(5)
    H, W = 150, 331                               # several chunks at level 0, a partial last chunk at every level
    cal, disp, Zm, img, ref_img, poses = _frames(H, W, seed=9)
    T_true = track.rigid_inv(poses[1]) @ poses[2]
    src, mod = to.source_pyramid(disp, cal), to.model_pyramid(Zm, cal)
    empty = to.model_pyramid(np.full_like(Zm, np.nan), cal)
    isrc, iref = po.pyramid(img), po.pyramid(ref_img)
    with track.Tracker(H, W) as tr:
        tr.source(cu(disp), cal)
        tr.intensity("source", img)
        tr.intensity("reference", ref_img)
        cases = [(T_true, 0.5, COS30, 2.0, 30.0)]
        cases += [(T_true @ _offset(rng, 1.0 * k, 0.05 * k), 0.25 * k, COS30, 2.0, 30.0) for k in range(1, 4)]
        cases += [(T_true, 0.5, COS30, 0.0, 1e9), (T_true, 0.5, COS30, 7.5, 3.0)]
        shift, behind = np.eye(4), np.eye(4)
        shift[0, 3], behind[2, 3] = 0.05, -100.0
        # every pixel gated out: no pair that near; q_z < 0; no gradient that steep
        cases += [(shift, 1e-9, COS30, 2.0, 30.0), (behind, 1.0, COS30, 2.0, 30.0), (T_true, 0.5, COS30, 1e6, 30.0)]
        for model, mref in (("rendered", mod), ("empty", empty)):
            tr.model(cu(Zm if model == "rendered" else np.full_like(Zm, np.nan)), cal)
            for k, (T, delta, cos_t, g_min, rho) in enumerate(cases):
                for level in range(3):
                    got = tr.step(level, T, delta, cos_t, (g_min, rho))
                    want = po.step(src, mref, isrc, iref, cal, level, T[:3].reshape(12), delta, cos_t, g_min, rho)
                    what = "%s model case %d level %d" % (model, k, level)
                    assert got[1:] == want[1:], "%s: counts %s vs %s" % (what, got[1:], want[1:])
                    assert np.array_equal(got[0].view(np.uint64), want[0].view(np.uint64)), what
                    geo = tr.step(level, T, delta, cos_t)
                    assert np.array_equal(got[0][:28].view(np.uint64), geo[0].view(np.uint64)), what + ": geometric half"
                    assert (got[1], 0, got[3]) == geo[1:], what
                    if model == "rendered" and k == 0:
                        assert got[2] > 0.2 * got[3], what
                    if model == "empty" or k >= 6:
                        assert got[2] == 0 and not got[0][28:].any(), what


def test_abi_refusals():
    lib = adcensus.lib()
    h = ctypes.c_void_p()
    assert lib.mccnn_track_create(ctypes.byref(h), 6, 7, 0) == 0
    s = torch.cuda.current_stream().cuda_stream
    sums, counts, gates = np.zeros(56), np.zeros(3, np.int64), np.array([2.0, 30.0])
    pose = np.eye(4)[:3].reshape(-1).copy()
    step = (h, 0, pose.ctypes.data, 0.5, 0.5, gates.ctypes.data, sums.ctypes.data, counts.ctypes.data, s)
    img = torch.zeros((6, 7, 3), dtype=torch.uint8, device="cuda")
    I = torch.empty(42, dtype=torch.float32, device="cuda")
    G = torch.empty(42, dtype=torch.float64, device="cuda")
    assert lib.mccnn_track_intensity_maps(h, 0, 0, I.data_ptr(), None, None, s) == -1      # no pyramid yet
    for which, nch, p in ((2, 1, img.data_ptr()), (-1, 1, img.data_ptr()), (0, 2, img.data_ptr()), (0, 0, img.data_ptr()),
                          (0, 1, None)):
        assert lib.mccnn_track_intensity(h, which, p, nch, s) == -1, (which, nch)
    d = torch.ones((6, 7), device="cuda")
    assert lib.mccnn_track_source(h, d.data_ptr(), 2.0, 2.0, 2.0, 1.0, 0.0, float("inf"), s) == 0
    assert lib.mccnn_track_model(h, d.data_ptr(), 2.0, 2.0, 2.0, s) == 0
    assert lib.mccnn_track_step(*step) == -1                               # no intensity pyramids
    assert lib.mccnn_track_intensity(h, 0, img.data_ptr(), 3, s) == 0
    assert lib.mccnn_track_step(*step) == -1                               # no reference
    assert lib.mccnn_track_intensity(h, 1, img.data_ptr(), 1, s) == 0
    bad_pose = pose.copy()
    bad_pose[5] = np.inf
    inf, nan = float("inf"), float("nan")
    bad_gates = [np.array(g) for g in ((-1.0, 30.0), (inf, 30.0), (nan, 30.0), (2.0, -0.5), (2.0, inf), (2.0, nan))]
    for k, v in ((0, None), (1, -1), (1, 3), (2, None), (2, bad_pose.ctypes.data), (3, 0.0), (3, nan), (4, 1.5),
                 *((5, g.ctypes.data) for g in bad_gates), (6, None), (7, None)):
        args = list(step)
        args[k] = v
        assert lib.mccnn_track_step(*args) == -1, "step argument %d = %r" % (k, v)
    assert lib.mccnn_track_step(*step) == 0
    assert lib.mccnn_track_intensity_maps(h, 0, 0, I.data_ptr(), G.data_ptr(), G.data_ptr(), s) == -1   # the source has no g
    assert lib.mccnn_track_intensity_maps(h, 1, 0, I.data_ptr(), None, G.data_ptr(), s) == -1
    assert lib.mccnn_track_intensity_maps(h, 1, 3, I.data_ptr(), G.data_ptr(), G.data_ptr(), s) == -1
    assert lib.mccnn_track_intensity_maps(h, 1, 0, None, G.data_ptr(), G.data_ptr(), s) == -1
    assert lib.mccnn_track_intensity_maps(h, 1, 0, I.data_ptr(), G.data_ptr(), G.data_ptr(), s) == 0
    lib.mccnn_track_destroy(h)
    cal = dataio.Calib(7.0, 3.0, 3.0, 0.5, 0.0, None, None)
    with track.Tracker(6, 7, photometric=LAMBDA) as tr:
        for kw in (dict(), dict(left=img.cpu().numpy()), dict(ref_left=img)):
            with pytest.raises(ValueError, match="give left and ref_left"):
                tr.track(d, cal, d, np.eye(4), np.eye(4), **kw)
        with pytest.raises(ValueError, match=r"left image: \(6, 7\) or \(6, 7, 3\) uint8 expected"):
            tr.intensity("source", np.zeros((6, 7, 2), np.uint8))
    with track.Tracker(6, 7) as tr:
        with pytest.raises(ValueError, match="photometric weight is 0"):
            tr.track(d, cal, d, np.eye(4), np.eye(4), left=img, ref_left=img)


def gpu_track_drive(disps, imgs, cal, voxel, trunc=None, max_depth=None, photometric=LAMBDA):
    """fuse_drive's tracked loop with the photometric term over maps already on hand, on the GPU: (poses, lost frame
    indices, the TSDF)"""
    H, W = disps[0].shape
    ts, tr = fusion.TSDF(voxel, trunc), track.Tracker(H, W, photometric=photometric)
    poses, lost = [], []
    for k, (d, img) in enumerate(zip(disps, imgs)):
        if k == 0:
            pose = np.eye(4)
        else:
            Z = ts.render(cal, poses[-1], H, W, 1, max_depth)
            images = dict(left=img, ref_left=imgs[k - 1]) if photometric else {}
            pose, _, is_lost = tr.track(cu(d), cal, Z, poses[-1], track.predict("track", poses), max_depth, **images)
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


def _street(tmp_path, H, W, **kw):
    drive, disps, _, truth = synth.write_kitti_posed_drive(str(tmp_path), n=5, H=H, W=W, **kw)
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    imgs = [png(dataio.raw_file(drive, dataio.RAW_LEFT, k)) for k in range(5)]
    return drive, disps, imgs, truth, cal


def test_tracked_street_is_the_oracle(tmp_path):
    """5 street frames at 64 x 192 with the term: every pose and the field bit for bit, and a second run with the same
    bits"""
    _, disps, imgs, _, cal = _street(tmp_path, 64, 192, planes=synth.STREET_PLANES, step=STREET_STEPS)
    want, wlost, ref = po.track_drive(track, disps, imgs, cal, 0.05, 0.2, max_depth=30.0, photometric=LAMBDA)
    runs = []
    for r in range(2):
        poses, lost, ts = gpu_track_drive(disps, imgs, cal, 0.05, 0.2, max_depth=30.0)
        assert lost == wlost
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
        out.append((float(np.linalg.norm(E[:3, 3])), math.degrees(track.rotation_angle(E[:3, :3])),
                    float(abs((P[:3, 3] - G[:3, 3]) @ G[:3, 2]))))
    return np.array(out)


# §25's bounds: every pose within v / 5 (v = 0.05 m) and 0.05 degrees of the truth, at KITTI's vertical field of view
BOUND_T, BOUND_R = 0.01, 0.05
ACC_H, ACC_W = 160, 320


def test_street_accuracy(tmp_path):
    """geometry alone loses the street or slides along it; with the term every frame is within §25's bounds"""
    _, disps, imgs, truth, cal = _street(tmp_path, ACC_H, ACC_W, planes=synth.STREET_PLANES, step=STREET_STEPS)
    poses, lost, ts = gpu_track_drive(disps, imgs, cal, 0.05, 0.2, photometric=0.0)
    e = _errors(poses, truth)
    print("street, geometric only: lost %s; max along the street %.5f m; per frame %s" % (lost, e[:, 2].max(),
                                                                                          e.round(5).tolist()))
    assert lost or e[:, 2].max() > 0.1
    ts.close()
    poses, lost, ts = gpu_track_drive(disps, imgs, cal, 0.05, 0.2)
    e = _errors(poses, truth)
    print("street, photometric %g: max %.5f m, %.5f deg; per frame %s" % (LAMBDA, e[:, 0].max(), e[:, 1].max(),
                                                                          e.round(5).tolist()))
    assert lost == [] and e[:, 0].max() < BOUND_T and e[:, 1].max() < BOUND_R
    ts.close()


def test_default_drive_accuracy(tmp_path):
    _, disps, imgs, truth, cal = _street(tmp_path, ACC_H, ACC_W)
    poses, lost, ts = gpu_track_drive(disps, imgs, cal, 0.05, 0.2)
    e = _errors(poses, truth)
    print("default drive, photometric %g: max %.5f m, %.5f deg; per frame %s" % (LAMBDA, e[:, 0].max(), e[:, 1].max(),
                                                                                 e.round(5).tolist()))
    assert lost == [] and e[:, 0].max() < BOUND_T and e[:, 1].max() < BOUND_R
    ts.close()


def _fuse(drive, out, extra, capsys):
    argv = ["kitti", "census", "-drive", drive, "-out", out, "-voxel", "0.08", "-disp_max", "64", "-mesh", "-poses",
            "track"] + extra
    assert fuse_tool.main(argv) == 0
    return capsys.readouterr().out.splitlines()


def test_fuse_raw_photometric_is_the_oracle(tmp_path, capsys, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    n, H, W, voxel = 4, 96, 192, 0.08
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=n, H=H, W=W, planes=synth.STREET_PLANES,
                                                   step=STREET_STEPS[:n])
    out = str(tmp_path / "out")
    lines = _fuse(drive, out, ["-photometric", str(LAMBDA)], capsys)
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
            preds.append(pred.cpu().numpy())
            lefts.append(left.cpu().numpy() if isinstance(left, torch.Tensor) else np.asarray(left))
    finally:
        run.close()
    want, wlost, ref = po.track_drive(track, preds, lefts, cal, voxel, photometric=LAMBDA)
    assert lines[:n] == ["%s %010d" % (name, k) + (" lost" if k in wlost else "") for k in range(n)]
    d = os.path.join(out, predict_raw.drive_name(drive))
    track.write_poses(str(tmp_path / "want.txt"), want)
    assert open(os.path.join(d, "poses.txt"), "rb").read() == open(str(tmp_path / "want.txt"), "rb").read()
    assert open(os.path.join(d, "mesh.ply"), "rb").read() == ref.mesh_ply(1)
    print("census street -photometric %g: lost %s" % (LAMBDA, wlost))


def test_photometric_zero_is_no_flag(tmp_path, capsys, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=3, H=48, W=160)
    outs = []
    for k, extra in enumerate(([], ["-photometric", "0"])):
        out = str(tmp_path / ("out%d" % k))
        lines = _fuse(drive, out, extra, capsys)
        d = os.path.join(out, predict_raw.drive_name(drive))
        outs.append((lines, open(os.path.join(d, "poses.txt"), "rb").read(), open(os.path.join(d, "mesh.ply"), "rb").read()))
    assert outs[0] == outs[1]
