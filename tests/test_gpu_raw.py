"""GPU: KITTI raw drives (DESIGN §21) -- mccnn_velo_depth_map bit for bit against the numpy restatement
(tests/raw_oracle.py) with duplicates, ties, image edges, min_depth, empty and ~1M-point scans; predict_raw's files against
frontend.predict and depth.depth / depth.point_cloud of its maps; depth_eval's raw scores against depth.metrics per frame
and 0 for the true disparity; and two ranks against one."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, depth, depth_eval, frontend, predict_raw, synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ro = _load("raw_oracle", "tests", "raw_oracle.py")
KITTI_P = np.array([[609.6954, -721.5377, -1.2513, -123.0418], [180.3842, 7.6448, -719.6515, -101.0167],
                    [0.9999, 0.0001, 0.0105, -0.2694]])          # a velodyne-to-image matrix of KITTI's shape


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(got, want, what):
    g = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    assert g.shape == want.shape, what
    bad = g.view(np.uint32) != np.asarray(want, np.float32).view(np.uint32)
    assert not bad.any(), "%s: %d of %d pixels differ" % (what, int(bad.sum()), bad.size)


def _kitti_scan(rng, n):
    """a scan shaped like a Velodyne HDL-64 sweep: all around the car, 1-80 m, some of it below the ground"""
    r = rng.uniform(1, 80, n)
    a = rng.uniform(-np.pi, np.pi, n)
    pts = np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-3, 2, n), rng.uniform(0, 1, n)], 1).astype(np.float32)
    return pts


def _with_duplicates(rng, pts, k):
    """k points copied exactly (equal z: the index breaks the tie) and k moved along their ray (same pixel, other z)"""
    src = rng.integers(0, len(pts), 2 * k)
    exact = pts[src[:k]]
    ray = pts[src[k:]].copy()
    ray[:, :3] *= rng.uniform(0.5, 1.5, (k, 1)).astype(np.float32)
    out = np.concatenate([pts, exact, ray])
    return out[rng.permutation(len(out))]


@pytest.mark.parametrize("H, W, n", [(375, 1242, 120000), (370, 1226, 130000), (1, 1, 5000), (7, 13, 3000),
                                     (256, 8, 20000)])
def test_velo_depth_map_is_the_oracle(H, W, n):
    rng = np.random.default_rng(H * 7 + W)
    pts = _with_duplicates(rng, _kitti_scan(rng, n), n // 10)
    P = KITTI_P.copy()
    P[0, 2] += (W - 1242) / 2
    P[1, 2] += (H - 375) / 2
    for min_depth in (0.0, 1e-3, 5.0):
        got = depth.velo_depth(cu(pts), P.ravel(), H, W, min_depth)
        same(got, ro.velo_depth_map(pts, P, H, W, min_depth), "%dx%d min_depth %g" % (H, W, min_depth))


def test_velo_depth_map_edges_ties_and_min_depth():
    H, W = 20, 31
    P = np.array([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, 1.0, 0]])
    rows = []
    # every pixel of every edge, and just outside it (projected coordinates 0 and W + 1 / H + 1), at a few depths
    for z in (0.5, 2.0, 7.25):
        for u in range(0, W + 2):
            for v in (0, 1, H, H + 1):
                rows.append((u * z, v * z, z))
        for v in range(0, H + 2):
            for u in (0, 1, W, W + 1):
                rows.append((u * z, v * z, z))
    # coordinates half-way between pixels (ties to even), and the depth rule's edges
    for u in np.arange(0.5, W + 1, 1.0):
        rows.append((u * 4.0, 3 * 4.0, 4.0))
    for z in (0.0, -0.0, -1.0, 1e-3, np.float32(1e-3) + np.float32(1e-10), np.inf, np.nan, 1e-30):
        rows.append((5 * z, 5 * z, z))
    pts = np.concatenate([np.array(rows, np.float32), np.zeros((len(rows), 1), np.float32)], 1)
    pts = np.concatenate([pts, pts, pts[::-1]])                      # every pixel hit three times with equal z
    for min_depth in (0.0, 1e-3, 2.0, 7.25):
        got = depth.velo_depth(cu(pts), P.ravel(), H, W, min_depth)
        want = ro.velo_depth_map(pts, P, H, W, min_depth)
        same(got, want, "min_depth %g" % min_depth)
        if min_depth < 7.25:
            assert (want[0] > 0).all() and (want[-1] > 0).all() and (want[:, 0] > 0).all() and (want[:, -1] > 0).all()


def test_velo_depth_map_empty_million_and_run_to_run():
    rng = np.random.default_rng(11)
    got = depth.velo_depth(torch.empty((0, 4), device="cuda"), KITTI_P.ravel(), 375, 1242)
    assert got.shape == (375, 1242) and not got.any()
    pts = _with_duplicates(rng, _kitti_scan(rng, 1_000_000), 100_000)
    a = depth.velo_depth(cu(pts), KITTI_P.ravel(), 375, 1242)
    b = depth.velo_depth(cu(pts), KITTI_P.ravel(), 375, 1242)
    same(a, ro.velo_depth_map(pts, KITTI_P, 375, 1242, depth.MIN_DEPTH), "1.2M points")
    same(b, a.cpu().numpy(), "second run")
    # an offset view of a larger buffer is copied to an aligned one
    flat = cu(np.concatenate([np.zeros(1, np.float32), pts[:1000].ravel()]))
    same(depth.velo_depth(flat[1:].view(1000, 4), KITTI_P.ravel(), 375, 1242),
         ro.velo_depth_map(pts[:1000], KITTI_P, 375, 1242, depth.MIN_DEPTH), "offset view")


def test_velo_depth_map_refusals():
    lib, s = adcensus.lib(), torch.cuda.current_stream().cuda_stream
    pts = torch.zeros((4, 4), device="cuda")
    out = torch.empty((5, 6), device="cuda")
    P = np.asarray(KITTI_P, np.float32).ravel()
    call = lambda **k: lib.mccnn_velo_depth_map(k.get("pts", pts.data_ptr()), k.get("n", 4), k.get("P", P.ctypes.data),
                                                k.get("H", 5), k.get("W", 6), k.get("min_depth", 0.0), out.data_ptr(), s)
    assert call() == 0
    bad_P = P.copy()
    bad_P[5] = np.nan
    for kw in (dict(n=-1), dict(pts=None), dict(pts=pts.data_ptr() + 4), dict(P=None), dict(P=bad_P.ctypes.data), dict(H=0),
               dict(W=0), dict(min_depth=-1.0), dict(min_depth=float("nan")), dict(min_depth=float("inf"))):
        assert call(**kw) == -1, kw
    assert call(H=1 << 16, W=1 << 15) == -2
    assert call(n=1 << 32) == -2
    assert call(pts=None, n=0) == 0
    with pytest.raises(adcensus.AdcensusError, match=r"pts must be \(N, 4\)"):
        depth.velo_depth(torch.zeros((4, 3), device="cuda"), P, 5, 6)
    with pytest.raises(ValueError, match="min_depth must be >= 0"):
        depth.velo_depth(pts, P, 5, 6, -1.0)


# ---- the drive tools ----

D = 64


@pytest.fixture(scope="module")
def raw(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("raw"))
    d1, g1 = synth.write_kitti_drive(root, drive=1, n=3, H=40, W=150, seed=51)
    d2, g2 = synth.write_kitti_drive(root, drive=2, n=2, H=40, W=150, seed=52)
    return dict(root=root, drives=[d1, d2], gts={d1: g1, d2: g2})


def _read(p):
    with open(p, "rb") as f:
        return f.read()


def _frontend_map(fr):
    l, r = (dataio.raw_file(fr.drive, w, fr.index) for w in (dataio.RAW_LEFT, dataio.RAW_RIGHT))
    return frontend.predict(l, r, dataset="kitti", arch="census", disp_max=D)


def test_predict_raw_files_equal_frontend_predict(raw, tmp_path, capsys):
    out = str(tmp_path / "o")
    names = predict_raw.predict_raw("kitti", "census", raw["drives"], out=out, disp=True, depth=True, ply=True, disp_max=D)
    lines = capsys.readouterr().out.splitlines()
    frames = predict_raw.drive_frames(raw["drives"])
    assert lines == names == [predict_raw.frame_name(f) for f in frames] and len(frames) == 5
    assert sorted(os.listdir(out)) == sorted(os.path.basename(d) for d in raw["drives"])
    for fr in frames:
        m = _frontend_map(fr)
        want = str(tmp_path / "want.png")
        dataio.write_png16(m, want)
        assert _read(predict_raw.out_file(out, fr, "disp")) == _read(want), fr
        cal = dataio.read_calib(predict_raw.date_dir(fr.drive), "kitti_raw")
        dataio.write_depth_png16(depth.depth(cu(m), cal).cpu().numpy(), want)
        assert _read(predict_raw.out_file(out, fr, "depth")) == _read(want), fr
        pts = depth.point_cloud(cu(m), cal, frontend.load_bytes(dataio.raw_file(fr.drive, dataio.RAW_LEFT, fr.index)))
        assert _read(predict_raw.out_file(out, fr, "points")) == depth.ply_bytes(pts.n) + pts.data.cpu().numpy().tobytes()
    with pytest.raises(ValueError, match="not empty"):
        predict_raw.predict_raw("kitti", "census", raw["drives"], out=out, disp=True, disp_max=D)


def test_predict_raw_every_and_confidence(raw, tmp_path, capsys):
    from mccnn_b200 import confidence

    out = str(tmp_path / "o")
    predict_raw.predict_raw("kitti", "census", raw["drives"][:1], out=out, disp=True, confidence=True, density=0.3, every=2,
                            disp_max=D)
    capsys.readouterr()
    frames = predict_raw.drive_frames(raw["drives"][:1], every=2)
    assert [f.index for f in frames] == [0, 2]
    assert sorted(os.listdir(os.path.join(out, os.path.basename(raw["drives"][0]), "disp"))) == ["0000000000.png",
                                                                                                 "0000000002.png"]
    for fr in frames:
        m = _frontend_map(fr)
        conf = np.fromfile(predict_raw.out_file(out, fr, "conf"), "<f4").reshape(m.shape)
        sparse = confidence.sparsify(cu(m), cu(conf), 0.3, 0.0).cpu().numpy()
        want = str(tmp_path / "want.png")
        dataio.write_png16(sparse, want)
        assert _read(predict_raw.out_file(out, fr, "disp")) == _read(want)


def test_depth_eval_raw_scores_the_true_disparity_exactly(raw, tmp_path, capsys):
    out = str(tmp_path / "o")
    frames = predict_raw.drive_frames(raw["drives"], velodyne=True)
    for fr in frames:
        p = predict_raw.out_file(out, fr, "disp")
        os.makedirs(os.path.dirname(p), exist_ok=True)
        dataio.write_png16(raw["gts"][fr.drive][fr.index], p)
    tool = _load("depth_eval_tool_raw", "tools", "depth_eval.py")
    tool.main(["raw", "score", out] + [a for d in raw["drives"] for a in ("-drive", d)])
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == len(frames) + 1
    res = depth_eval.score_raw(frames, out, verbose=False)
    for row, line in zip(res.rows, lines):
        m = depth.DepthMetrics(*row)
        assert m.rmse == 0 and m.abs_rel == 0 and m.rmse_log == 0 and m.a1 == 1 and m.coverage == 1 and m.n > 100
    assert lines[-1] == depth_eval.line("mean", res.mean)


@pytest.mark.parametrize("crop", ["none", "garg"])
def test_depth_eval_raw_predict_equals_depth_metrics_per_frame(raw, tmp_path, capsys, crop):
    lst = tmp_path / "split.txt"
    frames = predict_raw.drive_frames(raw["drives"], velodyne=True)[::-1]
    lst.write_text("".join(predict_raw.frame_name(f) + "\n" for f in frames))
    tool = _load("depth_eval_tool_raw2", "tools", "depth_eval.py")
    tool.main(["raw", "predict", "kitti", "census", "-list", str(lst), "-data_root", raw["root"], "-disp_max", str(D),
               "-crop", crop, "-max_depth", "50"])
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == len(frames) + 1
    rows = []
    for fr, line in zip(frames, lines):
        cal = dataio.read_calib(predict_raw.date_dir(fr.drive), "kitti_raw")
        m = cu(_frontend_map(fr))
        scan = dataio.read_velodyne(dataio.raw_file(fr.drive, dataio.RAW_SCAN, fr.index))
        Z = depth.velo_depth(cu(scan), cal, 40, 150)
        if crop == "garg":
            t, b, l, r = depth_eval.crop_box("garg", 40, 150)
            keep = torch.zeros_like(Z)
            keep[t:b, l:r] = 1
            Z = Z * keep
        gt = depth.depth(Z, cal)
        rows.append(list(depth.metrics(m, gt, cal, 1e-3, 50.0)))
        assert line == depth_eval.line(predict_raw.frame_name(fr), rows[-1])
    mean = [sum(r[k] for r in rows) / len(rows) for k in range(len(depth_eval.RAW_COLUMNS))]
    assert lines[-1] == depth_eval.line("mean", mean)


# ---- two ranks give one rank's files and means ----

def _rank_main(rank, store, raw, out, result):
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method="file://" + store, rank=rank, world_size=2)
    try:
        names = predict_raw.predict_raw("kitti", "census", raw["drives"], out=out, disp=True, depth=True, ply=True,
                                        disp_max=D, verbose=False)
        frames = predict_raw.drive_frames(raw["drives"], velodyne=True)
        res = depth_eval.evaluate_raw("kitti", "census", frames, disp_max=D, verbose=False)
        if rank == 0:
            with open(result, "w") as f:
                json.dump(dict(names=names, rows=res.rows, mean=res.mean), f)
    finally:
        dist.destroy_process_group()


def _tree(out):
    got = {}
    for d, _, files in os.walk(out):
        for f in files:
            got[os.path.relpath(os.path.join(d, f), out)] = _read(os.path.join(d, f))
    return got


def test_two_ranks_give_the_files_and_means_of_one(raw, tmp_path):
    import torch.multiprocessing as mp

    one = str(tmp_path / "one")
    names = predict_raw.predict_raw("kitti", "census", raw["drives"], out=one, disp=True, depth=True, ply=True, disp_max=D,
                                    verbose=False)
    res = depth_eval.evaluate_raw("kitti", "census", predict_raw.drive_frames(raw["drives"], velodyne=True), disp_max=D,
                                  verbose=False)
    two, result = str(tmp_path / "two"), str(tmp_path / "result.json")
    mp.start_processes(_rank_main, args=(str(tmp_path / "store"), raw, two, result), nprocs=2, join=True,
                       start_method="spawn")
    with open(result) as f:
        got = json.load(f)
    assert got["names"] == names
    assert got["rows"] == res.rows and got["mean"] == res.mean
    a, b = _tree(one), _tree(two)
    assert sorted(a) == sorted(b) and len(a) == 15
    assert all(a[k] == b[k] for k in a)
