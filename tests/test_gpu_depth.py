"""GPU: metric depth, point clouds and depth metrics (mc-cnn_b200/depth.py, csrc/depth.cu; DESIGN §20) -- depth, X and Y
bit for bit against the numpy float32 restatement (tests/depth_oracle.py) at KITTI and Middlebury sizes and at block edges;
the point cloud's bytes against numpy's packed row-major selection, with and without conf / density, at counts that cross
the scan's blocks, and past 2^31 bytes at sampled vertices; the metrics against the float64 oracle and run to run; and the
command-line tools on synthetic KITTI 2012 / 2015 and MiddEval3 trees with calibration files written here."""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import confidence, dataio, depth, evaluate, frontend, synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


do = _load("depth_oracle", "tests", "depth_oracle.py")
oc = _load("confidence_oracle", "tests", "confidence_oracle.py")

KITTI = dataio.Calib(721.5377, 609.5593, 172.854, 387.5744 / 721.5377, 0.0, None, None)
MB = dataio.Calib(1758.23, 829.15, 552.78, 0.178089, 147.24, None, None)
CHUNK = 2048                                        # pixels per block of csrc/depth.cu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(got, want, what):
    g = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    w = np.asarray(want).reshape(g.shape)
    bad = ~((g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w)))
    assert not bad.any(), "%s: %d of %d elements differ" % (what, int(bad.sum()), bad.size)


def disparities(rng, H, W, cal, lo=0.5, hi=200.0):
    """a map with the special values of the depth rule scattered over it"""
    d = rng.uniform(lo, hi, (H, W)).astype(np.float32)
    special = np.array([0.0, -cal.doffs, np.nan, np.inf, -np.inf, -1.0, 1e-30, -cal.doffs + 1e-3], np.float32)
    m = rng.random((H, W)) < 0.1
    d[m] = special[rng.integers(0, len(special), int(m.sum()))]
    return d


SHAPES = [(375, 1242), (994, 1482), (1, 1), (3, 255), (3, 256), (3, 257), (255, 8), (256, 8), (257, 8), (2, 1023),
          (2, 1024), (1, 2049)]


@pytest.mark.parametrize("H, W", SHAPES)
@pytest.mark.parametrize("cal, max_depth", [(KITTI, None), (KITTI, 80.0), (MB, None)], ids=["kitti", "kitti-cap", "mb"])
def test_depth_is_the_float32_restatement(H, W, cal, max_depth):
    d = disparities(np.random.default_rng(H * 7 + W), H, W, cal)
    Z, X, Y = depth.depth(cu(d), cal, max_depth=max_depth, xy=True)
    Zw, Xw, Yw = do.depth32(d, cal, max_depth)
    same(Z, Zw, "Z")
    same(X, Xw, "X")
    same(Y, Yw, "Y")
    same(depth.depth(cu(d), cal, max_depth=max_depth), Zw, "Z alone")
    with np.errstate(invalid="ignore"):
        ok = ~np.isnan(Zw) & (d.astype(np.float64) + cal.doffs > 1)     # away from the cancellation of d + doffs
    assert np.allclose(Zw[ok], do.depth64(d, cal, max_depth)[ok], rtol=2e-7, atol=0)


def test_depth_refusals():
    d = cu(np.ones((4, 4), np.float32))
    for bad in (KITTI._replace(f=0.0), KITTI._replace(baseline=-0.5), KITTI._replace(cx=float("nan"))):
        with pytest.raises(mccnn_b200.adcensus.AdcensusError, match="invalid argument"):
            depth.depth(d, bad)
    with pytest.raises(ValueError, match="max_depth"):
        depth.depth(d, KITTI, max_depth=0.0)


def _cloud_cases():
    rng = np.random.default_rng(5)
    H, W = 9, 1000                                  # 9000 pixels: five blocks, the last one partial
    dense = rng.uniform(1, 100, (H, W)).astype(np.float32)
    none = np.zeros((H, W), np.float32)
    one = none.copy()
    one[6, 777] = 3.5
    half = np.where(rng.random((H, W)) < 0.5, dense, np.float32(np.nan))
    edges = none.copy()                             # one valid pixel at each block's first and last index
    for b in range(0, H * W, CHUNK):
        edges.flat[b] = 2.0
        edges.flat[min(b + CHUNK, H * W) - 1] = 4.0
    return {"none": none, "one": one, "dense": dense, "half": half, "edges": edges}


@pytest.mark.parametrize("case", ["none", "one", "dense", "half", "edges"])
@pytest.mark.parametrize("colour", ["rgb", "grey"])
def test_point_cloud_bytes(case, colour):
    d = _cloud_cases()[case]
    H, W = d.shape
    rng = np.random.default_rng(6)
    left = rng.integers(0, 256, (H, W, 3) if colour == "rgb" else (H, W), dtype=np.uint8)
    pts = depth.point_cloud(cu(d), KITTI, left)
    want = do.cloud_records(d, KITTI, left)
    assert pts.n * 15 == len(want) == pts.data.numel()
    assert pts.data.cpu().numpy().tobytes() == want
    pm = depth.point_cloud(cu(d), KITTI, left, max_depth=10.0)
    assert pm.data.cpu().numpy().tobytes() == do.cloud_records(d, KITTI, left, 10.0)


@pytest.mark.parametrize("density", [1e-4, 0.3, 1.0])
def test_point_cloud_keeps_sparsify_pixels(density):
    rng = np.random.default_rng(7)
    H, W = 37, 301
    d = disparities(rng, H, W, MB, lo=-100.0)
    conf = rng.integers(0, 40, (H, W)).astype(np.float32) / 4      # ties, broken by the row-major index
    left = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    pts = depth.point_cloud(cu(d), MB, cu(left), conf=cu(conf), density=density)
    keep = np.zeros(H * W, bool)
    keep[oc.order(conf)[:confidence.n_keep(density, H, W)]] = True
    sparse = np.where(keep.reshape(H, W), d, np.float32(np.nan))
    assert pts.data.cpu().numpy().tobytes() == do.cloud_records(sparse, MB, left)


def test_point_cloud_past_2_31_bytes():
    H = W = 12000                                   # every pixel valid: 144e6 records, 2.16e9 bytes
    g = torch.Generator(device="cuda").manual_seed(8)
    d = torch.rand((H, W), device="cuda", generator=g) * 200 + 1
    left = torch.randint(0, 256, (H, W), device="cuda", dtype=torch.uint8, generator=g)
    pts = depth.point_cloud(d, KITTI, left)
    assert pts.n == H * W and pts.data.numel() == 15 * H * W > 2 ** 31
    n = H * W
    rec_at = lambda b: np.array([b // 15 + k for k in (-1, 0, 1)])
    idx = np.concatenate([[0, 1, n - 1], rec_at(2 ** 29), rec_at(2 ** 30), rec_at(2 ** 31), rec_at(2 ** 31 + 7),
                          np.random.default_rng(9).integers(0, n, 200)])
    idx = np.unique(idx[(idx >= 0) & (idx < n)])
    ys, xs = idx // W, idx % W
    dv = d[torch.from_numpy(ys).cuda(), torch.from_numpy(xs).cuda()].cpu().numpy()
    lv = left[torch.from_numpy(ys).cuda(), torch.from_numpy(xs).cuda()].cpu().numpy()
    z = np.float32(do.fB32(KITTI)) / (dv + np.float32(0))
    f, cx, cy = np.float32(KITTI.f), np.float32(KITTI.cx), np.float32(KITTI.cy)
    X = ((xs.astype(np.float32) - cx) * z) / f
    Y = ((ys.astype(np.float32) - cy) * z) / f
    rows = torch.from_numpy(idx[:, None] * 15 + np.arange(15)[None, :]).cuda()
    got = pts.data[rows].cpu().numpy()
    rec = np.empty(len(idx), np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))
    rec["xyz"] = np.stack([X, Y, z], 1)
    rec["rgb"] = np.repeat(lv[:, None], 3, 1)
    assert got.tobytes() == rec.tobytes()


@pytest.mark.parametrize("H, W", [(375, 1242), (994, 1482), (3, 2049), (1, 1)])
@pytest.mark.parametrize("cal, lo, hi", [(KITTI, 1e-3, 80.0), (MB, 1e-3, None), (KITTI, 5.0, 30.0)], ids=["kitti", "mb", "band"])
def test_metrics_equal_the_float64_oracle(H, W, cal, lo, hi):
    rng = np.random.default_rng(H + W)
    gt = disparities(rng, H, W, cal, lo=1.0, hi=150.0)
    gt[rng.random((H, W)) < 0.3] = 0.0 if cal is KITTI else np.inf
    pred = np.where(rng.random((H, W)) < 0.9, gt * rng.uniform(0.7, 1.4, (H, W)).astype(np.float32), disparities(rng, H, W, cal))
    pred = pred.astype(np.float32)
    c1, s1 = depth.counts(cu(pred), cu(gt), cal, lo, hi)
    c2, s2 = depth.counts(cu(pred), cu(gt), cal, lo, hi)
    assert torch.equal(c1, c2) and s1.cpu().numpy().tobytes() == s2.cpu().numpy().tobytes()
    got = depth.metrics_of(c1.cpu(), s1.cpu())._asdict()
    want = do.metrics64(pred, gt, cal, lo, hi)
    for k in do.NAMES:
        if np.isnan(want[k]):
            assert np.isnan(got[k]), k
        else:
            assert got[k] == pytest.approx(want[k], rel=1e-12, abs=0), k


def test_metrics_of_a_depth_map_read_back():
    rng = np.random.default_rng(10)
    H, W = 40, 300
    gt = rng.uniform(5, 100, (H, W)).astype(np.float32)
    pred = (gt * rng.uniform(0.8, 1.2, (H, W))).astype(np.float32)
    Z = depth.depth(cu(pred), KITTI)
    a = depth.metrics(cu(pred), cu(gt), KITTI)
    b = depth.metrics(Z, cu(gt), KITTI, is_depth=True)
    assert a == b


# ---- the command-line tools on synthetic trees ----

KITTI_CALIB = ("P0: {f} 0 {cx} 0 0 {f} {cy} 0 0 0 1 0\nP1: {f} 0 {cx} {tx} 0 {f} {cy} 0 0 0 1 0\n"
               "P2: {f} 0 {cx} 44.85 0 {f} {cy} 0 0 0 1 0\nP3: {f} 0 {cx} -339.5 0 {f} {cy} 0 0 0 1 0\n")
KITTI15_CALIB = ("S_rect_02: {w} {h}\nP_rect_02: {f} 0 {cx} 44.85728 0 {f} {cy} 0.2 0 0 1 0.003\n"
                 "P_rect_03: {f} 0 {cx} -339.5242 0 {f} {cy} 2.2 0 0 1 0.003\n")


def write_calibs(root, dataset):
    """a calibration file beside every image pair of the raw tree, of that image's size"""
    from mccnn_b200 import predict_kitti as pk

    for action in ("test", "submit"):
        for left, _, _ in pk.pair_files(root, dataset, action):
            h, w = pk._header(left)[0]
            p = pk.calib_file(left, dataset)
            os.makedirs(os.path.dirname(p), exist_ok=True)
            text = KITTI_CALIB if dataset == "kitti" else KITTI15_CALIB
            with open(p, "w") as f:
                f.write(text.format(f=700.0 + w / 10, cx=w / 2, cy=h / 2, tx=-0.54 * 700, w=w, h=h))


def write_mb_calibs(root):
    from mccnn_b200 import mb_eval as me
    from mccnn_b200 import preprocess

    for s in me.training_scenes(root):
        d = me.scene_dir(root, s)
        h, w = preprocess._image_size(os.path.join(d, "im0.png"))
        ndisp = preprocess._ndisp(os.path.join(d, "calib.txt"))
        with open(os.path.join(d, "calib.txt"), "w") as f:
            f.write("cam0=[120 0 %g; 0 120 %g; 0 0 1]\ncam1=[120 0 %g; 0 120 %g; 0 0 1]\ndoffs=3.5\nbaseline=160.2\nwidth=%d\n"
                    "height=%d\nndisp=%d\nisint=0\n" % (w / 2, h / 2, w / 2 + 3.5, h / 2, w, h, ndisp))


@pytest.fixture(scope="module")
def raw(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("depth"))
    for ds, seed in (("kitti", 91), ("kitti2015", 92)):
        unzip = synth.write_kitti_raw(root, ds, n_tr=2, n_te=2, H=40, widths=(150, 141), seed=seed)
        synth.write_kitti_eval_maps(unzip, ds, seed=seed + 10)
        write_calibs(root, ds)
    mb_unzip = synth.write_mb_raw(root, seed=93)
    synth.write_mb_eval_gt(mb_unzip, seed=94)
    write_mb_calibs(root)
    return root


def _read(p):
    with open(p, "rb") as f:
        return f.read()


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015", "mb"])
def test_run_main_predict_calib_ply(raw, tmp_path, monkeypatch, capsys, dataset):
    from mccnn_b200 import mb_eval as me
    from mccnn_b200 import predict_kitti as pk

    if dataset == "mb":
        s = me.training_scenes(raw)[0]
        d = me.scene_dir(raw, s)
        lp, rp, calp = os.path.join(d, "im0.png"), os.path.join(d, "im1.png"), os.path.join(d, "calib.txt")
    else:
        lp, rp, _ = pk.pair_files(raw, dataset, "test")[0]
        calp = pk.calib_file(lp, dataset)
    rm = _load("run_main", "tools", "run_main.py")
    base = [dataset, "census", "-a", "predict", "-left", lp, "-right", rp, "-disp_max", "12"]
    plain, flagged = tmp_path / "plain", tmp_path / "flagged"
    for d_, extra in ((plain, []), (flagged, ["-calib", calp, "-ply", "-confidence"])):
        d_.mkdir()
        monkeypatch.chdir(d_)
        rm.main(base + extra)
    out = capsys.readouterr().out
    for name in ("disp.bin", "left.bin", "right.bin"):
        assert _read(plain / name) == _read(flagged / name), name
    assert sorted(os.listdir(plain)) == ["disp.bin", "left.bin", "right.bin"]
    cal = dataio.read_calib(calp, dataset)
    disp = np.fromfile(str(flagged / "disp.bin"), "<f4")
    img = frontend.load_bytes(lp)
    H, W = img.shape[:2]
    Z = depth.depth(cu(disp.reshape(H, W)), cal)
    assert _read(flagged / "depth.bin") == Z.cpu().numpy().astype("<f4").tobytes()
    pts = depth.point_cloud(cu(disp.reshape(H, W)), cal, img)
    assert _read(flagged / "points.ply") == depth.ply_bytes(pts.n) + pts.data.cpu().numpy().tobytes()
    assert "Writing points.ply, %d points" % pts.n in out
    # -density keeps the confident pixels in both
    dens = tmp_path / "dens"
    dens.mkdir()
    monkeypatch.chdir(dens)
    rm.main(base + ["-calib", calp, "-ply", "-confidence", "-density", "0.25"])
    conf = np.fromfile(str(dens / "conf.bin"), "<f4").reshape(H, W)
    sparse = confidence.sparsify(cu(disp.reshape(H, W)), cu(conf), 0.25)
    assert _read(dens / "depth.bin") == depth.depth(sparse, cal).cpu().numpy().tobytes()
    xyz, _ = depth.read_ply(str(dens / "points.ply"))
    assert len(xyz) <= confidence.n_keep(0.25, H, W)


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015"])
def test_predict_kitti_submit_depth_ply(raw, tmp_path, capsys, dataset):
    from mccnn_b200 import kitti_eval as ke
    from mccnn_b200 import predict_kitti as pk

    plain, out = str(tmp_path / "plain"), str(tmp_path / "out")
    pk.predict_kitti("submit", dataset, arch="census", data_root=raw, out=plain, disp_max=12)
    pk.predict_kitti("submit", dataset, arch="census", data_root=raw, out=out, disp_max=12, depth=True, ply=True)
    capsys.readouterr()
    assert sorted(os.listdir(out)) == sorted(os.listdir(plain) + ["depth_0", "points_0"])
    ev = evaluate.Evaluator(dataset, "census")
    try:
        for i, pair in enumerate(pk.pair_files(raw, dataset, "submit")):
            sub = ke.submission_file(out, dataset, i)
            assert _read(sub) == _read(ke.submission_file(plain, dataset, i))
            left, right, _ = pk.decode(pair)
            x = frontend.make_batch_cuda(left, right, ev.dev)
            ev.prepare([tuple(x.shape[2:]) + (12,)])
            pred = ev.stereo_predict(x, 12)
            cal = dataio.read_calib(pk.calib_file(pair[0], dataset), dataset)
            fz, fp = pk.depth_files(out, i)
            want = str(tmp_path / "want.png")
            dataio.write_depth_png16(depth.depth(pred, cal).cpu().numpy(), want)
            assert _read(fz) == _read(want)
            pts = depth.point_cloud(pred, cal, left)
            assert _read(fp) == depth.ply_bytes(pts.n) + pts.data.cpu().numpy().tobytes()
    finally:
        ev.close()


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015", "mb"])
def test_depth_eval_predict_and_score(raw, tmp_path, capsys, dataset):
    from mccnn_b200 import depth_eval as de
    from mccnn_b200 import mb_eval as me
    from mccnn_b200 import predict_kitti as pk

    tool = _load("depth_eval_tool", "tools", "depth_eval.py")
    tool.main(["predict", dataset, "-arch", "census", "-data_root", raw, "-disp_max", "12"])
    lines = capsys.readouterr().out.strip().splitlines()
    pairs = de.training_pairs(raw, dataset)
    assert len(lines) == len(pairs) + 1 and lines[-1].startswith("mean\t")
    ev = evaluate.Evaluator(dataset, "census")
    try:
        for (name, left, right, cal, gts), line in zip(pairs, lines):
            if dataset == "mb":
                from mccnn_b200 import preprocess

                x = preprocess._mb_views(dict(groups=[([left, right], (2,))], half=False), "gray", ev.dev)[0]
                x = torch.from_numpy(np.ascontiguousarray(x)).to(ev.dev)
                D = preprocess._ndisp(os.path.join(os.path.dirname(left), "calib.txt"))
            else:
                x = frontend.make_batch_cuda(frontend.load_bytes(left), frontend.load_bytes(right), ev.dev)
                D = 12
            ev.prepare([tuple(x.shape[2:]) + (D,)])
            pred = ev.stereo_predict(x, D)
            vals = []
            for g in gts:
                gt = cu(de._read_gt(g))
                vals += list(depth.metrics(pred, gt, cal, depth.MIN_DEPTH, de.max_depth_of(dataset)))
            assert line == de.line(name, vals)
    finally:
        ev.close()
    # score: from the disparity maps the other tools write, and for KITTI from depth PNGs
    out = str(tmp_path / "out")
    if dataset == "mb":
        me.evaluate_training("census", None, data_root=raw, out=out, verbose=False)
        tool.main(["score", "mb", out, "-data_root", raw])
        assert len(capsys.readouterr().out.strip().splitlines()) == len(pairs) + 1
    else:
        pk.predict_kitti("test", dataset, arch="census", data_root=raw, out=out, disp_max=12, depth=True, verbose=False)
        res = de.score_dir(dataset, out, data_root=raw, source="depth", verbose=False)
        for i, row in enumerate(res.rows):
            Z = dataio.read_depth_png16(pk.depth_files(out, i)[0])
            want = [v for g in pairs[i][4] for v in depth.metrics(cu(Z), cu(de._read_gt(g)), pairs[i][3], is_depth=True)]
            assert de.line(i, row) == de.line(i, want)
