"""GPU: Middlebury training (dataset mb) -- the pair-table sampler bit for bit against oracle/train.py's warp_affine on
ragged sources, the pair-table trainer against the X0 / X1 creators, determinism of the mb draws, and whole runs of
tools/train_mb.py on a synthetic raw Middlebury tree preprocessed by preprocess_mb."""
import os
import subprocess
import sys
import zipfile

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, preprocess, synth, t7, train  # noqa: E402
from oracle import train as ot  # noqa: E402

DEV = torch.device("cuda", 0)
SIZES = [(3, 4), (5, 7), (1, 9), (17, 33), (40, 96), (1000, 1500)]


def _planes(rng, sizes):
    return [tuple(torch.from_numpy(rng.standard_normal(s).astype(np.float32)).to(DEV) for _ in range(2)) for s in sizes]


def test_pair_sampler_bit_exact_on_ragged_pairs():
    rng = np.random.default_rng(0)
    planes = _planes(rng, SIZES)
    ws, per = 11, 96
    o = train.options("mb", "fast", hflip=1, vflip=1, trans=2.0)
    recs = []
    for k, (H, W) in enumerate(SIZES):
        # centres inside, across every border and wholly outside the pair's own H x W
        rows = np.stack([np.full(per, 1), rng.uniform(-12, H + 12, per), rng.uniform(-12, W + 12, per),
                         rng.uniform(0, 8, per)], 1).astype(np.float32)
        w = train.make_warps(train.draw_params(train.Stream(k), o, per), rows, ws,
                             pairs=(np.full(per, k), np.full(per, k)))
        w["m"][:8, 2] += np.float32(W + 30.0)                                      # wholly outside
        w["m"][8:16, 5] -= np.float32(H + 30.0)
        recs.append(w)
    w = np.concatenate(recs)
    w["image"][:5] = [-1, len(SIZES), 1 << 30, -(1 << 30), len(SIZES) + 7]      # bad pair indices: NaN patches
    got = train.sample_patches_pairs(planes, w, ws).cpu().numpy()
    host = [(a.cpu().numpy(), b.cpu().numpy()) for a, b in planes]
    for i, r in enumerate(w):
        if not 0 <= r["image"] < len(SIZES):
            assert np.isnan(got[i]).all(), i
            continue
        want = ot.warp_affine(host[r["image"]][r["view"]], r["m"], ws)
        want = (want * r["contrast"] + r["brightness"]).astype(np.float32)
        assert np.array_equal(got[i].view(np.int32), want.view(np.int32)), (i, r["image"])


def test_pair_sampler_refuses_bad_tables():
    from mccnn_b200.adcensus import AdcensusError

    rng = np.random.default_rng(1)
    planes = _planes(rng, [(4, 5)])
    w = np.zeros(1, train.WARP_DTYPE)
    t = train.pair_table(planes)
    for field, v, msg in (("H", 0, "invalid argument"), ("W", 40000, "size limit"), ("x1", 0, "invalid argument")):
        bad = t.copy()
        bad[field] = v
        table = torch.from_numpy(bad.view(np.uint8)).to(DEV)
        out = torch.empty((1, 3, 3), device=DEV)
        import ctypes

        from mccnn_b200.adcensus import _check, _stream, lib
        with pytest.raises(AdcensusError, match=msg):
            _check(lib().mccnn_train_sample_pairs(ctypes.c_void_p(table.data_ptr()), 1,
                                                  ctypes.c_void_p(torch.from_numpy(w.view(np.uint8)).to(DEV).data_ptr()),
                                                  1, 3, ctypes.c_void_p(out.data_ptr()), _stream(out)), "pairs")


@pytest.mark.parametrize("arch", ["fast", "slow"])
def test_pair_trainer_equals_stacked_trainer(arch):
    rng = np.random.default_rng(2)
    kw = dict(l1=3, fm=32, bs=32) if arch == "fast" else dict(l1=2, fm=32, l2=1, nh2=128, bs=32)
    o = train.options("kitti", arch, **kw)
    n_img, H, W = 3, 40, 90
    X0, X1 = (torch.from_numpy(rng.standard_normal((n_img, 1, H, W)).astype(np.float32)).to(DEV) for _ in range(2))
    a = train.Trainer(o, X0, X1, chunk=16, loss_cap=64, device=0)
    b = train.Trainer(o, chunk=16, loss_cap=64, device=0, planes=[(X0[i, 0], X1[i, 0]) for i in range(n_img)])
    s = train.Stream(5)
    layers = train.init_net(s, o)
    for tr in (a, b):
        tr.set_layers(*layers)
    for _ in range(3):
        rows = np.stack([rng.integers(1, n_img + 1, 16 * 16), rng.integers(0, H, 256), rng.integers(0, W, 256),
                         rng.uniform(0, 30, 256)], 1).astype(np.float32)
        w = train.make_warps(train.draw_params(s, o, 256), rows, a.ws)
        for tr in (a, b):
            tr.run(w, o["lr"])
    for what in (train.TRAIN_PARAMS, train.TRAIN_MOMENTA, train.TRAIN_LOSS, train.TRAIN_PATCHES):
        x, y = a.get(what).cpu().numpy(), b.get(what).cpu().numpy()
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), what
    a.close()
    b.close()


def _ragged_set(root):
    """a data.mb.imperfect_gray of four images with 1 to 3 lights, 1 to 3 exposures and different sizes"""
    d = os.path.join(str(root), "data.mb.imperfect_gray")
    os.makedirs(d)
    rng = np.random.default_rng(3)
    groups = {1: [(3, 30, 70)] * 3, 2: [(1, 20, 41)], 3: [(2, 44, 90)] * 2, 4: [(3, 25, 60)]}
    rows = []
    for i, gs in groups.items():
        for j, (ne, h, w) in enumerate(gs, 2):
            dataio.tofile(os.path.join(d, "x_%d_%d.bin" % (i, j)), rng.standard_normal((ne, 2, 1, h, w)).astype(np.float32))
        h, w = gs[0][1:]
        rows.append(np.stack([np.full(200, i), rng.integers(0, h, 200), rng.integers(0, w, 200), rng.uniform(0, 10, 200)], 1))
    dataio.tofile(os.path.join(d, "meta.bin"), np.array([(g[0][1], g[0][2], 16) for g in groups.values()], np.int32))
    dataio.tofile(os.path.join(d, "nnz_tr.bin"), np.concatenate(rows).astype(np.float32))
    return train.MbTrainSet(str(root), "imperfect", "train_tr")


def _mb_run(ts, planes, o, seed, chunks=3, n=8):
    s = train.Stream(seed)
    perm = train.randperm(s, len(ts.nnz))
    tr = train.Trainer(o, chunk=n, loss_cap=64, device=0, planes=planes)
    tr.set_layers(*train.init_net(s, o))
    h = o["bs"] // 2
    for c in range(chunks):
        rows = ts.nnz[perm[c * n * h:(c + 1) * n * h] - 1]
        tr.run(ts.warps(s, o, rows, tr.ws), o["lr"])
    out = [tr.get(w).cpu().numpy() for w in (train.TRAIN_PARAMS, train.TRAIN_LOSS)]
    tr.close()
    return out


@pytest.mark.parametrize("arch", ["fast", "slow"])
def test_mb_runs_are_deterministic(arch, tmp_path):
    ts = _ragged_set(tmp_path)
    planes = ts.upload(0)
    assert len(planes) == ts.n_pairs == 9 + 1 + 4 + 3
    kw = dict(l1=3, fm=32, bs=16) if arch == "fast" else dict(l1=2, fm=32, l2=1, nh2=128, bs=16)
    o = train.options("mb", arch, d_exp=0.5, d_light=0.5, **kw)
    a, b, c = _mb_run(ts, planes, o, 1), _mb_run(ts, planes, o, 1), _mb_run(ts, planes, o, 2)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))
    assert not np.array_equal(a[0], c[0])
    assert np.isfinite(a[1][:24]).all() and (a[1][:24] > 0).all()


@pytest.fixture(scope="module")
def mb_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("mb"))
    synth.write_mb_raw(root, seed=7)
    preprocess.preprocess_mb(root, "imperfect", "gray")
    return root


def _tool(args, cwd):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train_mb.py")] + args, capture_output=True,
                          text=True, cwd=cwd, timeout=1800)


def _fresh(mb_root, tmp_path):
    """a copy of the preprocessed set (links to the data files), so that each run writes its own net/ and out/"""
    src = os.path.join(mb_root, "data.mb.imperfect_gray")
    dst = os.path.join(str(tmp_path), "data.mb.imperfect_gray")
    os.makedirs(dst)
    for f in os.listdir(src):
        os.symlink(os.path.join(src, f), os.path.join(dst, f))
    return str(tmp_path)


def test_train_tr_end_to_end(mb_root, tmp_path):
    from mccnn_b200 import evaluate

    root = _fresh(mb_root, tmp_path)
    o = train.options("mb", "fast")
    r = _tool(["mb", "fast", "-a", "train_tr", "-data_root", root], ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = r.stdout.splitlines()
    assert lines[0].startswith("mb fast -a train_tr")
    nl = len(train.net_lines(o))
    assert lines[1:1 + nl] == train.net_lines(o) and lines[1] == "conv(in=1, out=64, k=3)"
    ep = [l.split("\t") for l in lines[1 + nl:15 + nl]]
    assert [int(e[0]) for e in ep] == list(range(1, 15))
    assert [float(e[2]) for e in ep] == [0.002] * 11 + [0.0002] * 3
    errs = [float(e[1]) for e in ep]
    assert errs[-1] < errs[0], errs
    test_lines = lines[15 + nl:]
    d = os.path.join(root, "data.mb.imperfect_gray")
    n_te = len(dataio.fromfile(os.path.join(d, "te.bin")).reshape(-1))
    assert len(test_lines) == n_te + 2 + 1 and all(len(l.split("\t")) == 2 for l in test_lines[:-1])
    fname = train.net_path(root, "mb", ["-a", "train_tr"], "fast")
    net = t7.load_net(fname)
    assert net.arch == "fast" and len(net.tower) == 5
    assert net.opt["d_exp"] == 0.2 and net.opt["ds"] == 2001 and net.opt["rect"] == "imperfect"
    trained_err = float(test_lines[-1])
    init = os.path.join(root, "init.t7")
    s = train.Stream(42)
    train.randperm(s, len(train.MbTrainSet(root, "imperfect", "train_tr").nnz))
    t7.save_net(init, *train.init_net(s, o))
    ev = evaluate.Evaluator("mb", "fast", net_fname=init, device=0)
    init_err = ev.test("test_te", data=evaluate.load_data("mb", root), verbose=False).mean
    ev.close()
    assert trained_err < init_err, (trained_err, init_err)
    r = _tool(["mb", "fast", "-a", "train_tr", "-data_root", root], ROOT)
    assert r.returncode != 0 and "already exists" in r.stderr


def test_slow_train_all_writes_submission(mb_root, tmp_path):
    root = _fresh(mb_root, tmp_path)
    out = os.path.join(root, "out")
    args = ["-a", "train_all", "-l1", "2", "-fm", "32", "-l2", "1", "-nh2", "128"]
    r = _tool(["mb", "slow"] + args + ["-data_root", root, "-out", out], ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert os.path.exists(train.net_path(root, "mb", args, "slow"))
    with zipfile.ZipFile(os.path.join(out, "submission.zip")) as z:
        names = set(z.namelist())
    for s in synth.MB_SUBMIT_NAMES:
        assert "trainingH/%s/disp0MC-CNN-acrt.pfm" % s in names and "testH/%sT/timeMC-CNN-acrt.txt" % s in names
