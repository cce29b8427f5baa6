"""GPU: training of the slow architecture (csrc/train.cu, mccnn_b200/train.py, tools/train_slow.py) against float64
autograd (oracle/train_slow.py), a float32 restatement of BCECriterion2 and of the update, determinism, the inference path
on the saved net, and whole runs on a synthetic KITTI set."""
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, preprocess, synth, t7, train  # noqa: E402
from oracle import train as ot  # noqa: E402
from oracle import train_slow as ots  # noqa: E402

DEV = torch.device("cuda", 0)


def _trainer(o, rng, n_img=2, H=40, W=90, chunk=64, loss_cap=64):
    X0, X1 = (torch.from_numpy(rng.standard_normal((n_img, 1, H, W)).astype(np.float32)).to(DEV) for _ in range(2))
    return train.Trainer(o, X0, X1, chunk=chunk, loss_cap=loss_cap, device=0)


def _warps(rng, n, ws, o, stream, n_img=2, H=40, W=90):
    rows = np.stack([rng.integers(1, n_img + 1, n), rng.integers(0, H, n), rng.integers(0, W, n), rng.uniform(0, 60, n)],
                    1).astype(np.float32)
    return train.make_warps(train.draw_params(stream, o, n), rows, ws)


def _f64(layers):
    return [(w.astype(np.float64), b.astype(np.float64)) for w, b in layers]


def test_buffer_ids_per_arch():
    rng = np.random.default_rng(0)
    o = train.options("kitti", "slow", l1=2, fm=16, l2=1, nh2=128, bs=8)
    tr = _trainer(o, rng)
    assert tr.size(train.TRAIN_ROWS) == 8 * 32 and tr.size(train.TRAIN_FC) == 8 * 128 + 8
    assert tr.size(train.TRAIN_NORM) == -1 and tr.size(train.TRAIN_HINGE) == -1
    assert tr.launches_per_step == 3 + 3 * 2 + 3 * 1
    tr.close()
    f = _trainer(train.options("kitti", l1=2, fm=16, bs=8), rng)
    assert f.size(train.TRAIN_ROWS) == -1 and f.size(train.TRAIN_SIGMOID) == -1 and f.launches_per_step == 7
    f.close()


@pytest.mark.parametrize("shape", [(4, 112, 4, 384, 128), (2, 32, 1, 128, 16)])
def test_step_matches_float64_autograd_along_a_run(shape):
    l1, fm, l2, nh2, bs = shape
    o = train.options("kitti", "slow", l1=l1, fm=fm, l2=l2, nh2=nh2, bs=bs)
    rng = np.random.default_rng(l1)
    tr = _trainer(o, rng)
    s = train.Stream(3)
    tr.set_layers(*train.init_slow(s, o))
    ws = tr.ws
    for point in range(3):
        tr.reset_losses()
        patches = tr.get(train.TRAIN_PATCHES).cpu().numpy().reshape(tr.N, 1, ws, ws) if point else \
            rng.standard_normal((tr.N, 1, ws, ws)).astype(np.float32)
        tower, head = tr.net()
        tr.step_patches(patches, 0.003)
        torch.cuda.synchronize()
        loss64, gt, gh, y64 = ots.step64_slow(patches.astype(np.float64), _f64(tower), _f64(head))
        assert abs(float(tr.get(train.TRAIN_LOSS)[0]) - loss64) <= 1e-4 * max(abs(loss64), 1e-3)
        assert np.abs(tr.get(train.TRAIN_SIGMOID).cpu().numpy() - y64).max() <= 1e-5
        got_t, got_h = tr.net(train.TRAIN_GRADS)
        for (aw, ab), (ww, wb) in zip(got_t + got_h, gt + gh):
            for a, b in ((aw, ww), (ab, wb)):
                scale = max(np.abs(b).max(), 1e-12)
                assert np.abs(a - b).max() <= 1e-4 * scale, (point, np.abs(a - b).max(), scale)
        tr.run(_warps(rng, 20 * bs // 2, ws, o, s), 0.003)                       # move along the run: 20 sampler steps
        torch.cuda.synchronize()
    tr.close()


def test_bce_and_sigmoid_stage():
    """gradInput bit for bit against BCECriterion2's expression sequence in float32 CUDA torch; the loss (which goes through
    log) against the same sequence, reporting its distance in ulps"""
    o = train.options("kitti", "slow")
    rng = np.random.default_rng(7)
    tr = _trainer(o, rng)
    tr.set_layers(*train.init_slow(train.Stream(8), o))
    tr.reset_losses()
    tr.step_patches(rng.standard_normal((tr.N, 1, tr.ws, tr.ws)).astype(np.float32), 0.003)
    y = tr.get(train.TRAIN_SIGMOID)
    z = tr.get(train.TRAIN_FC)[-o["bs"]:]
    assert torch.equal(y, 1 / (1 + torch.exp(-z)))
    bs = float(o["bs"])
    t = torch.arange(o["bs"], device=DEV).remainder(2).float()
    eps = 1e-12
    term1 = torch.ones_like(y).add(t, alpha=-1)
    term2 = torch.ones_like(y).add(y, alpha=-1).add(eps)
    term1 = term1.div(term2)
    term3 = y.clone().add(eps)
    g = t.clone().div(term3).add(term1, alpha=-1).div(bs).mul(-1)
    assert torch.equal(tr.get(train.TRAIN_BCE_GRAD), g)
    l2 = torch.ones_like(y).add(y, alpha=-1).add(eps).log().mul(torch.ones_like(y).add(t, alpha=-1))
    l3 = y.clone().add(eps).log().mul(t).add(l2).div(bs).cpu().numpy()
    s = np.float32(0)
    for v in l3:                                                                 # the row order the kernel sums in
        s = np.float32(s + v)
    want = np.float32(-s)
    got = np.float32(tr.get(train.TRAIN_LOSS)[0].item())
    ulps = abs(int(got.view(np.int32)) - int(want.view(np.int32)))
    print("BCECriterion2 loss: %d ulp from torch's log" % ulps)
    assert ulps <= 4, ulps
    tr.close()


def test_update_bit_exact():
    o = train.options("kitti", "slow", l1=2, fm=16, l2=2, nh2=128, bs=8, mom=0.9)
    rng = np.random.default_rng(5)
    tr = _trainer(o, rng)
    n = tr.size(train.TRAIN_PARAMS)
    p0 = (rng.standard_normal(n) * 0.1).astype(np.float32)
    v0 = rng.standard_normal(n).astype(np.float32) * np.float32(1e-3)
    tr.set(train.TRAIN_PARAMS, p0)
    tr.set(train.TRAIN_MOMENTA, v0)
    lr = 0.0123
    tr.step_patches(rng.standard_normal((tr.N, 1, tr.ws, tr.ws)).astype(np.float32), lr)
    g = tr.get(train.TRAIN_GRADS).cpu().numpy()
    assert np.abs(g[-(128 + 1):]).max() > 0                                     # the head's gradients are in the vector
    p1, v1 = ot.update32(p0, v0, g, o["mom"], lr)
    assert np.array_equal(tr.get(train.TRAIN_MOMENTA).cpu().numpy(), v1)
    assert np.array_equal(tr.get(train.TRAIN_PARAMS).cpu().numpy(), p1)
    tr.close()


def _short_run(seed):
    o = train.options("kitti", "slow", l1=3, fm=48, l2=2, nh2=256, bs=32)
    rng = np.random.default_rng(0)
    tr = _trainer(o, rng)
    s = train.Stream(seed)
    tr.set_layers(*train.init_slow(s, o))
    r2 = np.random.default_rng(seed)
    for _ in range(3):
        tr.run(_warps(r2, 50 * o["bs"] // 2, tr.ws, o, s), 0.003)
    p = tr.get(train.TRAIN_PARAMS).cpu().numpy()
    tr.close()
    return p


def test_same_seed_same_bits():
    a, b, c = _short_run(1), _short_run(1), _short_run(2)
    assert np.array_equal(a, b)
    assert not np.array_equal(a, c)


def test_train_and_test_are_tied(tmp_path):
    """the saved net through FeatureTower(arch='slow') and ScorerHead reproduces the trainer's sigmoid outputs"""
    from mccnn_b200 import feature_tower, scorer_head

    o = train.options("kitti", "slow")
    rng = np.random.default_rng(9)
    tr = _trainer(o, rng)
    s = train.Stream(10)
    tr.set_layers(*train.init_slow(s, o))
    tr.run(_warps(rng, 30 * o["bs"] // 2, tr.ws, o, s), 0.003)                   # away from the init
    tower, head = tr.net()                                                       # the weights the next step reads
    tr.step_patches(tr.get(train.TRAIN_PATCHES).reshape(tr.N, 1, tr.ws, tr.ws), 0.003)
    torch.cuda.synchronize()
    y = tr.get(train.TRAIN_SIGMOID).cpu().numpy()
    x = tr.get(train.TRAIN_PATCHES).reshape(tr.N, 1, tr.ws, tr.ws)
    fname = os.path.join(str(tmp_path), "net.t7")
    t7.save_net(fname, tower, head)
    tr.close()
    net = t7.load_net(fname)
    assert net.arch == "slow"
    ft = feature_tower.FeatureTower(net.tower, arch="slow", device=0)
    c = ft.forward(x)[:, :, tr.ws // 2, tr.ws // 2]                              # (N, fm): the centre, padding-free
    ft.close()
    featL = c[0::2].t().reshape(o["fm"], 1, o["bs"]).contiguous()               # row r: patch 2r (left) ...
    featR = c[1::2].t().reshape(o["fm"], 1, o["bs"]).contiguous()               # ... and patch 2r + 1 (right)
    hd = scorer_head.ScorerHead(net.head, device=0)
    volL, _ = hd.volumes(featL, featR, 1, want_right=False)
    torch.cuda.synchronize()
    hd.close()
    got = volL[0, 0, 0].cpu().numpy()
    assert np.abs(got - y).max() <= 1e-4, np.abs(got - y).max()


def _kitti_set(root, dataset):
    d = synth.write_kitti_set(str(root), dataset, n_tr=6, n_te=2, H=48, width=130, widths=(130, 121), seed=1)
    disp = dataio.fromfile(os.path.join(d, "dispnoc.bin"))
    x0 = dataio.fromfile(os.path.join(d, "x0.bin"))
    te = dataio.fromfile(os.path.join(d, "te.bin")).reshape(-1)
    is_te = np.zeros(len(disp), bool)
    is_te[te - 1] = True
    nnz_tr, nnz_te = preprocess.kitti_nnz(torch.from_numpy(disp).to(DEV), torch.from_numpy(x0[:len(disp)]).to(DEV), is_te)
    dataio.tofile(os.path.join(d, "nnz_tr.bin"), nnz_tr.cpu().numpy())
    dataio.tofile(os.path.join(d, "nnz_te.bin"), nnz_te.cpu().numpy())
    return d, len(nnz_tr)


def _tool(args, cwd):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train_slow.py")] + args, capture_output=True,
                          text=True, cwd=cwd, timeout=1800)


def test_train_tr_end_to_end(tmp_path):
    from mccnn_b200 import evaluate

    d, n_rows = _kitti_set(tmp_path, "kitti")
    o = train.options("kitti", "slow")
    r = _tool(["kitti", "slow", "-a", "train_tr", "-data_root", str(tmp_path)], ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = r.stdout.splitlines()
    assert lines[0].startswith("kitti slow -a train_tr")
    nl = len(train.net_lines(o))
    assert lines[1:1 + nl] == train.net_lines(o)
    ep = [l.split("\t") for l in lines[1 + nl:15 + nl]]
    assert [int(e[0]) for e in ep] == list(range(1, 15))
    assert [float(e[2]) for e in ep] == [0.003] * 11 + [0.0003] * 3
    errs = [float(e[1]) for e in ep]
    assert errs[-1] < errs[0], errs
    test_lines = lines[15 + nl:]
    n_te = len(dataio.fromfile(os.path.join(d, "te.bin")).reshape(-1))
    assert len(test_lines) == n_te + 1 and all(len(l.split("\t")) == 2 for l in test_lines[:-1])
    fname = train.net_path(str(tmp_path), "kitti", ["-a", "train_tr"], "slow")
    net = t7.load_net(fname)
    assert net.arch == "slow" and len(net.tower) == 4 and len(net.head) == 5
    trained_err = float(test_lines[-1])
    init = os.path.join(str(tmp_path), "init.t7")
    s = train.Stream(42)
    train.randperm(s, n_rows)
    t7.save_net(init, *train.init_slow(s, o))
    ev = evaluate.Evaluator("kitti", "slow", net_fname=init, device=0)
    init_err = ev.test("test_te", data_root=str(tmp_path), verbose=False).mean
    ev.close()
    assert trained_err < init_err, (trained_err, init_err)
    r = _tool(["kitti", "slow", "-a", "train_tr", "-data_root", str(tmp_path)], ROOT)
    assert r.returncode != 0 and "already exists" in r.stderr


def test_train_all_writes_submission(tmp_path):
    _kitti_set(tmp_path, "kitti2015")
    out = os.path.join(str(tmp_path), "out")
    args = ["-a", "train_all", "-l1", "2", "-fm", "32", "-l2", "1", "-nh2", "128"]
    r = _tool(["kitti2015", "slow"] + args + ["-data_root", str(tmp_path), "-out", out], ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert os.path.exists(os.path.join(out, "submission.zip"))
    assert len(os.listdir(os.path.join(out, "disp_0"))) == 2
    assert os.path.exists(train.net_path(str(tmp_path), "kitti2015", args, "slow"))
