"""GPU: training of the fast architecture (csrc/train.cu, mccnn_b200/train.py, tools/train.py) against oracle/train.py, the
reference's own Normalize2 / Margin2 kernels and float64 autograd, plus determinism and a whole run on a synthetic KITTI set."""
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

DEV = torch.device("cuda", 0)


def _images(rng, n, H, W):
    return [rng.standard_normal((n, 1, H, W)).astype(np.float32) for _ in range(2)]


def _warps(rng, n_samples, n_img, H, W, ws, o, stream):
    rows = np.stack([rng.integers(1, n_img + 1, n_samples), rng.integers(0, H, n_samples), rng.integers(0, W, n_samples),
                     rng.uniform(0, 60, n_samples)], 1).astype(np.float32)
    return train.make_warps(train.draw_params(stream, o, n_samples), rows, ws)


def test_sampler_bit_exact_kitti_size():
    rng = np.random.default_rng(0)
    H, W = 350, 1242
    X0, X1 = _images(rng, 2, H, W)
    o = train.options("kitti", hflip=1, vflip=1, trans=2.0, d_vtrans=1.0, d_rotate=3.0, d_hshear=0.2, rotate=20.0)
    w = _warps(rng, 2560, 2, H, W, 9, o, train.Stream(1))                     # 10240 patches
    # edge cases: patches across every border, wholly outside, far outside
    w["m"][:64, 2] += np.float32(-3.0)
    w["m"][64:128, 2] += np.float32(W + 2.0)
    w["m"][128:192, 5] += np.float32(-H - 8.0)
    w["m"][192:256, 5] += np.float32(5000.0)
    got = train.sample_patches(torch.from_numpy(X0).to(DEV), torch.from_numpy(X1).to(DEV), w, 9).cpu().numpy()
    for i, r in enumerate(w):
        src = (X1 if r["view"] else X0)[r["image"], 0]
        want = ot.warp_affine(src, r["m"], 9)
        want = (want * r["contrast"] + r["brightness"]).astype(np.float32)
        assert np.array_equal(got[i].view(np.int32), want.view(np.int32)), i


def _trainer(o, rng, n_img=2, H=40, W=90, chunk=64, loss_cap=64):
    X0, X1 = (torch.from_numpy(x).to(DEV) for x in _images(rng, n_img, H, W))
    return train.Trainer(o, X0, X1, chunk=chunk, loss_cap=loss_cap, device=0)


def _check_step(tr, o, patches, layers):
    loss64, grads = ot.step64(patches.astype(np.float64), [(w.astype(np.float64), b.astype(np.float64)) for w, b in layers],
                              o["m"], o["pow"])
    got = tr.layers(train.TRAIN_GRADS)
    assert abs(float(tr.get(train.TRAIN_LOSS)[0]) - loss64) <= 1e-4 * max(abs(loss64), 1e-3)
    for (gw, gb), (ww, wb) in zip(got, grads):
        for a, b in ((gw, ww), (gb, wb)):
            scale = max(np.abs(b).max(), 1e-12)
            assert np.abs(a - b).max() <= 1e-4 * scale, (np.abs(a - b).max(), scale)


@pytest.mark.parametrize("shape,pow_", [((4, 64, 128), 1), ((4, 64, 128), 2), ((3, 32, 16), 1), ((3, 32, 16), 2)])
def test_step_matches_float64_autograd_along_a_run(shape, pow_):
    l1, fm, bs = shape
    o = train.options("kitti", l1=l1, fm=fm, bs=bs, pow=pow_)
    rng = np.random.default_rng(l1 + pow_)
    tr = _trainer(o, rng)
    s = train.Stream(3)
    layers = train.init_weights(s, l1, fm)
    tr.set_layers(layers)
    ws = tr.ws
    for point in range(3):
        tr.reset_losses()
        patches = tr.get(train.TRAIN_PATCHES).cpu().numpy().reshape(tr.N, 1, ws, ws) if point else \
            rng.standard_normal((tr.N, 1, ws, ws)).astype(np.float32)
        layers = tr.layers()
        tr.step_patches(patches, 0.002)
        torch.cuda.synchronize()
        _check_step(tr, o, patches, layers)
        # move along the run: 20 sampler steps
        tr.run(_warps(rng, 20 * bs // 2, 2, 40, 90, ws, o, s), 0.002)
        torch.cuda.synchronize()
    tr.close()


def test_head_stages_equal_reference_kernels():
    from oracle import refdriver

    if not os.path.exists(refdriver.REF_LIB):
        pytest.skip("oracle/_ref/libadcensus_ref.so not built")
    ref = refdriver.ShimLibrary()
    for pow_ in (1, 2):
        o = train.options("kitti", pow=pow_)
        rng = np.random.default_rng(pow_)
        tr = _trainer(o, rng)
        tr.set_layers(train.init_weights(train.Stream(4), o["l1"], o["fm"]))
        tr.step_patches(rng.standard_normal((tr.N, 1, tr.ws, tr.ws)).astype(np.float32), 0.002)
        N, fm, bs = tr.N, o["fm"], o["bs"]
        tower = tr.get(train.TRAIN_TOWER)
        F = tower[-N * fm:].reshape(N, fm, 1, 1).contiguous()
        norm = torch.empty((N, 1, 1, 1), device=DEV)
        out = torch.empty_like(F)
        ref.call("Normalize_forward", F, norm, out)
        assert torch.equal(norm.reshape(-1), tr.get(train.TRAIN_NORM))
        assert torch.equal(out.reshape(-1), tr.get(train.TRAIN_NORMALIZED))
        # StereoJoin1 (cmul + sum over the planes): THC's reduction order is not restated, fp32 sums of 64 terms
        join = tr.get(train.TRAIN_JOIN)
        want = (out[0::2] * out[1::2]).sum(1).reshape(-1)
        assert torch.allclose(join, want, rtol=0, atol=1e-6)
        tmp = torch.empty(bs // 2, device=DEV)
        gin = torch.empty((bs, 1, 1, 1), device=DEV)
        ref.call("Margin2", join.reshape(bs, 1, 1, 1).contiguous(), tmp, gin, o["m"], pow_)
        assert torch.equal(tmp, tr.get(train.TRAIN_HINGE))
        assert torch.equal(gin.reshape(-1).div_(bs // 2), tr.get(train.TRAIN_JOIN_GRAD))
        gout = tr.get(train.TRAIN_NORM_GRAD_OUT).reshape(N, fm, 1, 1).contiguous()
        gF = torch.empty_like(F)
        ref.call("Normalize_backward_input", gout, F, norm, gF)
        assert torch.equal(gF.reshape(-1), tr.get(train.TRAIN_DZ)[-N * fm:])
        tr.close()


def test_update_bit_exact():
    o = train.options("kitti", l1=2, fm=16, bs=8, mom=0.9)
    rng = np.random.default_rng(5)
    tr = _trainer(o, rng)
    n = tr.size(train.TRAIN_PARAMS)
    p0 = rng.standard_normal(n).astype(np.float32)
    v0 = rng.standard_normal(n).astype(np.float32) * np.float32(1e-3)
    tr.set(train.TRAIN_PARAMS, p0)
    tr.set(train.TRAIN_MOMENTA, v0)
    lr = 0.0123
    tr.step_patches(rng.standard_normal((tr.N, 1, tr.ws, tr.ws)).astype(np.float32), lr)
    g = tr.get(train.TRAIN_GRADS).cpu().numpy()
    p1, v1 = ot.update32(p0, v0, g, o["mom"], lr)
    assert np.array_equal(tr.get(train.TRAIN_MOMENTA).cpu().numpy(), v1)
    assert np.array_equal(tr.get(train.TRAIN_PARAMS).cpu().numpy(), p1)
    tr.close()


def _short_run(seed):
    o = train.options("kitti", l1=3, fm=32, bs=32)
    rng = np.random.default_rng(0)
    tr = _trainer(o, rng)
    s = train.Stream(seed)
    tr.set_layers(train.init_weights(s, o["l1"], o["fm"]))
    r2 = np.random.default_rng(seed)
    for _ in range(3):
        tr.run(_warps(r2, 50 * o["bs"] // 2, 2, 40, 90, tr.ws, o, s), 0.002)
    p = tr.get(train.TRAIN_PARAMS).cpu().numpy()
    tr.close()
    return p


def test_same_seed_same_bits():
    a, b, c = _short_run(1), _short_run(1), _short_run(2)
    assert np.array_equal(a, b)
    assert not np.array_equal(a, c)


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
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train.py")] + args, capture_output=True, text=True,
                          cwd=cwd, timeout=1800)


def test_train_tr_end_to_end(tmp_path):
    from mccnn_b200 import evaluate

    d, n_rows = _kitti_set(tmp_path, "kitti")
    steps = train.steps_per_epoch(n_rows, 128)
    assert 100 <= steps <= 1000, steps
    r = _tool(["kitti", "fast", "-a", "train_tr", "-data_root", str(tmp_path)], ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = r.stdout.splitlines()
    assert lines[0].startswith("kitti fast -a train_tr")
    assert lines[1:10] == train.net_lines(train.options("kitti"))
    ep = [l.split("\t") for l in lines[10:24]]
    assert [int(e[0]) for e in ep] == list(range(1, 15))
    errs = [float(e[1]) for e in ep]
    assert [float(e[2]) for e in ep] == [0.002] * 11 + [0.0002] * 3
    assert errs[-1] < errs[0]
    test_lines = lines[24:]
    n_te = len(dataio.fromfile(os.path.join(d, "te.bin")).reshape(-1))
    assert len(test_lines) == n_te + 1 and all(len(l.split("\t")) == 2 for l in test_lines[:-1])
    fname = train.net_path(str(tmp_path), "kitti", ["-a", "train_tr"])
    net = t7.load_net(fname)
    assert net.arch == "fast" and len(net.tower) == 4
    trained_err = float(test_lines[-1])
    init = os.path.join(str(tmp_path), "init.t7")
    s = train.Stream(42)
    train.randperm(s, n_rows)
    t7.save_net(init, train.init_weights(s, 4, 64))
    ev = evaluate.Evaluator("kitti", "fast", net_fname=init, device=0)
    init_err = ev.test("test_te", data_root=str(tmp_path), verbose=False).mean
    ev.close()
    assert trained_err < init_err, (trained_err, init_err)
    # the same command again is refused: the net exists
    r = _tool(["kitti", "fast", "-a", "train_tr", "-data_root", str(tmp_path)], ROOT)
    assert r.returncode != 0 and "already exists" in r.stderr


def test_train_all_writes_submission(tmp_path):
    _kitti_set(tmp_path, "kitti2015")
    out = os.path.join(str(tmp_path), "out")
    r = _tool(["kitti2015", "fast", "-a", "train_all", "-data_root", str(tmp_path), "-out", out, "-l1", "2", "-fm", "32"],
              ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert os.path.exists(os.path.join(out, "submission.zip"))
    assert len(os.listdir(os.path.join(out, "disp_0"))) == 2
    assert os.path.exists(train.net_path(str(tmp_path), "kitti2015", ["-a", "train_all", "-l1", "2", "-fm", "32"]))
