"""GPU: the margin confidence, the LR map, sparse maps and the sparsification counts (mc-cnn_b200/confidence.py,
csrc/confidence.cu) -- the kernel against the numpy restatement (tests/confidence_oracle.py) bit for bit, also on a volume
past 2^31 elements; the fused pipeline's disp unchanged by conf / lr across presets, -sm_terminate / -sm_skip values, CBCA
and overlap modes, with conf and lr equal to what the returned volumes give; the operator chain equal to run_volumes; and
the command-line tools on synthetic sets."""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, confidence, evaluate, frontend, pipeline, scorer_head, synth  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


oc = _load("confidence_oracle", "tests", "confidence_oracle.py")
sc = _load("stage_chain", "tests", "stage_chain.py")


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def same(got, want, what):
    g = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    w = want.detach().cpu().numpy() if isinstance(want, torch.Tensor) else np.asarray(want)
    g = g.reshape(w.shape)
    bad = ~((g == w) | (np.isnan(g) & np.isnan(w)))
    assert not bad.any(), "%s: %d of %d elements differ" % (what, int(bad.sum()), bad.size)


def _tied_volume(rng, D, H, W):
    vol = (rng.integers(0, 12, (D, H, W)) / 8).astype(np.float32)
    for d in range(D):
        vol[d, :, :min(d, W)] = np.nan
    vol[rng.random((D, H, W)) < 0.05] = np.inf
    vol[:, 0, W - 1] = np.nan
    return vol


# ---- the kernel ----

@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 70, 228, 400, 512])
def test_margin_kernel_equals_the_oracle(D):
    rng = np.random.default_rng(D)
    H, W = 5, 131                                       # W not a multiple of the 128-thread block
    vol = _tied_volume(rng, D, H, W)
    disp, conf = confidence.margin(cu(vol))
    wd, wc = oc.margin(vol)
    same(disp, wd, "disp D %d" % D)
    same(conf, wc, "conf D %d" % D)
    same(disp, adcensus.argmin(cu(vol)[None])[0, 0], "disp vs argmin D %d" % D)


def test_margin_kernel_past_2_31_elements():
    D, H, W = 512, 1100, 3900                           # 2.2e9 elements, 8.8 GB
    assert D * H * W > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(5)
    vol = torch.rand((D, H, W), device="cuda", generator=g).mul_(64).floor_()       # many ties
    disp, conf = confidence.margin(vol)
    rng = np.random.default_rng(6)
    ys = np.concatenate([[0, H - 1, H - 1], rng.integers(0, H, 200)])
    xs = np.concatenate([[0, W - 1, 0], rng.integers(0, W, 200)])
    yt, xt = torch.from_numpy(ys).cuda(), torch.from_numpy(xs).cuda()
    curves = vol[:, yt, xt].cpu().numpy()               # (D, n): every pixel's last planes lie past 2^31
    del vol
    wd, wc = oc.margin(curves[:, None, :])
    same(disp[yt, xt], wd[0], "disp at sampled pixels")
    same(conf[yt, xt], wc[0], "conf at sampled pixels")


# ---- the fused pipeline ----

C, PH, PW, PD = 32, 24, 130, 32                         # W 130: pitch 132 > W
PRESETS = [("kitti", "fast"), ("kitti", "slow"), ("mb", "fast"), ("mb", "slow")]


def _variants(dataset, arch):
    idle = pipeline.idle_steps(pipeline.make_params(dataset, arch))
    return [(t, s) for t, s in sc.VARIANTS if t not in idle and s not in idle]


@pytest.fixture(scope="module")
def pair():
    p = synth.make_pair(PH, PW, C, PD, seed=21)
    return tuple(cu(p[k]) for k in ("featL", "featR", "imgL", "imgR"))


@pytest.mark.parametrize("overlap", [0, 1, 2])
@pytest.mark.parametrize("cbca", ["exact", "fast"])
@pytest.mark.parametrize("dataset,arch", PRESETS)
def test_pipeline_conf_and_lr(pair, dataset, arch, cbca, overlap):
    base = pipeline.make_params(dataset, arch)
    sp = pipeline.StereoPipeline(C, PD + 4, PH + 2, PW + 3, base, cbca_mode=cbca)     # run below the created shape
    sp.set_overlap(overlap)
    nan = float("nan")
    full = lambda *s: torch.full(s, nan, device="cuda")
    for t, s in _variants(dataset, arch):
        what = "%s %s %s overlap %d %s" % (dataset, arch, cbca, overlap, sc.variant_id((t, s)))
        sp.set_params(pipeline.make_params(dataset, arch, sm_terminate=t, sm_skip=s))
        dp = full(PH, PW)
        sp.run_shape(*pair, disp_max=PD, disp=dp)
        n0 = sp.launches_per_run
        d1, conf = full(PH, PW), full(PH, PW)
        sp.run_shape(*pair, disp_max=PD, disp=d1, conf=conf)
        assert sp.launches_per_run == n0, what
        d0, vl, vr = full(PH, PW), full(PD, PH, PW), full(PD, PH, PW)
        sp.run_shape(*pair, disp_max=PD, disp=d0, volL=vl, volR=vr)
        torch.cuda.synchronize()
        same(dp, d0, what + ": disp with and without the volumes")
        torch.cuda.synchronize()
        same(d1, d0, what + ": disp with conf")
        wd, wc = oc.margin(vl.cpu().numpy())
        same(conf, wc, what + ": conf vs the margin of volL")
        if base.lr_check:
            d2, conf2, lr = full(PH, PW), full(PH, PW), full(PH, PW)
            sp.run_shape(*pair, disp_max=PD, disp=d2, conf=conf2, lr=lr)
            d3, lr3 = full(PH, PW), full(PH, PW)
            sp.run_shape(*pair, disp_max=PD, disp=d3, lr=lr3)
            want = torch.zeros((1, 1, PH, PW), device="cuda")
            adcensus.outlier_detection(adcensus.argmin(vl[None]), adcensus.argmin(vr[None]), want, PD)
            torch.cuda.synchronize()
            same(d2, d0, what + ": disp with conf and lr")
            same(d3, d0, what + ": disp with lr")
            same(conf2, wc, what + ": conf with lr")
            same(lr, want, what + ": lr")
            same(lr3, want, what + ": lr alone")
        else:
            lr = full(PH, PW)
            with pytest.raises(adcensus.AdcensusError, match="LR check"):
                sp.run_shape(*pair, disp_max=PD, disp=d1, lr=lr)
            one = torch.full((PH, PW), nan, device="cuda")
            p = [x.data_ptr() for x in pair]
            rc = adcensus.lib().mccnn_pipeline_run_shape_conf(sp._h, PH, PW, PD, *p, one.data_ptr(), None, lr.data_ptr(),
                                                              None, None, None)
            torch.cuda.synchronize()
            assert rc == -1 and torch.isnan(one).all() and torch.isnan(lr).all(), what
    sp.close()


@pytest.mark.parametrize("arch", ["slow", "ad", "census"])
def test_operator_chain_equals_run_volumes(pair, arch):
    """pipeline.stereo_predict's conf / lr equal mccnn_pipeline_run_volumes_conf's in exact mode"""
    dataset = "kitti"
    H, W, D = PH, PW, PD
    x = torch.stack([pair[2], pair[3]])[:, None].contiguous()
    head = feats = None
    over = {}
    if arch == "slow":
        rng = np.random.default_rng(8)
        head = scorer_head.ScorerHead(osh.make_weights(rng, 16, 128, 2))
        f = torch.nn.functional.normalize(torch.randn((2, 16, H, W), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)), dim=1)
        feats = f.contiguous()
        over = dict(border=2)
    opt = pipeline.make_params(dataset, arch, **over)
    conf, lr = torch.empty((H, W), device="cuda"), torch.empty((H, W), device="cuda")
    d = pipeline.stereo_predict(x, feats, opt, D, arch=arch, head=head, conf=conf, lr=lr)
    vols = torch.empty((2, D, H, W), device="cuda")
    adcensus.fill_nan(vols)
    if arch == "ad":
        adcensus.ad(x[0:1], x[1:2], vols[0:1], -1)
        adcensus.ad(x[1:2], x[0:1], vols[1:2], 1)
    elif arch == "census":
        adcensus.census(x[0:1], x[1:2], vols[0:1], -1)
        adcensus.census(x[1:2], x[0:1], vols[1:2], 1)
    else:
        vl, vr = head.volumes(feats[0].contiguous(), feats[1].contiguous(), D)
        vols[0:1].copy_(vl)
        vols[1:2].copy_(vr)
        adcensus.fix_border(vols[0:1], opt.border, -1)
        adcensus.fix_border(vols[1:2], opt.border, 1)
    sp = pipeline.StereoPipeline(C, D, H, W, opt, cbca_mode="exact")
    conf2, lr2 = torch.empty((H, W), device="cuda"), torch.empty((H, W), device="cuda")
    d2 = sp.run_volumes(vols[0], vols[1], x[0, 0], x[1, 0], disp_max=D, conf=conf2, lr=lr2)
    torch.cuda.synchronize()
    same(d2, d[0, 0], arch + " disp")
    same(conf2, conf, arch + " conf")
    same(lr2, lr, arch + " lr")
    sp.close()
    if head is not None:
        head.close()


# ---- sparsify and the counts ----

@pytest.mark.parametrize("H,W", [(375, 1242), (1988, 2964)])
def test_sparsify_and_counts_equal_numpy(H, W):
    rng = np.random.default_rng(H)
    disp = (rng.random((H, W)) * 200).astype(np.float32)
    conf = (rng.integers(0, 50, (H, W)) / 7).astype(np.float32)        # ties
    conf[rng.random((H, W)) < 0.01] = 0
    gt = np.where(rng.random((H, W)) < 0.4, disp + rng.normal(0, 3, (H, W)), 0).astype(np.float32)
    for density in (0.5, 0.123, 1.0, 1e-7):
        n = confidence.n_keep(density, H, W)
        for invalid in (0.0, float("inf"), float("nan")):
            got = confidence.sparsify(cu(disp), cu(conf), density, invalid)
            same(got, oc.sparsify(disp, conf, n, invalid), "sparsify %s %g %g" % ((H, W), density, invalid))
    M, B, bad = confidence.counts(cu(disp), cu(conf), cu(gt), 3.0)
    assert (M, B, bad) == oc.counts(disp, conf, gt, 3.0)
    res = confidence.sparsification(cu(disp), cu(conf), cu(gt), 1.0)
    want = oc.counts(disp, conf, gt, 1.0)
    assert (res.M, res.B, res.bad) == want
    assert (res.curve, res.auc, res.auc_opt) == tuple(oc.curve(*want))
    z = np.zeros_like(gt)
    r0 = confidence.sparsification(cu(disp), cu(conf), cu(z), 3.0)
    assert (r0.M, r0.B, r0.bad) == (0, 0, [0] * 20) and np.isnan(r0.auc)


def test_sparsify_refuses_what_it_cannot_keep():
    lib = adcensus.lib()
    a = torch.zeros((4, 5), device="cuda")
    for n in (0, 21, -1):
        assert lib.mccnn_sparsify(a.data_ptr(), a.data_ptr(), a.data_ptr(), 4, 5, n, 0.0, None) == -1
    assert lib.mccnn_sparsify(None, a.data_ptr(), a.data_ptr(), 4, 5, 3, 0.0, None) == -1
    assert lib.mccnn_sparsification_counts(a.data_ptr(), a.data_ptr(), a.data_ptr(), 4, 5, 3.0, None, None) == -1
    assert lib.mccnn_margin_confidence(a.data_ptr(), None, a.data_ptr(), 1, 4, 5, None) == -1


# ---- the command-line tools on synthetic sets ----

@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("confidence"))
    synth.write_kitti_set(root, "kitti", n_tr=3, n_te=2, H=24, width=120, widths=(120, 111), seed=71)
    synth.write_mb_set(root, n=6, shapes=((24, 64, 16), (28, 72, 20)), seed=72)
    return root


@pytest.mark.parametrize("dataset", ["kitti", "mb"])
def test_run_main_predict_confidence(tmp_path, monkeypatch, capsys, dataset):
    from PIL import Image

    H, W, D, shift = 26, 72, 10, 4
    base = synth.natural_image(np.random.default_rng(73), H, W + shift)
    u8 = np.clip((base - base.min()) / (base.max() - base.min()) * 255.0, 0, 255).astype(np.uint8)
    lp, rp = str(tmp_path / "l.png"), str(tmp_path / "r.png")
    Image.fromarray(np.ascontiguousarray(u8[:, :W])).save(lp)
    Image.fromarray(np.ascontiguousarray(u8[:, shift:])).save(rp)
    monkeypatch.chdir(tmp_path)
    rm = _load("run_main", "tools", "run_main.py")
    rm.main([dataset, "census", "-a", "predict", "-left", lp, "-right", rp, "-disp_max", str(D), "-confidence"])
    lines = capsys.readouterr().out.splitlines()
    names = ["conf"] + (["lr"] if dataset == "kitti" else [])
    assert lines == ["Writing %s.bin, 1 x 1 x %d x %d" % (n, H, W) for n in names]
    assert not os.path.exists(tmp_path / "lr.bin") or dataset == "kitti"
    vl = np.fromfile(str(tmp_path / "left.bin"), "<f4").reshape(D, H, W)
    vr = np.fromfile(str(tmp_path / "right.bin"), "<f4").reshape(D, H, W)
    same(np.fromfile(str(tmp_path / "conf.bin"), "<f4"), oc.margin(vl)[1].ravel(), "conf.bin")
    if dataset == "kitti":
        want = torch.zeros((1, 1, H, W), device="cuda")
        adcensus.outlier_detection(adcensus.argmin(cu(vl)[None]), adcensus.argmin(cu(vr)[None]), want, D)
        same(np.fromfile(str(tmp_path / "lr.bin"), "<f4"), want.cpu().numpy().ravel(), "lr.bin")


@pytest.mark.parametrize("dataset", ["kitti", "mb"])
def test_sparsification_err_equals_test_te(sets, capsys, dataset):
    rm = _load("run_main", "tools", "run_main.py")
    rm.main([dataset, "census", "-a", "test_te", "-data_root", sets])
    errs = [l.split("\t")[1] for l in capsys.readouterr().out.strip().splitlines()[:-1]]
    spt = _load("sparsification", "tools", "sparsification.py")
    res = spt.main([dataset, "census", "-a", "test_te", "-data_root", sets])
    lines = capsys.readouterr().out.strip().splitlines()
    assert len(lines) == len(errs) + 1 and lines[-1].startswith("mean\t")
    for line, err, (id_, r) in zip(lines, errs, res):
        f = line.split("\t")
        assert f[0] == str(id_) and f[1] == err
        assert float(f[3]) <= float(f[2]) and r.auc_opt <= r.auc
        assert f[2] == evaluate.lua_num(r.auc) and f[3] == evaluate.lua_num(r.auc_opt)


# ---- sparse maps from the prediction tools ----

@pytest.fixture(scope="module")
def raw(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("sparse"))
    unzip = synth.write_kitti_raw(root, "kitti", n_tr=2, n_te=2, seed=81)
    synth.write_kitti_eval_maps(unzip, "kitti", seed=82)
    mb_unzip = synth.write_mb_raw(root, seed=83)
    synth.write_mb_eval_gt(mb_unzip, seed=84)
    return root


def test_kitti_eval_predict_density_then_score(raw, capsys, tmp_path):
    from mccnn_b200 import dataio
    from mccnn_b200 import kitti_eval as ke

    ktool = _load("kitti_eval_tool", "tools", "kitti_eval.py")
    out = str(tmp_path / "out")
    ktool.main(["predict", "kitti", "-arch", "census", "-data_root", raw, "-density", "0.5", "-out", out])
    printed = capsys.readouterr().out
    ktool.main(["score", "kitti", out, "-data_root", raw])
    assert capsys.readouterr().out == printed
    res = ke.score_dir("kitti", out, data_root=raw, verbose=False)
    for i, f in enumerate(ke.training_files(raw, "kitti")):
        est = dataio.read_png16_raw(ke.submission_file(out, "kitti", i))
        gt = dataio.read_png16_raw(f[3])
        assert (est > 0).sum() <= -(-est.size // 2)
        want = ((est > 0) & (gt > 0)).sum() / (gt > 0).sum()
        assert res.pairs[i]["density"] == pytest.approx(want, rel=1e-12)


def test_predict_kitti_submit_density(raw, capsys, tmp_path, monkeypatch):
    from mccnn_b200 import dataio
    from mccnn_b200 import predict_kitti as pk

    out = str(tmp_path / "out")
    pk.predict_kitti("submit", "kitti", arch="census", data_root=raw, out=out, density=0.5)
    capsys.readouterr()
    ev = evaluate.Evaluator("kitti", "census")
    try:
        for i, pair in enumerate(pk.pair_files(raw, "kitti", "submit")):
            left, right, _ = pk.decode(pair)
            x = frontend.make_batch_cuda(left, right, ev.dev)
            H, W = x.shape[2:]
            ev.prepare([(H, W, pk.DISP_MAX)])
            conf = torch.empty((H, W), device=ev.dev)
            pred = ev.stereo_predict(x, pk.DISP_MAX, conf=conf).cpu().numpy()
            kept = np.zeros(H * W, bool)
            kept[oc.order(conf.cpu().numpy())[:-(-H * W // 2)]] = True
            kept = kept.reshape(H, W)
            png = dataio.read_png16_raw(os.path.join(out, "%06d_10.png" % i))
            assert kept.sum() == -(-H * W // 2)
            assert np.array_equal(png > 0, kept & (pred * np.float32(256) >= 1)), "pair %d" % i
    finally:
        ev.close()


def test_mb_eval_predict_density(raw, capsys, tmp_path):
    from mccnn_b200 import mb_eval as me

    out = str(tmp_path / "out")
    res = me.evaluate_training("census", None, data_root=raw, out=out, density=0.8)
    printed = capsys.readouterr().out
    again = me.score_dir(out, data_root=raw)
    assert capsys.readouterr().out == printed
    for s, ev_ in zip(res.scenes, res.evals):
        disp = me._read_topdown(me.find_map(out, s))
        assert np.isfinite(disp).sum() == -(-disp.size * 8 // 10)
        assert np.isposinf(disp[~np.isfinite(disp)]).all()
    assert all(x.tobytes() == y.tobytes() for a, b in zip(again.evals, res.evals) for x, y in zip(a, b))
    # the counts behind the invalid share are the SDK oracle's on the written sparse map (scene 0, at F)
    from mccnn_b200 import preprocess
    from oracle import mb_evaldisp as od

    s0 = res.scenes[0]
    gt_f, mask_f = me.gt_files(raw, s0, "F")
    c, _, _ = od.evaldisp(me._read_topdown(me.find_map(out, s0)), me._read_topdown(gt_f), preprocess._read_grey(mask_f),
                          preprocess._ndisp(os.path.join(me.scene_dir(raw, s0), "calib.txt")))
    assert np.array_equal(c, res.evals[0].counts)
    assert res.rows[0]["all_invalid"] > 0
