"""GPU: main.lua's -sm_terminate / -sm_skip (main.lua:953-1082) through every layer -- the fused pipeline's entry points in
both CBCA modes and both overlap modes against the reference's own kernels (tests/stage_chain.reference_chain, where
oracle/_ref has been built) and the CPU oracle chain (stage_chain.oracle_chain); the operator path; set_params; the launch
count; and tools/run_main.py, tools/ablation.py and Evaluator on synthetic sets."""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import evaluate, pipeline, scorer_head, search, synth  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


sc = _load("stage_chain", "tests", "stage_chain.py")
IDS = [sc.variant_id(v) for v in sc.VARIANTS]


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def same(got, want, what):
    g = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    w = want.detach().cpu().numpy() if isinstance(want, torch.Tensor) else np.asarray(want)
    g, w = g.reshape(w.shape), w
    bad = ~((g == w) | (np.isnan(g) & np.isnan(w)))
    assert not bad.any(), "%s: %d of %d elements differ" % (what, int(bad.sum()), bad.size)


def shim():
    from oracle import refdriver

    return refdriver.ShimLibrary(refdriver.REF_LIB) if os.path.exists(refdriver.REF_LIB) else None


# (dataset, arch, overrides): the KITTI accurate preset (LR check, CBCA x4, arms of 5) and a Middlebury preset (no LR check,
# arms of 5, mb's five-layer border) on StereoJoin volumes
EDGE_PRESETS = {"kitti": ("kitti", "accurate_cbca4", {}), "mb": ("mb", "census", dict(cbca_i1=2, cbca_i2=4, border=5))}
EH, EW, EC, ED = 37, 203, 32, 40


@pytest.fixture(scope="module")
def edge_pair():
    return synth.make_pair(EH, EW, EC, ED, seed=9)


@pytest.mark.parametrize("ds", ["kitti", "mb"])
def test_exact_every_variant_at_a_tile_edge(oracle, edge_pair, ds):
    """run_shape and run_volumes in exact mode (both overlap modes) bit-identical to the reference's kernels and the oracle,
    for the full chain, every skip and every terminate; left/right volumes as -a predict writes them"""
    dataset, arch, over = EDGE_PRESETS[ds]
    p = edge_pair
    fL, fR, iL, iR = cu(p["featL"]), cu(p["featR"]), cu(p["imgL"]), cu(p["imgR"])
    base = pipeline.make_params(dataset, arch, **over)
    raw_L, raw_R = oracle.stereo_join(p["featL"], p["featR"], ED)
    oracle.fix_border(raw_L, base.border, -1)
    oracle.fix_border(raw_R, base.border, 1)
    sps = {}
    for ov in (2, 0):
        sps[ov] = pipeline.StereoPipeline(EC, ED + 8, EH + 3, EW + 5, base, cbca_mode="exact")   # run below the created shape
        sps[ov].set_overlap(ov)
    ref = shim()
    for t, s in sc.VARIANTS:
        what = "%s %s" % (ds, sc.variant_id((t, s)))
        opt = pipeline.make_params(dataset, arch, sm_terminate=t, sm_skip=s, **over)
        want, wL, wR = sc.oracle_chain(oracle, p["imgL"], p["imgR"], ED, opt, t, s, featL=p["featL"], featR=p["featR"],
                                       want_vols=True)
        if ref is not None:
            rd, rL, rR = sc.reference_chain(ref, torch.stack([iL, iR])[:, None], torch.stack([fL, fR]), opt, ED, t, s,
                                            want_vols=True)
            same(rd, want, what + ": reference kernels vs oracle (disp)")
            same(rL, wL, what + ": reference kernels vs oracle (left)")
        for ov, sp in sps.items():
            sp.set_params(opt)
            vl, vr = torch.empty((ED, EH, EW), device="cuda"), torch.empty((ED, EH, EW), device="cuda")
            d = sp.run_shape(fL, fR, iL, iR, disp_max=ED, volL=vl, volR=vr)
            torch.cuda.synchronize()
            same(d, want, "%s overlap %d: run_shape disp" % (what, ov))
            same(vl, wL, "%s overlap %d: run_shape left volume" % (what, ov))
            same(vr, wR, "%s overlap %d: run_shape right volume" % (what, ov))
            d2 = sp.run_volumes(cu(raw_L), cu(raw_R), iL, iR, disp_max=ED)
            torch.cuda.synchronize()
            same(d2, want, "%s overlap %d: run_volumes disp" % (what, ov))
            if not base.lr_check:                               # mb: the right volume is optional
                same(sp.run_volumes(cu(raw_L), None, iL, iR, disp_max=ED), want, what + ": run_volumes without volR")
    for sp in sps.values():
        sp.close()


def test_default_mode_variants_at_a_tile_edge(edge_pair):
    """default (constant-work) CBCA: every variant of the KITTI preset within the default-mode rule of the exact mode"""
    dataset, arch, over = EDGE_PRESETS["kitti"]
    p = edge_pair
    fL, fR, iL, iR = cu(p["featL"]), cu(p["featR"]), cu(p["imgL"]), cu(p["imgR"])
    sps = {m: pipeline.StereoPipeline(EC, ED, EH, EW, pipeline.make_params(dataset, arch, **over), cbca_mode=m)
           for m in ("exact", "fast")}
    for t, s in sc.VARIANTS:
        out = {}
        for m, sp in sps.items():
            sp.set_params(pipeline.make_params(dataset, arch, sm_terminate=t, sm_skip=s, **over))
            vl = torch.empty((ED, EH, EW), device="cuda")
            out[m] = (sp.run(fL, fR, iL, iR, volL=vl).clone(), vl)
        torch.cuda.synchronize()
        (de, ve), (df, vf) = out["exact"], out["fast"]
        assert bool((torch.isnan(ve) == torch.isnan(vf)).all())
        assert bool((torch.isnan(ve) | ((vf - ve).abs() <= 1e-4 * ve.abs().clamp(min=1.0))).all()), (t, s)
        frac = float(((df - de).abs() > 1e-4 * de.abs().clamp(min=1.0)).float().mean())
        assert frac < 5e-3, "%s: %.4f of the map changed" % (sc.variant_id((t, s)), frac)
    for sp in sps.values():
        sp.close()


def test_full_size_skip_variants():
    """BASELINE's full size (370 x 1226, D 228, the bench preset): every skip variant bit-identical in exact mode to the
    reference's kernels (or, without oracle/_ref, to the operator chain); in the default mode, volumes within 1e-4 and the
    disparity map within 1e-4 on >= 1 - 1e-4 of the pixels"""
    H, W, C, D = 370, 1226, 64, 228
    p = synth.make_pair(H, W, C, D, seed=2)
    fL, fR, iL, iR = cu(p["featL"]), cu(p["featR"]), cu(p["imgL"]), cu(p["imgR"])
    base = pipeline.make_params("kitti", "accurate_cbca4")
    sps = {m: pipeline.StereoPipeline(C, D, H, W, base, cbca_mode=m) for m in ("exact", "fast")}
    ref = shim()
    for s in sc.SKIP:
        opt = pipeline.make_params("kitti", "accurate_cbca4", sm_skip=s)
        if ref is not None:
            want = sc.reference_chain(ref, torch.stack([iL, iR])[:, None], torch.stack([fL, fR]), opt, D, "", s)
        else:
            want = pipeline.stereo_predict(torch.stack([iL, iR])[:, None], torch.stack([fL, fR]), opt, D)
        want = want.reshape(H, W)
        got = {}
        for m, sp in sps.items():
            sp.set_params(opt)
            got[m] = sp.run(fL, fR, iL, iR).clone()
        torch.cuda.synchronize()
        same(got["exact"], want, "skip %s: exact mode at full size" % s)
        frac = float(((got["fast"] - want).abs() > 1e-4 * want.abs().clamp(min=1.0)).float().mean())
        assert frac <= 1e-4, "skip %s: default mode changed %.3g of the map (bar 1e-4)" % (s, frac)
        del want
    for sp in sps.values():
        sp.close()


def _batch_inputs(n, H, W, C, D):
    return [synth.make_pair(H, W, C, D, seed=30 + i) for i in range(n)]


@pytest.mark.parametrize("variant", [("sgm", "median"), ("cnn", ""), ("", "cbca"), ("mismatch", "")],
                         ids=lambda v: "%s_%s" % v)
def test_batch_entry_points_give_the_bits_of_run_shape(variant):
    t, s = variant
    H, W, C, D = 30, 96, 16, 24
    opt = pipeline.make_params("kitti", "accurate_cbca4", sm_terminate=t, sm_skip=s)
    pairs = _batch_inputs(3, H, W, C, D)
    sp = pipeline.StereoPipeline(C, D, H, W, opt, cbca_mode="exact")
    dev_pairs = [(cu(q["featL"]), cu(q["featR"]), cu(q["imgL"]), cu(q["imgR"])) for q in pairs]
    want = [sp.run_shape(*dp, disp_max=D).clone() for dp in dev_pairs]
    got_b = sp.run_batch(dev_pairs)
    host = [tuple(torch.from_numpy(np.ascontiguousarray(q[k], np.float32)).pin_memory()
                  for k in ("featL", "featR", "imgL", "imgR")) for q in pairs]
    got_h = sp.run_host_batch(host)
    got_1 = sp.run_host(*host[0])
    torch.cuda.synchronize()
    for i in range(3):
        same(got_b[i], want[i], "run_batch pair %d" % i)
        same(got_h[i], want[i], "run_host_batch pair %d" % i)
    same(got_1, want[0], "run_host")
    sp.close()


def test_set_params_round_trip_and_launch_counts():
    H, W, C, D = 30, 96, 16, 24
    q = synth.make_pair(H, W, C, D, seed=40)
    args = (cu(q["featL"]), cu(q["featR"]), cu(q["imgL"]), cu(q["imgR"]))
    sp = pipeline.StereoPipeline(C, D, H, W, pipeline.make_params("kitti", "accurate_cbca4"))
    sp.run(*args)
    torch.cuda.synchronize()
    o = sp.params
    # default parameters: the parent's count -- volumes 4, cross 2 + pack 2, per direction CBCA + 7 per SGM iteration +
    # argmin, LR check 3, subpixel / median / bilateral 3
    assert sp.launches_per_run == 4 + 4 + 2 * (o.cbca_i1 + 7 * o.sgm_i + o.cbca_i2 + 1) + 3 + 3
    counts = {}
    for t, s in sc.VARIANTS[1:] + [("", "")]:
        opt = pipeline.make_params("kitti", "accurate_cbca4", sm_terminate=t, sm_skip=s)
        sp.set_params(opt)
        got = sp.run(*args).clone()
        torch.cuda.synchronize()
        counts[(t, s)] = sp.launches_per_run
        fresh = pipeline.StereoPipeline(C, D, H, W, opt)
        same(got, fresh.run(*args), "set_params to %s" % sc.variant_id((t, s)))
        torch.cuda.synchronize()
        assert fresh.launches_per_run == counts[(t, s)]
        fresh.close()
    full = counts[("", "")]
    assert full == 4 + 4 + 2 * (o.cbca_i1 + 7 * o.sgm_i + o.cbca_i2 + 1) + 3 + 3
    assert counts[("cnn", "")] == 4 + 1                  # the volumes and the left argmin: nothing else is read
    assert counts[("", "cbca")] == full - 4 - 2 * (o.cbca_i1 + o.cbca_i2)
    assert counts[("", "sgm")] == full - 2 * 7 * o.sgm_i
    assert counts[("", "occlusion")] == full - 3 - (o.cbca_i1 + 7 * o.sgm_i + o.cbca_i2 + 1)   # no direction +1
    assert counts[("", "bilateral")] == counts[("", "median")] == counts[("median", "")] == full - 1
    sp.close()


def test_operator_path_census_and_slow_volumes(oracle):
    """pipeline.stereo_predict, arch census (KITTI preset) and arch slow (a random ScorerHead, Middlebury preset)"""
    H, W, D = 20, 61, 12
    rng = np.random.default_rng(50)
    imgL, imgR = (synth._standardise(synth.natural_image(rng, H, W)).astype(np.float32) for _ in range(2))
    xb = cu(np.stack([imgL, imgR])[:, None])
    fm = 16
    feats = torch.relu(cu(rng.standard_normal((2, fm, H, W))))
    head = scorer_head.ScorerHead(osh.make_weights(rng, fm, 128, 2))
    vl, vr = head.volumes(feats[0].contiguous(), feats[1].contiguous(), D)
    torch.cuda.synchronize()
    for t, s in sc.VARIANTS:
        what = sc.variant_id((t, s))
        opt = pipeline.make_params("kitti", "census", sm_terminate=t, sm_skip=s)
        got, gL, gR = pipeline.stereo_predict(xb, None, opt, D, want_vols=True, arch="census")
        want, wL, wR = sc.oracle_chain(oracle, imgL, imgR, D, opt, t, s, arch="census", want_vols=True)
        same(got, want, "census %s disp" % what)
        same(gL, wL, "census %s left" % what)
        same(gR, wR, "census %s right" % what)
        opt = pipeline.make_params("mb", "slow", sm_terminate=t, sm_skip=s, cbca_i2=3)
        got = pipeline.stereo_predict(xb, feats, opt, D, arch="slow", head=head)
        hl, hr = vl.cpu().numpy().reshape(D, H, W).copy(), vr.cpu().numpy().reshape(D, H, W).copy()
        oracle.fix_border(hl, opt.border, -1)
        oracle.fix_border(hr, opt.border, 1)
        want = sc.oracle_chain(oracle, imgL, imgR, D, opt, t, s, arch="volumes", volL=hl, volR=hr)
        same(got, want, "slow %s disp" % what)
    head.close()


# ---- the command-line tools on synthetic sets ----

@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("stages"))
    synth.write_kitti_set(root, "kitti", n_tr=3, n_te=2, H=24, width=120, widths=(120, 111), seed=61)
    synth.write_mb_set(root, n=6, shapes=((24, 64, 16), (28, 72, 20)), seed=62)
    return root


def _oracle_errs(oracle, data, dataset, opt, t, s):
    from mccnn_b200 import dataio

    errs = []
    for ex in data.examples("test_te"):
        x, disp_max, _, _, img_width = data.example(ex)
        d = sc.oracle_chain(oracle, x[0, 0], x[1, 0], disp_max, opt, t, s, arch="census")
        errs.append(dataio.bad_pixel_rate(d, data.ground_truth(ex, img_width), dataio.ERR_AT[dataset]))
    return errs


@pytest.mark.parametrize("dataset", ["kitti", "mb"])
def test_run_main_test_te_skip_sgm(oracle, sets, dataset, capsys):
    rm = _load("run_main", "tools", "run_main.py")
    rm.main([dataset, "census", "-a", "test_te", "-data_root", sets, "-sm_skip", "sgm"])
    lines = capsys.readouterr().out.strip().splitlines()
    opt = pipeline.make_params(dataset, "census", sm_skip="sgm")
    errs = _oracle_errs(oracle, evaluate.load_data(dataset, sets), dataset, opt, "", "sgm")
    assert len(lines) == len(errs) + 1
    for line, e in zip(lines, errs):
        assert line.split("\t")[1] == evaluate.lua_num(e)
    assert lines[-1] == evaluate.lua_num(sum(errs) / len(errs))


@pytest.mark.parametrize("dataset", ["kitti", "mb"])
def test_run_main_predict_terminate_cbca1(oracle, tmp_path, monkeypatch, dataset):
    from PIL import Image

    from mccnn_b200 import frontend

    H, W, D, shift = 26, 72, 10, 4
    base = synth.natural_image(np.random.default_rng(70), H, W + shift)
    u8 = np.clip((base - base.min()) / (base.max() - base.min()) * 255.0, 0, 255).astype(np.uint8)
    lp, rp = str(tmp_path / "l.png"), str(tmp_path / "r.png")
    Image.fromarray(np.ascontiguousarray(u8[:, :W])).save(lp)
    Image.fromarray(np.ascontiguousarray(u8[:, shift:])).save(rp)
    monkeypatch.chdir(tmp_path)
    rm = _load("run_main", "tools", "run_main.py")
    rm.main([dataset, "census", "-a", "predict", "-left", lp, "-right", rp, "-disp_max", str(D), "-sm_terminate", "cbca1"])
    batch = frontend.make_batch(lp, rp)
    opt = pipeline.make_params(dataset, "census", sm_terminate="cbca1")
    want, wL, wR = sc.oracle_chain(oracle, batch[0, 0], batch[1, 0], D, opt, "cbca1", "", arch="census", want_vols=True)
    for name, ref in (("right.bin", wR), ("left.bin", wL), ("disp.bin", want)):
        data = np.fromfile(str(tmp_path / name), "<f4")
        assert data.size == ref.size
        same(data, ref.ravel(), name)


@pytest.mark.parametrize("dataset", ["kitti", "mb"])
def test_ablation_lines_equal_single_variant_evaluators(sets, dataset, capsys):
    ab = _load("ablation", "tools", "ablation.py")
    res = ab.main([dataset, "census", "-", "-data_root", sets])
    captured = capsys.readouterr()
    lines = captured.out.strip().splitlines()
    variants = search.ablation_variants(pipeline.make_params(dataset, "census"))
    assert len(variants) == (15 if dataset == "kitti" else 12)
    assert [l.split("\t")[0] for l in lines] == [l for l, _ in variants] and len(res) == len(variants)
    for (label, ov), line, (_, score) in zip(variants, lines, res):
        ev = evaluate.Evaluator(dataset, "census", **ov)
        try:
            mean = ev.test("test_te", data_root=sets, verbose=False).mean
            want = float("%.14g" % mean)
            assert score == want, "%s: ablation %r, Evaluator %r" % (label, score, want)
            assert line.split("\t")[1] == evaluate.lua_num(want)
        except ValueError as e:                              # NaN prediction: main.lua:1224 would assert
            assert "NaN" in str(e) and np.isnan(score) and line.split("\t")[1] == "nan"
            assert label in captured.err
        finally:
            ev.close()
