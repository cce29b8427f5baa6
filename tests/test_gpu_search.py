"""GPU: the pieces of the test_te parameter search.

* mccnn_pipeline_set_params: a re-targeted pipeline gives the bits of one created with the parameters (disparity map and both
  volumes), over seeded grid points, in both CBCA modes and overlap on / off, at the created shape and below it, with a
  blur_sigma that grows the Gaussian buffer, L1 crossing the constant-work CBCA's arm limit, and run_batch's twin lanes;
* mccnn_pipeline_run_volumes: from StereoJoin + fix_border volumes it equals run_shape, from census volumes and from the
  scorer head's volumes (exact mode) the operator chain pipeline.stereo_predict -- also with volR = NULL on Middlebury;
* search.Searcher.score equals '%.14g' of Evaluator(...).test('test_te').mean and its per-example errors, and arch 'slow'
  runs the scorer head once per example however many points are scored;
* tools/hs.py end to end (random, then hillclimb_fast on the same log), and a candidate with a NaN prediction.
"""
import importlib.util
import os
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, evaluate, feature_tower, pipeline, scorer_head, search, synth, t7  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = 64
CREATED = (32, 96, 40)        # (H, W, D)
SMALL = (24, 77, 30)


def _hs():
    spec = importlib.util.spec_from_file_location("hs", os.path.join(ROOT, "tools", "hs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def world(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("search"))
    # D = 228 on KITTI: widths >= 228 + border + 1 keep every fix_border'ed volume finite on its valid part
    synth.write_kitti_set(root, "kitti", n_tr=6, n_te=1, H=32, width=300, widths=(300, 263, 281), seed=21)
    synth.write_mb_set(root, n=6, shapes=((32, 96, 24), (40, 110, 40)), seed=22)
    rng = np.random.default_rng(23)
    layers = {"fast": (oft.make_weights(rng, l1=3, fm=64), None),
              "slow": (oft.make_weights(rng, l1=3, fm=16), osh.make_weights(rng, 16, 128, 2))}
    nets = {}
    for arch, (tower, head) in layers.items():
        nets[arch] = os.path.join(root, "net_%s.t7" % arch)
        t7.save_net(nets[arch], tower, head)
    return dict(root=root, layers=layers, nets=nets)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pair(shape, seed):
    h, w, d = shape
    p = synth.make_pair(h, w, C, d, seed=seed)
    return _t(p["featL"]), _t(p["featR"]), _t(p["imgL"]), _t(p["imgR"])


def _outputs(shape):
    h, w, d = shape
    nan = float("nan")
    return (torch.full((h, w), nan, device="cuda"), torch.full((d, h, w), nan, device="cuda"),
            torch.full((d, h, w), nan, device="cuda"))


def _run(sp, ins, shape):
    disp, vl, vr = _outputs(shape)
    if shape == (sp.H, sp.W, sp.D):
        sp.run(*ins, disp=disp, volL=vl, volR=vr)
    else:
        sp.run_shape(*ins, disp_max=shape[2], disp=disp, volL=vl, volR=vr)
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (disp, vl, vr)]


def _configure(sp, cbca, overlap):
    sp.set_cbca_mode(cbca)
    sp.set_overlap(overlap)


def _same(got, want, what, names=("disp", "volL", "volR")):
    for g, w, name in zip(got, want, names):
        assert g.shape == w.shape, "%s %s: shape %s vs %s" % (what, name, g.shape, w.shape)
        assert np.array_equal(g, w, equal_nan=True), "%s: %s differs" % (what, name)


def _points(dataset, arch, n, seed, forced=()):
    """n valid seeded grid points of search.grid(dataset, arch) as dicts, after the `forced` ones"""
    params = search.grid(dataset, arch)
    rng = random.Random(seed)
    out = [dict(f) for f in forced]
    while len(out) < n:
        ps = dict(search.point(params, search.propose("random", params, rng)))
        if search.valid(ps):
            out.append(ps)
    return out


PRESETS = [("kitti", "slow"), ("kitti", "census"), ("mb", "census")]


@pytest.mark.parametrize("overlap", [0, 2])
@pytest.mark.parametrize("cbca", ["fast", "exact"])
@pytest.mark.parametrize("dataset,arch", PRESETS)
def test_set_params_equals_a_fresh_pipeline(dataset, arch, cbca, overlap):
    kitti = dataset == "kitti"
    forced = []
    if kitti:          # arms across the constant-work limit (L1 6 -> exact kernels, then back), the largest Gaussian
        forced = [dict(L1=6, blur_sigma=10.0, pi1=1.0, pi2=32.0), dict(L1=5, cbca_i1=2, cbca_i2=2, pi1=1.0, pi2=32.0),
                  dict(L1=6, cbca_i1=4, cbca_i2=0, blur_sigma=1.0)]
    else:
        forced = [dict(blur_sigma=10.0, pi1=1.0, pi2=32.0)]
    points = _points(dataset, arch, 10, seed=11 + PRESETS.index((dataset, arch)), forced=forced)
    base = pipeline.make_params(dataset, arch, blur_sigma=1.0)          # smallest Gaussian: 10.0 must grow the buffer
    sp = pipeline.StereoPipeline(C, CREATED[2], CREATED[0], CREATED[1], base)
    _configure(sp, cbca, overlap)
    ins = {s: _pair(s, seed=s[1]) for s in (CREATED, SMALL)}
    for k, pt in enumerate(points):
        opt = pipeline.make_params(dataset, arch, **pt)
        shape = SMALL if k % 3 == 1 else CREATED
        fresh = pipeline.StereoPipeline(C, shape[2], shape[0], shape[1], opt)
        _configure(fresh, cbca, overlap)
        want = _run(fresh, ins[shape], shape)
        fresh.close()
        sp.set_params(opt)
        _same(_run(sp, ins[shape], shape), want, "%s %s point %d %s at %s" % (dataset, arch, k, pt, shape))
    # the twin lanes of run_batch follow set_params: a batch at the created shape, then re-targeted again
    pairs = [_pair(CREATED, seed=s) for s in (1, 2, 3)]
    for pt in points[-2:]:
        opt = pipeline.make_params(dataset, arch, **pt)
        sp.set_params(opt)
        got = sp.run_batch(pairs)
        torch.cuda.synchronize()
        fresh = pipeline.StereoPipeline(C, CREATED[2], CREATED[0], CREATED[1], opt)
        _configure(fresh, cbca, overlap)
        for j, pr in enumerate(pairs):
            want = _run(fresh, pr, CREATED)[0]
            assert np.array_equal(got[j].cpu().numpy(), want, equal_nan=True), "run_batch pair %d after set_params" % j
        fresh.close()
    sp.close()


def test_set_params_rejects_bad_parameters():
    sp = pipeline.StereoPipeline(C, 16, 16, 32, pipeline.make_params("kitti", "fast"))
    for bad in (dict(border=32), dict(cbca_i1=-1), dict(sgm_i=-1)):
        with pytest.raises(adcensus.AdcensusError, match="invalid argument"):
            sp.set_params(pipeline.make_params("kitti", "fast", **bad))
    sp.set_params(pipeline.make_params("kitti", "fast", border=31))                    # border + 1 == created W
    sp.close()


def _join_volumes(featL, featR, d, border):
    _, h, w = featL.shape
    vols = torch.empty((2, d, h, w), device="cuda")
    adcensus.fill_nan(vols)
    adcensus.StereoJoin(featL[None], featR[None], vols[0:1], vols[1:2])
    adcensus.fix_border(vols[0:1], border, -1)
    adcensus.fix_border(vols[1:2], border, 1)
    return vols[0:1], vols[1:2]


@pytest.mark.parametrize("shape", [CREATED, SMALL])
def test_run_volumes_from_stereo_join_equals_run_shape(shape):
    opt = pipeline.make_params("kitti", "fast")
    sp = pipeline.StereoPipeline(C, CREATED[2], CREATED[0], CREATED[1], opt)
    ins = _pair(shape, seed=5)
    want = _run(sp, ins, shape)
    vl, vr = _join_volumes(ins[0], ins[1], shape[2], opt.border)
    keep = (vl.clone(), vr.clone())
    disp, ol, orr = _outputs(shape)
    sp.run_volumes(vl, vr, ins[2], ins[3], disp_max=shape[2], disp=disp, outL=ol, outR=orr)
    torch.cuda.synchronize()
    _same([x.cpu().numpy() for x in (disp, ol, orr)], want, "run_volumes vs run_shape at %s" % (shape,))
    assert torch.equal(torch.nan_to_num(vl, 7.0), torch.nan_to_num(keep[0], 7.0)), "run_volumes modified volL"
    assert torch.equal(torch.nan_to_num(vr, 7.0), torch.nan_to_num(keep[1], 7.0)), "run_volumes modified volR"
    sp.close()


def _chain_case(world, dataset, arch, shape, seed):
    """x_batch, features, head and Params of one pair for the operator chain"""
    h, w, d = shape
    rng = np.random.default_rng(seed)
    views, _ = synth._scene_views(rng, h, w, d)
    xb = _t(views[:, None])
    feats = head = None
    opt = pipeline.make_params(dataset, arch)
    if arch == "slow":
        tl, hl = world["layers"]["slow"]
        tower = feature_tower.FeatureTower(tl, arch="slow")
        head = scorer_head.ScorerHead(hl)
        feats = tower.forward(xb)
        opt = pipeline.make_params(dataset, arch, border=3)
    return xb, feats, head, opt


@pytest.mark.parametrize("dataset,arch", [("kitti", "census"), ("kitti", "slow"), ("mb", "census"), ("mb", "slow")])
def test_run_volumes_equals_the_operator_chain(world, dataset, arch):
    shape = (32, 96, 40)
    h, w, d = shape
    xb, feats, head, opt = _chain_case(world, dataset, arch, shape, seed=31)
    want_d, want_l, want_r = pipeline.stereo_predict(xb, feats, opt, d, want_vols=True, arch=arch, head=head)
    torch.cuda.synchronize()
    if arch == "census":
        vols = torch.empty((2, d, h, w), device="cuda")
        adcensus.fill_nan(vols)
        adcensus.census(xb[0:1], xb[1:2], vols[0:1], -1)
        adcensus.census(xb[1:2], xb[0:1], vols[1:2], 1)
        vl, vr = vols[0:1], vols[1:2]
    else:
        vl, vr = head.volumes(feats[0].contiguous(), feats[1].contiguous(), d)
        adcensus.fix_border(vl, opt.border, -1)
        adcensus.fix_border(vr, opt.border, 1)
    sp = pipeline.StereoPipeline(1, 48, 40, 128, opt, cbca_mode="exact")        # created larger than the run
    cases = [(vr, True)] + ([(None, False)] if not opt.lr_check else [])
    for volR, want_right in cases:
        disp, ol, orr = _outputs(shape)
        sp.run_volumes(vl, volR, xb[0, 0], xb[1, 0], disp_max=d, disp=disp, outL=ol, outR=orr if want_right else None)
        torch.cuda.synchronize()
        what = "%s %s run_volumes (volR %s)" % (dataset, arch, "given" if volR is not None else "NULL")
        _same([disp.cpu().numpy(), ol.cpu().numpy()], [want_d[0, 0].cpu().numpy(), want_l[0].cpu().numpy()], what,
              ("disp", "volL"))
        if want_right:
            _same([orr.cpu().numpy()], [want_r[0].cpu().numpy()], what, ("volR",))
    sp.close()


def _evaluator_result(world, dataset, arch, pt):
    net = world["nets"].get(arch)
    ev = evaluate.Evaluator(dataset, arch, net_fname=net, **pt)
    try:
        return ev.test("test_te", data_root=world["root"], verbose=False)
    except ValueError as e:
        assert "NaN" in str(e)
        return None
    finally:
        ev.close()


@pytest.mark.parametrize("dataset,arch", [("kitti", "fast"), ("kitti", "slow"), ("kitti", "census"), ("mb", "fast"),
                                          ("mb", "slow")])
def test_score_equals_the_evaluator(world, dataset, arch):
    s = search.Searcher(dataset, arch, net_fname=world["nets"].get(arch), data_root=world["root"])
    assert s.sp.cbca_mode == ("fast" if arch == "fast" else "exact") or os.environ.get("ADCENSUS_CBCA_EXACT")
    n = len(s.examples)
    assert n == len(evaluate.load_data(dataset, world["root"]).examples("test_te"))
    for pt in _points(dataset, arch, 3, seed=41):
        res = _evaluator_result(world, dataset, arch, pt)
        if res is None:
            with pytest.raises(search.NaNPrediction):
                s.score(pt)
            continue
        score, errs = s.score(pt)
        assert score == float("%.14g" % res.mean), "%s %s %s: %r vs %r" % (dataset, arch, pt, score, res.mean)
        want = [e[3] for e in res.examples]
        assert np.array_equal(np.array(errs), np.array(want), equal_nan=True), (errs, want)
    if arch == "slow":
        assert s.head_calls == n, "the scorer head ran %d times for %d examples" % (s.head_calls, n)
        assert s.cache_bytes == 4 * sum((2 if s.opt.lr_check else 1) * d * h * w for h, w, d in s.shapes)
    s.close()


def _log_points(path, dataset, arch):
    params = search.grid(dataset, arch)
    with open(path) as f:
        lines = f.read().splitlines()
    res = search.parse_log(lines, dataset, arch, params)
    assert len(res) == len(lines)
    return lines, res


def test_hs_end_to_end(world, tmp_path, capsys):
    hs = _hs()
    log = str(tmp_path / "hs.log")
    net = world["nets"]["fast"]
    s = search.Searcher("kitti", "fast", net_fname=net, data_root=world["root"])
    common = ["kitti", "fast", "test_te", net, "-data_root", world["root"], "-log", log]
    hs.main(["random"] + common + ["-n", "3", "-seed", "1"], searcher=s)
    first = capsys.readouterr()
    hs.main(["hillclimb_fast"] + common + ["-n", "2", "-seed", "2"], searcher=s)
    second = capsys.readouterr()
    lines, res = _log_points(log, "kitti", "fast")
    skipped = (first.err + second.err).count("skipped")
    assert len(lines) + skipped == 5 and len(res) >= 1
    assert (first.out + second.out).splitlines() == lines
    params = search.grid("kitti", "fast")
    xs = [search.recover(params, ps) for _, ps in res]
    for line, (score, _), x in zip(lines, res, xs):
        ps = search.point(params, x)
        assert line == search.format_line(score, "kitti", "fast", ps, net)
        assert score == s.score(dict(ps))[0]
    n_random = len(first.out.splitlines())
    for k in range(n_random, len(res)):
        best = search.recover(params, min(res[:k])[1])          # the log's minimum when point k was proposed
        assert all(abs(a - b) <= 1 for a, b in zip(xs[k], best)), "hillclimb point %d is not a neighbour" % k
    s.close()


def test_nan_prediction_is_refused_and_skipped(world, tmp_path, capsys):
    s = search.Searcher("kitti", "census", data_root=world["root"])
    orig = s.predict
    left = {"n": 1}

    def fake(i):                    # example 1's stage yields a prediction with an all-NaN pixel column, once
        d = orig(i)
        if i == 1 and left["n"]:
            left["n"] -= 1
            d = d.clone()
            d[:, 7] = float("nan")
        return d

    s.predict = fake
    pt = _points("kitti", "census", 1, seed=3)[0]
    with pytest.raises(search.NaNPrediction) as e:
        s.score(pt)
    assert e.value.example_id == s.ids[1]
    assert s.score(pt)[0] == s.score(pt)[0]                # and the next call is a normal one
    left["n"] = 1
    hs = _hs()
    log = str(tmp_path / "hs.log")
    hs.main(["random", "kitti", "census", "test_te", "-", "-data_root", world["root"], "-log", log, "-n", "3",
             "-seed", "4"], searcher=s)
    out = capsys.readouterr()
    assert out.err.count("skipped") == 1 and "prediction contains NaN" in out.err
    lines, _ = _log_points(log, "kitti", "census")
    assert len(lines) == 2 and out.out.splitlines() == lines
    s.close()
