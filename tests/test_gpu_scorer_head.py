"""GPU parity of the fused wgmma scorer head (csrc/scorer_head.cu) against the CPU oracle (oracle/scorer_head.py, pinned
to the PyTorch restatement of main.lua:958-984 / SpatialConvolution1_fw.lua by tests/golden/scorer_head.npz).
Bar: the north star's 1e-4 for float work (output is a sigmoid in (0, 1): absolute), NaN pattern identical."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, scorer_head  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402
from oracle import tower_head_cases as cases  # noqa: E402


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to("cuda:0")


def check(got, want, bar):
    got = got.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN pattern differs"
    m = ~np.isnan(want)
    err = float(np.abs(got[m] - want[m]).max())
    assert err <= bar, "max abs error %.3g (bar %.1g)" % (err, bar)
    return err


def test_golden_fixture():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "scorer_head.npz"))
    layers = [(g["w%d" % i], g["b%d" % i]) for i in range(5)]
    head = scorer_head.ScorerHead(layers)
    vL, vR = head.volumes(cu(g["featL"]), cu(g["featR"]), int(g["D"]))
    torch.cuda.synchronize()
    check(vL, g["volL"], 1e-4)
    check(vR, g["volR"], 1e-4)
    head.close()


@pytest.mark.parametrize("fm,nh2,l2,H,W,D", [
    (112, 384, 4, 5, 300, 40),     # kitti net, three tiles per row, ragged last tile
    (112, 384, 3, 2, 130, 130),    # kitti2015 / mb depth (l2 = 3), D reaches past the first tile
    (64, 256, 2, 3, 128, 9),       # one 256-wide instruction per step
    (8, 128, 1, 2, 77, 5),         # smallest legal shapes
])
def test_against_oracle(fm, nh2, l2, H, W, D):
    rng = np.random.default_rng(fm + l2)
    layers = osh.make_weights(rng, fm, nh2, l2)
    fL = np.maximum(rng.standard_normal((fm, H, W)), 0).astype(np.float32)
    fR = np.maximum(rng.standard_normal((fm, H, W)), 0).astype(np.float32)
    head = scorer_head.ScorerHead(layers)
    vL, vR = head.volumes(cu(fL), cu(fR), D)
    torch.cuda.synchronize()
    wantL = osh.head_volume(fL, fR, D, layers, -1)[None]
    wantR = osh.head_volume(fL, fR, D, layers, 1)[None]
    e = check(vL, wantL, 1e-4)
    check(vR, wantR, 1e-4)
    assert e < 2e-5, "the bf16-split path should sit two orders inside the bar, got %.3g" % e
    # plain bf16 operands (nterms = 1): the fast, not fp32-grade mode
    v1, _ = head.volumes(cu(fL), cu(fR), D, nterms=1, want_right=False)
    torch.cuda.synchronize()
    check(v1, wantL, 2e-2)
    head.close()


def bits(t):
    """the float32 tensor's bit patterns: equality of these is bitwise equality, NaNs included"""
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("case", cases.HEAD_SWEEP, ids=lambda c: "seed%d" % c[0])
def test_sweep(case):
    """fm 8 .. 192 (192 fills layer 1's K = 384, 24 and 120 give an odd number of layer-1 K steps), nh2 128 / 256 / 384,
    l2 1 .. 4, W around the 64-pixel tile, D = 1 .. W + 5, feature scales 0.01 .. 30; both modes, each with the left volume
    only, the right volume only and both.  At scale 30 the features round far in plain bf16, so nterms = 1 is compared with
    the oracle's bf16 model there (oracle/tower_head_cases.py) at the same 2e-2.  At that scale the three-term split itself
    (hi.whi + lo.whi + hi.wlo, computed exactly in float64) is 3e-5 .. 4e-5 off the oracle, so nterms = 3 is held to the
    1e-4 bar there and to 2e-5 only at scales up to 1, as elsewhere in this file."""
    seed, fm, nh2, l2, H, W, D, scale = case
    layers, fL, fR = cases.head_case(seed, fm, nh2, l2, H, W, scale)
    wantL, wantR = cases.head_want(fL, fR, D, layers)
    if scale > 1:
        bfL = cases.head_volume_bf16(fL, fR, D, layers)
        want1 = (bfL, cases.right_from_left(bfL))
    else:
        want1 = (wantL, wantR)
    head = scorer_head.ScorerHead(layers)
    worst = {3: 0.0, 1: 0.0}
    for nterms in (3, 1):
        runs = {}
        for wl, wr in ((True, True), (True, False), (False, True)):
            vL, vR = head.volumes(cu(fL), cu(fR), D, nterms=nterms, want_left=wl, want_right=wr)
            torch.cuda.synchronize()
            assert (vL is not None) == wl and (vR is not None) == wr
            runs[wl, wr] = (vL, vR)
            for v, w3, w1 in ((vL, wantL, want1[0]), (vR, wantR, want1[1])):
                if v is None:
                    continue
                assert v.shape == (1, D, H, W)
                if nterms == 3:
                    e = check(v, w3[None], 1e-4)
                    if scale <= 1:
                        assert e < 2e-5, "the bf16-split path should sit two orders inside the bar, got %.3g" % e
                else:
                    e = check(v, w1[None], 2e-2)
                worst[nterms] = max(worst[nterms], e)
        bL, bR = runs[True, True]
        assert torch.equal(bits(runs[True, False][0]), bits(bL)) and torch.equal(bits(runs[False, True][1]), bits(bR))
        for d in range(min(D, W)):
            assert torch.equal(bits(bR[0, d, :, :W - d]), bits(bL[0, d, :, d:])), "volR[d, y, x - d] != volL[d, y, x]"
    print("seed %d: max err %.3g (nterms 3), %.3g (nterms 1)" % (seed, worst[3], worst[1]))
    head.close()


def _free_device_memory():
    import gc

    gc.collect()
    torch.cuda.empty_cache()
    adcensus.lib().adcensus_trim_scratch()
    return torch.cuda.mem_get_info()[0]


def _samples(rng, H, W, D, n):
    """n valid (d, y, x) of a left volume: every tile row of the first and of the ragged last 64-pixel tile; d in 0, 1, 63, 64,
    65, D - 1 at x = d, x = W - 1 and a random x, each in rows 0, H - 1 and a random row; the rest uniform"""
    ds, ys, xs = [], [], []
    for x in list(range(min(64, W))) + list(range((W - 1) // 64 * 64, W)):
        ds.append(int(rng.integers(0, min(D - 1, x) + 1)))
        ys.append(int(rng.integers(0, H)))
        xs.append(x)
    for d in sorted({0, 1, 63, 64, 65, D - 1}):
        if d >= min(D, W):
            continue
        for y in (0, H - 1, int(rng.integers(0, H))):
            for x in (d, W - 1, int(rng.integers(d, W))):
                ds.append(d)
                ys.append(y)
                xs.append(x)
    k = n - len(ds)
    d = rng.integers(0, min(D, W), k)
    x = d + (rng.random(k) * (W - d)).astype(np.int64)
    y = rng.integers(0, H, k)
    return np.concatenate([ds, d]), np.concatenate([ys, y]), np.concatenate([xs, x])


@pytest.mark.parametrize("name,seed,fm,nh2,l2,H,W,D", [
    ("kitti", 51, 112, 384, 4, 350, 1242, 228),
    ("mb", 52, 112, 384, 3, 4, 3000, 400),
])
def test_full_size(name, seed, fm, nh2, l2, H, W, D):
    """The kitti net at 350 x 1242, D = 228, and the mb / kitti2015 depth at 4 x 3000, D = 400: 32768 stratified entries
    against the oracle; over the whole volumes the structural NaN pattern, volR[d, y, x - d] == volL[d, y, x] bitwise and
    every score in [0, 1]; one-row runs equal the full run's rows bitwise."""
    need = 4 * (2 * D * H * W + 2 * fm * H * W)
    if _free_device_memory() < 2 * need:
        pytest.skip("needs %.1f GB of free device memory" % (2 * need / 1e9))
    layers, fL, fR = cases.head_case(seed, fm, nh2, l2, H, W)
    head = scorer_head.ScorerHead(layers)
    fLd, fRd = cu(fL), cu(fR)
    vL, vR = head.volumes(fLd, fRd, D)
    vL, vR = vL[0], vR[0]
    dev = vL.device
    dd = torch.arange(D, device=dev)[:, None, None]
    xx = torch.arange(W, device=dev)[None, None, :]
    assert torch.equal(torch.isnan(vL), (xx < dd).expand(D, H, W)), "left volume: NaN pattern is not x < d"
    assert torch.equal(torch.isnan(vR), (xx >= W - dd).expand(D, H, W)), "right volume: NaN pattern is not x >= W - d"
    valid = vL[~torch.isnan(vL)]
    assert float(valid.min()) >= 0.0 and float(valid.max()) <= 1.0
    del valid
    for d in range(min(D, W)):
        assert torch.equal(bits(vR[d, :, :W - d]), bits(vL[d, :, d:])), "d = %d: volR[d, y, x - d] != volL[d, y, x]" % d
    rng = np.random.default_rng(seed)
    d, y, x = _samples(rng, H, W, D, 32768)
    assert len(d) >= 32768 and (x >= d).all() and (x < W).all()
    got = vL[torch.from_numpy(d).to(dev), torch.from_numpy(y).to(dev), torch.from_numpy(x).to(dev)].cpu().numpy()
    want = osh.head_samples(fL, fR, layers, d, y, x)
    e = float(np.abs(got - want).max())
    assert e <= 1e-4, "%s: max abs error %.3g over %d samples" % (name, e, len(d))
    assert e < 2e-5, "the bf16-split path should sit two orders inside the bar, got %.3g" % e
    for row in sorted({0, H // 2, H - 1}):
        cL, cR = head.volumes(fLd[:, row:row + 1].contiguous(), fRd[:, row:row + 1].contiguous(), D)
        assert torch.equal(bits(cL[0]), bits(vL[:, row:row + 1])) and torch.equal(bits(cR[0]), bits(vR[:, row:row + 1])), \
            "%s: a one-row run differs from row %d of the full run" % (name, row)
    print("%s: %d x %d, D = %d: max err %.3g over %d samples" % (name, H, W, D, e, len(d)))
    head.close()
    del vL, vR, fLd, fRd
    _free_device_memory()


def test_rejects_unsupported_shapes():
    rng = np.random.default_rng(0)
    with pytest.raises(Exception):
        scorer_head.ScorerHead(osh.make_weights(rng, 8, 100, 2))       # nh2 not a multiple of 128


def test_arch_slow_chain_from_images(oracle):
    """main.lua's arch 'slow' flow end to end on the GPU: images -> feature tower (wgmma) -> scorer head (wgmma) ->
    fix_border -> cross / cbca / sgm2 / post (pipeline.stereo_predict(arch='slow')).  The stages after the head are integer /
    exact-order work: from the head's own volumes they must equal the oracle chain bit for bit."""
    from mccnn_b200 import feature_tower, pipeline, synth
    from oracle import feature_tower as oft

    H, W, D, fm, nh2 = 40, 150, 24, 16, 128
    rng = np.random.default_rng(3)
    p = synth.make_pair(H, W, 4, D, seed=9)
    x = np.stack([p["imgL"], p["imgR"]])[:, None].astype(np.float32)
    tower = feature_tower.FeatureTower(oft.make_weights(rng, l1=3, fm=fm), arch="slow")
    head = scorer_head.ScorerHead(osh.make_weights(rng, fm, nh2, 2))
    opt = pipeline.make_params("kitti", "slow")
    xb = cu(x)
    feats = tower.forward(xb)
    disp, vl, vr = pipeline.stereo_predict(xb, feats, opt, D, want_vols=True, arch="slow", head=head)
    hl, hr = head.volumes(feats[0].contiguous(), feats[1].contiguous(), D)
    torch.cuda.synchronize()
    want, wl, wr = oracle.stereo_predict_chain(p["imgL"], p["imgR"], D, oracle.Params(**opt.as_dict()), arch="volumes",
                                               volL=hl[0].cpu().numpy(), volR=hr[0].cpu().numpy(), want_vols=True)
    for got, ref, what in ((vl, wl, "left volume"), (vr, wr, "right volume"), (disp, want, "disparity map")):
        g = got.cpu().numpy().reshape(ref.shape)
        assert np.array_equal(g, ref, equal_nan=True), what + " differs from the oracle chain"
    tower.close()
    head.close()
