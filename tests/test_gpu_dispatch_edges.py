"""GPU: every kernel variant of StereoJoin, SGM, CBCA (exact and constant-work), AD / census and the post-processing operators
at the edges of its dispatch, bit for bit against the CPU oracle (NaN positions included) -- the constant-work CBCA within
its 1e-4 contract, against the oracle and a float64 tap-sum reference -- and, where oracle/_ref/libadcensus_ref.so has been
built, median2d, mean2d, sgm2, cross and cbca against the reference's own kernels too.  The cases, and the variant each one selects, are in
tests/dispatch_cases.py; tests/test_dispatch_cases.py checks on the CPU that they reach every variant and that their inputs
tell a correct kernel from a subtly wrong one.  Every case is small (well under 1 GB of device memory)."""
import ctypes
import importlib.util
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, pipeline, rowband, synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("dispatch_cases", os.path.join(ROOT, "tests", "dispatch_cases.py"))
dc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(dc)
_spec = importlib.util.spec_from_file_location("stage_chain", os.path.join(ROOT, "tests", "stage_chain.py"))
sc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sc)
EINVAL, ELIMIT = -1, -2


def dev():
    return torch.device("cuda:0")


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev())


def at_offset(a, off):
    """a copy of `a` on the device whose data starts `off` floats after a fresh (aligned) allocation"""
    a = np.ascontiguousarray(a, dtype=np.float32)
    buf = torch.empty(a.size + off, device=dev())
    t = buf[off:].view(a.shape)
    t.copy_(cu(a))
    return t


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


def same(a, b, what=""):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else b
    a = a.reshape(b.shape)
    if not np.array_equal(a, b, equal_nan=True):
        bad = ~((a == b) | (np.isnan(a) & np.isnan(b)))
        idx = np.argwhere(bad)[:5]
        raise AssertionError("%s: %d / %d elements differ, first %s: got %s want %s" % (
            what, bad.sum(), bad.size, idx.tolist(), a[bad][:5], b[bad][:5]))
    z = b == 0                                                      # signed zeros are different bits
    assert np.array_equal(np.signbit(a[z]), np.signbit(b[z])), what + ": signs of zeros differ"


@pytest.fixture(scope="module")
def ref():
    """the reference's own kernels through the shim, where they have been built; else None"""
    from oracle import refdriver

    return refdriver.ShimLibrary(refdriver.REF_LIB) if os.path.exists(refdriver.REF_LIB) else None


# ---------------------------------------------------------------------------------------------------------- StereoJoin

def _features(c):
    rng = np.random.default_rng(c.D * 131 + c.W)
    return rng.standard_normal((2, c.C, c.H, c.W)).astype(np.float32)


@pytest.mark.parametrize("c", dc.SJ_CASES, ids=dc.sj_id)
def test_stereo_join_operator(oracle, c):
    """adcensus.StereoJoin: volumes bit-identical; entries with x < d (left) / x >= W - d (right) untouched"""
    fL, fR = _features(c)
    wantL, wantR = oracle.stereo_join(fL, fR, c.D)
    outL = torch.full((1, c.D, c.H, c.W), 7.0, device=dev())
    outR = torch.full((1, c.D, c.H, c.W), 9.0, device=dev())
    adcensus.StereoJoin(at_offset(fL[None], c.feat_off), at_offset(fR[None], c.feat_off), outL, outR)
    same(outL, np.where(np.isnan(wantL), np.float32(7.0), wantL), "left volume")
    same(outR, np.where(np.isnan(wantR), np.float32(9.0), wantR), "right volume")


@pytest.mark.parametrize("c", [c for c in dc.SJ_CASES if dc.sj_pitched_ok(c.W, c.feat_off, dc.sj_ld(c.W))], ids=dc.sj_id)
def test_stereo_join_pitched(oracle, c):
    """mccnn_stereo_join_pitched: left volume NaN where x < d, right volume untouched where x >= W - d, nothing but the
    left volume's clipped NaN in the padding columns"""
    fL, fR = _features(c)
    wantL, wantR = oracle.stereo_join(fL, fR, c.D)
    ld = dc.sj_ld(c.W)
    outL = torch.full((c.D, c.H, ld), 7.0, device=dev())
    outR = torch.full((c.D, c.H, ld), 9.0, device=dev())
    tL, tR = at_offset(fL, c.feat_off), at_offset(fR, c.feat_off)
    rc = adcensus.lib().mccnn_stereo_join_pitched(vp(tL), vp(tR), vp(outL), vp(outR), c.C, c.D, c.H, c.W, ld, adcensus._stream(tL))
    assert rc == 0, rc
    oL, oR = outL.cpu().numpy(), outR.cpu().numpy()
    padL = oL[:, :, c.W:]
    assert (np.isnan(padL) | (padL == 7.0)).all() and (oR[:, :, c.W:] == 9.0).all(), "padding columns hold data"
    same(oL[:, :, :c.W], wantL, "left volume")
    same(oR[:, :, :c.W], np.where(np.isnan(wantR), np.float32(9.0), wantR), "right volume")


# ------------------------------------------------------------------------------------------------------------------ SGM

@pytest.mark.parametrize("c", dc.SGM_CASES, ids=dc.sgm_id)
@pytest.mark.parametrize("direction", [-1, 1])
def test_sgm2(oracle, ref, c, direction):
    """adcensus.sgm2 (four single passes, accumulator read) and mccnn_sgm2_band for each pass mask with zero_out on (the
    hpair kernel, a ZERO pass) and off, against oracle.sgm2 / oracle.sgm2_band"""
    x0, x1, vol = dc.sgm_inputs(c, direction)
    args = c.params + (direction,)
    H, W, D = vol.shape
    iL, iR = cu(x0), cu(x1)
    cost = at_offset(vol, c.in_off)
    init = np.random.default_rng(D + W).standard_normal((H, W, D)).astype(np.float32)
    zeros = np.zeros((H, W, D), np.float32)
    got_op = None
    for acc0, what in ((zeros, "zero"), (init, "non-zero")):
        want = oracle.sgm2(x0, x1, vol, *args, out=acc0.copy())
        out = at_offset(acc0, c.out_off)
        adcensus.sgm2(iL[None], iR[None], cost[None], out[None], None, *args)
        same(out, want, "adcensus.sgm2, %s accumulator" % what)
        got_op = out if got_op is None else got_op
    ops = rowband.CudaOps(dev())
    pi1, pi2, tau_so, alpha1, q1, q2 = c.params
    opt = SimpleNamespace(pi1=pi1, pi2=pi2, tau_so=tau_so, alpha1=alpha1, sgm_q1=q1, sgm_q2=q2)
    for mask in dc.SGM_MASKS:
        for zero_out in (True, False):
            acc0 = zeros if zero_out else init
            want = oracle.sgm2_band(x0, x1, vol, acc0.copy(), W, 0, 0, *args, mask)
            out = at_offset(acc0, c.out_off)
            ops.sgm_band(iL, iR, cost, out, H, W, 0, 0, opt, direction, mask, zero_out)
            same(out, want, "mccnn_sgm2_band mask %d zero_out %d" % (mask, zero_out))
    if ref is not None and D <= 400:                                # the reference's output_s[400] (adcensus.cu)
        out = torch.zeros((1, H, W, D), device=dev())
        tmp = torch.empty((W, D), device=dev())
        ref.call("sgm2", iL[None], iR[None], cu(vol)[None], out, tmp, *args)
        same(got_op, out, "adcensus.sgm2 vs the live reference")


# ----------------------------------------------------------------------------------------------------- post-processing

@pytest.mark.parametrize("kind", dc.MEDIAN_KINDS)
@pytest.mark.parametrize("k", dc.MEDIAN_K)
def test_median2d(oracle, ref, kind, k):
    """k = 5 (counting kernel, sort for windows holding NaN or -0) and the sort kernel, on images larger and smaller
    than the window"""
    for H, W in dc.MEDIAN_SHAPES:
        img = dc.median_image(kind, H, W)
        got = adcensus.median2d(cu(img)[None, None], k)
        same(got, oracle.median2d(img, k), "median2d k=%d %dx%d" % (k, H, W))
        if ref is not None:
            same(got, ref.call("median2d", cu(img)[None, None], k)[0], "median2d k=%d %dx%d vs the live reference" % (k, H, W))


@pytest.mark.parametrize("c", dc.MEAN2D_CASES, ids=lambda c: "ks%d_%s" % (c.ksize, c.regime))
def test_mean2d(oracle, ref, c):
    """a random asymmetric kernel in each regime of adcensus_mean2d; NaN pixels; alpha2 on a quantisation step, tiny, +inf"""
    img, kern = dc.mean2d_inputs(c)
    got = adcensus.mean2d(cu(img)[None, None], cu(kern), c.alpha2)
    same(got, oracle.mean2d(img, kern, c.alpha2), "mean2d")
    if ref is not None:
        same(got, ref.call("mean2d", cu(img)[None, None], cu(kern), c.alpha2)[0], "mean2d vs the live reference")


@pytest.mark.parametrize("kernel", sorted(dc.INTERP_OCC_W))
def test_interpolate_occlusion_wide_rows(oracle, kernel):
    """the row kernel up to W = 4096 and the per-pixel kernel above; rows without label 0, label 1 at both ends"""
    W, H = dc.INTERP_OCC_W[kernel], 5
    rng = np.random.default_rng(W)
    d0 = rng.integers(0, 60, (H, W)).astype(np.float32)
    lab = rng.choice(np.array([0, 1, 2], np.float32), p=[0.05, 0.6, 0.35], size=(H, W))
    lab[1][lab[1] == 0] = 2                                          # no label 0: occluded pixels keep their value
    lab[2] = 1                                                       # all occluded
    lab[[0, 1, 3, 4], 0] = 1
    lab[[0, 1, 3, 4], -1] = 1
    lab[4, 1:-1] = 2
    lab[4, W // 2] = 0                                               # one match in the middle of a row
    got = adcensus.interpolate_occlusion(cu(d0)[None, None], cu(lab)[None, None])
    same(got, oracle.interpolate_occlusion(d0, lab), "interpolate_occlusion W=%d" % W)


def test_outlier_detection_disp_max_above_width(oracle):
    H, W, D = 6, 20, 50
    rng = np.random.default_rng(4)
    d0 = np.where(rng.random((H, W)) < 0.5, rng.integers(0, 6, (H, W)), rng.integers(0, D, (H, W))).astype(np.float32)
    d1 = rng.integers(0, 6, (H, W)).astype(np.float32)
    want = oracle.outlier_detection(d0, d1, D)
    assert set(np.unique(want)) == {0.0, 1.0, 2.0}
    outlier = torch.zeros((1, 1, H, W), device=dev())
    adcensus.outlier_detection(cu(d0)[None, None], cu(d1)[None, None], outlier, D)
    same(outlier, want, "outlier_detection")


@pytest.mark.parametrize("D", [1, 2, 3, 4, 5])
def test_argmin_edges(oracle, D):
    """first minimum with NaN skipped: all-NaN and all-+inf columns give 0, -inf wins, ties go to the first index"""
    H, W = 6, 11
    rng = np.random.default_rng(D)
    vol = rng.integers(0, 3, (D, H, W)).astype(np.float32)
    vol[rng.random((D, H, W)) < 0.2] = np.nan
    vol[rng.random((D, H, W)) < 0.1] = np.inf
    vol[rng.random((D, H, W)) < 0.1] = -np.inf
    vol[:, 0, :3] = np.nan
    vol[:, 1, :2] = np.inf
    want = oracle.spatial_argmin(vol)
    same(adcensus.argmin(cu(vol)[None]), want - 1, "argmin")
    out = torch.empty((1, 1, H, W), device=dev())
    adcensus.spatial_argmin(cu(vol)[None], out)
    same(out, want, "spatial_argmin")
    ld = W + 5
    pv = torch.full((D, H, ld), -np.inf, device=dev())             # a read of the padding would win
    pv[:, :, :W] = cu(vol)
    disp = torch.empty((H, W), device=dev())
    assert adcensus.lib().mccnn_argmin_pitched(vp(pv), vp(disp), D, H, W, ld, adcensus._stream(pv)) == 0
    same(disp, want - 1, "mccnn_argmin_pitched")


@pytest.mark.parametrize("c", dc.TRANSPOSE_CASES, ids=lambda c: "D%dH%dW%d_off%d" % c)
def test_transposes(oracle, c):
    """mccnn_transpose_* plain (64- and 32-tile kernels, both LONGROWS orientations) and pitched (float4 or not)"""
    D, H, W = c.D, c.H, c.W
    vol = np.random.default_rng(D * W).standard_normal((D, H, W)).astype(np.float32)
    hwd = oracle.transpose_dhw_to_hwd(vol)
    lib, s = adcensus.lib(), adcensus._stream
    src, dst = at_offset(vol, c.off), at_offset(np.zeros((H, W, D)), c.off)
    assert lib.mccnn_transpose_dhw_to_hwd(vp(src), vp(dst), D, H, W, s(src)) == 0
    same(dst, hwd, "dhw -> hwd")
    src, dst = at_offset(hwd, c.off), at_offset(np.zeros((D, H, W)), c.off)
    assert lib.mccnn_transpose_hwd_to_dhw_div4(vp(src), vp(dst), D, H, W, s(src)) == 0
    same(dst, oracle.transpose_hwd_to_dhw_div4(hwd), "hwd -> dhw / 4")
    ld = dc.sj_ld(W)
    padded = np.full((D, H, ld), np.inf, np.float32)
    padded[:, :, :W] = vol
    src, dst = at_offset(padded, c.off), at_offset(np.zeros((H, W, D)), c.off)
    assert lib.mccnn_transpose_dhw_pitched_to_hwd(vp(src), vp(dst), D, H, W, ld, s(src)) == 0
    same(dst, hwd, "pitched dhw -> hwd")
    src, dst = at_offset(hwd, c.off), at_offset(np.zeros((D, H, ld)), c.off)
    assert lib.mccnn_transpose_hwd_to_dhw_pitched_div4(vp(src), vp(dst), D, H, W, ld, s(src)) == 0
    same(dst.cpu().numpy()[:, :, :W], oracle.transpose_hwd_to_dhw_div4(hwd), "hwd -> pitched dhw / 4")


# ----------------------------------------------------------------------------------------------------------------- CBCA

def _exact_kind(i, c):
    kind = dc.CBCA_KINDS[i % len(dc.CBCA_KINDS)]
    return "stereojoin" if kind == "post_sgm" and c.H > c.W else kind


@pytest.mark.parametrize("i,c", list(enumerate(dc.CBCA_EXACT_CASES)), ids=[dc.cbca_id(c) for c in dc.CBCA_EXACT_CASES])
def test_cbca_exact(oracle, ref, i, c):
    """adcensus_cbca (device gate), adcensus_cbca_ex and mccnn_pack_arms + mccnn_cbca_packed (host bound): bit-identical to
    oracle.cbca on the arms the case aggregates (clipped at an understated bound), zero signs included; cross and cbca
    against the reference's own kernels where built"""
    x0c, x1c, a0, a1 = dc.cbca_arms(c)
    vol = dc.cbca_volume(_exact_kind(i, c), c.H, c.W, c.D, c.direction)
    want = oracle.cbca(a0, a1, vol, c.direction)
    out = torch.full((1, c.D, c.H, c.W), 5.0, device=dev())
    t0, t1, tv = cu(x0c)[None], cu(x1c)[None], cu(vol)[None]
    if c.entry == "gate":
        adcensus.cbca(t0, t1, tv, out, c.direction)
    elif c.entry == "ex":
        adcensus.cbca(t0, t1, tv, out, c.direction, max_arm=c.max_arm)
    else:
        packed = torch.zeros(2 * c.H * c.W + 1, dtype=torch.int32, device=dev())
        lib, s = adcensus.lib(), adcensus._stream(tv)
        assert lib.mccnn_pack_arms(vp(t0), vp(t1), vp(packed), c.H, c.W, s) == 0
        assert lib.mccnn_cbca_packed(vp(packed), vp(t0), vp(t1), vp(tv), vp(out), c.D, c.H, c.W, c.direction, c.max_arm, s) == 0
    same(out, want, "cbca %s" % c.entry)
    if ref is not None:
        img = dc.cbca_image(c.H, c.W, c.L, 7 * c.H + 3 * c.W + c.L)
        rc = torch.empty((1, 4, c.H, c.W), device=dev())
        ref.call("cross", cu(img)[None], rc, c.L, dc.CBCA_TAU1)
        oc = torch.empty((1, 4, c.H, c.W), device=dev())
        adcensus.cross(cu(img)[None], oc, c.L, dc.CBCA_TAU1)
        same(oc, rc, "cross vs the live reference")
        if c.arms != "clip":
            ro = torch.empty((1, c.D, c.H, c.W), device=dev())
            ref.call("cbca", t0, t1, tv, ro, c.direction)
            same(out, ro, "cbca %s vs the live reference" % c.entry)


def _run_fast(entry, x0c, x1c, vol, c):
    """one aggregation through mccnn_cbca_fast_pitched or mccnn_pack_arms_hv + mccnn_cbca_fast_pitched_packed on (D, H, ld)
    volumes whose padding holds 123 (input) / -7 (output): returns the (D, H, W) result; the padding must stay -7"""
    D, H, W = vol.shape
    vin = torch.full((D, H, c.ld), 123.0, device=dev())
    vin[:, :, :W] = cu(vol)
    vout = torch.full((D, H, c.ld), -7.0, device=dev())
    a0, a1 = cu(x0c), cu(x1c)
    lib, s = adcensus.lib(), adcensus._stream(vin)
    if entry == "pitched":
        rc = lib.mccnn_cbca_fast_pitched(vp(a0), vp(a1), vp(vin), vp(vout), D, H, W, c.ld, c.direction, c.max_arm, s)
    else:
        hv = torch.zeros(4 * H * W, dtype=torch.int32, device=dev())
        assert lib.mccnn_pack_arms_hv(vp(a0), vp(a1), vp(hv), H, W, s) == 0
        rc = lib.mccnn_cbca_fast_pitched_packed(vp(hv), vp(vin), vp(vout), D, H, W, c.ld, c.direction, c.max_arm, s)
    assert rc == 0, rc
    o = vout.cpu().numpy()
    assert (o[:, :, W:] == -7.0).all(), "%s: padding columns were written" % entry
    return o[:, :, :W]


def _rel_err(got, want):
    m = ~np.isnan(want)
    return float((np.abs(got[m] - want[m]) / np.maximum(1.0, np.abs(want[m]))).max()) if m.any() else 0.0


@pytest.mark.parametrize("c", dc.CBCA_FAST_CASES, ids=dc.fast_id)
def test_cbca_fast(oracle, record_property, c):
    """every constant-work kernel through both fast entries, on every volume kind: relative error <= 1e-4 max(1, |want|)
    against oracle.cbca and the float64 tap sums, NaN pattern identical, padding columns untouched"""
    x0c, x1c, _, _ = dc.cbca_arms(dc.CbcaCase(c.H, c.W, c.D, c.L, c.direction, "ex", c.max_arm, None, "cross"))
    vol = dc.cbca_volume(c.kind, c.H, c.W, c.D, c.direction)
    want, want64 = oracle.cbca(x0c, x1c, vol, c.direction), dc.cbca_f64(x0c, x1c, vol, c.direction)
    for entry in ("pitched", "packed"):
        got = _run_fast(entry, x0c, x1c, vol, c)
        assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN pattern differs" % entry
        e32, e64 = _rel_err(got, want), _rel_err(got, want64)
        record_property("max_rel_err_f64_%s_%s" % (c.kind, entry), e64)
        assert e32 <= 1e-4 and e64 <= 1e-4, "%s: max relative error %.3g (oracle), %.3g (float64)" % (entry, e32, e64)


def test_cbca_fast_four_iterations_on_census(oracle):
    """mb census's eight iterations of arms of 5 on a census volume: the error does not build up past the bar"""
    c = dc.FastCase(70, 257, 40, 5, -1, 5, "ws4", 264, "census3")
    x0c, x1c, _, _ = dc.cbca_arms(dc.CbcaCase(c.H, c.W, c.D, c.L, c.direction, "ex", 5, None, "cross"))
    want = got = dc.cbca_volume(c.kind, c.H, c.W, c.D, c.direction)
    for _ in range(8):
        want = oracle.cbca(x0c, x1c, want, c.direction)
        got = _run_fast("packed", x0c, x1c, got, c)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert _rel_err(got, want) <= 1e-4


@pytest.mark.parametrize("r", dc.CBCA_FAST_REFUSALS, ids=lambda r: "W%d_ld%d_off%d.%d_alias%d_arm%d" % r[:6])
def test_cbca_fast_refusals(r):
    """ld < W, ld % 4, a base off 16 bytes and vol_in == vol_out are EINVAL, a halo above 13 ELIMIT, for both entries"""
    W, ld, in_off, out_off, aliased, max_arm, want = r
    assert dc.cbca_fast_refusal(W, ld, in_off, out_off, aliased, max_arm) == want
    D, H = 4, 8
    code = {"EINVAL": EINVAL, "ELIMIT": ELIMIT, None: 0}[want]
    vin = at_offset(np.zeros((D, H, ld)), in_off)
    vout = vin if aliased else at_offset(np.zeros((D, H, ld)), out_off)
    arms = cu(dc.clip_arms(np.zeros((4, H, W), np.float32), 1))
    hv = torch.zeros(4 * H * W, dtype=torch.int32, device=dev())
    lib, s = adcensus.lib(), adcensus._stream(vin)
    assert lib.mccnn_pack_arms_hv(vp(arms), vp(arms), vp(hv), H, W, s) == 0
    assert lib.mccnn_cbca_fast_pitched(vp(arms), vp(arms), vp(vin), vp(vout), D, H, W, ld, -1, max_arm, s) == code
    assert lib.mccnn_cbca_fast_pitched_packed(vp(hv), vp(vin), vp(vout), D, H, W, ld, -1, max_arm, s) == code
    torch.cuda.synchronize()


# the pipeline: mb census (arms of 5, 8 + 8 iterations) in the default mode against the exact mode
MB_H, MB_W, MB_D = 70, 257, 40


@pytest.fixture(scope="module")
def mb_census_pair(oracle):
    p = synth.make_pair(MB_H, MB_W, 1, MB_D, seed=21)
    volL = oracle.census(p["imgL"], p["imgR"], MB_D, -1)
    volR = oracle.census(p["imgR"], p["imgL"], MB_D, 1)
    return p, volL, volR


@pytest.mark.parametrize("terminate", ["cbca1", ""])
def test_pipeline_mb_census_fast_vs_exact(oracle, mb_census_pair, terminate):
    """run_volumes on census volumes: after cbca1's 8 iterations (and after the full chain) the default mode's left volume
    is within 1e-4 of the exact mode's, NaN pattern identical, and the map differs on < 5e-3 of the pixels; the exact mode
    after cbca1 is bit-identical to the oracle chain"""
    p, volL, volR = mb_census_pair
    opt = pipeline.make_params("mb", "census", sm_terminate=terminate)
    iL, iR = cu(p["imgL"]), cu(p["imgR"])
    out = {}
    for m in ("exact", "fast"):
        sp = pipeline.StereoPipeline(1, MB_D, MB_H, MB_W, opt, cbca_mode=m)
        vl = torch.empty((MB_D, MB_H, MB_W), device=dev())
        d = sp.run_volumes(cu(volL), cu(volR), iL, iR, outL=vl)
        torch.cuda.synchronize()
        out[m] = (d.cpu().numpy(), vl.cpu().numpy())
        sp.close()
    (de, ve), (df, vf) = out["exact"], out["fast"]
    assert np.array_equal(np.isnan(ve), np.isnan(vf)), "NaN pattern differs"
    assert _rel_err(vf, ve) <= 1e-4
    frac = float((np.abs(df - de) > 1e-4 * np.maximum(1.0, np.abs(de))).mean())
    assert frac < 5e-3, "%.4f of the map changed" % frac
    if terminate == "cbca1":
        want, wL, _ = sc.oracle_chain(oracle, p["imgL"], p["imgR"], MB_D, opt, "cbca1", "", arch="volumes", volL=volL,
                                      volR=volR, want_vols=True)
        same(ve, wL, "exact mode after cbca1 vs the oracle chain")
        same(de, want, "exact mode map after cbca1 vs the oracle chain")


def test_pipeline_nan_in_valid_route(oracle):
    """border > 0 and D > W - border - 1: fix_border leaves NaN at valid positions, and both modes run the generic kernel:
    the left volume after cbca1 bit-identical to the oracle chain, and the default mode equal to the exact mode"""
    H, W, C, D = 21, 40, 8, 40
    opt = pipeline.make_params("kitti", "accurate_cbca4", sm_terminate="cbca1")
    assert dc.pipe_cbca_route(True, opt.L1, opt.border, D, W) == "generic"
    p = synth.make_pair(H, W, C, D, seed=5)
    want, wL, _ = sc.oracle_chain(oracle, p["imgL"], p["imgR"], D, opt, "cbca1", "", featL=p["featL"], featR=p["featR"],
                                  want_vols=True)
    assert np.isnan(wL).any() and not np.isnan(wL).all()
    got = {}
    for m in ("exact", "fast"):
        sp = pipeline.StereoPipeline(C, D, H, W, opt, cbca_mode=m)
        vl = torch.empty((D, H, W), device=dev())
        d = sp.run(cu(p["featL"]), cu(p["featR"]), cu(p["imgL"]), cu(p["imgR"]), volL=vl)
        torch.cuda.synchronize()
        got[m] = (d.clone(), vl.clone())
        sp.close()
        same(vl, wL, "%s mode: left volume after cbca1" % m)
        same(d, want, "%s mode: map after cbca1" % m)
    same(got["fast"][1], got["exact"][1], "fast == exact")


# ------------------------------------------------------------------------------------------------------------ AD / census

@pytest.mark.parametrize("c", dc.AD_CENSUS_CASES, ids=lambda c: "H%dW%dD%d_nch%d%s" % (c.H, c.W, c.D, c.nch, "_nan" * c.nan))
def test_ad_census(oracle, c):
    """census (nch 1, 3 and the runtime-nch kernel at 2 and 4) and AD bit for bit: NaN pixels, one row, one column,
    W = 128k +- 1, D at the chunk edges (8 for AD, 16 for census) and D > W"""
    a, b = dc.ad_census_images(c)
    for direction in (-1, 1):
        o = torch.full((1, c.D, c.H, c.W), 3.0, device=dev())
        adcensus.census(cu(a)[None], cu(b)[None], o, direction)
        same(o, oracle.census(a, b, c.D, direction), "census nch %d (%s)" % (c.nch, dc.census_kernel(c.nch)))
        o = torch.full((1, c.D, c.H, c.W), 3.0, device=dev())
        adcensus.ad(cu(a[:1])[None], cu(b[:1])[None], o, direction)
        same(o, oracle.ad(a[0], b[0], c.D, direction), "ad")


def test_census_refuses_five_channels():
    a = torch.zeros((5, 6, 20), device=dev())
    o = torch.full((4, 6, 20), 3.0, device=dev())
    assert dc.census_kernel(5) == "ELIMIT"
    assert adcensus.lib().adcensus_census(vp(a), vp(a), vp(o), 4, 5, 6, 20, -1, adcensus._stream(a)) == ELIMIT
    torch.cuda.synchronize()
    assert bool((o == 3.0).all())
