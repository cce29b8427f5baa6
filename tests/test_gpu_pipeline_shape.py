"""GPU: one StereoPipeline created at the largest shape runs smaller shapes (mccnn_pipeline_run_shape) with the same
results, bit for bit, as a pipeline created at each shape -- in both CBCA modes and overlap modes 0 and 2 -- and a plain
run afterwards still reproduces the created shape's result.  The accurate_cbca4 preset has CBCA blocks before and after
SGM, so the TMA-staged CBCA's tensor maps are re-encoded for every shape change; mb slow's arms of up to 14 pixels run the
exact CBCA kernels in both modes, with no tensor maps at all."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, pipeline, synth  # noqa: E402

C, D, H, W = 64, 32, 48, 130
SHAPES = [(48, 130, 32), (40, 117, 24), (48, 96, 32), (17, 64, 9)]      # (H, W, D); 117 is odd
OPT = pipeline.make_params("kitti", "accurate_cbca4")


def _inputs(h, w, d, seed):
    p = synth.make_pair(h, w, C, d, seed=seed)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t(p["featL"]), t(p["featR"]), t(p["imgL"]), t(p["imgR"])


def _configure(sp, cbca, overlap):
    sp.set_cbca_mode(cbca)
    sp.set_overlap(overlap)


def _outputs(h, w, d):
    nan = float("nan")
    return (torch.full((h, w), nan, device="cuda"), torch.full((d, h, w), nan, device="cuda"),
            torch.full((d, h, w), nan, device="cuda"))


def _fresh(shape, ins, opt, cbca, overlap):
    h, w, d = shape
    sp = pipeline.StereoPipeline(C, d, h, w, opt)
    _configure(sp, cbca, overlap)
    disp, vl, vr = _outputs(h, w, d)
    sp.run(*ins, disp=disp, volL=vl, volR=vr)
    torch.cuda.synchronize()
    out = [t.cpu().numpy() for t in (disp, vl, vr)]
    sp.close()
    return out


def _same(got, want, what):
    for g, w_, name in zip(got, want, ("disp", "volL", "volR")):
        assert g.shape == w_.shape, "%s %s: shape %s vs %s" % (what, name, g.shape, w_.shape)
        assert np.array_equal(g, w_, equal_nan=True), "%s %s differs from a pipeline created at that shape" % (what, name)


@pytest.mark.parametrize("overlap", [0, 2])
@pytest.mark.parametrize("cbca", ["fast", "exact"])
@pytest.mark.parametrize("dataset,arch", [("kitti", "accurate_cbca4"), ("mb", "slow")])
def test_run_shape_matches_a_pipeline_of_that_shape(dataset, arch, cbca, overlap):
    opt = pipeline.make_params(dataset, arch)
    inputs = {s: _inputs(*s, seed=7 * s[0] + s[1] + s[2]) for s in SHAPES}
    want = {s: _fresh(s, inputs[s], opt, cbca, overlap) for s in SHAPES}
    sp = pipeline.StereoPipeline(C, D, H, W, opt)
    _configure(sp, cbca, overlap)
    first = None
    for s in SHAPES + SHAPES[::-1][1:]:                        # interleaved: every shape change re-encodes the maps
        h, w, d = s
        disp, vl, vr = _outputs(h, w, d)
        sp.run_shape(*inputs[s], disp_max=d, disp=disp, volL=vl, volR=vr)
        torch.cuda.synchronize()
        got = [t.cpu().numpy() for t in (disp, vl, vr)]
        _same(got, want[s], "run_shape %s" % (s,))
        if first is None:
            first = got
    # a plain run at the created shape after the smaller ones
    disp, vl, vr = _outputs(H, W, D)
    sp.run(*inputs[SHAPES[0]], disp=disp, volL=vl, volR=vr)
    torch.cuda.synchronize()
    _same([t.cpu().numpy() for t in (disp, vl, vr)], first, "run after run_shape")
    sp.close()


def test_run_shape_exact_mode_matches_the_oracle(oracle):
    h, w, d = SHAPES[1]
    p = synth.make_pair(h, w, C, d, seed=3)
    want, wL, wR = oracle.stereo_predict(p["featL"], p["featR"], p["imgL"], p["imgR"], d,
                                         oracle.Params(**OPT.as_dict()), want_vols=True)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    sp = pipeline.StereoPipeline(C, D, H, W, OPT, cbca_mode="exact")
    disp, vl, vr = _outputs(h, w, d)
    sp.run_shape(t(p["featL"]), t(p["featR"]), t(p["imgL"]), t(p["imgR"]), disp_max=d, disp=disp, volL=vl, volR=vr)
    torch.cuda.synchronize()
    _same([x.cpu().numpy() for x in (disp, vl, vr)], [want, wL, wR], "exact run_shape vs oracle")
    sp.close()


def test_run_shape_rejects_what_does_not_fit():
    sp = pipeline.StereoPipeline(C, D, H, W, OPT)
    lib = adcensus.lib()
    for (h, w, d) in [(H + 1, W, D), (H, W + 1, D), (H, W, D + 1), (H, W + 3, D)]:
        ins = _inputs(h, w, min(d, D), seed=1)
        disp, vl, vr = _outputs(h, w, d)
        with pytest.raises(adcensus.AdcensusError, match="size limit exceeded"):
            sp.run_shape(*ins, disp_max=d, disp=disp, volL=vl, volR=vr)
        torch.cuda.synchronize()
        assert torch.isnan(disp).all() and torch.isnan(vl).all() and torch.isnan(vr).all()
    # border + 1 > W and sizes < 1: invalid arguments, nothing launched
    h, w, d = 8, OPT.border, 4
    ins = _inputs(h, 16, d, seed=2)
    small = [x[..., :w].contiguous() for x in ins]
    disp, vl, vr = _outputs(h, w, d)
    with pytest.raises(adcensus.AdcensusError, match="invalid argument"):
        sp.run_shape(*small, disp_max=d, disp=disp, volL=vl, volR=vr)
    one = ctypes.c_void_p(disp.data_ptr())
    for (hh, ww, dd) in [(0, 16, 4), (8, 16, 0), (8, 0, 4)]:
        assert lib.mccnn_pipeline_run_shape(sp._h, hh, ww, dd, one, one, one, one, one, None, None, None) == -1
    torch.cuda.synchronize()
    assert torch.isnan(disp).all() and torch.isnan(vl).all()
    # C differs from the created C: refused before the library is called
    h, w, d = SHAPES[2]
    fL, fR, iL, iR = _inputs(h, w, d, seed=4)
    disp, vl, vr = _outputs(h, w, d)
    with pytest.raises(adcensus.AdcensusError, match="featL must be"):
        sp.run_shape(fL[:32].contiguous(), fR[:32].contiguous(), iL, iR, disp_max=d, disp=disp, volL=vl)
    with pytest.raises(adcensus.AdcensusError, match="volR must be"):
        sp.run_shape(fL, fR, iL, iR, disp_max=d - 1, disp=disp, volL=None, volR=vr)
    torch.cuda.synchronize()
    assert torch.isnan(disp).all() and torch.isnan(vl).all() and torch.isnan(vr).all()
    sp.close()
