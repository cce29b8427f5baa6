"""GPU, one device: the row-band split with N > 1 ranks on the CUDA operators, its ranks as threads of one process
(tests/rank_threads.py), each on a stream of its own.  This runs on one H100 what otherwise needs two GPUs: the halo
exchanges of both CBCA blocks, the SGM wavefront (mccnn_sgm2_rows on bands below the top, line states in and out column
chunk by column chunk), sub-pixel refinement against a band's own volume, the median and bilateral filters on row slices
with halos, and write_outputs from several ranks.  Every comparison is bit for bit (equal or both NaN; for volumes also
the signs of zeros):

a. stereo_predict_rowband from features against the CPU oracle's whole-image pipeline, at splits that reach 1-row bands,
   both exchange regimes of the second CBCA block, the thinnest legal band, and column chunks of 1, 7, W and W + 5;
b. at the bench size against the fused pipeline in exact mode;
c. band_predict for every architecture: the map and each rank's rows of both volumes against pipeline.stereo_predict;
d. predict_pair writes frontend.predict's three files byte for byte;
e. mccnn_sgm2_rows, chained over three row bands and three column chunks, at every (K, VEC) instantiation, against
   oracle.sgm2; and its argument refusals.
"""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rank_threads import run_ranks  # noqa: E402
from test_gpu_rowband_predict import ARCHS, _assert_same_files, _frontend_files, _images, _net  # noqa: E402

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, frontend, pipeline, rowband, synth  # noqa: E402
import dispatch_cases as dc  # noqa: E402

EINVAL, ELIMIT = -1, -2


def dev():
    return torch.device("cuda", 0)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev())


def same(a, b, what):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    assert a.shape == b.shape, "%s: shape %s, expected %s" % (what, a.shape, b.shape)
    if not np.array_equal(a, b, equal_nan=True):
        bad = ~((a == b) | (np.isnan(a) & np.isnan(b)))
        idx = np.argwhere(bad)[:5]
        raise AssertionError("%s: %d / %d elements differ, first %s: got %s want %s" % (
            what, bad.sum(), bad.size, idx.tolist(), a[bad][:5], b[bad][:5]))
    z = b == 0                                                       # signed zeros are different bits
    assert np.array_equal(np.signbit(a[z]), np.signbit(b[z])), what + ": signs of zeros differ"


def regime(opt, H, world):
    """the second CBCA block's exchanges at this split: 'one' (n * halo rows once), 'per_iteration', None (none)"""
    halo, n = rowband.cbca_halo(opt)[1], int(opt.cbca_i2)
    if halo == 0 or n == 0:
        return None
    band_min = min(b - a for a, b in (rowband.split(H, world, p) for p in range(world)))
    return "one" if n * halo <= band_min else "per_iteration"


# ------------------------------------------------------------------------------------ a. from features, against the oracle

# name -> ((dataset, arch), H, W, C, D, world, chunks, regime of the second CBCA block).  H <= W: oracle.sgm2 needs it.
ORACLE_CASES = {
    "kitti_fast_1row_bands": (("kitti", "fast"), 5, 40, 8, 10, 5, None, None),
    "kitti2015_slow_one_exchange": (("kitti2015", "slow"), 50, 72, 8, 14, 3, None, "one"),
    "kitti2015_slow_per_iteration": (("kitti2015", "slow"), 47, 72, 8, 14, 3, None, "per_iteration"),
    "mb_slow_thinnest_band": (("mb", "slow"), 27, 48, 8, 9, 2, None, "per_iteration"),
    "accurate_cbca4": (("kitti", "accurate_cbca4"), 37, 52, 8, 12, 3, None, "one"),
    "accurate_cbca4_chunks1": (("kitti", "accurate_cbca4"), 37, 52, 8, 12, 3, 1, "one"),
    "accurate_cbca4_chunks7": (("kitti", "accurate_cbca4"), 37, 52, 8, 12, 3, 7, "one"),
    "accurate_cbca4_chunksW": (("kitti", "accurate_cbca4"), 37, 52, 8, 12, 3, 52, "one"),
    "accurate_cbca4_chunksW+5": (("kitti", "accurate_cbca4"), 37, 52, 8, 12, 3, 57, "one"),
}


def _rowband_threads(opt, featL, featR, imgL, imgR, D, world, chunks=None):
    torch.cuda.synchronize()                                         # the inputs are read on every rank's stream
    ops = rowband.CudaOps(dev())
    return run_ranks(world, lambda comm: rowband.stereo_predict_rowband(ops, featL, featR, imgL, imgR, D, opt, comm=comm,
                                                                        chunks=chunks).cpu(), device=dev())


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_rowband_matches_the_oracle(oracle, case):
    preset, H, W, C, D, world, chunks, want_regime = ORACLE_CASES[case]
    opt = pipeline.make_params(*preset)
    assert regime(opt, H, world) == want_regime
    if preset == ("mb", "slow"):
        assert opt.L1 == 14 and min(b - a for a, b in (rowband.split(H, world, p) for p in range(world))) == 13
    p = synth.make_pair(H, W, C, D, seed=H + 3 * D)
    want = oracle.stereo_predict(p["featL"], p["featR"], p["imgL"], p["imgR"], D, oracle.Params(**opt.as_dict()))
    outs = _rowband_threads(opt, cu(p["featL"]), cu(p["featR"]), cu(p["imgL"]), cu(p["imgR"]), D, world, chunks)
    for r, got in enumerate(outs):
        same(got, want, "%s: rank %d of %d" % (case, r, world))


class _CountingOps(rowband.CudaOps):
    def __init__(self, device):
        super().__init__(device)
        self.calls = []

    def __getattribute__(self, name):
        attr = object.__getattribute__(self, name)
        if callable(attr) and not name.startswith("_"):
            object.__getattribute__(self, "calls").append(name)
        return attr


def test_a_band_thinner_than_the_halo_is_refused_before_any_launch():
    """mb slow (L1 14, halo 13) on two bands of 12 and 13 rows"""
    opt = pipeline.make_params("mb", "slow")
    H, W, C, D = 25, 48, 8, 9
    p = synth.make_pair(H, W, C, D, seed=1)
    fL, fR, iL, iR = cu(p["featL"]), cu(p["featR"]), cu(p["imgL"]), cu(p["imgR"])
    torch.cuda.synchronize()
    ops = [_CountingOps(dev()) for _ in range(2)]
    with pytest.raises(AssertionError, match="thinner than the CBCA halo"):
        run_ranks(2, lambda comm: rowband.stereo_predict_rowband(ops[comm.rank], fL, fR, iL, iR, D, opt, comm=comm),
                  device=dev())
    assert [o.calls for o in ops] == [[], []]


# ------------------------------------------------------------------------------------------------------- b. bench size

@pytest.mark.parametrize("world", [2, 3])
def test_bench_size_matches_the_fused_pipeline(world):
    """kitti accurate_cbca4 at 370 x 1226, D 228 (bench.py's workload) against StereoPipeline in exact mode"""
    H, W, C, D = 370, 1226, 64, 228
    opt = pipeline.make_params("kitti", "accurate_cbca4")
    g = torch.Generator(device=dev()).manual_seed(11)
    featL = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev(), generator=g), dim=0)
    featR = torch.nn.functional.normalize(torch.randn((C, H, W), device=dev(), generator=g), dim=0)
    img = synth.natural_image(np.random.default_rng(11), H, W + 16)
    st = lambda x: cu((x - x.mean()) / x.std(ddof=1))
    imgL, imgR = st(img[:, 16:]), st(img[:, :W])
    sp = pipeline.StereoPipeline(C, D, H, W, opt, device=0, cbca_mode="exact")
    try:
        want = sp.run(featL, featR, imgL, imgR).cpu()
    finally:
        sp.close()
    for r, got in enumerate(_rowband_threads(opt, featL, featR, imgL, imgR, D, world)):
        same(got, want, "bench size, rank %d of %d" % (r, world))


# ---------------------------------------------------------------------------- c, d. from the images, every architecture

H_IMG, W_IMG, D_IMG, WORLD = 61, 203, 24, 3


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("rowband_threads")
    lp, rp = _images(tmp, H_IMG, W_IMG)
    nets = {arch: _net(str(tmp / ("%s.t7" % arch)), arch) for arch in ("fast", "slow")}
    return tmp, lp, rp, nets


@pytest.mark.parametrize("arch", ARCHS)
def test_band_predict_matches_the_whole_image(pair, arch):
    """each rank builds its own feature tower and scorer head, as it would on its own GPU"""
    tmp, lp, rp, nets = pair
    xb = torch.from_numpy(frontend.make_batch(lp, rp)).to(dev())
    opt = pipeline.make_params("kitti", arch)
    method = frontend.StereoMethod("kitti", arch, nets.get(arch))
    tower, head = method.stages(dev())
    feats = tower.forward(xb) if tower is not None else None
    want, wantL, wantR = pipeline.stereo_predict(xb, feats, opt, D_IMG, want_vols=True, arch=arch, head=head)
    torch.cuda.synchronize()
    method.close()
    del feats

    def rank(comm):
        m = frontend.StereoMethod("kitti", arch, nets.get(arch))
        t, h = m.stages(dev())
        try:
            d, vl, vr = rowband.band_predict(rowband.CudaOps(dev()), xb, D_IMG, opt, arch, t, h, comm, want_vols=True)
            return d.cpu(), vl.cpu(), vr.cpu()
        finally:
            torch.cuda.current_stream().synchronize()
            m.close()

    for r, (d, vl, vr) in enumerate(run_ranks(WORLD, rank, device=dev())):
        y0, y1 = rowband.split(H_IMG, WORLD, r)
        same(d, want[0, 0], "%s rank %d: disparity map" % (arch, r))
        same(vl, wantL[0, :, y0:y1], "%s rank %d: left volume rows [%d, %d)" % (arch, r, y0, y1))
        same(vr, wantR[0, :, y0:y1], "%s rank %d: right volume rows [%d, %d)" % (arch, r, y0, y1))


@pytest.mark.parametrize("arch", ARCHS)
def test_predict_pair_writes_frontend_predict_files(pair, arch):
    tmp, lp, rp, nets = pair
    net = nets.get(arch)
    want = _frontend_files(tmp / arch, lp, rp, arch, D_IMG, net)
    out = str(tmp / arch / "rowband")
    run_ranks(WORLD, lambda comm: rowband.predict_pair(lp, rp, "kitti", arch, disp_max=D_IMG, net_fname=net, comm=comm,
                                                       device=dev(), out_dir=out), device=dev())
    _assert_same_files(out, want)


# ---------------------------------------------------------------------------- e. mccnn_sgm2_rows at its dispatch edges

SGM_H = 7
SGM_BANDS = [(0, 1), (1, 4), (4, 7)]


def _sgm_rows_cases():
    """D as tests/dispatch_cases.SGM_CASES chooses it for every (K, VEC) instantiation, with its misaligned cost volume and
    accumulator; W at least H (oracle.sgm2) and 4 (three column chunks)"""
    out, seen = [], set()
    for c in dc.SGM_CASES:
        key = (c.D, c.in_off, c.out_off)
        if key not in seen:
            seen.add(key)
            out.append(c._replace(H=SGM_H, W=max(c.W, 9)))
    assert {(c.K, c.vec) for c in out} == set(dc.SGM_INSTANTIATIONS)
    return out


SGM_ROWS_CASES = _sgm_rows_cases()


def _at_offset(a, off):
    a = np.ascontiguousarray(a, dtype=np.float32)
    buf = torch.empty(a.size + off, device=dev())
    t = buf[off:].view(a.shape)
    t.copy_(cu(a))
    return t


def _opt(params):
    pi1, pi2, tau_so, alpha1, q1, q2 = params
    return pipeline.make_params("kitti", "fast", pi1=pi1, pi2=pi2, tau_so=tau_so, alpha1=alpha1, sgm_q1=q1, sgm_q2=q2)


@pytest.mark.parametrize("params", [dc.SGM_TIE, dc.SGM_TEN], ids=["tie", "ten"])
@pytest.mark.parametrize("direction", [-1, 1])
@pytest.mark.parametrize("c", SGM_ROWS_CASES, ids=lambda c: "D%d_K%d%s_off%d.%d" % (c.D, c.K, "vec" if c.vec else "", c.in_off,
                                                                                   c.out_off))
def test_sgm2_rows_chained(oracle, c, direction, params):
    """band_chain's schedule on one thread: the horizontal pair per band (zero_out, accumulator not initialised), then the
    down and the up pass band by band, each over the column chunks [0, 1), [1, W/2), [W/2, W), the line state of a band's
    last row handed to the next.  State buffers start as NaN; a call leaves the columns of state_out outside its chunk as
    they were.  The accumulator equals oracle.sgm2 of the whole image."""
    c = c._replace(params=params)
    x0, x1, vol = dc.sgm_inputs(c, direction)
    H, W, D = vol.shape
    assert dc.sgm_vec(D, c.in_off, c.out_off) == c.vec
    want = oracle.sgm2(x0, x1, vol, *params, direction)
    opt, ops = _opt(params), rowband.CudaOps(dev())
    tab = ops.sgm_tables(cu(x0), cu(x1), D, opt, direction)
    costs = [_at_offset(vol[a:b], c.in_off) for a, b in SGM_BANDS]
    accs = [_at_offset(np.full((b - a, W, D), np.nan, np.float32), c.out_off) for a, b in SGM_BANDS]
    for (a, b), cost, acc in zip(SGM_BANDS, costs, accs):
        ops.sgm_rows(tab, cost, acc, H, a, opt, direction, 3, True, 0, W, None, None)
    chunks = [(0, 1), (1, W // 2), (W // 2, W)]
    for sd, order in ((2, [0, 1, 2]), (3, [2, 1, 0])):
        st_in = None
        for i in order:
            st_out = None if i == order[-1] else torch.full((W, adcensus.lib().mccnn_sgm_state_pitch(D)), float("nan"),
                                                            device=dev())
            for xa, xb in chunks:
                before = st_out.clone() if st_out is not None else None
                ops.sgm_rows(tab, costs[i], accs[i], H, SGM_BANDS[i][0], opt, direction, 1 << sd, False, xa, xb, st_in, st_out)
                if st_out is not None:
                    outside = torch.ones(W, dtype=torch.bool, device=dev())
                    outside[xa:xb] = False
                    same(st_out[outside], before[outside], "pass %d band %d chunk [%d, %d): state_out outside the chunk"
                         % (sd, i, xa, xb))
            st_in = st_out
    same(torch.cat(accs), want, "sgm2 chained over row bands")


# ---------------------------------------------------------------------------------------- f. mccnn_sgm2_rows refusals

def test_sgm2_rows_refusals():
    """every check of mccnn_sgm2_rows, one argument wrong per call: the code comes back and nothing is written"""
    Ht, W, D = 7, 12, 40
    rng = np.random.default_rng(0)
    x0, x1 = cu(rng.random((Ht, W))), cu(rng.random((Ht, W)))
    opt = _opt(dc.SGM_TIE)
    ops = rowband.CudaOps(dev())
    tab = ops.sgm_tables(x0, x1, D, opt, -1)
    pitch = adcensus.lib().mccnn_sgm_state_pitch(D)
    cost = cu(rng.random((3, W, D)))
    acc = torch.full((3, W, D), 7.0, device=dev())
    st_in = torch.full((W, pitch), 5.0, device=dev())
    st_out = torch.full((W, pitch), 9.0, device=dev())
    torch.cuda.synchronize()
    base = dict(tab=tab.data_ptr(), input=cost.data_ptr(), output=acc.data_ptr(), H=3, W=W, D=D, Ht=Ht, yoff=2,
                pi1=opt.pi1, pi2=opt.pi2, tau_so=opt.tau_so, alpha1=opt.alpha1, q1=opt.sgm_q1, q2=opt.sgm_q2, direction=-1,
                pass_mask=4, zero_out=0, xa=0, xb=W, state_in=st_in.data_ptr(), state_out=st_out.data_ptr())

    def call(**over):
        a = dict(base, **over)
        return adcensus.lib().mccnn_sgm2_rows(*a.values(), adcensus._stream(cost))

    checks = [
        (EINVAL, dict(tab=None)), (EINVAL, dict(input=None)), (EINVAL, dict(output=None)),
        (EINVAL, dict(output=cost.data_ptr())),
        (EINVAL, dict(H=0)), (EINVAL, dict(W=0)), (EINVAL, dict(D=0)), (EINVAL, dict(Ht=2)),
        (EINVAL, dict(yoff=-1)), (EINVAL, dict(yoff=5)),
        (EINVAL, dict(direction=0)), (EINVAL, dict(direction=2)),
        (EINVAL, dict(pass_mask=0)), (EINVAL, dict(pass_mask=16)), (EINVAL, dict(pass_mask=20)),
        (EINVAL, dict(xa=-1)), (EINVAL, dict(xb=W + 1)), (EINVAL, dict(xa=5, xb=5)), (EINVAL, dict(xa=6, xb=5)),
        (EINVAL, dict(pass_mask=12)), (EINVAL, dict(pass_mask=12, state_in=None)),
        (EINVAL, dict(state_in=None)),                                    # down pass below the top without the state above
        (EINVAL, dict(pass_mask=8, state_in=None)),                       # up pass above the bottom without the state below
        (ELIMIT, dict(D=513)),
    ]
    for want_rc, over in checks:
        rc = call(**over)
        torch.cuda.synchronize()
        assert rc == want_rc, "%s: returned %d, expected %d" % (over, rc, want_rc)
        assert (acc == 7.0).all() and (st_in == 5.0).all() and (st_out == 9.0).all(), "%s: wrote its buffers" % over
    # the same calls with nothing wrong are accepted: the codes above come from the one argument changed
    for over in (dict(), dict(pass_mask=8, yoff=4), dict(pass_mask=4, yoff=0, state_in=None),
                 dict(pass_mask=8, yoff=4, state_in=None), dict(pass_mask=3, zero_out=1, state_in=None, state_out=None)):
        assert call(**over) == 0, over
    torch.cuda.synchronize()
