"""GPU: every cost-volume kernel family on a volume past 2^31 elements (D = 400, H = 2000, W = 3002: 2.40e9 floats, 9.6 GB),
compared at sampled places with a reference computed on the host from the few rows or columns the place depends on
(tests/large_volumes.py; tests/test_large_volume_refs.py proves those references on the CPU at a small shape).

The samples hold, for every layout a kernel reads or writes -- (D, H, W), the pitched (D, H, ld) with ld = 3004 (two
padding columns) or (H, W, D) -- the elements just before and at the flat indices 2^29 (2^31 bytes), 2^30 (2^32 bytes)
and 2^31, the last element, and a few seeded random ones.  H = 1999 makes H * W % 4 != 0 (StereoJoin's cp.async kernel
instead of its TMA one); D = 399 runs the scalar variants of SGM and of the pitched transposes.

Inputs are made on the device from seeded generators in the value kinds of tests/dispatch_cases.py; only images,
features, arms and the sampled rows / columns travel to the host.  Each test holds at most two volumes (19.2 GB) plus
small tensors, and skips, saying how much it needs, when the device has less free memory."""
import ctypes
import gc
import importlib.util
import os
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, scorer_head  # noqa: E402
from oracle import scorer_head as osh  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


dc = _load("dispatch_cases")
lv = _load("large_volumes")
same = _load("test_gpu_dispatch_edges").same

D, H, W = 400, 2000, 3002
LD = (W + 3) // 4 * 4                  # 3004: the pitch the pipeline uses, two padding columns
H_ODD, D_ODD = 1999, 399
NAN = float("nan")


def dev():
    return torch.device("cuda:0")


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


def stream(t):
    return adcensus._stream(t)


def gen(seed):
    return torch.Generator(device=dev()).manual_seed(seed)


def vol_bytes(*shape):
    return 4 * int(np.prod(shape))


def free_device_memory():
    gc.collect()
    torch.cuda.empty_cache()                                # memory cached by earlier tests counts as used otherwise
    adcensus.lib().adcensus_trim_scratch()
    return torch.cuda.mem_get_info()[0]


@pytest.fixture
def room(record_property):
    """need(bytes): skip unless the device has that much free memory.  Frees memory before and after the test and
    reports the test's peak of torch-allocated device memory and its wall time."""
    free_device_memory()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()

    def need(nbytes):
        free = free_device_memory()
        if free < nbytes:
            pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (nbytes / 1e9, free / 1e9))

    yield need
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    record_property("peak_device_bytes", peak)
    print("\n  peak %.1f GB allocated, %.1f s" % (peak / 1e9, time.time() - t0))
    free_device_memory()


def rows_of(vol, rows, width=None):
    """vol[:, rows, :width] of a (D, H, X) device volume, on the host"""
    idx = torch.as_tensor(list(rows), device=vol.device)
    return vol.index_select(1, idx)[..., :width].cpu().numpy()


def nan_triangle_(vol, direction):
    """NaN where StereoJoin writes nothing: x < d (direction -1) or x >= W - d (+1), on a (D, H, W) view"""
    Dv, _, Wv = vol.shape
    d = torch.arange(Dv, device=vol.device)[:, None, None]
    x = torch.arange(Wv, device=vol.device)[None, None, :]
    vol.masked_fill_((x < d) if direction < 0 else (x >= Wv - d), NAN)
    return vol


def quantised_(vol, g, levels, step):
    """in place: values k * step, k uniform in 0 .. levels - 1 (census: levels 244, step 1/3; SGM: 64, 0.125)"""
    return vol.uniform_(0, levels, generator=g).floor_().mul_(step)


def sample_rows(shapes, axis, extent, seed):
    return lv.sample_rows([(s, 0) for s in shapes], axis, extent, np.random.default_rng(seed))


# ---------------------------------------------------------------------------------------------------------- StereoJoin

@pytest.mark.parametrize("Hs", [H, H_ODD], ids=["tma", "cp_async"])
def test_stereo_join(oracle, room, Hs):
    """adcensus_StereoJoin on (D, H, W) and mccnn_stereo_join_pitched on (D, H, ld): both volumes bit for bit against
    oracle.stereo_join on the sampled rows; x < d NaN (pitched left) or untouched, x >= W - d untouched, padding untouched"""
    C = 16
    assert dc.sj_tma(Hs, W, (0, 0, 0, 0)) == (Hs % 2 == 0) and dc.sj_pitched_ok(W, 0, LD)
    room(2 * vol_bytes(D, Hs, LD) + 2 * vol_bytes(C, Hs, W) + 1e9)
    g = gen(1)
    fL = torch.nn.functional.normalize(torch.randn((C, Hs, W), generator=g, device=dev()), dim=0)
    fR = torch.nn.functional.normalize(torch.randn((C, Hs, W), generator=g, device=dev()), dim=0)
    hL, hR = fL.cpu().numpy(), fR.cpu().numpy()
    rows = sample_rows([(D, Hs, W), (D, Hs, LD)], 1, Hs, Hs)
    want = [lv.stereo_join_row(oracle, hL, hR, D, y) for y in rows]
    wantL, wantR = np.stack([w[0] for w in want], 1), np.stack([w[1] for w in want], 1)
    bufL, bufR = torch.empty(D * Hs * LD, device=dev()), torch.empty(D * Hs * LD, device=dev())

    oL, oR = bufL[:D * Hs * W].view(1, D, Hs, W).fill_(7.0), bufR[:D * Hs * W].view(1, D, Hs, W).fill_(9.0)
    adcensus.StereoJoin(fL[None], fR[None], oL, oR)
    same(rows_of(oL[0], rows), np.where(np.isnan(wantL), np.float32(7.0), wantL), "adcensus_StereoJoin left")
    same(rows_of(oR[0], rows), np.where(np.isnan(wantR), np.float32(9.0), wantR), "adcensus_StereoJoin right")

    pL, pR = bufL.view(D, Hs, LD).fill_(7.0), bufR.view(D, Hs, LD).fill_(9.0)
    rc = adcensus.lib().mccnn_stereo_join_pitched(vp(fL), vp(fR), vp(pL), vp(pR), C, D, Hs, W, LD, stream(pL))
    assert rc == 0, rc
    gL, gR = rows_of(pL, rows), rows_of(pR, rows)
    same(gL[..., :W], wantL, "mccnn_stereo_join_pitched left")
    same(gR[..., :W], np.where(np.isnan(wantR), np.float32(9.0), wantR), "mccnn_stereo_join_pitched right")
    assert bool((pL[:, :, W:] == 7.0).all()) and bool((pR[:, :, W:] == 9.0).all()), "padding columns were written"


# ------------------------------------------------------------------------------------------------------------- fills

def test_fill_invalid_small():
    """mccnn_fill_invalid on a small pair: NaN exactly where x < d (left) / x >= W - d (right), every other entry kept"""
    Ds, Hs, Ws = 40, 37, 66
    vL, vR = torch.full((Ds, Hs, Ws), 5.0, device=dev()), torch.full((Ds, Hs, Ws), 5.0, device=dev())
    assert adcensus.lib().mccnn_fill_invalid(vp(vL), vp(vR), Ds, Hs, Ws, stream(vL)) == 0
    wL, wR = lv.fill_invalid_rows(np.full((Ds, Hs, Ws), 5.0, np.float32), Ws, 5.0)
    same(vL, wL, "left")
    same(vR, wR, "right")


def test_fills_and_fix_border(oracle, room):
    """mccnn_fill_invalid (the rule on the sampled rows), mccnn_fix_border both directions (oracle.fix_border on the
    sampled rows as they were before), and mccnn_fill_nan over all but the first and the last two floats of a volume
    (a 4-byte head, the float4 body and a 2-float tail): NaN exactly there, the sentinel elsewhere"""
    room(2 * vol_bytes(D, H, W) + 3e9)
    lib = adcensus.lib()
    N = D * H * W
    vL, vR = torch.full((D, H, W), 5.0, device=dev()), torch.full((D, H, W), 5.0, device=dev())
    rows = sample_rows([(D, H, W)], 1, H, 2)
    assert lib.mccnn_fill_invalid(vp(vL), vp(vR), D, H, W, stream(vL)) == 0
    wL, wR = lv.fill_invalid_rows(np.full((D, len(rows), W), 5.0, np.float32), W, 5.0)
    same(rows_of(vL, rows), wL, "mccnn_fill_invalid left")
    same(rows_of(vR, rows), wR, "mccnn_fill_invalid right")

    g = gen(2)
    for v, direction in ((vL, -1), (vR, 1)):
        v.uniform_(-1, 1, generator=g)
        before = rows_of(v, rows)
        assert lib.mccnn_fix_border(vp(v), D, H, W, 4, direction, stream(v)) == 0
        same(rows_of(v, rows), oracle.fix_border(before, 4, direction), "mccnn_fix_border direction %+d" % direction)

    flat = vL.view(-1).fill_(5.0)
    assert lib.mccnn_fill_nan(ctypes.c_void_p(flat.data_ptr() + 4), N - 3, stream(flat)) == 0
    idx = sorted(set(lv.threshold_flats((N,))) | {0, 1, 2, 3, 4, 5, N - 6, N - 5, N - 4, N - 3, N - 2}
                 | set(np.random.default_rng(3).integers(0, N, 200).tolist()))
    got = flat[torch.as_tensor(idx, device=dev())].cpu().numpy()
    want = np.where((np.array(idx) >= 1) & (np.array(idx) < N - 2), np.float32(np.nan), np.float32(5.0))
    same(got, want, "mccnn_fill_nan")
    assert bool(flat[1:N - 2].isnan().all()), "mccnn_fill_nan left an entry"


# ------------------------------------------------------------------------------------------------------- AD / census

@pytest.mark.parametrize("kind,nch,direction", [("census", 1, -1), ("census", 3, 1), ("ad", 1, -1), ("ad", 1, 1)])
def test_ad_census(oracle, room, kind, nch, direction):
    """adcensus_census (1 and 3 channels) and adcensus_ad: the sampled rows bit for bit against oracle.census / oracle.ad
    on the image rows y - 4 .. y + 4; images on a grid of 1/3 with 2% NaN pixels (dispatch_cases.ad_census_images)"""
    room(vol_bytes(D, H, W) + 2e9)
    g = gen(10 + nch + (direction > 0))
    imgs = torch.randn((2, nch, H, W), generator=g, device=dev()).mul_(3).round_().div_(3)
    nan_at = torch.randint(0, imgs.numel(), (imgs.numel() // 50,), generator=g, device=dev())
    imgs.view(-1)[nan_at] = NAN
    a, b = imgs.cpu().numpy()
    out = torch.full((1, D, H, W), 3.0, device=dev())
    rows = sample_rows([(D, H, W)], 1, H, 4)
    if kind == "census":
        adcensus.census(imgs[0][None], imgs[1][None], out, direction)
        want = [lv.cost_row(oracle, a, b, D, y, direction, kind) for y in rows]
    else:
        adcensus.ad(imgs[0][None], imgs[1][None], out, direction)
        want = [lv.cost_row(oracle, a[0], b[0], D, y, direction, kind) for y in rows]
    same(rows_of(out[0], rows), np.stack(want, 1), "%s nch %d direction %+d" % (kind, nch, direction))


# ----------------------------------------------------------------------------------------------------------------- CBCA

EXACT_ARM = {"win1": 2, "win4": 5, "loop8": 9, "loop13": 14, "generic": 15}     # one max_arm per exact kernel
FAST_ARM = {"ws1": 2, "ws4": 5, "tma8": 9, "tma13": 14}


def cbca_arms(oracle, L, seed):
    """cross() arms (tau1 0.5, L1 = L) of two dispatch_cases.cbca_image images: (host x0c, x1c, device x0c, x1c)"""
    x0c = oracle.cross(dc.cbca_image(H, W, L, seed), L, dc.CBCA_TAU1)
    x1c = oracle.cross(dc.cbca_image(H, W, L, seed + 1), L, dc.CBCA_TAU1)
    assert dc.pack_maxlen(x0c, x1c) == L
    return x0c, x1c, torch.from_numpy(x0c).to(dev()), torch.from_numpy(x1c).to(dev())


@pytest.mark.parametrize("entry,kernel", [("packed", k) for k in dc.CBCA_EXACT_KERNELS] + [("gate", "loop8")])
def test_cbca_exact(oracle, room, entry, kernel):
    """mccnn_pack_arms + mccnn_cbca_packed at one max_arm per exact kernel, and adcensus_cbca (the device gate), both
    directions, on a census-valued volume with StereoJoin's NaN triangle: the sampled rows bit for bit against oracle.cbca
    on the rows [y - halo, y + halo]"""
    L = EXACT_ARM[kernel]
    assert (dc.cbca_packed_kernel(L) if entry == "packed" else dc.cbca_gate(L)) == kernel
    room(2 * vol_bytes(D, H, W) + 2e9)
    x0c, x1c, t0, t1 = cbca_arms(oracle, L, 20 + L)
    lib = adcensus.lib()
    vin, vout = torch.empty((D, H, W), device=dev()), torch.empty((D, H, W), device=dev())
    rows = sample_rows([(D, H, W)], 1, H, 5)
    packed = torch.zeros(lib.mccnn_packed_arms_bytes(H, W) // 4, dtype=torch.int32, device=dev())
    for direction in (-1, 1):
        nan_triangle_(quantised_(vin, gen(30 + direction), 244, 1.0 / 3), direction)
        vout.fill_(5.0)
        if entry == "gate":
            adcensus.cbca(t0[None], t1[None], vin[None], vout[None], direction)
        else:
            s = stream(vin)
            assert lib.mccnn_pack_arms(vp(t0), vp(t1), vp(packed), H, W, s) == 0
            assert lib.mccnn_cbca_packed(vp(packed), vp(t0), vp(t1), vp(vin), vp(vout), D, H, W, direction, L, s) == 0
        want = [lv.cbca_row(oracle, x0c, x1c, lambda a, b: rows_of(vin, range(a, b)), y, L - 1, direction) for y in rows]
        same(rows_of(vout, rows), np.stack(want, 1), "cbca %s %s direction %+d" % (entry, kernel, direction))


def _rel_err(got, want):
    m = ~np.isnan(want)
    return float((np.abs(got[m] - want[m]) / np.maximum(1.0, np.abs(want[m]))).max()) if m.any() else 0.0


@pytest.mark.parametrize("i,kernel", list(enumerate(dc.CBCA_FAST_KERNELS)), ids=list(dc.CBCA_FAST_KERNELS))
def test_cbca_fast(oracle, room, record_property, i, kernel):
    """mccnn_cbca_fast_pitched and mccnn_pack_arms_hv + mccnn_cbca_fast_pitched_packed at one max_arm per constant-work
    kernel, directions alternating, on census-valued (D, H, ld) volumes whose padding holds 123 (input) / -7 (output): the
    sampled rows within 1e-4 max(1, |want|)
    of oracle.cbca and of the float64 tap sums (on the planes of the threshold elements), NaN positions identical, the
    output's padding untouched"""
    L, direction = FAST_ARM[kernel], (-1 if i % 2 == 0 else 1)
    assert dc.cbca_fast_kernel(L) == kernel and dc.cbca_fast_refusal(W, LD, 0, 0, False, L) is None
    room(2 * vol_bytes(D, H, LD) + 2e9)
    x0c, x1c, t0, t1 = cbca_arms(oracle, L, 40 + L)
    lib = adcensus.lib()
    vin, vout = torch.full((D, H, LD), 123.0, device=dev()), torch.empty((D, H, LD), device=dev())
    # census3 values: a plane read in place of another is off by O(1), far outside the bar (on the offset_gradient kind,
    # 3000 + 40 x + [-1, 1], it would be off by 1e-5 relative and pass)
    nan_triangle_(quantised_(vin[:, :, :W], gen(50 + i), 244, 1.0 / 3), direction)
    rows = sample_rows([(D, H, LD)], 1, H, 6)
    planes = sorted({p[0] for p in lv.positions((D, H, LD))} | {0, 1, D // 2})
    want = [lv.cbca_row(oracle, x0c, x1c, lambda a, b: rows_of(vin, range(a, b), W), y, L - 1, direction, dc.cbca_f64,
                        planes) for y in rows]
    want32, want64 = np.stack([w[0] for w in want], 1), np.stack([w[1] for w in want], 1)
    hv = torch.zeros(lib.mccnn_packed_hv_bytes(H, W) // 4, dtype=torch.int32, device=dev())
    for entry in ("pitched", "packed"):
        vout.fill_(-7.0)
        s = stream(vin)
        if entry == "pitched":
            rc = lib.mccnn_cbca_fast_pitched(vp(t0), vp(t1), vp(vin), vp(vout), D, H, W, LD, direction, L, s)
        else:
            assert lib.mccnn_pack_arms_hv(vp(t0), vp(t1), vp(hv), H, W, s) == 0
            rc = lib.mccnn_cbca_fast_pitched_packed(vp(hv), vp(vin), vp(vout), D, H, W, LD, direction, L, s)
        assert rc == 0, rc
        assert bool((vout[:, :, W:] == -7.0).all()), "%s: padding columns were written" % entry
        got = rows_of(vout, rows, W)
        assert np.array_equal(np.isnan(got), np.isnan(want32)), "%s: NaN pattern differs" % entry
        e32 = _rel_err(got, want32)
        e64 = _rel_err(got[planes].astype(np.float64), want64[planes])
        record_property("max_rel_err_%s" % entry, max(e32, e64))
        assert e32 <= 1e-4 and e64 <= 1e-4, "%s: max relative error %.3g (oracle), %.3g (float64)" % (entry, e32, e64)


# ------------------------------------------------------------------------------------------------------------------ SGM

def sgm_inputs(Dv, direction, seed):
    """SGM_TIE images (0 .. 1 on a grid of 0.25, one NaN pixel each) and an (H, W, D) volume of multiples of 0.125 in
    0 .. 7.875 with StereoJoin's NaN triangle (dispatch_cases.sgm_inputs' kinds); host copies of the images"""
    g = gen(seed)
    imgs = torch.randint(0, 5, (2, H, W), generator=g, device=dev()).float().mul_(0.25)
    for k in range(2):
        imgs[k, int(torch.randint(0, H, (1,), generator=g, device=dev())), int(torch.randint(0, W, (1,), generator=g, device=dev()))] = NAN
    cost = quantised_(torch.empty((H, W, Dv), device=dev()), g, 64, 0.125)
    d = torch.arange(Dv, device=dev())[None, None, :]
    x = torch.arange(W, device=dev())[None, :, None]
    cost.masked_fill_((x < d) if direction < 0 else (x >= W - d), NAN)
    return imgs[0].contiguous(), imgs[1].contiguous(), cost, imgs.cpu().numpy()


@pytest.mark.parametrize("entry,Dv,direction", [("ckpt", D, -1), ("ckpt", D_ODD, 1), ("sgm2", D, 1), ("sgm2", D_ODD, -1),
                                                ("rows", D, -1)])
def test_sgm(oracle, room, entry, Dv, direction):
    """mccnn_sgm2_ckpt (checkpoints in a scratch of mccnn_sgm2_ckpt_bytes), adcensus_sgm2, and mccnn_sgm2_rows chained over
    two row bands split just after the 2^31st element's row: at every crossing of the sampled rows and columns (which
    include the pixels of the (H, W, D) threshold elements) bit for bit against the oracle's 1-row and 1-column bands,
    signs of zeros included"""
    params = dc.SGM_TIE
    assert dc.sgm_vec(Dv, 0, 0) == (Dv % 4 == 0)
    lib = adcensus.lib()
    ck = lib.mccnn_sgm2_ckpt_bytes(H, W, Dv) if entry == "ckpt" else 0
    room(2 * vol_bytes(H, W, Dv) + ck + lib.mccnn_sgm_tables_bytes(H, W, Dv) + 1e9)
    iL, iR, cost, (x0, x1) = sgm_inputs(Dv, direction, 60 + Dv + direction)
    s = stream(cost)
    ysplit = lv.positions((H, W, Dv))[5][0] + 1                     # band 0 holds the 2^31st element, and more than 2^31
    if entry == "ckpt":
        assert ck > 0, "mccnn_sgm2_ckpt would fall back to the 11-pass kernels"
        scratch = torch.empty(ck // 4, device=dev())
        out = torch.full_like(cost, NAN)
        assert lib.mccnn_sgm2_ckpt(vp(iL), vp(iR), vp(cost), vp(out), vp(scratch), ck, H, W, Dv, *params, direction, s) == 0
        del scratch
    elif entry == "sgm2":
        out = torch.zeros_like(cost)
        adcensus.sgm2(iL[None], iR[None], cost[None], out[None], None, *params, direction)
    else:
        out = torch.full_like(cost, NAN)
        tab = torch.empty(lib.mccnn_sgm_tables_bytes(H, W, Dv), dtype=torch.uint8, device=dev())
        assert lib.mccnn_sgm_tables_build(vp(iL), vp(iR), vp(tab), H, W, Dv, params[2], direction, s) == 0
        assert ysplit * W * Dv > 1 << 31
        bands = [(0, ysplit), (ysplit, H)]
        pitch = lib.mccnn_sgm_state_pitch(Dv)
        state = torch.empty((W, pitch), device=dev())

        def run(a, b, mask, zero_out, st_in, st_out):
            rc = lib.mccnn_sgm2_rows(vp(tab), vp(cost[a:b]), vp(out[a:b]), b - a, W, Dv, H, a, *params, direction, mask,
                                     zero_out, 0, W, None if st_in is None else vp(st_in),
                                     None if st_out is None else vp(st_out), s)
            assert rc == 0, rc

        for a, b in bands:
            run(a, b, 3, 1, None, None)                             # right, left: band-local
        run(0, ysplit, 4, 0, None, state)                           # down: band 0, then band 1 from its last row
        run(ysplit, H, 4, 0, state, None)
        run(ysplit, H, 8, 0, None, state)                           # up: band 1, then band 0
        run(0, ysplit, 8, 0, state, None)
        del tab
    torch.cuda.synchronize()
    shape = (H, W, Dv)
    ys = sample_rows([shape], 0, H, 7)
    xs = sample_rows([shape], 1, W, 8)
    if entry == "rows":
        ys = sorted(set(ys) | {ysplit - 1, ysplit})
    want = lv.sgm_crossings(oracle, x0, x1, lambda y: cost[y].cpu().numpy(), lambda x: cost[:, x].cpu().numpy(), ys, xs,
                            params, direction)
    yi, xi = torch.as_tensor(ys, device=dev()), torch.as_tensor(xs, device=dev())
    got = out.index_select(0, yi).index_select(1, xi).cpu().numpy()
    same(got, np.stack([np.stack([want[y, x] for x in xs]) for y in ys]), "%s D=%d direction %+d" % (entry, Dv, direction))


# ----------------------------------------------------------------------------------------------------------- transposes

def gather(t, pos):
    """t[pos] for a list of index tuples, by torch indexing (64-bit), on the host"""
    idx = [torch.as_tensor(c, device=t.device) for c in zip(*pos)]
    return t[tuple(idx)].cpu().numpy()


def element_samples(shape, seed, n=1000):
    rng = np.random.default_rng(seed)
    return lv.positions(shape) + [tuple(int(rng.integers(0, e)) for e in shape) for _ in range(n)]


def logical(layout, shape, seed):
    """(d, h, w) of the threshold and random elements of a (D, H, X) ('dhw') or (H, W, D) ('hwd') volume; padding dropped"""
    out = []
    for p in element_samples(shape, seed):
        d, h, w = p if layout == "dhw" else (p[2], p[0], p[1])
        if w < W:
            out.append((d, h, w))
    return out


def at(layout, pos):
    return pos if layout == "dhw" else [(h, w, d) for d, h, w in pos]


@pytest.mark.parametrize("Dv", [D, D_ODD])
def test_transposes(room, Dv):
    """mccnn_transpose_dhw_to_hwd, _hwd_to_dhw_div4 and both pitched forms: at the threshold elements of the input and of
    the output layout and at random ones, out == in (x 1/4) exactly, by torch indexing of the input"""
    assert dc.transpose_pitched_vec(Dv, LD, 0) == (Dv % 4 == 0)
    room(2 * vol_bytes(Dv, H, LD) + 1e9)
    lib = adcensus.lib()
    N = Dv * H * W
    a, b = torch.empty(Dv * H * LD, device=dev()), torch.empty(Dv * H * LD, device=dev())
    dhw, hwd, pitched = a[:N].view(Dv, H, W), b[:N].view(H, W, Dv), a.view(Dv, H, LD)
    s = stream(a)

    def check(src, src_layout, dst, dst_layout, scale, what):
        pos = logical(src_layout, tuple(src.shape), Dv) + logical(dst_layout, tuple(dst.shape), Dv + 1)
        same(gather(dst, at(dst_layout, pos)), gather(src, at(src_layout, pos)) * np.float32(scale), what)

    dhw.uniform_(-1, 1, generator=gen(70))
    assert lib.mccnn_transpose_dhw_to_hwd(vp(dhw), vp(hwd), Dv, H, W, s) == 0
    check(dhw, "dhw", hwd, "hwd", 1.0, "dhw -> hwd")
    assert lib.mccnn_transpose_hwd_to_dhw_div4(vp(hwd), vp(dhw), Dv, H, W, s) == 0
    check(hwd, "hwd", dhw, "dhw", 0.25, "hwd -> dhw / 4")
    pitched.fill_(float("inf"))
    pitched[:, :, :W].uniform_(-1, 1, generator=gen(71))
    assert lib.mccnn_transpose_dhw_pitched_to_hwd(vp(pitched), vp(hwd), Dv, H, W, LD, s) == 0
    check(pitched, "dhw", hwd, "hwd", 1.0, "pitched dhw -> hwd")
    assert lib.mccnn_transpose_hwd_to_dhw_pitched_div4(vp(hwd), vp(pitched), Dv, H, W, LD, s) == 0
    check(hwd, "hwd", pitched, "dhw", 0.25, "hwd -> pitched dhw / 4")


# ------------------------------------------------------------------------------------------------ arg-min and sub-pixel

def test_argmin_subpixel(oracle, room):
    """mccnn_argmin_pitched on (D, H, ld) with -inf in the padding, mccnn_argmin and adcensus_spatial_argmin on (D, H, W),
    and adcensus_subpixel_enchancement with c2 past 2^31 (d0 set so that the pixels of the threshold elements read them):
    on the D-columns of those pixels and of random ones, the first minimum with NaN skipped and the sub-pixel value as
    oracle.subpixel_enchancement states it, exactly"""
    room(vol_bytes(D, H, LD) + 1e9)
    lib = adcensus.lib()
    buf = torch.full((D * H * LD,), -float("inf"), device=dev())
    pv = buf.view(D, H, LD)
    g = gen(80)
    for d0 in range(0, D, 40):                                    # integers 0 .. 7 with 20% NaN, ties common
        blk = quantised_(pv[d0:d0 + 40, :, :W], g, 8, 1.0)
        blk.masked_fill_(torch.rand(blk.shape, generator=g, device=dev()) < 0.2, NAN)
    vc = buf[:D * H * W].view(D, H, W)                            # the same storage read as a contiguous (D, H, W) volume
    rng = np.random.default_rng(81)
    rand_pix = [(int(rng.integers(0, H)), int(rng.integers(0, W))) for _ in range(300)]
    pix_p = sorted({(p[1], p[2]) for p in lv.positions((D, H, LD)) if p[2] < W} | set(rand_pix))
    pix_c = sorted({(p[1], p[2]) for p in lv.positions((D, H, W))} | set(rand_pix))

    def cols(vol, pix):
        ys, xs = (torch.as_tensor(c, device=dev()) for c in zip(*pix))
        return vol[:, ys, xs].cpu().numpy()

    disp = torch.empty((H, W), device=dev())
    assert lib.mccnn_argmin_pitched(vp(pv), vp(disp), D, H, W, LD, stream(pv)) == 0
    same(gather(disp, pix_p), lv.argmin_columns(cols(pv, pix_p)), "mccnn_argmin_pitched")
    assert lib.mccnn_argmin(vp(vc), vp(disp), D, H * W, stream(vc)) == 0
    want = lv.argmin_columns(cols(vc, pix_c))
    same(gather(disp, pix_c), want, "mccnn_argmin")
    out = torch.empty((1, 1, H, W), device=dev())
    adcensus.spatial_argmin(vc[None], out)
    same(gather(out[0, 0], pix_c), want + 1, "adcensus_spatial_argmin")

    d0 = torch.randint(0, D, (H, W), generator=g, device=dev()).float()
    for p in lv.positions((D, H, W)):
        d0[p[1], p[2]] = float(min(max(p[0], 1), D - 2))
    sub = adcensus.subpixel_enchancement(d0[None, None], vc[None], D)
    d0s = gather(d0, pix_c)[None]
    want = oracle.subpixel_enchancement(d0s, cols(vc, pix_c)[:, None, :], D)[0]
    same(gather(sub[0, 0], pix_c), want, "adcensus_subpixel_enchancement")


# --------------------------------------------------------------------------------------------------------- scorer head

@pytest.mark.parametrize("nterms,bar", [(3, 1e-4), (1, 2e-2)])
def test_scorer_head(room, nterms, bar):
    """mccnn_scorer_head_forward (the smallest net: fm 8, nh2 128, l2 1) into both volumes: at the threshold elements of
    each volume and at 1000 random valid entries within `bar` of oracle.scorer_head.head_samples (float64), the caller's
    NaN fill untouched where x < d (left) / x >= W - d (right)"""
    fm, nh2, l2 = 8, 128, 1
    room(2 * vol_bytes(D, H, W) + 2 * vol_bytes(fm, H, W) + 1e9)
    rng = np.random.default_rng(90 + nterms)
    layers = osh.make_weights(rng, fm, nh2, l2)
    g = gen(91)
    fL = torch.randn((fm, H, W), generator=g, device=dev()).clamp_(min=0)
    fR = torch.randn((fm, H, W), generator=g, device=dev()).clamp_(min=0)
    hL, hR = fL.cpu().numpy(), fR.cpu().numpy()
    head = scorer_head.ScorerHead(layers)
    try:
        vL, vR = head.volumes(fL, fR, D, nterms=nterms)
        torch.cuda.synchronize()
    finally:
        head.close()
    vL, vR = vL[0], vR[0]
    k = 1000
    d = rng.integers(0, D, k)
    x = d + (rng.random(k) * (W - d)).astype(np.int64)
    y = rng.integers(0, H, k)
    pos = lv.positions((D, H, W))
    for vol, right in ((vL, False), (vR, True)):
        samples = pos + [(int(a), int(b), int(c - d_ if right else c)) for a, b, c, d_ in zip(d, y, x, d)]
        sd, sy, sx = (np.array(c) for c in zip(*samples))
        xl = sx + sd if right else sx                                    # the left-volume column of the same score
        valid = xl < W if right else sx >= sd
        got = gather(vol, samples)
        assert np.isnan(got[~valid]).all(), "%s volume: the NaN fill was written" % ("right" if right else "left")
        want = osh.head_samples(hL, hR, layers, sd[valid], sy[valid], xl[valid])
        err = float(np.abs(got[valid] - want).max())
        assert err <= bar, "%s volume, nterms %d: max abs error %.3g (bar %.1g)" % ("right" if right else "left", nterms, err, bar)
    rows = sample_rows([(D, H, W)], 1, H, 92)
    dd, xx = np.arange(D)[:, None, None], np.arange(W)[None, None, :]
    assert np.array_equal(np.isnan(rows_of(vL, rows)), np.broadcast_to(xx < dd, (D, len(rows), W)))
    assert np.array_equal(np.isnan(rows_of(vR, rows)), np.broadcast_to(xx >= W - dd, (D, len(rows), W)))
