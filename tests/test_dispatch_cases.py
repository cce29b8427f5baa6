"""CPU: the cases of tests/test_gpu_dispatch_edges.py select what they claim and reach every kernel variant, and their inputs
have teeth.  The selection rules are tests/dispatch_cases.py's restatement of the dispatchers in csrc/; the teeth are
computed with the oracle, in the style of test_kernel_mistakes.py: a kernel carrying the mistake would not pass the GPU
test on these inputs."""
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("dispatch_cases", os.path.join(ROOT, "tests", "dispatch_cases.py"))
dc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(dc)


# ------------------------------------------------------------------------------------------------------------ the rules

def test_sj_ns_table():
    """NS = 1 for D <= 8, then one more tile per 16 disparities up to 120; beyond, D is split into equal chunks"""
    for D in range(1, 121):
        assert dc.sj_ns(D) == -(-(D + 8) // 16)
    assert [dc.sj_ns(D) for D in (8, 9, 56, 57, 104, 105, 120, 121, 240, 241, 400)] == [1, 2, 4, 5, 7, 8, 8, 5, 8, 6, 7]


def test_sgm_and_post_thresholds():
    assert [dc.sgm_k(D) for D in (1, 32, 33, 64, 65, 128, 129, 256, 257, 512)] == [1, 1, 2, 2, 4, 4, 8, 8, 16, 16]
    assert not dc.sgm_vec(64, 0, 0) and dc.sgm_vec(128, 0, 0) and not dc.sgm_vec(128, 1, 0) and not dc.sgm_vec(130, 0, 0)
    assert [dc.mean2d_regime(k) for k in (1, 67, 69, 149, 151)] == ["tile", "tile", "tile_big", "tile_big", "pixel"]
    assert dc.interp_occ_kernel(4096) == "row" and dc.interp_occ_kernel(4097) == "pixel"
    # hpair needs both horizontal passes, a known-zero accumulator and two columns
    assert dc.sgm_launches(33, 3, 15, True) == [("hpair", 2, False), ("pass", 2, False, 2, False), ("pass", 2, False, 3, False)]
    assert dc.sgm_launches(129, 1, 15, True)[0] == ("pass", 8, False, 0, True)
    assert dc.sgm_launches(128, 9, 1, True) == [("pass", 4, True, 0, True)]
    assert dc.sgm_launches(128, 9, 15, False)[0] == ("pass", 4, True, 0, False)


# ------------------------------------------------------------------------------------------------------------- coverage

@pytest.mark.parametrize("c", dc.SJ_CASES, ids=dc.sj_id)
def test_sj_case_selects_its_variant(c):
    assert dc.sj_ns(c.D) == c.ns
    assert dc.sj_tma(c.H, c.W, (c.feat_off, c.feat_off, 0, 0)) == c.tma
    if dc.sj_pitched_ok(c.W, c.feat_off, dc.sj_ld(c.W)):
        assert dc.sj_tma(c.H, c.W, (c.feat_off, c.feat_off, 0, 0), dc.sj_ld(c.W)) == c.tma


def test_sj_cases_reach_every_variant():
    op = {(c.ns, c.tma) for c in dc.SJ_CASES}
    pitched = {(c.ns, c.tma) for c in dc.SJ_CASES if dc.sj_pitched_ok(c.W, c.feat_off, dc.sj_ld(c.W))}
    every = {(ns, t) for ns in range(1, 9) for t in (True, False)}
    assert op == every and pitched == every
    for ns in range(1, 9):                                              # the smallest and largest single-chunk D
        Ds = {c.D for c in dc.SJ_CASES if c.ns == ns}
        assert max(1, 16 * ns - 23) in Ds and 16 * ns - 8 in Ds
        assert dc.sj_ns(16 * ns - 7) != ns and (ns == 1 or dc.sj_ns(16 * ns - 24) != ns)
    assert any(c.D > c.W for c in dc.SJ_CASES) and any(c.D > 120 for c in dc.SJ_CASES)
    assert {1, 128} <= {c.C for c in dc.SJ_CASES} and any(c.C % 2 and c.C > 1 for c in dc.SJ_CASES)
    plain_hw = {c.ns for c in dc.SJ_CASES if (c.H * c.W) % 4 and dc.sj_pitched_ok(c.W, c.feat_off, dc.sj_ld(c.W))}
    plain_off1 = {c.ns for c in dc.SJ_CASES if c.feat_off == 1 and (c.H * c.W) % 4 == 0}
    assert plain_hw == set(range(1, 9)) and plain_off1 == set(range(1, 9))


@pytest.mark.parametrize("c", dc.SGM_CASES, ids=dc.sgm_id)
def test_sgm_case_selects_its_variant(c):
    assert (dc.sgm_k(c.D), dc.sgm_vec(c.D, c.in_off, c.out_off)) == (c.K, c.vec)
    assert c.H <= c.W


def test_sgm_cases_reach_every_instantiation():
    every = set(dc.SGM_INSTANTIATIONS)
    op, hpair, zero_pass, misaligned = set(), set(), set(), set()
    for c in dc.SGM_CASES:
        for kern in dc.sgm_launches(c.D, c.W, 15, False, c.in_off, c.out_off):        # adcensus.sgm2
            assert kern[0] == "pass" and not kern[4]
            op.add(kern[1:3])
        for mask in dc.SGM_MASKS:                                                     # mccnn_sgm2_band with zero_out
            for kern in dc.sgm_launches(c.D, c.W, mask, True, c.in_off, c.out_off):
                if kern[0] == "hpair":
                    hpair.add(kern[1:3])
                elif kern[4]:
                    zero_pass.add(kern[1:3])
        if (c.in_off or c.out_off) and c.D % 4 == 0:
            misaligned.add(c.K)
            assert not c.vec and dc.sgm_vec(c.D, 0, 0)
    assert op == every and hpair == every and zero_pass == every
    assert misaligned == {4, 8, 16}
    Ds = {c.D for c in dc.SGM_CASES}
    assert {1, 31, 32, 33, 64, 65, 127, 128, 129, 250, 256, 257, 510, 512} <= Ds
    assert {c.D for c in dc.SGM_CASES if c.in_off or c.out_off} == {128, 256, 512}
    assert {1, 2, 3} <= {c.W for c in dc.SGM_CASES} and {1, 2} == {c.H for c in dc.SGM_CASES}
    assert any(c.W % 2 and c.W > 3 for c in dc.SGM_CASES)
    assert {c.params[2] for c in dc.SGM_CASES} == {0.25, 10.0}
    for p in (dc.SGM_TIE, dc.SGM_TEN):
        assert p[4] * p[5] != 1 and p[3] != 1


def test_post_cases_reach_every_regime():
    assert {c.regime for c in dc.MEAN2D_CASES} == set(dc.MEAN2D_REGIMES)
    for c in dc.MEAN2D_CASES:
        assert dc.mean2d_regime(c.ksize) == c.regime
        assert c.W % 32 and c.H % 8
    alphas = {c.alpha2 for c in dc.MEAN2D_CASES}
    assert np.inf in alphas and min(alphas) < 0.01
    assert {dc.interp_occ_kernel(W) for W in dc.INTERP_OCC_W.values()} == {"row", "pixel"}
    assert all(dc.interp_occ_kernel(W) == k for k, W in dc.INTERP_OCC_W.items())
    assert {dc.median_kernel(k) for k in dc.MEDIAN_K} == {"median5", "sort"}
    assert any(H < 11 and W < 11 for H, W in dc.MEDIAN_SHAPES)
    plain = set()
    for c in dc.TRANSPOSE_CASES:
        plain.add(dc.transpose_kernel(c.D, c.H * c.W, c.off, c.off))               # mccnn_transpose_dhw_to_hwd
        plain.add(dc.transpose_kernel(c.H * c.W, c.D, c.off, c.off))               # mccnn_transpose_hwd_to_dhw_div4
    assert plain == {(t, lr) for t in (32, 64) for lr in (False, True)}
    pitched = {dc.transpose_pitched_vec(c.D, dc.sj_ld(c.W), c.off) for c in dc.TRANSPOSE_CASES}
    assert pitched == {True, False}
    assert any(c.off and c.D % 4 == 0 for c in dc.TRANSPOSE_CASES) and any(c.D % 4 for c in dc.TRANSPOSE_CASES)


# ---------------------------------------------------------------------------------------------------------------- teeth

@pytest.mark.parametrize("c", [c for c in dc.SGM_CASES if c.D > 1 and c.W > 2], ids=dc.sgm_id)
@pytest.mark.parametrize("direction", [-1, 1])
def test_sgm_class_ties_decide_the_result(oracle, c, direction):
    """tau_so one ulp either way moves |dI| == tau_so (and the NaN pixel's differences, and for tau_so = 10 the
    out-of-image D2) into another penalty class: a '<' / '<=' slip in the class tables changes sgm2 on every case with
    more than one disparity and more than two columns (with D = 1, or a 1 x 1 or 1 x 2 image holding a NaN pixel, no
    penalty reaches the result)"""
    x0, x1, vol = dc.sgm_inputs(c, direction)
    pi1, pi2, tau, alpha1, q1, q2 = c.params
    run = lambda t: oracle.sgm2(x0, x1, vol, pi1, pi2, t, alpha1, q1, q2, direction)
    want = run(tau)
    t = np.float32(tau)
    for moved in (np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(0))):
        assert not np.array_equal(run(float(moved)), want, equal_nan=True), "tau_so %r" % float(moved)


@pytest.mark.parametrize("c", dc.MEAN2D_CASES, ids=lambda c: "ks%d" % c.ksize)
def test_mean2d_transposed_kernel_changes_the_result(oracle, c):
    img, kern = dc.mean2d_inputs(c)
    want = oracle.mean2d(img, kern, c.alpha2)
    assert not np.array_equal(oracle.mean2d(img, np.ascontiguousarray(kern.T), c.alpha2), want, equal_nan=True)
    assert np.isnan(want).any() and not np.isnan(want).all()


def median5_nan_skipping(img):
    """post.cu's median5_kernel before it handled NaN: the n/2-th smallest by counting ranks, out-of-image taps +inf;
    a NaN is neither below nor equal to anything, so it never counts"""
    H, W = img.shape
    out = np.empty_like(img)
    with np.errstate(invalid="ignore"):
        for y in range(H):
            for x in range(W):
                v, n = [], 0
                for i in range(25):
                    xx, yy = x - 2 + i // 5, y - 2 + i % 5
                    ok = 0 <= xx < W and 0 <= yy < H
                    v.append(img[yy, xx] if ok else np.float32(np.inf))
                    n += ok
                v = np.array(v, np.float32)
                res = np.float32(0)
                for i in range(25):
                    if (v < v[i]).sum() <= n // 2 < (v <= v[i]).sum():
                        res = v[i]
                out[y, x] = res
    return out


def test_nan_skipping_median_disagrees_with_the_reference(oracle):
    img = dc.median_image("nan", 9, 13)
    want = oracle.median2d(img, 5)
    got = median5_nan_skipping(img)
    assert (~((got == want) | (np.isnan(got) & np.isnan(want)))).sum() > 20
    img = dc.median_image("signed_zero", 9, 13)                       # equal values, different bits: the sort picks
    want, got = oracle.median2d(img, 5), median5_nan_skipping(img)
    assert np.array_equal(got, want) and (np.signbit(got) != np.signbit(want)).sum() > 10
    for kind in ("ties", "inf"):                                      # the counting is right without NaN and -0
        img = dc.median_image(kind, 9, 13)
        assert np.array_equal(median5_nan_skipping(img), oracle.median2d(img, 5), equal_nan=True)


# ----------------------------------------------------------------------------------------------------------------- CBCA

def test_cbca_tables():
    assert [dc.cbca_gate(m) for m in (1, 2, 3, 5, 6, 9, 10, 14, 15, 1 << 20)] == \
        ["win1", "win1", "win4", "win4", "loop8", "loop8", "loop13", "loop13", "generic", "generic"]
    for m in range(1, 40):
        assert dc.cbca_gate(m) == dc.cbca_packed_kernel(m)                     # the gate and the halo table agree
    assert [dc.cbca_fast_kernel(m) for m in (1, 2, 3, 5, 6, 9, 10, 14, 15)] == \
        ["ws1", "ws1", "ws4", "ws4", "tma8", "tma8", "tma13", "tma13", "ELIMIT"]
    assert [dc.cbca_ex_clamp(m) for m in (1, 14, 15)] == [1, 14, 0]
    assert [dc.cbca_dchunk("ws4", D) for D in (20, 21, 40, 41, 228)] == [20, 11, 20, 14, 19]
    assert [dc.cbca_dchunk(k, 100) for k in ("win1", "loop13", "tma8")] == [14, 16, 20]
    assert dc.pipe_cbca_route(True, 5, 4, 35, 40) == "fast" and dc.pipe_cbca_route(False, 5, 4, 35, 40) == "packed"
    assert dc.pipe_cbca_route(True, 5, 4, 36, 40) == "generic" and dc.pipe_cbca_route(False, 5, 4, 36, 40) == "generic"
    assert dc.pipe_cbca_route(True, 14, 5, 20, 100) == "packed" and dc.pipe_cbca_route(True, 5, 0, 200, 100) == "fast"
    assert dc.pipe_cbca_route(True, 6, 4, 20, 100) == "packed"


@pytest.mark.parametrize("c", dc.CBCA_EXACT_CASES, ids=dc.cbca_id)
def test_cbca_exact_case_selects_its_kernel(oracle, c):
    """the arms' longest length is the case's L exactly (large runs, L1 = L), and the entry selects the claimed kernel"""
    x0c, x1c, a0, a1 = dc.cbca_arms(c)
    m = dc.pack_maxlen(x0c, x1c)
    if c.arms == "negative":
        assert m == 1 << 20 and c.entry == "gate"
    else:
        assert m == c.L
    k = dc.cbca_gate(m) if c.entry == "gate" else dc.cbca_packed_kernel(c.max_arm)
    assert k == c.kernel
    if c.arms == "clip":
        assert c.entry == "ex" and c.max_arm < c.L and dc.cbca_ex_clamp(c.max_arm) == c.max_arm
        assert dc.pack_maxlen(a0, a1) == c.max_arm
    elif c.max_arm is not None:
        assert c.max_arm >= c.L


def test_cbca_exact_cases_reach_every_kernel_and_boundary():
    pairs = {(c.entry, c.kernel) for c in dc.CBCA_EXACT_CASES if c.arms == "cross"}
    assert pairs == {(e, k) for e in ("gate", "ex", "packed") for k in dc.CBCA_EXACT_KERNELS}
    for lo, hi in dc.CBCA_BOUNDARIES:                                        # both sides of every boundary, every entry
        for e in ("gate", "ex", "packed"):
            Ls = {c.L for c in dc.CBCA_EXACT_CASES if c.entry == e and c.arms == "cross" and c.max_arm in (None, c.L)}
            assert {lo, hi} <= Ls, (e, lo, hi)
    over = {c.entry for c in dc.CBCA_EXACT_CASES if c.max_arm and c.max_arm > c.L}
    assert over == {"ex", "packed"}
    assert any(dc.cbca_packed_kernel(c.max_arm) != dc.cbca_gate(c.L) for c in dc.CBCA_EXACT_CASES if c.max_arm and c.max_arm > c.L)
    assert {c.entry for c in dc.CBCA_EXACT_CASES if c.arms == "clip"} == {"ex"}
    assert {c.kernel for c in dc.CBCA_EXACT_CASES if c.arms == "negative"} == {"generic"}
    assert {1, 127, 128, 129, 257} <= {c.W for c in dc.CBCA_EXACT_CASES}
    assert {1, 31, 32, 33, 63, 64, 65} <= {c.H for c in dc.CBCA_EXACT_CASES}
    assert any(c.D > c.W for c in dc.CBCA_EXACT_CASES)
    for k in ("win1", "win4"):                             # whole tiles in the invalid triangle (the loop kernels copy per column)
        for direction in (-1, 1):
            assert any("whole" in dc.cbca_copy_paths(k, c.D, c.W, direction) and "partial" in dc.cbca_copy_paths(k, c.D, c.W, direction)
                       for c in dc.CBCA_EXACT_CASES if c.kernel == k and c.direction == direction and c.W > 1), (k, direction)


@pytest.mark.parametrize("c", dc.CBCA_FAST_CASES, ids=dc.fast_id)
def test_cbca_fast_case_selects_its_kernel(c):
    assert dc.cbca_fast_kernel(c.max_arm) == c.kernel and c.max_arm == c.L
    assert dc.cbca_fast_refusal(c.W, c.ld, 0, 0, False, c.max_arm) is None and c.ld > c.W + 3
    assert c.kind in dc.CBCA_KINDS and (c.kind != "post_sgm" or c.H <= c.W)


def test_cbca_fast_cases_reach_every_kernel_and_edge():
    cases = dc.CBCA_FAST_CASES
    assert {c.kernel for c in cases} == set(dc.CBCA_FAST_KERNELS)
    assert {(c.kernel, c.direction) for c in cases} == {(k, d) for k in dc.CBCA_FAST_KERNELS for d in (-1, 1)}
    for k in dc.CBCA_FAST_KERNELS:
        mine = [c for c in cases if c.kernel == k]
        assert {127, 128, 129, 257} <= {c.W for c in mine}, k
        Ds = {c.D for c in mine}
        assert {20, 21, 40, 41} <= Ds, k                                         # one, two and three chunks
        for direction in (-1, 1):                                               # whole chunks copied, and partial ones
            paths = set()
            for c in mine:
                if c.direction == direction:
                    paths |= dc.cbca_copy_paths(k, c.D, c.W, direction)
            assert paths == {"whole", "partial"}, (k, direction)
    assert {c.kind for c in cases} == set(dc.CBCA_KINDS)
    for kind in dc.CBCA_KINDS:                                                  # every kind through a ws and a tma kernel
        ks = {c.kernel[:2] for c in cases if c.kind == kind}
        assert ks == {"ws", "tm"}, kind
    assert 228 in {c.D for c in cases if c.kernel.startswith("ws")} and dc.cbca_dchunk("ws4", 228) == 19
    assert {1, 31, 32, 33, 63, 64, 65} <= {c.H for c in cases} and 1 in {c.W for c in cases}
    assert {r[6] for r in dc.CBCA_FAST_REFUSALS} == {"EINVAL", "ELIMIT", None}
    for W, ld, i, o, a, m, want in dc.CBCA_FAST_REFUSALS:
        assert dc.cbca_fast_refusal(W, ld, i, o, a, m) == want


def test_ad_census_cases_reach_every_edge():
    cs = dc.AD_CENSUS_CASES
    assert {dc.census_kernel(c.nch) for c in cs} == {"nch1", "nch3", "nch_rt"} and 4 in {c.nch for c in cs}
    assert dc.census_kernel(5) == "ELIMIT"
    assert any(c.H == 1 for c in cs) and any(c.W == 1 for c in cs) and any(c.nan for c in cs)
    Ws = {c.W % 128 for c in cs if c.W > 1}
    assert {0, 1, 127} <= Ws
    Ds = {c.D for c in cs}
    assert {8, 9, 16, 17} <= Ds and any(c.D > c.W for c in cs)


# ---------------------------------------------------------------------------------------------------------------- teeth

def _tap_sum(a0, a1, vol, direction, rows=1, cols=1):
    """adcensus.cu:343-377 in float32 with one accumulator per output, rows and columns visited in the given order
    (1 ascending, the reference's; -1 descending)"""
    D, H, W = vol.shape
    out = np.array(vol, np.float32)
    ys, xs = np.mgrid[0:H, 0:W]
    m = max(dc.pack_maxlen(a0, a1), 1)
    for d in range(D):
        sh = d * direction
        xpc = np.clip(xs + sh, 0, W - 1)
        ok = (xs + sh >= 0) & (xs + sh < W)
        up = np.minimum(ys - a0[2], ys - a1[2][ys, xpc])
        dn = np.minimum(a0[3] - ys, a1[3][ys, xpc] - ys)
        acc = np.zeros((H, W), np.float32)
        cnt = np.zeros((H, W), np.int64)
        for dy in range(-m + 1, m)[::rows]:
            yy = np.clip(ys + dy, 0, H - 1)
            lft = np.minimum(xs - a0[0][yy, xs], xpc - a1[0][yy, xpc])
            rgt = np.minimum(a0[1][yy, xs] - xs, a1[1][yy, xpc] - xpc)
            rin = (dy > -up) & (dy < dn)
            for dx in range(-m + 1, m)[::cols]:
                tap = rin & (dx > -lft) & (dx < rgt)
                v = vol[d][yy, np.clip(xs + dx, 0, W - 1)]
                acc = np.where(tap, (acc + v).astype(np.float32), acc)
                cnt += tap
        with np.errstate(invalid="ignore", divide="ignore"):
            out[d] = np.where(ok, acc / cnt.astype(np.float32), out[d])
    return out


TEETH_CASES = [c for c in dc.CBCA_EXACT_CASES if c.entry == "ex" and c.arms == "cross" and c.H > 1 and c.W > 1]


@pytest.mark.parametrize("c", TEETH_CASES, ids=dc.cbca_id)
def test_cbca_summation_order_changes_the_bits(oracle, c):
    """the exact cases' volumes tell the reference's order (rows, then columns, ascending) from any other: a kernel that
    summed a run or the rows the other way round would not be bit-identical"""
    x0c, x1c, a0, a1 = dc.cbca_arms(c)
    vol = dc.cbca_volume("stereojoin", c.H, c.W, min(c.D, 24), c.direction)
    want = oracle.cbca(a0, a1, vol, c.direction)
    assert np.array_equal(_tap_sum(a0, a1, vol, c.direction), want, equal_nan=True)     # the restatement is right
    for rows, cols in ((1, -1), (-1, 1)):
        assert not np.array_equal(_tap_sum(a0, a1, vol, c.direction, rows, cols), want, equal_nan=True), (rows, cols)


@pytest.mark.parametrize("c", [c for c in dc.CBCA_EXACT_CASES if c.L == 3 and c.arms == "cross"], ids=dc.cbca_id)
def test_cbca_gate_off_by_one_changes_the_result(oracle, c):
    """arms of 3 aggregated by win<1> (a window of +-1 column and row: arms cut at 2), as a gate one off would do"""
    x0c, x1c, a0, a1 = dc.cbca_arms(c)
    vol = dc.cbca_volume("stereojoin", c.H, c.W, min(c.D, 24), c.direction)
    want = oracle.cbca(a0, a1, vol, c.direction)
    cut = oracle.cbca(dc.clip_arms(a0, 2), dc.clip_arms(a1, 2), vol, c.direction)
    assert not np.array_equal(cut, want, equal_nan=True)
