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
