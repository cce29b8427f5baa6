"""Kernel-variant selection of the hot path, restated in Python, and the cases of tests/test_gpu_dispatch_edges.py.

Most operators are not one kernel: a dispatcher picks a template instantiation or a fallback from D, W, H, pointer alignment
or shared-memory size.  Each rule below is a plain statement of one such dispatcher, next to the C function it restates, and
every case carries the variant it is meant to select.  tests/test_dispatch_cases.py checks, without a GPU, that each case
selects what it claims and that the lists reach every variant; the GPU test then runs each case against the oracle.

Pointer offsets are in floats from a 16-byte aligned allocation (torch's allocator aligns far more than that), so a
case's offset decides the alignment the dispatcher sees.
"""
from collections import namedtuple

import numpy as np

# ---------------------------------------------------------------------------------------------------------- StereoJoin

def sj_ns(D):
    """stereo_join.cu sj_ns: D in equal chunks of at most 120, the smallest tile count (DC = 16 NS - 8) that covers one"""
    nchunk = -(-D // 120)
    dc = -(-D // nchunk)
    return -(-(dc + 8) // 16)


def sj_tma(H, W, ptr_offsets, ldo=None):
    """stereo_join_tma.cu adc_stereo_join_tma_ok and its caller stereo_join.cu adc_stereo_join: the TMA-load kernel runs
    when H * W % 4 == 0, all four pointers are 16-byte aligned and the output pitch is a multiple of 4 (or W)"""
    ldo = W if ldo is None else ldo
    return (H * W) % 4 == 0 and all((4 * o) % 16 == 0 for o in ptr_offsets) and (ldo % 4 == 0 or ldo == W)


def sj_pitched_ok(W, feat_off, ld):
    """stereo_join.cu mccnn_stereo_join_pitched: W even, ld % 4 == 0, features 8-byte and outputs 16-byte aligned"""
    return W % 2 == 0 and ld % 4 == 0 and (4 * feat_off) % 8 == 0


def sj_ld(W):
    """row pitch of the pitched volumes in these tests: a multiple of 4 with at least 4 columns of padding"""
    return (W + 3) // 4 * 4 + 4


# H, W, C, D, feat_off (floats, both feature tensors); ns and tma: the operator's (adcensus_StereoJoin) selection
SJCase = namedtuple("SJCase", "H W C D feat_off ns tma")


def _sj_cases():
    cases = []
    cs = (1, 5, 128, 64, 3, 128, 17, 1)
    for ns in range(1, 9):
        lo, hi = max(1, 16 * ns - 23), 16 * ns - 8            # the D that select ns with one chunk
        C = cs[ns - 1]
        for D in (lo, hi):
            wb = D + 6 if D == lo else max(2, D // 2)            # the largest D of each NS runs with D > W
            even = wb + wb % 2
            odd_rows = wb // 4 * 4 + 2                           # W % 4 == 2: H * W % 4 != 0 for odd H, W still even
            cases += [SJCase(4, even, C, D, 0, ns, True),        # TMA
                      SJCase(3, odd_rows, C, D, 0, ns, False),   # plain: H * W % 4 != 0
                      SJCase(4, even, C, D, 1, ns, False),       # plain: features 4 bytes off (the operator only)
                      SJCase(2, even, C, D, 2, ns, False)]       # plain: features 8 bytes off
    cases += [SJCase(2, 130, 3, 121, 0, 5, True),                # two chunks of 61
              SJCase(3, 66, 7, 240, 0, 8, False),                # two chunks of 120, D > W
              SJCase(2, 250, 1, 241, 2, 6, False),               # three chunks of 81
              SJCase(5, 9, 9, 100, 0, 7, False)]                 # -disp_max 100, odd W, D > W
    return cases


SJ_CASES = _sj_cases()


def sj_id(c):
    return "H%dW%dC%dD%d_off%d" % (c.H, c.W, c.C, c.D, c.feat_off)


# ------------------------------------------------------------------------------------------------------------------ SGM

def sgm_k(D):
    """sgm.cu adc_sgm2_passes: K disparity slots per lane"""
    return 1 if D <= 32 else 2 if D <= 64 else 4 if D <= 128 else 8 if D <= 256 else 16


def sgm_vec(D, in_off, out_off):
    """sgm.cu adc_sgm2_passes: float4 traffic for K >= 4 when D % 4 == 0 and both volume pointers are 16-byte aligned"""
    return sgm_k(D) >= 4 and D % 4 == 0 and (4 * in_off) % 16 == 0 and (4 * out_off) % 16 == 0


def sgm_launches(D, W, pass_mask, zero_out, in_off=0, out_off=0):
    """sgm.cu launch_all: the kernels one call launches, in order: ("hpair", K, VEC) for sgm_hpair_kernel, or
    ("pass", K, VEC, SD, ZERO) for sgm_pass_kernel.  adcensus.sgm2 is pass_mask 15 without zero_out."""
    K, vec = sgm_k(D), sgm_vec(D, in_off, out_off)
    out = []
    if pass_mask & 3 == 3 and zero_out and W >= 2:
        out.append(("hpair", K, vec))
    else:
        if pass_mask & 1:
            out.append(("pass", K, vec, 0, bool(zero_out)))
        if pass_mask & 2:
            out.append(("pass", K, vec, 1, False))
    for sd in (2, 3):
        if pass_mask & (1 << sd):
            out.append(("pass", K, vec, sd, False))
    return out


SGM_INSTANTIATIONS = [(1, False), (2, False), (4, False), (4, True), (8, False), (8, True), (16, False), (16, True)]

# penalty parameters (pi1, pi2, tau_so, alpha1, sgm_q1, sgm_q2): q1 * q2 != 1 and alpha1 != 1, so every one of the
# three classes and the alpha1 scaling of the vertical passes gives a different penalty
SGM_TIE = (1.32, 24.25, 0.25, 2.0, 3.0, 2.0)      # images quantised to 0.25: |dI| == tau_so is common
SGM_TEN = (1.32, 24.25, 10.0, 1.5, 4.0, 1.25)     # the out-of-image difference D2 = 10 falls on tau_so

# H, W, D, in_off, out_off (floats), params, K, VEC.  H <= W: oracle.sgm2 (the reference) needs it.
SGMCase = namedtuple("SGMCase", "H W D in_off out_off params K vec")
SGM_CASES = [
    SGMCase(1, 1, 1, 0, 0, SGM_TIE, 1, False),
    SGMCase(2, 5, 1, 0, 0, SGM_TIE, 1, False),
    SGMCase(2, 37, 31, 0, 0, SGM_TIE, 1, False),
    SGMCase(1, 40, 32, 0, 0, SGM_TIE, 1, False),        # every lane full
    SGMCase(2, 3, 33, 0, 0, SGM_TIE, 2, False),         # W = 3: hpair meets at column 1
    SGMCase(2, 70, 64, 0, 0, SGM_TIE, 2, False),
    SGMCase(1, 2, 65, 0, 0, SGM_TIE, 4, False),         # W = 2: hpair meets at column 1
    SGMCase(2, 131, 127, 0, 0, SGM_TIE, 4, False),
    SGMCase(2, 133, 128, 0, 0, SGM_TIE, 4, True),
    SGMCase(1, 1, 129, 0, 0, SGM_TIE, 8, False),        # W = 1: no hpair, H = 1
    SGMCase(2, 255, 250, 0, 0, SGM_TIE, 8, False),
    SGMCase(2, 261, 256, 0, 0, SGM_TIE, 8, True),       # every lane full
    SGMCase(2, 263, 257, 0, 0, SGM_TIE, 16, False),
    SGMCase(1, 515, 510, 0, 0, SGM_TIE, 16, False),
    SGMCase(2, 517, 512, 0, 0, SGM_TIE, 16, True),      # every lane full
    SGMCase(2, 133, 128, 1, 0, SGM_TIE, 4, False),      # misaligned cost volume: the scalar fallback of a VEC-eligible D
    SGMCase(2, 261, 256, 0, 1, SGM_TIE, 8, False),      # misaligned accumulator
    SGMCase(1, 517, 512, 1, 1, SGM_TIE, 16, False),
    SGMCase(2, 45, 40, 0, 0, SGM_TEN, 2, False),
    SGMCase(2, 137, 132, 0, 0, SGM_TEN, 8, True),
]

SGM_MASKS = (15, 1, 2, 4, 8)


def sgm_id(c):
    return "H%dW%dD%d_off%d.%d_tau%g" % (c.H, c.W, c.D, c.in_off, c.out_off, c.params[2])


def sgm_inputs(c, direction, seed=0):
    """(x0, x1, vol): two (H, W) images and an (H, W, D) cost volume.  Images on a grid of 0.25 (tau_so = 0.25) or of
    1 (tau_so = 10), so |dI| falls below, on and above tau_so, with one NaN pixel each (its differences are the third
    class too).  The volume keeps StereoJoin's NaN triangle (x < d for direction -1, x >= W - d for +1): sgm.cu is
    bit-identical to the reference only where each pixel's valid disparities form a prefix."""
    rng = np.random.default_rng(seed + 1000 * c.D + 7 * c.W + (direction > 0))
    step, levels = (0.25, 5) if c.params[2] < 1 else (1.0, 25)
    x0, x1 = (rng.integers(0, levels, (2, c.H, c.W)) * step).astype(np.float32)
    for x in (x0, x1):
        x[rng.integers(0, c.H), rng.integers(0, c.W)] = np.nan
    vol = (rng.integers(0, 64, (c.H, c.W, c.D)) * 0.125).astype(np.float32)
    d, xs = np.arange(c.D)[None, :], np.arange(c.W)[:, None]
    vol[:, (xs < d) if direction < 0 else (xs >= c.W - d)] = np.nan
    return x0, x1, vol


def mean2d_inputs(c, seed=0):
    """(img, kernel): a quantised image with a few NaN pixels and a random (asymmetric) float32 kernel"""
    rng = np.random.default_rng(seed + c.ksize)
    img = (rng.integers(0, 8, (c.H, c.W)) * 0.25).astype(np.float32)
    img.flat[rng.choice(img.size, 3, replace=False)] = np.nan
    kern = (rng.random((c.ksize, c.ksize)) + 0.05).astype(np.float32)
    return img, kern


def median_image(kind, H, W, seed=0):
    """tied integers; with +-inf; with 10% NaN (and with both); zeros of both signs"""
    rng = np.random.default_rng(seed + 31 * H + W)
    img = rng.integers(0, 4, (H, W)).astype(np.float32)
    if kind == "signed_zero":
        img[rng.random((H, W)) < 0.4] = -0.0
        img[img == 2] = 0.0
    if "inf" in kind:
        img[rng.random((H, W)) < 0.15] = np.inf
        img[rng.random((H, W)) < 0.15] = -np.inf
    if "nan" in kind:
        img[rng.random((H, W)) < 0.1] = np.nan
    return img


MEDIAN_KINDS = ("ties", "inf", "nan", "nan_inf", "signed_zero")
MEDIAN_SHAPES = ((9, 13), (1, 1), (2, 7), (4, 3), (37, 41))    # images smaller than every window, and larger


# ----------------------------------------------------------------------------------------------------- post-processing
M2_TX, M2_TY = 32, 8                                # post.cu mean2d_tile_kernel's tile


def mean2d_regime(ksize):
    """post.cu adcensus_mean2d: the tile kernel when tile + halo + weights fit in 200 KB of shared memory (above 48 KB
    with an opt-in), else the per-pixel kernel"""
    r = ksize // 2
    smem = ((M2_TY + 2 * r) * (M2_TX + 2 * r) + ksize * ksize) * 4
    return "tile" if smem <= 48 * 1024 else "tile_big" if smem <= 200 * 1024 else "pixel"


MEAN2D_REGIMES = ("tile", "tile_big", "pixel")
# H, W, ksize, alpha2, regime: W and H not multiples of the 32 x 8 tile
Mean2dCase = namedtuple("Mean2dCase", "H W ksize alpha2 regime")
MEAN2D_CASES = [
    Mean2dCase(37, 45, 7, 0.5, "tile"),              # alpha2 on a quantisation step: |dI| == alpha2 is common
    Mean2dCase(13, 70, 7, 1e-3, "tile"),             # alpha2 small: equal neighbours only
    Mean2dCase(9, 33, 67, float("inf"), "tile"),     # the largest kernel that fits in 48 KB
    Mean2dCase(21, 50, 69, 0.75, "tile_big"),        # the smallest that does not
    Mean2dCase(19, 41, 71, float("inf"), "tile_big"),
    Mean2dCase(10, 39, 149, 1.0, "tile_big"),        # the largest tile kernel
    Mean2dCase(11, 35, 151, 0.5, "pixel"),           # the smallest per-pixel one
    Mean2dCase(17, 23, 161, float("inf"), "pixel"),
]


def interp_occ_kernel(W):
    """post.cu adcensus_interpolate_occlusion: one block per row when 3 W ints fit in 48 KB, else one thread per pixel"""
    return "row" if 3 * W * 4 <= 48 * 1024 else "pixel"


INTERP_OCC_W = {"row": 4096, "pixel": 4097}


def transpose_kernel(R, Cn, in_off, out_off):
    """post.cu adc_transpose (R x Cn -> Cn x R): (tile, LONGROWS); the 64-tile float4 kernel when R and Cn are multiples
    of 4 and both pointers 16-byte aligned, else the 32-tile one; LONGROWS when R >= Cn"""
    vec = R % 4 == 0 and Cn % 4 == 0 and (4 * in_off) % 16 == 0 and (4 * out_off) % 16 == 0
    return (64 if vec else 32), R >= Cn


def transpose_pitched_vec(D, ld, off):
    """post.cu adc_transpose_dhw_pitched_to_hwd / adc_transpose_hwd_to_dhw_pitched_div4: float4 when D % 4 == 0,
    ld % 4 == 0 and both pointers 16-byte aligned"""
    return D % 4 == 0 and ld % 4 == 0 and (4 * off) % 16 == 0


# D, H, W, off (floats, input and output).  mccnn_transpose_dhw_to_hwd transposes R = D by Cn = H W,
# mccnn_transpose_hwd_to_dhw_div4 the other way round, so each case runs both LONGROWS orientations unless D == H W.
TransposeCase = namedtuple("TransposeCase", "D H W off")
TRANSPOSE_CASES = [
    TransposeCase(8, 4, 8, 0),
    TransposeCase(68, 8, 12, 0),       # two 64-tiles along D
    TransposeCase(128, 3, 4, 0),       # D > H W
    TransposeCase(13, 5, 7, 0),        # D % 4 != 0
    TransposeCase(70, 9, 15, 0),
    TransposeCase(8, 4, 8, 1),         # misaligned
    TransposeCase(128, 3, 4, 2),
]


def median_kernel(ksize):
    """post.cu adcensus_median2d: k = 5 has its own kernel"""
    return "median5" if ksize == 5 else "sort"


MEDIAN_K = (1, 3, 5, 7, 9, 11)
