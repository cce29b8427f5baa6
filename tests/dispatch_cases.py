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


# ----------------------------------------------------------------------------------------------------------------- CBCA
# Exact kernels (cross_cbca.cu): tile (columns, rows) and disparities per CTA
CBCA_EXACT_KERNELS = ("win1", "win4", "loop8", "loop13", "generic")
# constant-work kernels (cbca_tma.cu): cbca_ws_kernel<1, 6>, <4, 4>, cbca_tma_kernel<8>, <13>
CBCA_FAST_KERNELS = ("ws1", "ws4", "tma8", "tma13")
CBCA_TILE = {"win1": (128, 32), "win4": (128, 32), "loop8": (64, 16), "loop13": (64, 16),
             "ws1": (128, 64), "ws4": (128, 64), "tma8": (128, 32), "tma13": (128, 32)}
CBCA_R = {"win1": 1, "win4": 4, "loop8": 8, "loop13": 13, "ws1": 1, "ws4": 4, "tma8": 8, "tma13": 13}


def _by_halo(halo, names):
    return names[0] if halo <= 1 else names[1] if halo <= 4 else names[2] if halo <= 8 else names[3] if halo <= 13 else names[4]


def cbca_gate(maxlen):
    """cross_cbca.cu adcensus_cbca: every candidate kernel is launched with a gate on the longest arm, held on the device
    (win<1> 0-2, win<4> 3-5, loop<8> 6-9, loop<13> 10-14, generic >= 15)"""
    return _by_halo(maxlen - 1, CBCA_EXACT_KERNELS)


def cbca_packed_kernel(max_arm):
    """cross_cbca.cu adc_cbca_packed (adcensus_cbca_ex, mccnn_cbca_packed, the pipeline's exact mode): the caller's bound,
    halo = max_arm - 1: <= 1 win<1>, <= 4 win<4>, <= 8 loop<8>, <= 13 loop<13>, else generic"""
    return _by_halo(max_arm - 1, CBCA_EXACT_KERNELS)


def cbca_ex_clamp(max_arm):
    """cross_cbca.cu adcensus_cbca_ex: the packed arm lengths are cut at max_arm when max_arm <= 14; beyond, the generic
    kernel reads the float arms themselves (no cut).  0 = no cut."""
    return max_arm if max_arm <= 14 else 0


def pack_maxlen(x0c, x1c):
    """cross_cbca.cu pack_arms_kernel: the longest arm length (x - left end, right end - x, y - upper end, lower end - y)
    of either image; 1 << 20 (the generic kernel) when any length is negative, i.e. the arms are not cross() outputs"""
    m = 0
    for xc in (x0c, x1c):
        H, W = xc.shape[1:]
        ys, xs = np.mgrid[0:H, 0:W]
        lens = np.stack([xs - xc[0], xc[1] - xs, ys - xc[2], xc[3] - ys]).astype(np.int64)
        if lens.min() < 0:
            return 1 << 20
        m = max(m, int(lens.max()))
    return m


def clip_arms(xc, bound):
    """the arms adcensus_cbca_ex aggregates over for a stated bound below the real arms: every length cut at `bound`"""
    H, W = xc.shape[1:]
    ys, xs = np.mgrid[0:H, 0:W]
    return np.stack([np.maximum(xc[0], xs - bound), np.minimum(xc[1], xs + bound),
                     np.maximum(xc[2], ys - bound), np.minimum(xc[3], ys + bound)]).astype(np.float32)


def cbca_fast_kernel(max_arm):
    """cbca_tma.cu adc_cbca_fast: halo = max_arm - 1: <= 1 cbca_ws<1>, <= 4 cbca_ws<4>, <= 8 cbca_tma<8>, <= 13
    cbca_tma<13>, otherwise ADCENSUS_ELIMIT"""
    return _by_halo(max_arm - 1, CBCA_FAST_KERNELS + ("ELIMIT",))


def cbca_fast_refusal(W, ld, in_off, out_off, aliased, max_arm):
    """cbca_tma.cu mccnn_cbca_fast_pitched / mccnn_cbca_fast_pitched_packed: EINVAL for vol_in == vol_out, ld < W,
    ld % 4 != 0 or a base not 16-byte aligned; ELIMIT for a halo above 13.  None: the call runs."""
    if aliased or ld < W or ld % 4 or (4 * in_off) % 16 or (4 * out_off) % 16 or max_arm < 1:
        return "EINVAL"
    return "ELIMIT" if max_arm - 1 > 13 else None


def cbca_dchunk(kernel, D):
    """disparities per CTA: launch_win 14, launch_tile 16, launch_tma 20, launch_ws equal chunks of at most 20
    (12 x 19 at D = 228); the generic kernel has no chunks"""
    if kernel in ("ws1", "ws4"):
        return -(-D // -(-D // 20))
    return {"win1": 14, "win4": 14, "loop8": 16, "loop13": 16, "tma8": 20, "tma13": 20}.get(kernel)


def cbca_nproc(x0, d0, dn, W, direction, TX):
    """the planes of a chunk that are aggregated (cbca_win_kernel, cbca_ws_kernel, cbca_tma_kernel: `nproc`; the loop and
    generic kernels copy column by column): a tile whose columns all have x + d * direction
    outside the image is a plain copy (adcensus.cu:353-354), and those planes form a suffix of the chunk"""
    n = 0
    while n < dn and not ((x0 + TX - 1 - (d0 + n) < 0) if direction < 0 else (x0 + d0 + n >= W)):
        n += 1
    return n


def cbca_copy_paths(kernel, D, W, direction):
    """{'whole', 'partial'}: some chunk of some tile column is copied entirely (nproc == 0; cbca_ws copies it before any
    staging) / only after some aggregated planes (0 < nproc < dn)"""
    TX = CBCA_TILE[kernel][0]
    dch = cbca_dchunk(kernel, D)
    out = set()
    for x0 in range(0, W, TX):
        for d0 in range(0, D, dch):
            dn = min(dch, D - d0)
            n = cbca_nproc(x0, d0, dn, W, direction, TX)
            if n == 0:
                out.add("whole")
            elif n < dn:
                out.add("partial")
    return out


def pipe_cbca_route(fast_mode, L1, border, D, W):
    """pipeline.cu run_chain: 'fast' (adc_cbca_fast) when the mode is fast, max(L1, 2) - 1 <= 4 (pipe_fast_cbca_ok) and
    not nan_in_valid; 'generic' (adc_cbca_packed with maxlen 1 << 20) when nan_in_valid = border > 0 and
    D > W - border - 1, in both modes; else 'packed' (the exact kernel of max(L1, 2))"""
    if border > 0 and D > W - border - 1:
        return "generic"
    return "fast" if fast_mode and max(L1, 2) - 1 <= 4 else "packed"


def cbca_image(H, W, L, seed):
    """a blocky quantised image whose cross() arms (tau1 = 0.5, L1 = L) are as long as L along the blocks' long side and
    short across them: the longest arm is exactly L when max(H, W) > L"""
    rng = np.random.default_rng(seed)
    bh, bw = (3, 2 * L + 2) if W > L else (2 * L + 2, 3)
    lv = rng.integers(0, 4, (H // bh + 2, W // bw + 2))
    oy, ox = rng.integers(0, bh), rng.integers(0, bw)
    img = np.kron(lv, np.ones((bh, bw)))[oy:oy + H, ox:ox + W]
    noise = rng.random((H, W)) < 0.05                                     # a few pixels that cut the arms
    img[noise] = rng.integers(0, 4, noise.sum())
    return img.astype(np.float32)


CBCA_TAU1 = 0.5

# H, W, D, L (L1 = the longest arm), direction, entry ('gate' adcensus_cbca, 'ex' adcensus_cbca_ex, 'packed'
# mccnn_pack_arms + mccnn_cbca_packed), max_arm (the stated bound; None for the gate), kernel, and `arms`: 'cross', 'clip'
# (bound below the arms: the expected result aggregates clipped arms) or 'negative' (one arm of negative length)
CbcaCase = namedtuple("CbcaCase", "H W D L direction entry max_arm kernel arms")

# the longest arm on each side of each boundary of the exact tables, and a shape for it (W in {1, 127, 128, 129, 257},
# H in {1, 31, 32, 33, 63, 64, 65}; D below 128 and above, where whole tiles lie in the invalid triangle)
CBCA_EXACT_SHAPES = {
    2: [(33, 129, 20), (1, 257, 150)],
    3: [(31, 127, 15), (65, 1, 9)],
    5: [(64, 128, 30), (32, 257, 150)],
    6: [(63, 129, 17), (1, 127, 40)],
    9: [(65, 128, 33), (33, 257, 131)],
    10: [(32, 127, 16), (64, 1, 5)],
    14: [(31, 129, 18), (1, 257, 135)],
    15: [(33, 128, 14), (65, 33, 40)],
}
CBCA_BOUNDARIES = ((2, 3), (5, 6), (9, 10), (14, 15))


def _cbca_exact_cases():
    cases = []
    for L, shapes in CBCA_EXACT_SHAPES.items():
        for i, (H, W, D) in enumerate(shapes):
            direction = -1 if i == 0 else 1
            k = cbca_packed_kernel(L)
            cases += [CbcaCase(H, W, D, L, direction, "gate", None, k, "cross"),
                      CbcaCase(H, W, D, L, -direction, "gate", None, k, "cross"),
                      CbcaCase(H, W, D, L, direction, "ex", L, k, "cross"),
                      CbcaCase(H, W, D, L, -direction, "packed", L, k, "cross")]
    # a stated bound above the real arms: a bigger kernel for short arms (both host-bound entries)
    for L, bound, (H, W, D) in ((2, 9, (33, 129, 20)), (3, 14, (31, 127, 15)), (6, 20, (63, 129, 17)),
                                (5, 13, (32, 257, 150))):
        for e, direction in (("ex", -1), ("packed", 1)):
            cases.append(CbcaCase(H, W, D, L, direction, e, bound, cbca_packed_kernel(bound), "cross"))
    # a stated bound below the real arms (adcensus_cbca_ex only): the lengths are cut at the bound
    for L, bound, (H, W, D) in ((6, 2, (63, 129, 17)), (9, 5, (65, 128, 33)), (15, 14, (33, 128, 14)),
                                (10, 7, (32, 127, 16))):
        for direction in (-1, 1):
            cases.append(CbcaCase(H, W, D, L, direction, "ex", bound, cbca_packed_kernel(bound), "clip"))
    # arms that are not cross() outputs: one negative length sends adcensus_cbca to the generic kernel
    for direction in (-1, 1):
        cases.append(CbcaCase(31, 129, 18, 5, direction, "gate", None, "generic", "negative"))
    return cases


CBCA_EXACT_CASES = _cbca_exact_cases()


def cbca_id(c):
    b = "" if c.max_arm is None else "_b%d" % c.max_arm
    return "%s_H%dW%dD%d_L%d%s_%s_%+d" % (c.entry, c.H, c.W, c.D, c.L, b, c.arms, c.direction)


def cbca_arms(c, seed=0):
    """(x0c, x1c) the arms case `c` hands to the kernel, and (a0, a1) the arms its expected result aggregates over"""
    from oracle import oracle as orc
    s = seed + 7 * c.H + 3 * c.W + c.L
    x0c = orc.cross(cbca_image(c.H, c.W, c.L, s), c.L, CBCA_TAU1)
    x1c = orc.cross(cbca_image(c.H, c.W, c.L, s + 1), c.L, CBCA_TAU1)
    if c.arms == "negative":
        x0c[0, c.H // 2, c.W // 2] = c.W // 2 + 1                        # left end right of the pixel: length -1
    a0, a1 = x0c, x1c
    if c.arms == "clip":
        a0, a1 = clip_arms(x0c, c.max_arm), clip_arms(x1c, c.max_arm)
    return x0c, x1c, a0, a1


# Constant-work cases: H, W, D, L, direction, max_arm, kernel, ld (row pitch), kind (the volume, see cbca_volume)
FastCase = namedtuple("FastCase", "H W D L direction max_arm kernel ld kind")
CBCA_KINDS = ("stereojoin", "census1", "census3", "ad", "post_sgm", "offset_gradient")


def _cbca_fast_cases():
    cases = []
    # per kernel: the largest arm it serves, and shapes at the tile and chunk edges
    shapes = {
        "ws1": [(64, 128, 20), (65, 129, 21), (1, 257, 228), (33, 1, 40), (63, 127, 41)],
        "ws4": [(64, 257, 228), (31, 128, 20), (65, 129, 40), (32, 127, 21), (1, 129, 41)],
        "tma8": [(32, 129, 20), (33, 257, 150), (63, 128, 21), (1, 127, 40), (64, 1, 41)],
        "tma13": [(33, 128, 20), (31, 257, 160), (65, 129, 41), (32, 127, 21), (1, 129, 40)],
    }
    arm = {"ws1": (2, 2), "ws4": (3, 5), "tma8": (6, 9), "tma13": (10, 14)}
    i = 0
    for k, sh in shapes.items():
        for j, (H, W, D) in enumerate(sh):
            L = arm[k][j % 2]
            direction = -1 if j % 2 == 0 else 1
            ld = (W + 3) // 4 * 4 + (4 if j % 2 else 8)                      # ld > W + 3
            for n in range(2):                                               # two volume kinds per shape
                kind = CBCA_KINDS[(i + n) % len(CBCA_KINDS)]
                if kind == "post_sgm" and H > W:
                    kind = "ad"
                cases.append(FastCase(H, W, D, L, direction if n == 0 else -direction, L, k, ld, kind))
            i += 2
    return cases


CBCA_FAST_CASES = _cbca_fast_cases()


def fast_id(c):
    return "%s_H%dW%dD%d_L%d_ld%d_%s_%+d" % (c.kernel, c.H, c.W, c.D, c.L, c.ld, c.kind, c.direction)


def cbca_volume(kind, H, W, D, direction, seed=0):
    """an (D, H, W) cost volume of `kind` with the NaN triangle (x < d for direction -1, x >= W - d for +1) and a finite
    valid part: StereoJoin of unit features ([-1, 1]); census of quantised images with 1 or 3 channels (0 .. 81); AD of
    the images; a post-SGM volume (sgm2 of a StereoJoin volume, / 4, as main.lua:1017 hands it to cbca_i2); and a large
    common offset (3000) with a steep gradient along x (40 per column), which stresses cancellation in row prefixes"""
    from oracle import oracle as orc
    rng = np.random.default_rng(seed + 17 * H + 5 * W + D + (direction > 0))
    d, xs = np.arange(D)[:, None, None], np.arange(W)[None, None, :]
    tri = (xs < d) if direction < 0 else (xs >= W - d)
    if kind in ("stereojoin", "post_sgm", "offset_gradient"):
        f = rng.standard_normal((2, 8, H, W)).astype(np.float32)
        f /= np.sqrt((f * f).sum(1, keepdims=True))
        vL, vR = orc.stereo_join(f[0], f[1], D)
        vol = vL if direction < 0 else vR
        if kind == "post_sgm":
            img = (rng.integers(0, 16, (2, H, W)) / 8.0).astype(np.float32)
            hwd = orc.sgm2(img[0], img[1], orc.transpose_dhw_to_hwd(vol), 1.32, 24.25, 0.08, 2.0, 3.0, 2.0, direction)
            vol = np.ascontiguousarray(hwd.transpose(2, 0, 1)) / np.float32(4)
        elif kind == "offset_gradient":
            vol = vol + np.float32(3000) + np.float32(40) * np.arange(W, dtype=np.float32)[None, None, :]
    elif kind in ("census1", "census3"):
        nch = 1 if kind == "census1" else 3
        a = (rng.integers(0, 6, (2, nch, H, W)) / 5.0).astype(np.float32)
        vol = orc.census(a[0], a[1], D, direction) if direction < 0 else orc.census(a[1], a[0], D, direction)
    elif kind == "ad":
        a = rng.standard_normal((2, H, W)).astype(np.float32)
        vol = orc.ad(a[0], a[1], D, direction) if direction < 0 else orc.ad(a[1], a[0], D, direction)
    else:
        raise ValueError(kind)
    vol = np.array(vol, np.float32)
    vol[np.broadcast_to(tri, vol.shape)] = np.nan
    return vol


def cbca_f64(x0c, x1c, vol, direction, planes=None):
    """adcensus.cu:343-377 in float64: the tap sums over each output's cross support, as (row runs, then rows); the
    order does not matter at this precision.  Entries with x + d * direction outside the image are copied.  `planes`:
    aggregate only these disparities (the others are copied)."""
    D, H, W = vol.shape
    out = np.array(vol, np.float64)
    ys, xs = np.mgrid[0:H, 0:W]
    v = np.nan_to_num(np.asarray(vol, np.float64), nan=0.0)
    m = int(max(pack_maxlen(x0c, x1c), 1))
    for d in (range(D) if planes is None else planes):
        sh = d * direction
        xp = xs + sh
        ok = (xp >= 0) & (xp < W)
        xpc = np.clip(xp, 0, W - 1)
        lft = np.minimum(xs - x0c[0], xpc - x1c[0][ys, xpc])           # run (x - L, x + R) of row yy, :362-363
        rgt = np.minimum(x0c[1] - xs, x1c[1][ys, xpc] - xpc)
        up = np.minimum(ys - x0c[2], ys - x1c[2][ys, xpc])              # rows (y - U, y + Dn), :359-360
        dn = np.minimum(x0c[3] - ys, x1c[3][ys, xpc] - ys)
        S = np.zeros((H, W))
        C = np.zeros((H, W))
        for dx in range(-m + 1, m):
            inrun = (dx > -lft) & (dx < rgt)
            S += np.where(inrun, np.roll(v[d], -dx, axis=1), 0.0)
            C += inrun
        T = np.zeros((H, W))
        N = np.zeros((H, W))
        for dy in range(-m + 1, m):
            inside = (dy > -up) & (dy < dn)
            T += np.where(inside, np.roll(S, -dy, axis=0), 0.0)
            N += np.where(inside, np.roll(C, -dy, axis=0), 0.0)
        with np.errstate(invalid="ignore", divide="ignore"):
            out[d] = np.where(ok, T / N, out[d])
    return out


# the fast entries' refusals: (W, ld, in_off, out_off, aliased, max_arm) -> expected return code
CBCA_FAST_REFUSALS = [
    (30, 28, 0, 0, False, 5, "EINVAL"),     # ld < W
    (30, 30, 0, 0, False, 5, "EINVAL"),     # ld % 4
    (30, 36, 1, 0, False, 5, "EINVAL"),     # vol_in 4 bytes off
    (30, 36, 0, 2, False, 5, "EINVAL"),     # vol_out 8 bytes off
    (30, 36, 0, 0, True, 5, "EINVAL"),      # vol_in == vol_out
    (30, 36, 0, 0, False, 15, "ELIMIT"),    # halo 14
    (30, 36, 0, 0, False, 14, None),        # halo 13: runs
]


# ------------------------------------------------------------------------------------------------------------ AD / census
AD_TILE, AD_DCH = (128, 8), 8                      # adcensus_cost.cu ad_kernel: 128 x 8 outputs, 8 disparities per CTA
CENSUS_TX, CENSUS_DCH = 128, 16                    # census_cost_kernel: 128 pixels of a row, 16 disparities per CTA


def census_kernel(nch):
    """adcensus_cost.cu adcensus_census: census_cost_kernel<1>, <3>, the runtime-nch <0> for 2 and 4, ELIMIT above 4"""
    return "ELIMIT" if nch > 4 else {1: "nch1", 3: "nch3"}.get(nch, "nch_rt")


# H, W, D, nch, nan (NaN pixels in the images)
AdCensusCase = namedtuple("AdCensusCase", "H W D nch nan")
AD_CENSUS_CASES = [
    AdCensusCase(1, 129, 8, 1, False),        # one row; D = one AD chunk
    AdCensusCase(1, 127, 9, 3, True),
    AdCensusCase(17, 1, 16, 1, True),         # one column; D = one census chunk, D > W
    AdCensusCase(9, 1, 17, 4, False),
    AdCensusCase(10, 128, 16, 4, True),       # the runtime-nch kernel at its limit
    AdCensusCase(9, 255, 17, 2, False),
    AdCensusCase(12, 256, 7, 3, True),
    AdCensusCase(7, 257, 33, 1, True),
    AdCensusCase(8, 383, 24, 4, False),
    AdCensusCase(11, 385, 9, 3, False),
]


def ad_census_images(c, seed=0):
    """(a, b): two (nch, H, W) images on a grid of 1/3 (census ties), with a few NaN pixels when c.nan"""
    rng = np.random.default_rng(seed + c.H * c.W + c.nch + c.D)
    a, b = (np.round(rng.standard_normal((2, c.nch, c.H, c.W)) * 3) / 3).astype(np.float32)
    if c.nan:
        for x in (a, b):
            x.reshape(-1)[rng.choice(x.size, max(1, x.size // 50), replace=False)] = np.nan
    return a, b
