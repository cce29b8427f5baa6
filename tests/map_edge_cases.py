"""Size rules of the distance field (csrc/tsdf.cu, csrc/keysort.cuh) and the tracker (csrc/track.cu), restated in Python,
and the cases of tests/test_gpu_map_edges.py.

Both layers launch kernels whose shape follows the frame: the field's allocation runs over m = H W (2K + 1) ray points in
blocks of 2048, scans the block counts on 1024 threads and walks the table with grid-stride loops capped at 8 blocks per SM;
the tracker reduces each pyramid level in chunks of 1024 pixels and the chunk sums padded to a power of two.  Each rule
below restates one of these next to the C it restates, and every case names the edges it is meant to hit.
tests/test_map_edge_cases.py checks, without a GPU, that each case hits what it claims, that the lists reach every edge,
and that the tracker's sums are order-sensitive on the cases' data; the GPU test runs each case against the numpy oracles
bit for bit."""
import math
from collections import namedtuple

import numpy as np

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, synth

# ------------------------------------------------------------------------------------------------- the distance field

THREADS = 256                    # keysort.cuh THREADS
ITEMS = 8                        # keysort.cuh ITEMS
CHUNK = THREADS * ITEMS          # keysort.cuh CHUNK: allocation points per block
SCAN_THREADS = 1024              # keysort.cuh SCAN_THREADS
MAX_K = 64                       # tsdf.cu mccnn_tsdf_create: K > 64 is ADCENSUS_ELIMIT
H100_SMS = (132, 114)            # H100 SXM, H100 PCIe


def K_of(voxel, trunc):
    """tsdf.cu mccnn_tsdf_create: K = ceil(trunc / (4 v)) in float64"""
    return int(math.ceil(float(trunc) / (4.0 * float(voxel))))


def points(H, W, K):
    """tsdf.cu run_add: m = H W J allocation points, J = 2K + 1 per pixel"""
    return H * W * (2 * K + 1)


def nblk(m):
    """tsdf.cu run_add: the blocks of alloc_count / alloc_fill / head_* / match_*, and the block counts scan_kernel adds up"""
    return -(-m // CHUNK)


def scan_per(n):
    """keysort.cuh scan_kernel: the block counts each of its 1024 threads adds up in a run"""
    return -(-n // SCAN_THREADS)


def grid_for(n, sms):
    """keysort.cuh grid_for: ceil(n / 256) blocks of 256 threads, at least 1, at most 8 per SM"""
    return max(1, min(-(-n // THREADS), sms * 8))


def grid_cap(sms):
    """the threads of grid_for's largest grid (270,336 on 132 SMs): a grid-stride loop over more elements wraps"""
    return sms * 8 * THREADS


def wraps(n, sms):
    return n > grid_for(n, sms) * THREADS


def hash_bits(n):
    """tsdf.cu mccnn_tsdf_render: the render's hash table has 2^bits slots, bits >= 10 and 2^bits >= 2 n"""
    bits = 10
    while (1 << bits) < 2 * n:
        bits += 1
    return bits


# ------------------------------------------------------------------------------------------ launches sized by the SM count
#
# Every grid that follows the SM count s (adc_num_sms, csrc/common.cu) is capped at a multiple of s, and the kernel covers
# the rest of its work with a grid-stride or persistent loop.  One row per cap: the C expression it restates, the blocks it
# launches, the elements one pass of the grid covers, and the launches it sizes.  tests/test_map_edge_cases.py checks the
# rows against every use of adc_num_sms in csrc/; tests/test_gpu_sm_counts.py runs each launch at forced SM counts.

def grid16(n, sms):
    """preprocess.cu / preprocess_mb.cu elementwise_grid: ceil(n / 256) blocks, at most 16 per SM"""
    return min(-(-n // THREADS), sms * 16)


def fill_nan_blocks(n, sms):
    """post.cu mccnn_fill_nan: the float4 body's blocks for n floats from a 16-byte aligned start, at least 1, at most 16 per SM"""
    return max(1, min(-(-(n // 4) // THREADS), sms * 16))


SEL_THREADS = 256                # confidence.cu SEL_THREADS


def sel_blocks(n, sms):
    """confidence.cu sel_blocks: ceil(n / 2048) blocks, at least 1, at most 4 per SM"""
    return max(1, min(-(-n // (SEL_THREADS * 8)), sms * 4))


def resident_ctas(ntile, sms):
    """feature_tower.cu: the resident conv's persistent CTAs, one per SM at most; each runs ceil(ntile / CTAs) tiles"""
    return min(ntile, sms)


# name; blocks(n, s); the elements one block covers in one pass; the elements per block of the uncapped grid; the (csrc
# file, sizing-line regex) of each use of adc_num_sms the row restates; the launches it sizes, as (file, kernel)
SmCap = namedtuple("SmCap", "name blocks per_block uncapped sites launches")

SM_CAPS = [
    SmCap("grid8", grid_for, THREADS, THREADS,
          [("keysort.cuh", r"long grid_for\(long long n\).*adc_num_sms\(\) \* 8"),
           ("depth.cu", r"long grid_for\(long n\).*adc_num_sms\(\) \* 8"),
           ("render.cu", r"long grid_for\(long n\).*adc_num_sms\(\) \* 8"),
           ("kitti_eval.cu", r"long grid_for\(long n\).*adc_num_sms\(\) \* 8"),
           ("rectify.cu", r"const int grid = .*adc_num_sms\(\) \* 8"),
           ("frontend.cu", r"const dim3 grid\(.*adc_num_sms\(\) \* 8\), 2\)"),
           ("frontend.cu", r"const int grid = .*adc_num_sms\(\) \* 8")],
          [("fusion.cu", "merge_table_kernel"), ("fusion.cu", "merge_frame_kernel"), ("tsdf.cu", "merge_table_kernel"),
           ("tsdf.cu", "merge_frame_kernel"), ("tsdf.cu", "hash_build_kernel"),
           ("depth.cu", "depth_kernel"), ("depth.cu", "velo_key_kernel"), ("depth.cu", "velo_decode_kernel"),
           ("render.cu", "volume_grey_kernel"), ("render.cu", "map_grey_kernel"), ("render.cu", "jet_kernel"),
           ("render.cu", "error_kernel"), ("kitti_eval.cu", "quantise_kernel"), ("kitti_eval.cu", "column_kernel"),
           ("rectify.cu", "rectify_kernel"), ("frontend.cu", "normalise_kernel"), ("frontend.cu", "error_count_kernel")]),
    SmCap("grid16", grid16, THREADS, THREADS,
          [("preprocess.cu", r"int elementwise_grid\(size_t n\).*adc_num_sms\(\) \* 16"),
           ("preprocess_mb.cu", r"int elementwise_grid\(long n\).*adc_num_sms\(\) \* 16")],
          [("preprocess.cu", "nonvisible_kernel"), ("preprocess.cu", "white_kernel"), ("preprocess_mb.cu", "half_rows_kernel"),
           ("preprocess_mb.cu", "half_cols_kernel"), ("preprocess_mb.cu", "half_disp_kernel"),
           ("preprocess_mb.cu", "mask_kernel")]),
    SmCap("fill_nan", fill_nan_blocks, 4 * THREADS, 4 * THREADS,
          [("post.cu", r"int cap = adc_num_sms\(\) \* 16;")],
          [("post.cu", "fill_nan_kernel")]),
    SmCap("sel", sel_blocks, SEL_THREADS, 8 * SEL_THREADS,
          [("confidence.cu", r"const long cap = \(long\)adc_num_sms\(\) \* 4;")],
          [("confidence.cu", "sparsify_write_kernel"), ("confidence.cu", "counts_mb_kernel"),
           ("confidence.cu", "counts_bad_kernel"), ("confidence.cu", "sel_hist_kernel")]),
    SmCap("resident", resident_ctas, 1, 1,
          [("feature_tower.cu", r"const int nb = ntile < adc_num_sms\(\) \? ntile : adc_num_sms\(\);")],
          [("feature_tower.cu", "conv3x3_resident_kernel")]),
]

# launches whose grids do not follow the SM count: mb_eval.cu sizes its grids from the pixel count, track.cu from the
# pyramid's chunks
SM_FREE = ("mb_eval.cu", "track.cu")


def sm_cap(name):
    return next(c for c in SM_CAPS if c.name == name)


def sm_passes(cap, n, s):
    """the passes of cap's grid-stride (or persistent) loop over n elements (tiles for the resident conv) at s SMs: above 1
    the loop wraps"""
    c = sm_cap(cap)
    return max(1, -(-n // (c.blocks(n, s) * c.per_block)))


def sm_cap_elements(cap, s):
    """the most elements at which cap's grid is still the uncapped one at s SMs: with one more the cap binds, and the loop
    takes one more pass (the selection's blocks loop over 2048 pixels each before the cap binds)"""
    c = sm_cap(cap)
    return c.blocks(1 << 40, s) * c.uncapped


# the KITTI-like camera of the full-size cases (2011_09_26's rectified left camera), and a proportional one otherwise
KITTI_H, KITTI_W = 375, 1242


def calib(H, W):
    if (H, W) == (KITTI_H, KITTI_W):
        return dataio.Calib(721.5377, 609.5593, 172.854, synth.POSED_B, 0.0, None, None)
    return dataio.Calib(0.58 * W, W / 2 - 0.25, H / 2 + 0.5, synth.POSED_B, 0.0, None, None)


# name; frame size; voxel and trunc (metres); image channels; the pose of each frame (steps of posed_camera_poses, then a
# translation of every frame after the first); the share of pixels with a depth; the edges the case claims
TsdfCase = namedtuple("TsdfCase", "name H W voxel trunc nch frames shift valid edges")


def _trunc_above(x):
    return float(np.nextafter(x, np.inf))


TSDF_CASES = [
    TsdfCase("m_multiple", 32, 64, 0.1, 0.4, 1, 2, 0.0, 0.95, ("m % 2048 == 0", "grey")),
    TsdfCase("m_plus_column", 32, 65, 0.1, 0.4, 3, 2, 0.0, 0.95, ("partial last block", "rgb")),
    TsdfCase("one_pixel", 1, 1, 0.1, 0.4, 1, 2, 0.0, 1.0, ("1x1",)),
    TsdfCase("kitti_K2", KITTI_H, KITTI_W, 0.1, 0.8, 1, 2, 0.0, 0.95,
             ("nblk > 1024", "scan per > 1", "K = 2", "hash bits > 10", "grey")),
    TsdfCase("kitti_K2_rgb", KITTI_H, KITTI_W, 0.1, 0.8, 3, 2, 0.0, 0.95, ("nblk > 1024", "scan per > 1", "rgb")),
    TsdfCase("K64", 96, 320, 0.125, 256 * 0.125, 1, 2, 0.0, 1.0,
             ("K = 64", "nblk > 1024", "scan per > 1", "hash bits > 10")),
    # fine voxels: about one brick per pixel, and the second frame 2 m to the side, so that the first frame's unique keys,
    # the table it leaves and the second frame's unique keys are all above grid_for's cap on both H100s
    TsdfCase("grid_wrap", KITTI_H, KITTI_W, 0.003, 0.012, 1, 2, 2.0, 1.0,
             ("U > grid cap", "table > grid cap", "hash bits > 10")),
]
# trunc = 256 v is the largest accepted; the next double above it is refused with ADCENSUS_ELIMIT before any allocation
K65 = (0.125, _trunc_above(256 * 0.125))


def tsdf_frames(case, seed=0):
    """[(disparity float32 (H, W), cal, image uint8 (H, W) or (H, W, 3), 4x4 pose)] of the case: exact disparities of the
    posed planes with a small multiplicative noise, (1 - valid) of the pixels NaN"""
    rng = np.random.default_rng(seed)
    cal = calib(case.H, case.W)
    out = []
    for k, P in enumerate(synth.posed_camera_poses(case.frames)):
        P = P.copy()
        if k:
            P[0, 3] += case.shift
        Z, _, grey = synth.posed_render(P, case.H, case.W, cal.f, cal.cx, cal.cy)
        d = (np.float32(cal.f * cal.baseline) / Z * (1 + 1e-4 * rng.standard_normal(Z.shape))).astype(np.float32)
        d[rng.random(d.shape) >= case.valid] = np.nan
        img = np.clip(np.rint(grey), 0, 255).astype(np.uint8)
        if case.nch == 3:
            img = np.stack([img, rng.integers(0, 256, img.shape, dtype=np.uint8), 255 - img], -1)
        out.append((d, cal, img, P))
    return out


def tsdf_size_edges(case):
    """the edges of a case that follow from its sizes alone"""
    K = K_of(case.voxel, case.trunc)
    m = points(case.H, case.W, K)
    e = {"K = %d" % K, "grey" if case.nch == 1 else "rgb"}
    if m % CHUNK == 0:
        e.add("m % 2048 == 0")
    else:
        e.add("partial last block")
    if (case.H, case.W) == (1, 1):
        e.add("1x1")
    if nblk(m) > SCAN_THREADS:
        e.add("nblk > 1024")
    if scan_per(nblk(m)) > 1:
        e.add("scan per > 1")
    return e


def tsdf_data_edges(U, table, sms):
    """the edges that follow from the data: U the largest unique-key count of one frame, `table` the brick counts the
    table holds before each frame after the first, and after the last"""
    e = set()
    if wraps(U, sms):
        e.add("U > grid cap")                     # merge_frame_kernel, launched on grid_for(m) >= grid_for(U)
    if any(wraps(n, sms) for n in table[:-1]):
        e.add("table > grid cap")                 # merge_table_kernel over the table's bricks
    if hash_bits(table[-1]) > 10:
        e.add("hash bits > 10")
    return e


# every edge the TSDF cases must reach between them
TSDF_EDGES = {"m % 2048 == 0", "partial last block", "1x1", "nblk > 1024", "scan per > 1", "K = 64", "grey", "rgb",
              "U > grid cap", "table > grid cap", "hash bits > 10"}

# ---------------------------------------------------------------------------------------------------------- the tracker

LEVELS = 3                       # MCCNN_TRACK_LEVELS
TRACK_CH = 1024                  # track.cu CH: pixels per chunk


def level_shape(H, W, l):
    """track.cu mccnn_track_create: h_l = ceil(H / 2^l), w_l = ceil(W / 2^l)"""
    return -(-H // (1 << l)), -(-W // (1 << l))


def chunks(H, W, l):
    """track.cu mccnn_track_step: n_l chunks of 1024 pixels, one block each"""
    h, w = level_shape(H, W, l)
    return -(-(h * w) // TRACK_CH)


def pad(n):
    """track.cu mccnn_track_step: P_l, the chunk sums padded with +0.0 to a power of two"""
    P = 1
    while P < n:
        P <<= 1
    return P


def last_chunk(H, W, l):
    """the pixels of level l's last chunk: threads beyond them have none"""
    h, w = level_shape(H, W, l)
    return h * w - (chunks(H, W, l) - 1) * TRACK_CH


def normal_sites(H, W, l):
    """track.cu normal_kernel: a normal needs the pixel's right and lower neighbours"""
    h, w = level_shape(H, W, l)
    return (h - 1) * (w - 1)


def photo_sites(H, W, l):
    """track.cu photo_term: 1 <= x0 and x0 + 1 <= w_l - 2 (likewise y), so w_l and h_l of at least 4"""
    h, w = level_shape(H, W, l)
    return max(0, w - 3) * max(0, h - 3)


TrackCase = namedtuple("TrackCase", "name H W nch edges")

TRACK_CASES = [
    TrackCase("kitti", KITTI_H, KITTI_W, 1, ("n = 455/115/29", "P = 512/128/32", "last chunk 854", "last chunk 12", "last chunk 562")),
    TrackCase("kitti_rgb", KITTI_H, KITTI_W, 3, ("n = 455/115/29", "rgb")),
    TrackCase("pow2", 64, 128, 1, ("n = P at level 0", "n = P at level 1")),
    TrackCase("pad_most", 96, 352, 1, ("n = P/2 + 1 at level 0",)),
    TrackCase("one_chunk", 32, 32, 1, ("one full chunk",)),
    TrackCase("one_pixel", 1, 1, 1, ("no normals",)),
    TrackCase("one_row", 1, 77, 1, ("no normals",)),
    TrackCase("one_column", 45, 1, 3, ("no normals",)),
    # the issue-style 3 x 7 has normals at levels 0 and 1 (2 x 4 keeps three sites); 2 x 7 has them at level 0 only
    TrackCase("tiny", 3, 7, 1, ("normals at level 0 only in part", "no photometric pixel")),
    TrackCase("tiny_flat", 2, 7, 1, ("normals at level 0 only",)),
    TrackCase("narrow", 40, 12, 1, ("no photometric pixel at level 2",)),
]


def track_edges(case):
    """the edges a tracker case reaches, from its size"""
    H, W = case.H, case.W
    n = [chunks(H, W, l) for l in range(LEVELS)]
    P = [pad(x) for x in n]
    e = {"rgb"} if case.nch == 3 else set()
    e.add("n = %s" % "/".join(map(str, n)))
    e.add("P = %s" % "/".join(map(str, P)))
    for l in range(LEVELS):
        if n[l] == P[l] and n[l] > 1:
            e.add("n = P at level %d" % l)
        if n[l] > 1 and n[l] == P[l] // 2 + 1:
            e.add("n = P/2 + 1 at level %d" % l)
        e.add("last chunk %d" % last_chunk(H, W, l))
    if n == [1, 1, 1] and level_shape(H, W, 0)[0] * level_shape(H, W, 0)[1] == TRACK_CH:
        e.add("one full chunk")
    sites = [normal_sites(H, W, l) for l in range(LEVELS)]
    if not any(sites):
        e.add("no normals")
    if sites[0] and not sites[1] and not sites[2]:
        e.add("normals at level 0 only")
    if sites[0] and sites[1] and not sites[2]:
        e.add("normals at level 0 only in part")
    photo = [photo_sites(H, W, l) for l in range(LEVELS)]
    if not any(photo):
        e.add("no photometric pixel")
    elif not photo[2]:
        e.add("no photometric pixel at level 2")
    return e


TRACK_EDGES = {"n = 455/115/29", "P = 512/128/32", "last chunk 12", "n = P at level 0", "n = P at level 1",
               "n = P/2 + 1 at level 0", "one full chunk", "no normals", "normals at level 0 only",
               "no photometric pixel", "no photometric pixel at level 2", "rgb"}


def track_frame(case, seed=0):
    """(cal, source disparity of posed frame 2, model depth of frame 1, frame 2's image, frame 1's image, the relative pose
    frame 2 -> frame 1): exact values with a small multiplicative noise, 8% holes in each map when the frame is large"""
    rng = np.random.default_rng(seed)
    H, W = case.H, case.W
    cal = calib(H, W)
    poses = synth.posed_camera_poses(3)
    Z2, _, g2 = synth.posed_render(poses[2], H, W, cal.f, cal.cx, cal.cy)
    Z1, _, g1 = synth.posed_render(poses[1], H, W, cal.f, cal.cx, cal.cy)
    holes = 0.08 if H * W >= 1024 else 0.0
    disp = (np.float32(cal.f * cal.baseline) / Z2 * (1 + 1e-4 * rng.standard_normal(Z2.shape))).astype(np.float32)
    disp[rng.random(disp.shape) < holes] = np.nan
    Zm = (Z1 * (1 + 1e-4 * rng.standard_normal(Z1.shape))).astype(np.float32)
    Zm[rng.random(Zm.shape) < holes] = np.nan
    Zm[~np.isfinite(Zm)] = np.nan
    imgs = []
    for g in (g2, g1):
        b = np.clip(np.rint(g), 0, 255).astype(np.uint8)
        if case.nch == 3:
            b = np.stack([b, rng.integers(0, 256, b.shape, dtype=np.uint8), 255 - b], -1)
        imgs.append(b)
    return cal, disp, Zm, imgs[0], imgs[1], np.linalg.inv(poses[1]) @ poses[2]


def track_poses(T_true, rng):
    """the relative poses each case steps at: the true one, and two off by up to 1 degree and 5 cm"""
    out = [T_true]
    for k in (1, 2):
        ax, dr = rng.standard_normal(3), rng.standard_normal(3)
        M = np.eye(4)
        M[:3, :3] = _rodrigues(math.radians(0.5 * k) * ax / np.linalg.norm(ax))
        M[:3, 3] = 0.025 * k * dr / np.linalg.norm(dr)
        out.append(T_true @ M)
    return out


def _rodrigues(w):
    th = float(np.linalg.norm(w))
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / th
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * (K @ K)


# the product-shaped drive: 3 frames at 375 x 1242 tracked with and without the photometric term
DRIVE = dict(n=3, H=KITTI_H, W=KITTI_W, voxel=0.2, trunc=0.8, max_depth=30.0)


def case_id(c):
    return c.name
