"""Run every launch sized by the SM count on seeded inputs and write the outputs to an .npz (a script, not a test module).

    python tests/sm_count_runs.py OUT.npz [CASE ...]

The process runs under whatever ADCENSUS_NUM_SMS it was started with (DESIGN §4); OUT.npz holds adcensus_num_sms() as
`num_sms` and each output of each case as `<case>/<name>`.  tests/test_gpu_sm_counts.py starts it at several SM counts,
compares every output with the numpy oracles and the runs with each other.  Each case lists its loops as (cap of
tests/map_edge_cases.py's SM_CAPS, launch, elements), so that the test can report which loops wrapped at each SM count."""
import importlib.util
import os
import sys
import tempfile
import zlib
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, synth  # noqa: E402


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mc = _load("map_edge_cases")

KITTI = dataio.Calib(721.5377, 609.5593, 172.854, 387.5744 / 721.5377, 0.0, None, None)
MB = dataio.Calib(1758.23, 829.15, 552.78, 0.178089, 147.24, None, None)
KITTI_P = np.array([[609.6954, -721.5377, -1.2513, -123.0418], [180.3842, 7.6448, -719.6515, -101.0167],
                    [0.9999, 0.0001, 0.0105, -0.2694]])
MB_H, MB_W = 1988, 2964          # a Middlebury full-size map
RAW_H, RAW_W = 512, 1392         # an unrectified KITTI raw image

# name; the family it belongs to; its parameters
Case = namedtuple("Case", "name kind args")


def rng_of(case):
    return np.random.default_rng(zlib.crc32(case.name.encode()))


CASES = [
    # grid8: 2048 s threads; at s = 1 the small cases wrap at least twice and the 1 x 2049 ones by one element
    Case("depth_64x100", "depth", dict(H=64, W=100, cal="kitti")),
    Case("depth_1x2049", "depth", dict(H=1, W=2049, cal="kitti")),
    Case("depth_mb", "depth", dict(H=MB_H, W=MB_W, cal="mb")),
    Case("velo_64x100", "velo", dict(H=64, W=100, n=5000)),
    Case("velo_kitti", "velo", dict(H=375, W=1242, n=120000)),
    Case("render_64x100", "render", dict(H=64, W=100, D=3)),
    Case("render_1x2049", "render", dict(H=1, W=2049, D=2)),
    Case("render_mb", "render", dict(H=MB_H, W=MB_W, D=2)),
    Case("kitti_eval_64x100", "kitti_eval", dict(H=64, W=100)),
    Case("kitti_eval_1x2049", "kitti_eval", dict(H=1, W=2049)),
    Case("kitti_eval_kitti", "kitti_eval", dict(H=375, W=1242)),
    Case("rectify_small", "rectify", dict(raw=(216, 80), rect=(192, 64), nch=1)),
    Case("rectify_raw_grey", "rectify", dict(raw=(RAW_W, RAW_H), rect=(1242, 375), nch=1)),
    Case("rectify_raw_rgb", "rectify", dict(raw=(RAW_W, RAW_H), rect=(1242, 375), nch=3)),
    Case("frontend_64x100", "frontend", dict(H=64, W=100, nch=1)),
    Case("frontend_1x2049", "frontend", dict(H=1, W=2049, nch=3)),
    Case("frontend_kitti_grey", "frontend", dict(H=375, W=1242, nch=1)),
    Case("frontend_kitti_rgb", "frontend", dict(H=375, W=1242, nch=3)),
    # grid16: 4096 s threads
    Case("preprocess_2x17x333", "preprocess", dict(n=2, H=17, W=333)),
    Case("preprocess_1x1x4097", "preprocess", dict(n=1, H=1, W=4097)),
    Case("preprocess_kitti", "preprocess", dict(n=1, H=350, W=1242)),
    Case("preprocess_mb_96x130", "preprocess_mb", dict(H=96, W=130)),
    Case("preprocess_mb_2x8194", "preprocess_mb", dict(H=2, W=8194)),
    Case("preprocess_mb_mb", "preprocess_mb", dict(H=MB_H, W=MB_W)),
    # fill_nan: 16384 s floats; each length at start offsets of 0..3 floats
    Case("fill_nan", "fill_nan", dict(ns=(40000, 16388, 16384, 5))),
    # sel: 1024 s threads, each block over 2048 pixels until the cap binds above 8192 s
    Case("confidence_96x200", "confidence", dict(H=96, W=200)),
    Case("confidence_1x8193", "confidence", dict(H=1, W=8193)),
    Case("confidence_mb", "confidence", dict(H=MB_H, W=MB_W)),
    # resident: s persistent CTAs over 128-pixel tiles
    Case("tower_24_tiles", "tower", dict(nimg=2, H=6, W=140)),
    Case("tower_2_tiles", "tower", dict(nimg=1, H=2, W=128)),
    Case("tower_kitti", "tower", dict(nimg=2, H=375, W=1242)),
    # the maps: merges (grid8) over three frames and more, and the TSDF render's hash build
    Case("fusion_merge", "fusion", dict(H=120, W=160, frames=4, voxel=0.02)),
    Case("tsdf_merge_render", "tsdf", dict(H=48, W=160, frames=3, voxel=0.028, trunc=0.112)),
]


def case(name):
    return next(c for c in CASES if c.name == name)


# ---------------------------------------------------------------------------------------------------------- the inputs

def _specials(rng, a, frac=0.01):
    flat = a.reshape(-1)
    for v in (np.nan, np.inf, -np.inf, 1e38, 2e38):
        flat[rng.random(flat.size) < frac] = v
    return a


def _camera(raw, rect, seed, rot):
    rng = np.random.default_rng(seed)
    (W, H), (Wo, Ho) = raw, rect
    f = 0.8 * max(W, H, 2)
    K = (f, 0.0, W / 2 - 0.3, 0.0, 1.01 * f, H / 2 + 0.2, 0.0, 0.0, 1.0)
    D = tuple(float(v) * (1 + 0.05 * rng.standard_normal()) for v in (-0.3, 0.12, 0.0012, 0.0005, -0.03))
    P = (f, 0.0, Wo / 2 - 0.25, 0.0, 0.0, f, Ho / 2 + 0.5, 0.0, 0.0, 0.0, 1.0, 0.0)
    R = tuple(synth._rodrigues(rot).reshape(-1))
    return dataio.CameraRect(K, D, R, P, (W, H), (Wo, Ho))


def tsdf_case(c):
    a = c.args
    return mc.TsdfCase(c.name, a["H"], a["W"], a["voxel"], a["trunc"], 1, a["frames"], 0.3, 0.95, ())


def inputs(c):
    """the case's seeded inputs, as numpy arrays (and calibrations)"""
    rng, a = rng_of(c), c.args
    if c.kind == "depth":
        cal = KITTI if a["cal"] == "kitti" else MB
        d = rng.uniform(0.5, 200.0, (a["H"], a["W"])).astype(np.float32)
        special = np.array([0.0, -cal.doffs, np.nan, np.inf, -np.inf, -1.0, 1e-30, -cal.doffs + 1e-3], np.float32)
        m = rng.random(d.shape) < 0.1
        d[m] = special[rng.integers(0, len(special), int(m.sum()))]
        return dict(d=d, cal=cal)
    if c.kind == "velo":
        n, H, W = a["n"], a["H"], a["W"]
        r, ang = rng.uniform(1, 80, n), rng.uniform(-np.pi, np.pi, n)
        pts = np.stack([r * np.cos(ang), r * np.sin(ang), rng.uniform(-3, 2, n), rng.uniform(0, 1, n)], 1).astype(np.float32)
        pts = np.concatenate([pts, pts[rng.integers(0, n, n // 10)]])             # exact duplicates: the index breaks ties
        P = KITTI_P.copy()
        P[0, 2] += (W - 1242) / 2
        P[1, 2] += (H - 375) / 2
        return dict(pts=pts[rng.permutation(len(pts))], P=P)
    if c.kind == "render":
        H, W, D = a["H"], a["W"], a["D"]
        vol = rng.integers(0, 6, (D, H, W)).astype(np.float32)
        _specials(rng, vol, 0.02)
        x = _specials(rng, rng.uniform(-5, 84, (H, W)).astype(np.float32))
        jet = rng.uniform(-2.75, 70.75, (H, W)).astype(np.float32)
        jet.reshape(-1)[rng.random(H * W) < 0.05] = 0
        x0 = rng.standard_normal((H, W)).astype(np.float32) * np.float32(1.5)
        gt = rng.uniform(0, 60, (H, W)).astype(np.float32)
        gt[rng.random((H, W)) < 0.3] = 0
        step = rng.choice(np.array([-3.5, -3, -0.3, 0, 3, 3.25, 7], np.float32), (H, W))
        return dict(vol=vol, x=x, jet=jet, x0=x0, pred=(gt + step).astype(np.float32), gt=gt)
    if c.kind == "kitti_eval":
        H, W = a["H"], a["W"]
        disp = rng.uniform(0, 120, (H, W)).astype(np.float32)
        bad = rng.random((H, W)) < 0.3
        bad[H // 2] = True                                                         # a whole invalid row
        kind = rng.integers(0, 3, (H, W))
        disp[bad & (kind == 0)] = 0
        disp[bad & (kind == 1)] = np.nan
        disp[bad & (kind == 2)] = -1
        noc = rng.integers(1, 100 * 256, (H, W)).astype(np.uint16)
        noc[rng.random((H, W)) < 0.3] = 0
        occ = np.where(noc == 0, rng.integers(0, 100 * 256, (H, W)), noc).astype(np.uint16)
        obj = (rng.random((H, W)) < 0.3).astype(np.uint8) * rng.integers(1, 5, (H, W)).astype(np.uint8)
        return dict(disp=disp, noc=noc, occ=occ, obj=obj)
    if c.kind == "rectify":
        (W, H), (Wo, Ho), nch = a["raw"], a["rect"], a["nch"]
        left, right = (_camera((W, H), (Wo, Ho), s, rot) for s, rot in ((1, (0.01, -0.02, 0.005)), (2, (-0.004, 0.01, 0.002))))
        P = list(right.P)
        P[3] = -P[0] * 0.5
        shape = (H, W) if nch == 1 else (H, W, 3)
        views = [rng.integers(0, 256, shape).astype(np.uint8) for _ in range(2)]
        return dict(rect=dataio.StereoRect(left, right._replace(P=tuple(P))), left=views[0], right=views[1])
    if c.kind == "frontend":
        shape = (a["H"], a["W"]) if a["nch"] == 1 else (a["H"], a["W"], 3)
        return dict(left=rng.integers(0, 256, shape, dtype=np.uint8), right=rng.integers(0, 256, shape, dtype=np.uint8))
    if c.kind == "preprocess":
        n, H, W = a["n"], a["H"], a["W"]
        y = (rng.integers(0, 200 * 256, (n, 1, H, W)) / np.float32(256)).astype(np.float32)
        y[rng.random(y.shape) < 0.3] = 0
        y[..., ::7] = np.floor(y[..., ::7] * 4) / 4                                # quarter steps: exact ties
        x0 = rng.standard_normal(y.shape).astype(np.float32)
        x0[rng.random(y.shape) < 0.01] = 255
        return dict(y=y, x0=x0)
    if c.kind == "preprocess_mb":
        H, W = a["H"], a["W"]
        img = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
        d = rng.uniform(0, 300, (H, W)).astype(np.float32)
        d[rng.random(d.shape) < 0.1] = np.inf
        d[rng.random(d.shape) < 0.02] = np.nan
        d0 = rng.uniform(0, min(W, 60), (H, W)).astype(np.float32)
        d0[rng.random(d0.shape) < 0.1] = np.inf
        d1 = (d0 + rng.choice(np.array([0, 0.5, 1, 1.5, 3], np.float32), (H, W))).astype(np.float32)
        dy = rng.uniform(-1.5, 1.5, (H, W)).astype(np.float32)
        return dict(img=img, d=d, d0=d0, d1=d1, dy=dy)
    if c.kind == "fill_nan":
        return dict(ns=a["ns"])
    if c.kind == "confidence":
        H, W = a["H"], a["W"]
        disp = (rng.random((H, W)) * 200).astype(np.float32)
        conf = (rng.integers(0, 50, (H, W)) / 7).astype(np.float32)               # ties
        gt = np.where(rng.random((H, W)) < 0.4, disp + rng.normal(0, 3, (H, W)), 0).astype(np.float32)
        return dict(disp=disp, conf=conf, gt=gt)
    if c.kind == "tower":
        from oracle import tower_head_cases as thc
        layers, x = thc.tower_case(zlib.crc32(c.name.encode()) % 1000, 1, 64, 4, a["nimg"], a["H"], a["W"])
        return dict(layers=layers, x=x)
    if c.kind == "fusion":
        H, W = a["H"], a["W"]
        cal = dataio.Calib(0.58 * W, W / 2 - 0.25, H / 2 + 0.5, synth.POSED_B, 0.0, None, None)
        frames = []
        for k, P in enumerate(synth.posed_camera_poses(a["frames"])):
            Z, _, grey = synth.posed_render(P, H, W, cal.f, cal.cx, cal.cy)
            d = (np.float32(cal.f * cal.baseline) / Z * (1 + 1e-3 * rng.standard_normal(Z.shape))).astype(np.float32)
            d[rng.random(d.shape) < 0.05] = np.nan
            img = np.stack([np.clip(np.rint(grey), 0, 255).astype(np.uint8),
                            rng.integers(0, 256, (H, W), dtype=np.uint8), rng.integers(0, 256, (H, W), dtype=np.uint8)], -1)
            frames.append((d, cal, img, P))
        return dict(frames=frames)
    if c.kind == "tsdf":
        return dict(frames=mc.tsdf_frames(tsdf_case(c)))
    raise ValueError(c.kind)


def map_sizes(c, inp):
    """(the largest unique-key count of one frame, [the table's keys before each frame after the first, and after the
    last]) of a fusion or TSDF case, by the numpy oracle's keys"""
    keys, U, table = np.zeros(0, np.uint64), [], []
    for d, cal, _, P in inp["frames"]:
        if len(keys):
            table.append(len(keys))
        if c.kind == "fusion":
            fo = _load("fusion_oracle")
            fk = np.unique(fo.voxel_keys(fo.world_points(d, cal, P)[0], c.args["voxel"])[0])
        else:
            fk = _load("tsdf_oracle").alloc_keys(d, cal, P, c.args["voxel"], c.args["trunc"])[0]
        U.append(len(fk))
        keys = np.union1d(keys, fk)
    return max(U), table + [len(keys)]


def tower_ntile(a):
    return a["nimg"] * a["H"] * -(-a["W"] // 128)


def loops(c, inp, sizes=None):
    """[(cap, launch, elements)] of the case's capped loops; `sizes` gives the fusion / TSDF case's data sizes (the largest
    unique-key count of a frame, the table before each frame after the first, the table at the end) from the oracle"""
    a = c.args
    if c.kind == "depth":
        return [("grid8", "disp_to_depth", a["H"] * a["W"])]
    if c.kind == "velo":
        return [("grid8", "velo_depth_map points", len(inp["pts"])), ("grid8", "velo_depth_map pixels", a["H"] * a["W"])]
    if c.kind == "render":
        hw = a["H"] * a["W"]
        return [("grid8", k, hw) for k in ("volume_grey", "map_grey", "grey2jet", "error_image")]
    if c.kind == "kitti_eval":
        hw = a["H"] * a["W"]
        return [("grid8", "kitti quantise", hw), ("grid8", "kitti column", hw), ("grid8", "kitti_error_count", hw)]
    if c.kind == "rectify":
        return [("grid8", "rectify", a["rect"][0] * a["rect"][1])]
    if c.kind == "frontend":
        return [("grid8", "frontend normalise", a["H"] * a["W"])]
    if c.kind == "preprocess":
        n = a["n"] * a["H"] * a["W"]
        return [("grid16", "remove_nonvisible", n), ("grid16", "remove_white", n)]
    if c.kind == "preprocess_mb":
        H, W = a["H"], a["W"]
        return [("grid16", "mb half rows", H * (W // 2) * 3), ("grid16", "mb half cols", (H // 2) * (W // 2) * 3),
                ("grid16", "mb half disp", (H // 2) * (W // 2)), ("grid16", "mb mask", H * W)]
    if c.kind == "fill_nan":
        # the float4 body covers the whole float4s after head = (4 - offset) % 4 floats from a 16-byte aligned allocation
        return [("fill_nan", "fill_nan n %d offset %d" % (n, o), (n - min(n, (4 - o) % 4)) // 4 * 4)
                for n in a["ns"] for o in range(4)]
    if c.kind == "confidence":
        hw = a["H"] * a["W"]
        return [("sel", k, hw) for k in ("sparsify write", "sparsification M", "sparsification bad", "select histograms")]
    if c.kind == "tower":
        return [("resident", "resident conv", tower_ntile(a))]
    if c.kind in ("fusion", "tsdf") and sizes:
        U, table = sizes
        return [("grid8", "%s merge_frame" % c.kind, U), ("grid8", "%s merge_table" % c.kind, max(table[:-1]))] + \
            ([("grid8", "tsdf hash_build", table[-1])] if c.kind == "tsdf" else [])
    return []


# --------------------------------------------------------------------------------------------------------- the GPU runs

def run(c, inp, tmp):
    """the case's outputs from the library, as {name: numpy array}"""
    import torch

    from mccnn_b200 import adcensus, confidence, depth, feature_tower, frontend, fusion, kitti_eval, predict_kitti, preprocess, \
        rectify, render

    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    npy = lambda t: t.cpu().numpy()
    a = c.args
    if c.kind == "depth":
        Z, X, Y = depth.depth(cu(inp["d"]), inp["cal"], xy=True)
        return dict(Z=npy(Z), X=npy(X), Y=npy(Y))
    if c.kind == "velo":
        return dict(depth=npy(depth.velo_depth(cu(inp["pts"]), inp["P"].ravel(), a["H"], a["W"], 1e-3)))
    if c.kind == "render":
        path = os.path.join(tmp, c.name + ".bin")
        inp["vol"].astype("<f4").tofile(path)
        return dict(volume_grey=npy(render.volume_file_grey(path, a["D"], a["H"], a["W"])),
                    map_grey=npy(render.map_grey(cu(inp["x"]), 70)),
                    grey2jet=npy(render.grey2jet(cu(inp["jet"]), 70, mask_blue=True)),
                    error_image=npy(render.error_image(cu(inp["x0"]), cu(inp["pred"]), cu(inp["gt"]), 3.0)))
    if c.kind == "kitti_eval":
        ipol = torch.full((a["H"], a["W"]), 7.0, device="cuda")
        got = kitti_eval.devkit_counts(cu(inp["disp"]), inp["noc"], inp["occ"], inp["obj"], ipol=ipol, device=0)
        return dict(ipol=npy(ipol), counts=npy(got.counts), sums=npy(got.sums),
                    error_counts=npy(predict_kitti.error_counts(cu(inp["disp"]), inp["noc"], 3.0)))
    if c.kind == "rectify":
        gl, gr, gv = rectify.rectify(inp["left"], inp["right"], inp["rect"], 0)
        return dict(left=npy(gl), right=npy(gr), valid=npy(gv))
    if c.kind == "frontend":
        return dict(x_batch=npy(frontend.make_batch_cuda(inp["left"], inp["right"], 0)))
    if c.kind == "preprocess":
        nv, w = cu(inp["y"]), cu(inp["y"])
        adcensus.remove_nonvisible(nv)
        adcensus.remove_white(cu(inp["x0"]), w)
        return dict(nonvisible=npy(nv), white=npy(w))
    if c.kind == "preprocess_mb":
        return dict(half_image=npy(preprocess.mb_half_image(cu(inp["img"][None])))[0],
                    half_disp=npy(preprocess.mb_half_disp(cu(inp["d"][None])))[0],
                    mask=npy(preprocess.mb_mask(cu(inp["d0"]), cu(inp["d1"]), cu(inp["dy"]))))
    if c.kind == "fill_nan":
        out = {}
        for n in a["ns"]:
            for o in range(4):
                buf = torch.full((n + 8,), 7.0, device="cuda")
                adcensus.fill_nan(buf[o:o + n])
                out["n%d_offset%d" % (n, o)] = npy(buf)
        return out
    if c.kind == "confidence":
        out = {}
        disp, conf, gt = cu(inp["disp"]), cu(inp["conf"]), cu(inp["gt"])
        for density in (0.5, 1e-7, 1.0):
            out["sparsify_%g" % density] = npy(confidence.sparsify(disp, conf, density, float("nan")))
        M, B, bad = confidence.counts(disp, conf, gt, 3.0)
        out["counts"] = np.array([M, B] + list(bad), np.int64)
        return out
    if c.kind == "tower":
        t = feature_tower.FeatureTower(inp["layers"], arch="fast")
        x = cu(inp["x"].astype(np.float32))
        out = dict(nterms3=npy(t.forward(x)), nterms1=npy(t.forward(x, nterms=1)))
        t.close()
        return out
    if c.kind == "fusion":
        fu = fusion.Fusion(a["voxel"])
        for d, cal, img, pose in inp["frames"]:
            fu.add(cu(d), cal, img, pose)
        t = fu.table()
        out = dict(keys=t.keys, n_pix=t.n_pix, n_frames=t.n_frames, sums=t.sums, colours=t.colours)
        st = fu.stats
        out["stats"] = np.array([st.pixels, st.outside, st.voxels], np.int64)
        for m in (1, 2, 3):
            p = os.path.join(tmp, "%s_m%d.ply" % (c.name, m))
            depth.write_ply(p, fu.cloud(m))
            out["ply_%d" % m] = np.fromfile(p, np.uint8)
        fu.close()
        return out
    if c.kind == "tsdf":
        ts = fusion.TSDF(a["voxel"], a["trunc"])
        for d, cal, img, pose in inp["frames"]:
            ts.add(cu(d), cal, img, pose)
        t = ts.table()
        out = dict(keys=t.keys, S=t.S, n=t.n, nc=t.nc, colours=t.colours)
        st = ts.stats
        out["stats"] = np.array([st.pixels, st.outside, st.bricks], np.int64)
        for m in (1, 2):
            p = os.path.join(tmp, "%s_m%d.ply" % (c.name, m))
            depth.write_mesh_ply(p, ts.mesh(m))
            out["mesh_%d" % m] = np.fromfile(p, np.uint8)
        cal, H, W = render_camera(inp["frames"][0][1], a["H"], a["W"])
        for k, (_, _, _, pose) in enumerate(inp["frames"]):
            out["render_%d" % k] = npy(ts.render(cal, pose, H, W, 1))
        out["render_min2"] = npy(ts.render(cal, inp["frames"][-1][3], H, W, 2))
        ts.close()
        return out
    raise ValueError(c.kind)


def render_camera(cal, H, W):
    """the TSDF case's render camera: half the frame's size, for the numpy render's sake"""
    q = 2
    return dataio.Calib(cal.f / q, (cal.cx + 0.5) / q - 0.5, (cal.cy + 0.5) / q - 0.5, cal.baseline, 0.0, None, None), \
        -(-H // q), -(-W // q)


def main(argv):
    import torch

    from mccnn_b200 import adcensus

    out, names = argv[0], argv[1:] or [c.name for c in CASES]
    torch.cuda.init()
    res = {"num_sms": np.array(adcensus.num_sms(), np.int64)}
    with tempfile.TemporaryDirectory() as tmp:
        for name in names:
            c = case(name)
            for k, v in run(c, inputs(c), tmp).items():
                res["%s/%s" % (name, k)] = np.asarray(v)
            torch.cuda.synchronize()
    np.savez(out, **res)
    print("sm_count_runs: %d cases at %d SMs" % (len(names), int(res["num_sms"])))


if __name__ == "__main__":
    main(sys.argv[1:])
