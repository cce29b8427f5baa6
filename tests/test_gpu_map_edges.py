"""GPU: the distance field (DESIGN §24) and the tracker (§25, §26) at full KITTI frames and at every chunk, scan and
grid-stride edge of tests/map_edge_cases.py, bit for bit against the numpy oracles (tests/tsdf_oracle.py,
tests/track_oracle.py, tests/track_photometric_oracle.py): the field's table, stats, mesh PLY bytes and renders; a table
whose grid-stride loops wrap, by its whole key array and sampled bricks; K = 64 run and K = 65 refused; the tracker's
vertex, normal and intensity pyramids, sums and counts at every level with and without gates; and a 3-frame drive at
375 x 1242 tracked with and without the photometric term."""
import ctypes
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, depth, fusion, synth, track  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mc = _load("map_edge_cases", "tests", "map_edge_cases.py")
to = _load("tsdf_oracle", "tests", "tsdf_oracle.py")
po = _load("track_photometric_oracle", "tests", "track_photometric_oracle.py")
tro = po.track_oracle
COS30 = math.cos(math.radians(30.0))
GATES = (2.0, 30.0)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def png(path):
    from PIL import Image

    with Image.open(path) as im:
        return np.array(im)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def same_bits(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, what
    assert np.array_equal(np.isnan(a), np.isnan(b)), "%s: NaN patterns differ" % what
    assert np.array_equal(a.view(np.uint64)[~np.isnan(a)], b.view(np.uint64)[~np.isnan(b)]), "%s: values differ" % what


# ------------------------------------------------------------------------------------------------- the distance field

def same_table(ts, ref, what):
    t = ts.table()
    assert np.array_equal(t.keys, ref.keys), "%s: keys differ (%d vs %d bricks)" % (what, len(t.keys), len(ref.keys))
    bad = t.S.reshape(-1, 512).view(np.uint64) != ref.S.view(np.uint64)
    assert not bad.any(), "%s: %d float64 S differ" % (what, int(bad.sum()))
    assert np.array_equal(t.n.reshape(-1, 512), ref.n), "%s: n" % what
    assert np.array_equal(t.nc.reshape(-1, 512), ref.nc), "%s: nc" % what
    assert np.array_equal(t.colours.reshape(-1, 512, 3), ref.col), "%s: colour sums" % what
    st = ts.stats
    assert (st.pixels, st.outside, st.bricks) == (ref.pixels, ref.outside, len(ref.keys)), what


def same_render(ts, ref, cal, pose, H, W, what, min_frames=1):
    got = ts.render(cal, pose, H, W, min_frames).cpu().numpy()
    want = ref.render(cal, pose, H, W, min_frames)
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: hit pixels differ" % what
    assert np.array_equal(got.view(np.uint32)[~np.isnan(got)], want.view(np.uint32)[~np.isnan(want)]), "%s: depths differ" % what
    return int(np.isfinite(want).sum())


def render_camera(cal, H, W):
    """the case's camera, or for frames above 10,000 pixels the same view at a quarter of the size: the numpy render
    marches every pixel through the field, and the render's edges are the table's, not the image's"""
    if H * W <= 10000:
        return cal, H, W
    q = 4
    return dataio.Calib(cal.f / q, (cal.cx + 0.5) / q - 0.5, (cal.cy + 0.5) / q - 0.5, cal.baseline, 0.0, None, None), \
        -(-H // q), -(-W // q)


@pytest.mark.parametrize("case", [c for c in mc.TSDF_CASES if c.name != "grid_wrap"], ids=mc.case_id)
def test_field_is_the_oracle(case, tmp_path):
    frames = mc.tsdf_frames(case)
    ts, ref = fusion.TSDF(case.voxel, case.trunc), to.Field(case.voxel, case.trunc)
    assert mc.K_of(case.voxel, case.trunc) == to.K_of(case.voxel, case.trunc)
    for k, (d, cal, img, P) in enumerate(frames):
        ts.add(cu(d), cal, img, P)
        ref.add(d, cal, img, P)
        same_table(ts, ref, "%s frame %d" % (case.name, k))
    if "hash bits > 10" in case.edges:
        assert mc.hash_bits(len(ref.keys)) > 10
    if len(ref.keys) <= 5000:                     # the oracle's mesh keeps 36 int64 slots per voxel
        for m in (1, 2):
            p = str(tmp_path / ("m%d.ply" % m))
            depth.write_mesh_ply(p, ts.mesh(m))
            assert open(p, "rb").read() == ref.mesh_ply(m), "%s: mesh PLY bytes differ at min_frames %d" % (case.name, m)
    rc, rh, rw = render_camera(frames[0][1], case.H, case.W)
    # a table of more than 5000 bricks (K = 64) is rendered once: the numpy render takes most of a minute there
    few = len(ref.keys) <= 5000
    hits = [same_render(ts, ref, rc, P, rh, rw, "%s render at pose %d" % (case.name, k))
            for k, (_, _, _, P) in enumerate(frames) if few or k == len(frames) - 1]
    if few:
        hits.append(same_render(ts, ref, rc, frames[-1][3], rh, rw, "%s render min_frames 2" % case.name, 2))
    print("%s: %d bricks, render hits %s of %d pixels" % (case.name, len(ref.keys), hits, rh * rw))
    if case.H * case.W > 1000:
        assert max(hits) > 0, "%s: the renders hit nothing" % case.name
    ts.close()


def test_k65_is_refused_before_any_allocation():
    lib = adcensus.lib()
    h = ctypes.c_void_p()
    voxel, trunc = mc.K65
    assert mc.K_of(voxel, trunc) == 65 and mc.K_of(voxel, 256 * voxel) == 64
    free0 = torch.cuda.mem_get_info()[0]
    assert lib.mccnn_tsdf_create(ctypes.byref(h), voxel, trunc, 0) == -2 and not h.value
    assert torch.cuda.mem_get_info()[0] == free0
    assert lib.mccnn_tsdf_create(ctypes.byref(h), voxel, 256 * voxel, 0) == 0 and h.value
    lib.mccnn_tsdf_destroy(h)
    with pytest.raises(ValueError, match="256 voxel"):
        fusion.TSDF(voxel, trunc)


def test_grid_stride_loops_wrap():
    """fine voxels on two 375 x 1242 frames 2 m apart: both frames' unique keys and the table the first leaves are above
    grid_for's cap on this device, so merge_frame_kernel and merge_table_kernel walk their grid-stride loops more than
    once.  The whole key array and the stats against the oracle's allocation; the voxels of the first and last bricks,
    those around the cap and 3000 random ones against the oracle's per-voxel rule"""
    case = next(c for c in mc.TSDF_CASES if c.name == "grid_wrap")
    n_sm = sms()
    cap = mc.grid_cap(n_sm)
    frames = mc.tsdf_frames(case)
    ts = fusion.TSDF(case.voxel, case.trunc)
    keys, tables, U, pixels, outside = np.zeros(0, np.uint64), [], [], 0, 0
    for d, cal, img, P in frames:
        before = len(keys)
        fk, pix, out = to.alloc_keys(d, cal, P, case.voxel, case.trunc)
        U.append(len(fk))
        pixels, outside = pixels + pix, outside + out
        keys = np.union1d(keys, fk).astype(np.uint64)
        tables.append(keys)
        ts.add(cu(d), cal, img, P)
        assert ts.stats.bricks == len(keys)
        if before:
            assert mc.wraps(before, n_sm), "the table before frame 2 (%d bricks) does not wrap at %d SMs" % (before, n_sm)
    print("grid_wrap on %d SMs (cap %d threads): U %s, table %d bricks, %.0fM voxels" % (n_sm, cap, U, len(keys),
                                                                                          len(keys) * 512 / 1e6))
    assert all(mc.wraps(u, n_sm) for u in U), (U, cap)
    st = ts.stats
    assert (st.pixels, st.outside, st.bricks) == (pixels, outside, len(keys))
    b = len(keys)
    h, lib = ts._handle(), adcensus.lib()
    dev = torch.device("cuda", 0)
    tk = torch.empty(b, dtype=torch.int64, device=dev)
    S = torch.empty((b, 512), dtype=torch.float64, device=dev)
    n, nc = (torch.empty((b, 512), dtype=torch.int32, device=dev) for _ in range(2))
    col = torch.empty((b, 512, 3), dtype=torch.int32, device=dev)
    assert lib.mccnn_tsdf_table(h, tk.data_ptr(), S.data_ptr(), n.data_ptr(), nc.data_ptr(), col.data_ptr(),
                                torch.cuda.current_stream().cuda_stream) == 0
    assert np.array_equal(tk.cpu().numpy().view(np.uint64), keys), "keys differ"
    rng = np.random.default_rng(0)
    pick = set(range(3)) | set(range(b - 3, b)) | set(range(max(0, cap - 4), min(b, cap + 4)))
    pick |= set(rng.choice(b, 3000, replace=False).tolist())
    idx = np.array(sorted(pick))
    ref = to.sampled_bricks(keys[idx], frames, tables, case.voxel, case.trunc)
    ti = torch.from_numpy(idx).to(dev)
    got_S = S.index_select(0, ti).cpu().numpy()
    assert np.array_equal(got_S.view(np.uint64), ref.S.view(np.uint64)), "S of sampled bricks"
    assert np.array_equal(n.index_select(0, ti).cpu().numpy(), ref.n), "n of sampled bricks"
    assert np.array_equal(nc.index_select(0, ti).cpu().numpy(), ref.nc), "nc of sampled bricks"
    assert np.array_equal(col.index_select(0, ti).cpu().numpy(), ref.col), "colour sums of sampled bricks"
    assert (ref.n > 0).sum() > 1000
    del tk, S, n, nc, col
    ts.close()


# ---------------------------------------------------------------------------------------------------------- the tracker

@pytest.mark.parametrize("case", mc.TRACK_CASES, ids=mc.case_id)
def test_tracker_is_the_oracle(case):
    H, W = case.H, case.W
    cal, disp, Zm, img, ref_img, T_true = mc.track_frame(case)
    src, mod = tro.source_pyramid(disp, cal), tro.model_pyramid(Zm, cal)
    isrc, iref = po.pyramid(img), po.pyramid(ref_img)
    edges = mc.track_edges(case)
    with track.Tracker(H, W) as tr:
        tr.source(cu(disp), cal)
        tr.model(cu(Zm), cal)
        tr.intensity("source", img)
        tr.intensity("reference", ref_img)
        for level in range(mc.LEVELS):
            for which, ref in (("source", src), ("model", mod)):
                V, N = tr.maps(which, level)
                same_bits(V, ref[level][0], "%s %s level %d vertices" % (case.name, which, level))
                same_bits(N, ref[level][1], "%s %s level %d normals" % (case.name, which, level))
            for which, ref in (("source", isrc), ("reference", iref)):
                I, gx, gy = tr.intensity_maps(which, level)
                same_bits(I, ref[level][0], "%s %s level %d intensity" % (case.name, which, level))
                if which == "reference":
                    same_bits(gx, ref[level][1], "%s level %d g_x" % (case.name, level))
                    same_bits(gy, ref[level][2], "%s level %d g_y" % (case.name, level))
        inliers = []
        for k, T in enumerate(mc.track_poses(T_true, np.random.default_rng(1))):
            p12 = T[:3].reshape(12)
            for level in range(mc.LEVELS):
                what = "%s pose %d level %d" % (case.name, k, level)
                got = tr.step(level, T, 0.5, COS30)
                want = tro.step(src, mod, cal, level, p12, 0.5, COS30)
                assert got[1:] == want[1:], "%s: counts %s vs %s" % (what, got[1:], want[1:])
                assert np.array_equal(got[0].view(np.uint64), want[0].view(np.uint64)), what
                gj = tr.step(level, T, 0.5, COS30, GATES)
                wj = po.step(src, mod, isrc, iref, cal, level, p12, 0.5, COS30, *GATES)
                assert gj[1:] == wj[1:], "%s gated: counts %s vs %s" % (what, gj[1:], wj[1:])
                assert np.array_equal(gj[0].view(np.uint64), wj[0].view(np.uint64)), what + " gated"
                if mc.normal_sites(H, W, level) == 0:       # no normal: every sum +0.0 bit for bit, no inlier
                    assert got[1] == 0 and not got[0].view(np.uint64).any(), what
                if mc.photo_sites(H, W, level) == 0:        # no photometric pixel
                    assert gj[2] == 0 and not gj[0][28:].view(np.uint64).any(), what
                inliers.append((got[1], gj[2]))
    print("%s: edges %s; (geometric, photometric) inliers per pose and level %s" % (case.name, sorted(edges), inliers))
    if H * W >= 1024:
        assert inliers[0][0] > 0 and inliers[0][1] > 0, case.name


# ----------------------------------------------------------------------------------------------- the product's drive

def gpu_track_drive(disps, imgs, cal, voxel, trunc, max_depth, photometric):
    H, W = disps[0].shape
    ts, tr = fusion.TSDF(voxel, trunc), track.Tracker(H, W, photometric=photometric)
    poses, lost = [], []
    for k, (d, img) in enumerate(zip(disps, imgs)):
        if k == 0:
            pose = np.eye(4)
        else:
            Z = ts.render(cal, poses[-1], H, W, 1, max_depth)
            images = dict(left=img, ref_left=imgs[k - 1]) if photometric else {}
            pose, _, is_lost = tr.track(cu(d), cal, Z, poses[-1], track.predict("track", poses), max_depth, **images)
            if is_lost:
                lost.append(k)
                poses.append(pose)
                continue
        ts.add(cu(d), cal, img, pose, max_depth=max_depth)
        poses.append(pose)
    tr.close()
    return poses, lost, ts


@pytest.mark.parametrize("photometric", [0.0, 0.01])
def test_kitti_sized_drive_is_the_oracle(photometric, tmp_path):
    """3 frames of the synthetic posed drive at 375 x 1242 tracked with -poses track: every pose and the field bit for bit"""
    D = mc.DRIVE
    drive, disps, _, truth = synth.write_kitti_posed_drive(str(tmp_path), n=D["n"], H=D["H"], W=D["W"])
    cal = dataio.read_calib(os.path.dirname(drive), "kitti_raw")
    imgs = [png(dataio.raw_file(drive, dataio.RAW_LEFT, k)) for k in range(D["n"])]
    want, wlost, ref = po.track_drive(track, disps, imgs, cal, D["voxel"], D["trunc"], max_depth=D["max_depth"],
                                      photometric=photometric)
    poses, lost, ts = gpu_track_drive(disps, imgs, cal, D["voxel"], D["trunc"], D["max_depth"], photometric)
    assert lost == wlost == []
    for k, (a, b) in enumerate(zip(poses, want)):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), "pose %d" % k
    same_table(ts, ref, "drive")
    err = [float(np.linalg.norm((track.rigid_inv(G) @ P)[:3, 3])) for P, G in zip(poses, truth)]
    print("375 x 1242 drive, photometric %g: translation errors %s m" % (photometric, np.round(err, 5).tolist()))
    ts.close()
