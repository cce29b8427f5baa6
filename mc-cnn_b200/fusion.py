"""The stereo depth of posed frames fused into one world-frame point cloud on the GPU (an addition beyond the reference;
DESIGN §23).

    fu = Fusion(voxel=0.1, device=0)
    fu.add(disp, cal, left, pose)              # pose: 4x4 (or its top 3x4) camera-to-world, float64
    pts = fu.cloud(min_frames=2)               # a depth.Cloud: one vertex per voxel seen by >= 2 frames
    depth.write_ply("map.ply", pts)
    t = fu.table()                             # numpy: keys, n_pix, n_frames, sums (n, 3), colours (n, 3)
    fu.stats                                   # FusionStats(pixels, outside, voxels)
    fu.close()

    fuse_drive("kitti", "census", ["/data/raw/2011_09_26/2011_09_26_drive_0002_sync"], out="O", voxel=0.1)
    # O/2011_09_26_drive_0002_sync/fused.ply, posed by the drive's OXTS records (dataio.raw_poses)

    ts = TSDF(voxel=0.1, trunc=None, device=0)  # a truncated signed distance field (DESIGN §24), trunc 4 voxel by default
    ts.add(disp, cal, left, pose)               # as Fusion.add
    m = ts.mesh(min_frames=1)                   # a depth.Mesh: vertex records and int32 faces on the device
    depth.write_mesh_ply("map.ply", m)
    Z = ts.render(cal, pose, H, W)              # CUDA (H, W) fp32 depth of the field seen from pose, NaN = no surface
    ts.table(); ts.stats; ts.close()            # TSDFTable numpy arrays, TSDFStats(pixels, outside, bricks, pool_bytes)
    fuse_drive(..., mesh=True, score=True)      # O/<drive>/mesh.ply, and each frame scored against its scan
    fuse_drive(..., mesh=True, poses="track")   # posed by tracking against the field (DESIGN §25): O/<drive>/poses.txt

A pixel contributes when §20's depth rule makes it valid (max_depth included).  Its camera point (X, Y, Z) is its
depth.point_cloud vertex; its world point w = R (X, Y, Z) + t is computed in float64 with each operation rounded once and
no FMA; its voxel is floor(w / voxel) per axis.  A voxel keeps n_pix, n_frames (frames that put a pixel in it), float64
sums of w and int64 sums of the colour bytes; a frame's partial adds its pixels in row-major order from +0.0 and the table
adds the frames' partials in the order they were added, so the result has the same bits on every run and GPU.  Points
whose voxel index lies outside [-2^20, 2^20) on some axis are counted in stats.outside and dropped.  The cloud has one
vertex per voxel with n_frames >= min_frames, in ascending key order: float32(sum / n_pix) and (C + n_pix // 2) // n_pix.
"""
import ctypes
import math
import os
from collections import namedtuple

import numpy as np
import torch

from . import adcensus, confidence as confidence_, dataio, depth, predict_kitti, predict_raw

KEY_BITS = 21
KEY_HALF = 1 << 20
FUSED = "fused.ply"
MESHED = "mesh.ply"
POSES = "poses.txt"
VOX = 512                                  # voxels per brick of the TSDF, local order (z, y, x)
MAX_TSDF_FRAMES = 1 << 23                  # the int32 colour sums of a voxel cannot overflow up to this many frames

FusionStats = namedtuple("FusionStats", "pixels outside voxels")
FusionStats.__doc__ = """pixels: the pixels added to the table, outside: the valid pixels dropped because their voxel lies outside the
key range, voxels: the table's voxel count"""
FusionTable = namedtuple("FusionTable", "keys n_pix n_frames sums colours")
FusionTable.__doc__ = """The table in ascending key order: keys (n,) uint64, n_pix and n_frames (n,) int64, sums (n, 3) float64 of the
world points, colours (n, 3) int64 sums of the R, G, B bytes"""
DriveSummary = namedtuple("DriveSummary", "drive frames pixels outside voxels vertices")
TSDFStats = namedtuple("TSDFStats", "pixels outside bricks pool_bytes")
TSDFStats.__doc__ = """pixels: the valid pixels integrated, outside: the ray points dropped because their brick lies outside the key
range, bricks: the table's brick count, pool_bytes: the bytes its brick pool holds"""
TSDFTable = namedtuple("TSDFTable", "keys S n nc colours")
TSDFTable.__doc__ = """The field in ascending brick-key order: keys (b,) uint64, then per voxel (b, 8, 8, 8) indexed (brick, z, y, x):
S float64, n and nc int32, and colours (b, 8, 8, 8, 3) int32 sums of the R, G, B bytes"""
MeshSummary = namedtuple("MeshSummary", "drive frames pixels outside bricks vertices faces scores poses lost traj",
                         defaults=(None, 0, None))
MeshSummary.__doc__ = """one drive's TSDF: frames integrated, pixels, outside, bricks, mesh vertices and faces; scores (with score);
poses (the drive's camera-to-world poses), lost (the frames tracking lost) and traj (track.TrajectoryMetrics against the
OXTS poses, with traj) when the frames were tracked"""


def check_voxel(voxel):
    if not (isinstance(voxel, (int, float)) and math.isfinite(voxel) and voxel > 0):
        raise ValueError("voxel must be a finite edge length > 0 in metres, got %r" % (voxel,))
    return float(voxel)


def check_min_frames(min_frames):
    if not (isinstance(min_frames, int) and min_frames >= 1):
        raise ValueError("min_frames must be an integer >= 1, got %r" % (min_frames,))
    return min_frames


def check_trunc(trunc, voxel):
    """the truncation in metres: 4 voxel when None, else finite, >= voxel and at most 256 voxel (2K + 1 <= 129 ray points
    per pixel)"""
    if trunc is None:
        return 4.0 * voxel
    if not (isinstance(trunc, (int, float)) and math.isfinite(trunc) and voxel <= trunc <= 256 * voxel):
        raise ValueError("trunc must be a finite length in [voxel, 256 voxel] (voxel %r) in metres, got %r" % (voxel, trunc))
    return float(trunc)


def pose12(pose):
    """the 12 float64 of a camera-to-world pose's [R | t], row-major: a 4x4 matrix whose last row is (0, 0, 0, 1), or its
    3x4 top; refuses other shapes and non-finite entries"""
    P = np.asarray(pose, np.float64)
    if P.shape == (4, 4):
        if not np.array_equal(P[3], [0.0, 0.0, 0.0, 1.0]):
            raise ValueError("a 4x4 pose's last row must be (0, 0, 0, 1), got %s" % (P[3],))
        P = P[:3]
    if P.shape != (3, 4):
        raise ValueError("a pose is 4x4 or 3x4, got %s" % (P.shape,))
    if not np.isfinite(P).all():
        raise ValueError("a pose must be finite")
    return np.ascontiguousarray(P.reshape(12))


def key_index(keys):
    """(ix, iy, iz) int64 arrays of voxel keys"""
    k = np.asarray(keys, np.uint64)
    m = np.uint64((1 << KEY_BITS) - 1)
    return tuple((((k >> np.uint64(s)) & m).astype(np.int64) - KEY_HALF) for s in (2 * KEY_BITS, KEY_BITS, 0))


class Fusion:
    """One world-frame voxel map on CUDA device `device` (mccnn_fusion_*): frames are added in order, the map read out as a
    cloud or a table (module docstring)."""

    def __init__(self, voxel, device=0):
        self.voxel = check_voxel(voxel)
        self.dev = torch.device("cuda", int(device))
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_fusion_create(ctypes.byref(self._h), self.voxel, self.dev.index),
                            "mccnn_fusion_create")
        self._totals = torch.zeros(2, dtype=torch.int64, device=self.dev)
        self.frames = 0

    def _handle(self):
        if not self._h:
            raise ValueError("the fusion map is closed")
        return self._h

    def add(self, disp, cal, left, pose, max_depth=None, conf=None, density=None):
        """Fuse one frame: `disp` its CUDA disparity map, `cal` its dataio.Calib, `left` its decoded left image ((H, W) or
        (H, W, 3) uint8, host or device), `pose` its camera-to-world matrix.  With `conf` and `density`, only the pixels
        confidence.sparsify keeps."""
        if (conf is None) != (density is None):
            raise ValueError("conf and density go together")
        h = self._handle()
        P = pose12(pose)
        name = "mccnn_fusion_add"
        d, H, W = depth._map(disp, "disp", name)
        if d.device != self.dev:
            raise ValueError("%s: disp is on %s, the map on %s" % (name, d.device, self.dev))
        rgb, nch = depth._colour(left, H, W, self.dev)
        cap = depth._cap(max_depth)
        stats = torch.empty(3, dtype=torch.int64, device=self.dev)
        with torch.cuda.device(self.dev):
            if conf is not None:
                d = confidence_.sparsify(d, conf, density)
            adcensus._check(adcensus.lib().mccnn_fusion_add(
                h, d.data_ptr(), rgb.data_ptr(), nch, H, W, depth._f32(cal.f), depth._f32(cal.cx), depth._f32(cal.cy),
                depth.fB(cal), depth._f32(cal.doffs), cap, P.ctypes.data, stats.data_ptr(), adcensus._stream(d)), name)
            self._totals += stats[:2]
        self.frames += 1

    @property
    def stats(self):
        """:data:`FusionStats` of every frame added so far (one device-to-host copy)"""
        p, o = (int(v) for v in self._totals.cpu().tolist())
        return FusionStats(p, o, int(adcensus.lib().mccnn_fusion_size(self._handle())))

    def cloud(self, min_frames=1):
        """the :data:`depth.Cloud` of the voxels seen by at least `min_frames` frames: one int64 is read back (the count),
        the records stay on the device"""
        check_min_frames(min_frames)
        h, lib = self._handle(), adcensus.lib()
        with torch.cuda.device(self.dev):
            s = torch.cuda.current_stream(self.dev).cuda_stream
            count = torch.empty(1, dtype=torch.int64, device=self.dev)
            adcensus._check(lib.mccnn_fusion_count(h, min_frames, count.data_ptr(), s), "mccnn_fusion_count")
            n = int(count.item())
            data = torch.empty(max(1, n) * depth.REC, dtype=torch.uint8, device=self.dev)
            adcensus._check(lib.mccnn_fusion_fill(h, min_frames, data.data_ptr(), n, s), "mccnn_fusion_fill")
        return depth.Cloud(data[:n * depth.REC], n)

    def table(self):
        """the :data:`FusionTable` as numpy arrays"""
        h, lib = self._handle(), adcensus.lib()
        n = int(lib.mccnn_fusion_size(h))
        with torch.cuda.device(self.dev):
            buf = torch.empty(max(1, 9 * n), dtype=torch.int64, device=self.dev)
            p, e = buf.data_ptr(), buf.element_size()
            adcensus._check(lib.mccnn_fusion_table(h, p, p + n * e, p + 2 * n * e, p + 3 * n * e, p + 6 * n * e,
                                                   torch.cuda.current_stream(self.dev).cuda_stream), "mccnn_fusion_table")
            a = buf[:9 * n].cpu().numpy()
        return FusionTable(a[:n].view(np.uint64).copy(), a[n:2 * n].copy(), a[2 * n:3 * n].copy(),
                           a[3 * n:6 * n].view(np.float64).reshape(3, n).T.copy(), a[6 * n:].reshape(3, n).T.copy())

    def close(self):
        if self._h:
            torch.cuda.synchronize(self.dev)
            adcensus.lib().mccnn_fusion_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TSDF:
    """One truncated signed distance field on CUDA device `device` (mccnn_tsdf_*, DESIGN §24): frames are added in order at
    their poses; the field is read out as a mesh, a depth map seen from any pose, or a table."""

    def __init__(self, voxel, trunc=None, device=0):
        self.voxel = check_voxel(voxel)
        self.trunc = check_trunc(trunc, self.voxel)
        self.dev = torch.device("cuda", int(device))
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_tsdf_create(ctypes.byref(self._h), self.voxel, self.trunc, self.dev.index),
                            "mccnn_tsdf_create")
        self._totals = torch.zeros(2, dtype=torch.int64, device=self.dev)
        self.frames = 0

    def _handle(self):
        if not self._h:
            raise ValueError("the TSDF is closed")
        return self._h

    def add(self, disp, cal, left, pose, max_depth=None, conf=None, density=None):
        """Integrate one frame; the arguments are :meth:`Fusion.add`'s."""
        if (conf is None) != (density is None):
            raise ValueError("conf and density go together")
        h = self._handle()
        if self.frames >= MAX_TSDF_FRAMES:
            raise ValueError("a TSDF takes at most 2^23 frames")
        P = pose12(pose)
        name = "mccnn_tsdf_add"
        d, H, W = depth._map(disp, "disp", name)
        if d.device != self.dev:
            raise ValueError("%s: disp is on %s, the field on %s" % (name, d.device, self.dev))
        rgb, nch = depth._colour(left, H, W, self.dev)
        cap = depth._cap(max_depth)
        stats = torch.empty(2, dtype=torch.int64, device=self.dev)
        with torch.cuda.device(self.dev):
            if conf is not None:
                d = confidence_.sparsify(d, conf, density)
            adcensus._check(adcensus.lib().mccnn_tsdf_add(
                h, d.data_ptr(), rgb.data_ptr(), nch, H, W, depth._f32(cal.f), depth._f32(cal.cx), depth._f32(cal.cy),
                depth.fB(cal), depth._f32(cal.doffs), cap, P.ctypes.data, stats.data_ptr(), adcensus._stream(d)), name)
            self._totals += stats
        self.frames += 1

    @property
    def stats(self):
        """:data:`TSDFStats` of every frame added so far (one device-to-host copy)"""
        h, lib = self._handle(), adcensus.lib()
        p, o = (int(v) for v in self._totals.cpu().tolist())
        return TSDFStats(p, o, int(lib.mccnn_tsdf_bricks(h)), int(lib.mccnn_tsdf_pool_bytes(h)))

    def mesh(self, min_frames=1):
        """the :data:`depth.Mesh` of the voxels seen by at least `min_frames` frames: two int64 are read back (the counts),
        the vertex records and faces stay on the device"""
        check_min_frames(min_frames)
        h, lib = self._handle(), adcensus.lib()
        with torch.cuda.device(self.dev):
            s = torch.cuda.current_stream(self.dev).cuda_stream
            counts = torch.empty(2, dtype=torch.int64, device=self.dev)
            adcensus._check(lib.mccnn_tsdf_mesh_count(h, min_frames, counts.data_ptr(), s), "mccnn_tsdf_mesh_count")
            nv, nf = (int(v) for v in counts.cpu().tolist())
            if nv >= 1 << 31:
                raise ValueError("the mesh has %d vertices; int32 faces index fewer than 2^31" % nv)
            data = torch.empty(max(1, nv) * depth.REC, dtype=torch.uint8, device=self.dev)
            faces = torch.empty((max(1, nf), 3), dtype=torch.int32, device=self.dev)
            adcensus._check(lib.mccnn_tsdf_mesh_fill(h, min_frames, data.data_ptr(), nv, faces.data_ptr(), nf, s),
                            "mccnn_tsdf_mesh_fill")
        return depth.Mesh(data[:nv * depth.REC], nv, faces[:nf])

    def render(self, cal, pose, H, W, min_frames=1, max_depth=None):
        """the CUDA (H, W) float32 depth map of the field seen from camera-to-world `pose` under `cal`'s f, cx, cy: each
        pixel's first zero crossing from positive to negative, NaN where none"""
        check_min_frames(min_frames)
        h = self._handle()
        P = pose12(pose)
        if not (int(H) >= 1 and int(W) >= 1):
            raise ValueError("H and W must be >= 1, got %r, %r" % (H, W))
        Z = torch.empty((int(H), int(W)), dtype=torch.float32, device=self.dev)
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_tsdf_render(
                h, min_frames, int(H), int(W), depth._f32(cal.f), depth._f32(cal.cx), depth._f32(cal.cy),
                depth._cap(max_depth), P.ctypes.data, Z.data_ptr(), torch.cuda.current_stream(self.dev).cuda_stream),
                "mccnn_tsdf_render")
        return Z

    def table(self):
        """the :data:`TSDFTable` as numpy arrays"""
        h, lib = self._handle(), adcensus.lib()
        b = int(lib.mccnn_tsdf_bricks(h))
        with torch.cuda.device(self.dev):
            keys = torch.empty(max(1, b), dtype=torch.int64, device=self.dev)
            S = torch.empty(max(1, b * VOX), dtype=torch.float64, device=self.dev)
            n, nc = (torch.empty(max(1, b * VOX), dtype=torch.int32, device=self.dev) for _ in range(2))
            col = torch.empty(max(1, 3 * b * VOX), dtype=torch.int32, device=self.dev)
            adcensus._check(lib.mccnn_tsdf_table(h, keys.data_ptr(), S.data_ptr(), n.data_ptr(), nc.data_ptr(), col.data_ptr(),
                                                 torch.cuda.current_stream(self.dev).cuda_stream), "mccnn_tsdf_table")
            get = lambda t, m: t[:m].cpu().numpy()
            return TSDFTable(get(keys, b).view(np.uint64).copy(), get(S, b * VOX).reshape(b, 8, 8, 8),
                             get(n, b * VOX).reshape(b, 8, 8, 8), get(nc, b * VOX).reshape(b, 8, 8, 8),
                             get(col, 3 * b * VOX).reshape(b, 8, 8, 8, 3))

    def close(self):
        if self._h:
            torch.cuda.synchronize(self.dev)
            adcensus.lib().mccnn_tsdf_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def fused_file(out, drive, mesh=False):
    return os.path.join(out, predict_raw.drive_name(drive), MESHED if mesh else FUSED)


def poses_file(out, drive):
    return os.path.join(out, predict_raw.drive_name(drive), POSES)


def check_drives(drives, out, mesh=False, tracked=False):
    """the refusals of fuse_drive that need no GPU: _extract drives and an existing fused.ply (mesh.ply with `mesh`; and
    poses.txt with `tracked`)"""
    for d in drives:
        if predict_raw.is_extract(d):
            raise ValueError("%s is an unrectified (_extract) drive: its OXTS records run at their own rate, not one per "
                             "image, so its frames cannot be posed; use the drive's _sync version" % d)
        f = fused_file(out, d, mesh)
        if os.path.exists(f):
            raise ValueError("%s exists; fusion does not overwrite a map" % f)
        if tracked and os.path.exists(poses_file(out, d)):
            raise ValueError("%s exists; tracking does not overwrite a trajectory" % poses_file(out, d))


def fuse_drive(dataset, arch, drives, net_fname=None, out="out", voxel=0.1, min_frames=1, max_depth=None, every=1,
               confidence=False, density=None, disp_max=predict_kitti.DISP_MAX, device=0, prefetch=True, verbose=True,
               mesh=False, trunc=None, score=False, crop="none", min_depth=depth.MIN_DEPTH, poses="oxts", traj=False,
               photometric=0.0, rho=30.0, grad_min=2.0, **overrides):
    """The stereo method over every `every`-th frame of each `_sync` drive in `drives`, in frame order on one device, each
    drive's frames fused into ``out/<drive>/fused.ply`` in its own world frame (dataio.raw_poses: the drive's first fused
    frame).  Prints ``<date>/<drive> <frame>`` per frame and one summary line per drive; returns the
    :data:`DriveSummary` list.  With `mesh`, the frames go into a :class:`TSDF` of truncation `trunc` instead, and
    ``out/<drive>/mesh.ply`` gets its mesh (a :data:`MeshSummary` per drive); with `score` as well, each frame's stereo
    depth and the field rendered at its pose are scored against its projected scan (depth_eval.lidar_gt, `crop`,
    `min_depth`, max_depth 80 m): one line per frame, the stereo then the fused lidar_* values, then the line of means.
    `poses` 'track' or 'refine' (with `mesh`) poses each frame after a drive's first by tracking it against the field
    rendered at the previous frame's pose (track.Tracker, DESIGN §25), predicted by constant velocity ('track', no OXTS
    needed) or by the OXTS increment ('refine'); a lost frame is printed ``<date>/<drive> <frame> lost``, keeps its
    prediction and is not integrated; ``out/<drive>/poses.txt`` gets the poses, and `traj` prints one line of
    track.trajectory_metrics against the OXTS poses per drive.  Scores are taken at the tracked poses.  `photometric`
    lambda > 0 (metres per grey level) adds the photometric term (DESIGN §26, gates `rho` and `grad_min`): each frame's
    left image is aligned to the previous frame's, which stays on the device.  Everything that can be refused is refused
    before any GPU work."""
    import torch.distributed as dist

    from . import depth_eval, track as track_

    if dataset not in predict_raw.DATASETS:
        raise ValueError("dataset must be 'kitti' or 'kitti2015', got %r" % (dataset,))
    voxel = check_voxel(voxel)
    check_min_frames(min_frames)
    depth._cap(max_depth)
    if int(disp_max) < 1:
        raise ValueError("disp_max must be at least 1, got %r" % (disp_max,))
    if density is not None:
        if not confidence:
            raise ValueError("density ranks pixels by their confidence: it needs confidence")
        confidence_.check_density(density)
    if not mesh and (trunc is not None or score):
        raise ValueError("trunc and score apply to the distance field: they need mesh")
    if poses not in track_.MODES:
        raise ValueError("poses must be 'oxts', 'track' or 'refine', got %r" % (poses,))
    tracked = poses != "oxts"
    if tracked and not mesh:
        raise ValueError("poses %r tracks each frame against the distance field: it needs mesh" % poses)
    if traj and not tracked:
        raise ValueError("traj compares tracked poses with the OXTS poses: it needs poses 'track' or 'refine'")
    photometric, rho, grad_min = track_.check_photometric(photometric, rho, grad_min)
    if photometric and not tracked:
        raise ValueError("photometric weighs a term of the tracking: it needs poses 'track' or 'refine'")
    if mesh:
        trunc = check_trunc(trunc, voxel)
    if score:
        depth_eval._check_raw(min_depth, depth.KITTI_MAX_DEPTH, crop)
    if dist.is_initialized() and dist.get_world_size() > 1:
        raise ValueError("fusion adds the frames in order on one device; run it in one process")
    if not drives:
        raise ValueError("no drive given")
    check_drives(drives, out, mesh, tracked)
    frames = predict_raw.drive_frames(drives, every, velodyne=score)
    oxts = {}
    if poses != "track" or traj:
        for d in drives:
            idx = [fr.index for fr in frames if fr.drive == d]
            oxts.update(zip(((d, i) for i in idx), dataio.raw_poses(d, idx)))
    files = predict_raw.pair_files(frames)
    shapes = predict_kitti.scan(files)
    cals = predict_raw.read_calibs(frames, shapes)
    run = predict_kitti.PairRunner(files, shapes, dataset, arch, net_fname, disp_max, device, 0, 1, prefetch, **overrides)

    def gt_of(i):
        fr = frames[i]
        return depth_eval.lidar_gt(dataio.read_velodyne(dataio.raw_file(fr.drive, dataio.RAW_SCAN, fr.index)),
                                   cals[predict_raw.date_dir(fr.drive)], *shapes[i], run.dev, min_depth, crop)

    out_sums = []
    fu = tracker = ref_left = None
    stereo = []                            # the drive's per-frame stereo counts (score)
    used = oxts if not tracked else {}     # each frame's pose
    try:
        run.prepare()
        for i, fr in enumerate(frames):
            if fu is None:
                fu = TSDF(voxel, trunc, run.dev.index) if mesh else Fusion(voxel, run.dev.index)
                first = i
                est, lost = [], []
            cal = cals[predict_raw.date_dir(fr.drive)]
            left, _, _, pred, conf = run.predict(i, conf=confidence)
            is_lost = False
            if tracked:
                if i == first:
                    pose = np.eye(4)
                else:
                    H, W = (int(v) for v in shapes[i])
                    if tracker is None or (tracker.H, tracker.W) != (H, W):
                        if tracker is not None:
                            tracker.close()
                        tracker = track_.Tracker(H, W, run.dev.index, photometric=photometric, rho=rho, grad_min=grad_min)
                    Z = fu.render(cal, est[-1], H, W, 1, max_depth)
                    O = [oxts[(fr.drive, f.index)] for f in frames[first:i + 1]] if poses == "refine" else None
                    images = dict(left=left, ref_left=ref_left) if photometric else {}
                    pose, _, is_lost = tracker.track(pred, cal, Z, est[-1], track_.predict(poses, est, O), max_depth, **images)
                if photometric:                # the next frame's reference, lost or not
                    ref_left = depth._colour(left, *(int(v) for v in shapes[i]), run.dev)[0]
                est.append(pose)
                used[(fr.drive, fr.index)] = pose
                if is_lost:
                    lost.append(fr.index)
            if not is_lost:
                fu.add(pred, cal, left, used[(fr.drive, fr.index)], max_depth=max_depth,
                       conf=conf if density is not None else None, density=density)
            if score:
                with torch.cuda.device(run.dev):
                    stereo.append(depth.counts(pred, gt_of(i), cal, min_depth, depth.KITTI_MAX_DEPTH))
            if verbose:
                print(predict_raw.frame_name(fr) + (" lost" if is_lost else ""), flush=True)
            if i + 1 == len(frames) or frames[i + 1].drive != fr.drive:
                name = "%s/%s" % (os.path.basename(predict_raw.date_dir(fr.drive)), predict_raw.drive_name(fr.drive))
                path = fused_file(out, fr.drive, mesh)
                os.makedirs(os.path.dirname(path), exist_ok=True)
                if mesh:
                    m = fu.mesh(min_frames)
                    depth.write_mesh_ply(path, m)
                    st = fu.stats
                    s = MeshSummary(name, fu.frames, st.pixels, st.outside, st.bricks, m.n, int(m.faces.shape[0]), None)
                    if verbose:
                        print("%s: frames %d pixels %d outside %d bricks %d vertices %d faces %d" % s[:7], flush=True)
                    if tracked:
                        track_.write_poses(poses_file(out, fr.drive), est)
                        s = s._replace(poses=est, lost=len(lost))
                        if traj:
                            s = s._replace(traj=track_.trajectory_metrics(
                                est, [oxts[(fr.drive, f.index)] for f in frames[first:i + 1]]))
                            if verbose:
                                print(track_.metrics_line(name, s.traj), flush=True)
                    if score:
                        s = s._replace(scores=_score_drive(fu, frames[first:i + 1], first, cals, shapes, used, stereo, gt_of,
                                                           min_frames, max_depth, min_depth, verbose))
                else:
                    pts = fu.cloud(min_frames)
                    depth.write_ply(path, pts)
                    st = fu.stats
                    s = DriveSummary(name, fu.frames, st.pixels, st.outside, st.voxels, pts.n)
                    if verbose:
                        print("%s: frames %d pixels %d outside %d voxels %d vertices %d" % s, flush=True)
                out_sums.append(s)
                stereo = []
                fu.close()
                fu = None
    finally:
        if fu is not None:
            fu.close()
        if tracker is not None:
            tracker.close()
        run.close()
    return out_sums


def _score_drive(ts, frames, first, cals, shapes, poses, stereo, gt_of, min_frames, max_depth, min_depth, verbose):
    """each frame's stereo counts and the field rendered at its pose, scored against its scan: one depth_eval line per
    frame (the stereo then the fused lidar_* values) and the line of means; returns depth_eval.Scores"""
    from . import depth_eval

    names, rows = [], []
    for k, fr in enumerate(frames):
        cal = cals[predict_raw.date_dir(fr.drive)]
        H, W = shapes[first + k]
        with torch.cuda.device(ts.dev):
            Z = ts.render(cal, poses[(fr.drive, fr.index)], H, W, min_frames, max_depth)
            c, s = depth.counts(Z, gt_of(first + k), cal, min_depth, depth.KITTI_MAX_DEPTH, is_depth=True)
            row = list(depth.metrics_of(*(t.cpu() for t in stereo[k]))) + list(depth.metrics_of(c.cpu(), s.cpu()))
        names.append(predict_raw.frame_name(fr))
        rows.append(row)
        if verbose:
            print(depth_eval.line(names[-1], row), flush=True)
    mean = [sum(r[j] for r in rows) / len(rows) for j in range(len(SCORE_COLUMNS))]
    if verbose:
        print(depth_eval.line("mean", mean), flush=True)
    return depth_eval.Scores(names, rows, mean)


SCORE_COLUMNS = ["stereo_lidar_%s" % m for m in depth.METRICS] + ["fused_lidar_%s" % m for m in depth.METRICS]
