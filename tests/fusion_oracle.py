"""numpy restatement of the fusion rule (mc-cnn_b200/fusion.py, csrc/fusion.cu), for tests/test_fusion.py and
tests/test_gpu_fusion.py.  Written from DESIGN §23:

* points: the pixels §20's depth rule makes valid (max_depth included), their fp32 camera point (X, Y, Z) of
  depth_oracle.depth32, and the world point w_k = ((R_k0 X + R_k1 Y) + R_k2 Z) + t_k in float64 (numpy's elementwise
  operations round once each and never fuse);
* voxel: i = floor(w / v) in float64; kept when every axis lies in [-2^20, 2^20), else counted as outside; the key
  ((ix + 2^20) << 42) | ((iy + 2^20) << 21) | (iz + 2^20);
* accumulation: per frame, each voxel's partial starts at +0.0 and adds its pixels in row-major order; the table's sum starts
  at +0.0 and adds the frame partials in frame order; n_pix, n_frames and the colour byte sums in int64;
* output: the voxels with n_frames >= min_frames in ascending key order, float32(S / n_pix) and (C + n_pix // 2) // n_pix,
  packed as §20's 15-byte PLY records."""
import importlib.util
import os

import numpy as np

_spec = importlib.util.spec_from_file_location("depth_oracle", os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                            "depth_oracle.py"))
depth_oracle = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(depth_oracle)

HALF = 1 << 20


def world_points(disp, cal, pose, max_depth=None):
    """(w (n, 3) float64, pixel index (n,)) of the valid pixels of `disp` in row-major order"""
    Z, X, Y = depth_oracle.depth32(disp, cal, max_depth)
    ok = ~np.isnan(Z).reshape(-1)
    idx = np.nonzero(ok)[0]
    p = [a.reshape(-1)[idx].astype(np.float64) for a in (X, Y, Z)]
    P = np.asarray(pose, np.float64).reshape(-1)[:12].reshape(3, 4)
    w = np.stack([((P[k, 0] * p[0] + P[k, 1] * p[1]) + P[k, 2] * p[2]) + P[k, 3] for k in range(3)], 1)
    return w, idx


def voxel_keys(w, voxel):
    """(keys uint64 of the kept points, kept mask, outside count)"""
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.floor(w / np.float64(voxel))
        keep = np.all((q >= -HALF) & (q < HALF), axis=1)
    i = q[keep].astype(np.int64) + HALF
    keys = (i[:, 0].astype(np.uint64) << np.uint64(42)) | (i[:, 1].astype(np.uint64) << np.uint64(21)) | i[:, 2].astype(np.uint64)
    return keys, keep, int((~keep).sum())


def _colours(rgb, idx):
    rgb = np.asarray(rgb, np.uint8)
    if rgb.ndim == 2:
        rgb = np.repeat(rgb[:, :, None], 3, axis=2)
    return rgb.reshape(-1, 3)[idx].astype(np.int64)


def _run_sums(vals, starts, ends):
    """per run [s, e) of `vals` (m, 3) float64: +0.0 plus the run's values added one by one in order"""
    out = np.zeros((len(starts), 3))
    lens = ends - starts
    long_ = lens >= 64
    for r in np.nonzero(long_)[0]:                       # np.add.accumulate is a sequential loop
        out[r] = 0.0 + np.add.accumulate(vals[starts[r]:ends[r]], axis=0)[-1]
    short = np.nonzero(~long_)[0]
    for k in range(int(lens[short].max()) if len(short) else 0):
        sel = short[lens[short] > k]
        out[sel] = out[sel] + vals[starts[sel] + k]
    return out


def frame_partials(disp, cal, rgb, pose, voxel, max_depth=None):
    """one frame's voxels in ascending key order: (keys, n_pix, sums (u, 3), colours (u, 3)), plus (pixels kept, outside)"""
    w, idx = world_points(disp, cal, pose, max_depth)
    keys, keep, outside = voxel_keys(w, voxel)
    w, idx = w[keep], idx[keep]
    order = np.argsort(keys, kind="stable")
    keys, w, idx = keys[order], w[order], idx[order]
    starts = np.nonzero(np.r_[True, keys[1:] != keys[:-1]])[0] if len(keys) else np.zeros(0, np.int64)
    ends = np.r_[starts[1:], len(keys)].astype(np.int64)
    col = _colours(rgb, idx)
    csum = np.add.reduceat(col, starts, axis=0) if len(keys) else np.zeros((0, 3), np.int64)
    return (keys[starts], (ends - starts).astype(np.int64), _run_sums(w, starts, ends), csum), (len(keys), outside)


class Table:
    """the table of the rule: keys, n_pix, n_frames, sums (n, 3) float64, colours (n, 3) int64, in ascending key order"""

    def __init__(self, voxel):
        self.voxel = float(voxel)
        self.keys = np.zeros(0, np.uint64)
        self.n_pix = np.zeros(0, np.int64)
        self.n_frames = np.zeros(0, np.int64)
        self.sums = np.zeros((0, 3))
        self.colours = np.zeros((0, 3), np.int64)
        self.pixels = self.outside = 0

    def add(self, disp, cal, rgb, pose, max_depth=None):
        (fk, fn, fs, fc), (kept, outside) = frame_partials(disp, cal, rgb, pose, self.voxel, max_depth)
        self.pixels += kept
        self.outside += outside
        keys = np.union1d(self.keys, fk).astype(np.uint64)
        n = len(keys)
        pt, pf = np.searchsorted(keys, self.keys), np.searchsorted(keys, fk)
        n_pix, n_frames = np.zeros(n, np.int64), np.zeros(n, np.int64)
        sums, colours = np.zeros((n, 3)), np.zeros((n, 3), np.int64)
        n_pix[pt], n_frames[pt], sums[pt], colours[pt] = self.n_pix, self.n_frames, self.sums, self.colours
        n_pix[pf] += fn
        n_frames[pf] += 1
        sums[pf] = sums[pf] + fs
        colours[pf] += fc
        self.keys, self.n_pix, self.n_frames, self.sums, self.colours = keys, n_pix, n_frames, sums, colours

    def vertices(self, min_frames=1):
        """(xyz (m, 3) float32, rgb (m, 3) uint8) of the voxels seen by at least min_frames frames"""
        m = self.n_frames >= min_frames
        n = self.n_pix[m]
        xyz = (self.sums[m] / n[:, None].astype(np.float64)).astype(np.float32)
        rgb = ((self.colours[m] + n[:, None] // 2) // n[:, None]).astype(np.uint8)
        return xyz, rgb

    def records(self, min_frames=1):
        """the packed 15-byte PLY records (bytes)"""
        xyz, rgb = self.vertices(min_frames)
        rec = np.zeros(len(xyz), np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))
        rec["xyz"], rec["rgb"] = xyz, rgb
        return rec.tobytes()
