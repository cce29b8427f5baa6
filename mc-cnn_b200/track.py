"""Frame-to-model tracking of posed stereo frames against the distance field, and trajectory metrics (an addition beyond the
reference; DESIGN §25).

    tr = Tracker(H, W, device=0)                       # iters=(10, 5, 4), delta=(1.0, 0.5, 0.25), theta=30
    Z = tsdf.render(cal, W_prev, H, W, 1, max_depth)   # the model seen from the previous frame's pose
    pose, inliers, lost = tr.track(disp, cal, Z, W_prev, W_pred, max_depth)
    tr.close()

    write_poses("poses.txt", poses); poses = read_poses("poses.txt")     # KITTI odometry format, 12 numbers per line
    trajectory_metrics(est, gt)                        # TrajectoryMetrics(ate, rpe_t, rpe_r, t_err, r_err, segments)

Each frame's vertices and normals (three levels, level l keeping the pixels (2^l x, 2^l y)) are aligned to the model's by
projective point-to-plane ICP, coarsest level first.  The GPU sums each step's normal equations in a fixed order
(csrc/track.cu); :func:`run_icp` solves them and updates the pose on the host in float64.  It is the one copy of that loop,
used by :class:`Tracker` and by the numpy restatement in tests/track_oracle.py alike.

With ``Tracker(H, W, photometric=0.01)`` and ``track(..., left=left, ref_left=prev_left)`` each step also aligns the
frame's left image to the previous frame's (DESIGN §26), which fixes motion along a street whose normals all lie across it.
"""
import ctypes
import math
from collections import namedtuple

import numpy as np
import torch

from . import adcensus, depth, fusion

LEVELS = 3
ITERS = (10, 5, 4)                 # ICP steps per level, coarsest to finest
DELTA = (1.0, 0.5, 0.25)           # the largest point distance of an inlier per level, metres, coarsest to finest
THETA = 30.0                       # the largest angle between an inlier's normals, degrees
LOST_SHARE = 0.1                   # a frame whose level-0 inliers are fewer than this share of its vertices is lost
EIG_RATIO = 1e-12                  # a solve is degenerate when the smallest eigenvalue is <= this times the largest
CONVERGED = 1e-6                   # a level ends when |omega| (rad) and |tau| (m) are both below this
NSUMS = 28
RHO = 30.0                         # the largest photometric residual of an inlier, grey levels (DESIGN §26)
GRAD_MIN = 2.0                     # the smallest intensity gradient of a photometric inlier, grey levels per level pixel
MODES = ("oxts", "track", "refine")

TrajectoryMetrics = namedtuple("TrajectoryMetrics", "ate rpe_t rpe_r t_err r_err segments")
TrajectoryMetrics.__doc__ = """ate: RMSE of the translations in metres (no alignment: both start at I); rpe_t, rpe_r: the mean
translation (metres) and angle (degrees) of the consecutive-frame relative error; t_err (%) and r_err (deg/m): the KITTI
odometry segment errors over 100 .. 800 m of ground-truth path, NaN without a segment; segments: their count"""
SEGMENT_LENGTHS = (100, 200, 300, 400, 500, 600, 700, 800)
SEGMENT_STEP = 10


def as4(pose):
    """a camera-to-world pose (4x4 or its 3x4 top) as a 4x4 float64 matrix (fusion.pose12's checks)"""
    M = np.eye(4)
    M[:3] = fusion.pose12(pose).reshape(3, 4)
    return M


def rigid_inv(P):
    """the inverse of a rigid 4x4 pose: [R^T | -R^T t]"""
    P = np.asarray(P, np.float64)
    M = np.eye(4)
    M[:3, :3] = P[:3, :3].T
    M[:3, 3] = -(P[:3, :3].T @ P[:3, 3])
    return M


def rodrigues(w):
    """the rotation matrix of the rotation vector w (angle |w| about w / |w|)"""
    w = np.asarray(w, np.float64)
    th = math.sqrt(float(w @ w))
    if th == 0.0:
        return np.eye(3)
    k = w / th
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    return np.eye(3) + math.sin(th) * K + (1.0 - math.cos(th)) * (K @ K)


def solve(sums, count):
    """xi = (omega, tau) with A xi = -b from one step's 28 sums, or None when the solve is degenerate: count < 6, a sum not
    finite, or the smallest eigenvalue of A <= EIG_RATIO times the largest"""
    s = np.asarray(sums, np.float64)
    if count < 6 or not np.isfinite(s).all():
        return None
    A = np.empty((6, 6))
    k = 0
    for a in range(6):
        for b in range(a, 6):
            A[a, b] = A[b, a] = s[k]
            k += 1
    ev = np.linalg.eigvalsh(A)
    if not ev[0] > EIG_RATIO * ev[-1]:
        return None
    return np.linalg.solve(A, -s[21:27])


def solve_joint(sums_g, sums_p, count_g, count_p, lam2):
    """:func:`solve` of the joint system A_g + lam2 A_p, b_g + lam2 b_p (lam2 = lambda^2, in m^2 per grey level^2) with
    count = the geometric plus the photometric inliers"""
    return solve(np.asarray(sums_g, np.float64) + lam2 * np.asarray(sums_p, np.float64), count_g + count_p)


def update(T, xi):
    """[Rodrigues(omega) | tau] T"""
    M = np.eye(4)
    M[:3, :3] = rodrigues(xi[:3])
    M[:3, 3] = xi[3:]
    return M @ T


def run_icp(step, T, iters=ITERS, delta=DELTA, theta=THETA, photometric=0.0):
    """The ICP levels from the coarsest to the finest from the relative pose T (4x4, source camera to model camera).
    step(level, pose12, delta, cos_theta) returns (sums, geometric inliers, photometric inliers, the level's source
    vertices), as :meth:`Tracker.step`.  Returns (T, level-0 inliers, lost): lost when a level-0 solve was degenerate or
    its inliers are fewer than LOST_SHARE of its vertices.  Each solve is :func:`solve`'s of the 28 geometric sums, or
    with `photometric` lambda > 0 (metres per grey level) :func:`solve_joint`'s of the 56 sums, geometric then
    photometric; the inliers of the lost rule stay the geometric ones (DESIGN §26)."""
    cos_t = math.cos(math.radians(theta))
    lam2 = photometric * photometric
    inliers, vertices, degenerate = 0, 0, False
    for i in range(LEVELS):
        level = LEVELS - 1 - i
        for _ in range(iters[i]):
            sums, ng, nph, nv = step(level, np.ascontiguousarray(T[:3].reshape(12)), delta[i], cos_t)
            if photometric:
                xi = solve_joint(sums[:NSUMS], sums[NSUMS:], ng, nph, lam2)
            else:
                xi = solve(sums[:NSUMS], ng)
            if level == 0:
                inliers, vertices = ng, nv
            if xi is None:
                degenerate |= level == 0
                break
            T = update(T, xi)
            if math.sqrt(float(xi[:3] @ xi[:3])) < CONVERGED and math.sqrt(float(xi[3:] @ xi[3:])) < CONVERGED:
                break
    return T, inliers, degenerate or inliers < LOST_SHARE * vertices


def predict(mode, poses, oxts=None):
    """the predicted pose of the frame after `poses` (the drive's poses so far, 4x4): constant velocity W_{k-1}
    inv(W_{k-2}) W_{k-1} for 'track' (I for the second frame), W_{k-1} inv(O_{k-1}) O_k for 'refine' (oxts: the OXTS
    poses of frames 0 .. k)"""
    k = len(poses)
    if mode == "refine":
        return poses[-1] @ rigid_inv(oxts[k - 1]) @ oxts[k]
    if k == 1:
        return np.eye(4)
    return poses[-1] @ rigid_inv(poses[-2]) @ poses[-1]


def check_params(iters, delta, theta):
    if not (len(iters) == LEVELS and all(isinstance(n, int) and n >= 1 for n in iters)):
        raise ValueError("iters must be %d integers >= 1 (coarsest level first), got %r" % (LEVELS, iters))
    if not (len(delta) == LEVELS and all(isinstance(d, (int, float)) and math.isfinite(d) and d > 0 for d in delta)):
        raise ValueError("delta must be %d finite distances > 0 in metres (coarsest level first), got %r" % (LEVELS, delta))
    if not (isinstance(theta, (int, float)) and 0 < theta <= 90):
        raise ValueError("theta must be an angle in (0, 90] degrees, got %r" % (theta,))
    return tuple(iters), tuple(float(d) for d in delta), float(theta)


def check_photometric(photometric, rho, grad_min):
    """(lambda, rho, g_min) as floats; each must be a finite number >= 0"""
    for name, v in (("photometric", photometric), ("rho", rho), ("grad_min", grad_min)):
        if not (isinstance(v, (int, float)) and not isinstance(v, bool) and math.isfinite(v) and v >= 0):
            raise ValueError("%s must be a finite number >= 0, got %r" % (name, v))
    return float(photometric), float(rho), float(grad_min)


class Tracker:
    """Pyramids of one frame size on CUDA device `device` (mccnn_track_*); :meth:`track` poses one frame against the
    model's depth map.  With `photometric` lambda > 0 (metres per grey level; 0, the default, is off), each step also
    aligns the frame's left image to the previous frame's (DESIGN §26), gated by `rho` (grey levels) and `grad_min`
    (grey levels per level pixel)."""

    def __init__(self, H, W, device=0, iters=ITERS, delta=DELTA, theta=THETA, photometric=0.0, rho=RHO, grad_min=GRAD_MIN):
        if not (isinstance(H, int) and isinstance(W, int) and H >= 1 and W >= 1):
            raise ValueError("H and W must be integers >= 1, got %r, %r" % (H, W))
        self.iters, self.delta, self.theta = check_params(iters, delta, theta)
        self.photometric, self.rho, self.grad_min = check_photometric(photometric, rho, grad_min)
        self.H, self.W = H, W
        self.dev = torch.device("cuda", int(device))
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_track_create(ctypes.byref(self._h), H, W, self.dev.index), "mccnn_track_create")
        # the step's host buffers, and their addresses taken once: ndarray.ctypes costs microseconds on every access
        self._sums, self._counts, self._gates = np.zeros(2 * NSUMS), np.zeros(3, np.int64), np.zeros(2)
        self._ptrs = (self._sums.ctypes.data, self._counts.ctypes.data, self._gates.ctypes.data)

    def _handle(self):
        if not self._h:
            raise ValueError("the tracker is closed")
        return self._h

    def _map(self, t, name, fn):
        m, H, W = depth._map(t, name, fn)
        if (H, W) != (self.H, self.W) or m.device != self.dev:
            raise ValueError("%s: %s is %dx%d on %s, the tracker %dx%d on %s" % (fn, name, H, W, m.device, self.H, self.W, self.dev))
        return m

    def _step(self, level, pose12, delta, cos_t, gates=None):
        sums, counts, g = self._ptrs
        if gates is not None:
            self._gates[:] = gates
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_track_step(
                self._handle(), level, pose12.ctypes.data, delta, cos_t, None if gates is None else g, sums, counts,
                torch.cuda.current_stream(self.dev).cuda_stream), "mccnn_track_step")
        return (self._sums[:NSUMS if gates is None else 2 * NSUMS].copy(), *self._counts.tolist())

    def intensity(self, which, img):
        """the intensity pyramid of the (H, W) or (H, W, 3) uint8 image `img` (host or device): which is 'source' (the
        frame's left image) or 'reference' (the previous frame's, with its gradients)"""
        t, nch = depth._colour(img, self.H, self.W, self.dev)
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_track_intensity(self._handle(), ("source", "reference").index(which),
                                                                 t.data_ptr(), nch, adcensus._stream(t)),
                            "mccnn_track_intensity")

    def intensity_maps(self, which, level):
        """(I float32, g_x, g_y float64) of a level, each (ceil(H / 2^l), ceil(W / 2^l)) numpy, the gradients NaN where
        undefined; the source has no gradients (None)"""
        hl, wl = -(-self.H // (1 << level)), -(-self.W // (1 << level))
        k = ("source", "reference").index(which)
        with torch.cuda.device(self.dev):
            I = torch.empty((hl, wl), dtype=torch.float32, device=self.dev)
            G = torch.empty((2, hl, wl), dtype=torch.float64, device=self.dev) if k else None
            adcensus._check(adcensus.lib().mccnn_track_intensity_maps(
                self._handle(), k, level, I.data_ptr(), G[0].data_ptr() if k else None, G[1].data_ptr() if k else None,
                torch.cuda.current_stream(self.dev).cuda_stream), "mccnn_track_intensity_maps")
            return (I.cpu().numpy(),) + ((G[0].cpu().numpy(), G[1].cpu().numpy()) if k else (None, None))

    def source(self, disp, cal, max_depth=None):
        """the source pyramid of the CUDA disparity map `disp`"""
        d = self._map(disp, "disp", "mccnn_track_source")
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_track_source(
                self._handle(), d.data_ptr(), depth._f32(cal.f), depth._f32(cal.cx), depth._f32(cal.cy), depth.fB(cal),
                depth._f32(cal.doffs), depth._cap(max_depth), adcensus._stream(d)), "mccnn_track_source")

    def model(self, Z, cal):
        """the model pyramid of the CUDA depth map `Z` (NaN = no surface)"""
        z = self._map(Z, "model depth", "mccnn_track_model")
        with torch.cuda.device(self.dev):
            adcensus._check(adcensus.lib().mccnn_track_model(
                self._handle(), z.data_ptr(), depth._f32(cal.f), depth._f32(cal.cx), depth._f32(cal.cy), adcensus._stream(z)),
                "mccnn_track_model")

    def maps(self, which, level):
        """(vertices, normals) of a level, each (3, ceil(H / 2^l), ceil(W / 2^l)) float64 numpy, NaN = none; which is
        'source' or 'model'"""
        hl, wl = -(-self.H // (1 << level)), -(-self.W // (1 << level))
        with torch.cuda.device(self.dev):
            V, N = (torch.empty((3, hl, wl), dtype=torch.float64, device=self.dev) for _ in range(2))
            adcensus._check(adcensus.lib().mccnn_track_maps(self._handle(), ("source", "model").index(which), level,
                                                            V.data_ptr(), N.data_ptr(),
                                                            torch.cuda.current_stream(self.dev).cuda_stream), "mccnn_track_maps")
            return V.cpu().numpy(), N.cpu().numpy()

    def step(self, level, pose, delta, cos_theta, gates=None):
        """one reduce at `level` for the relative pose `pose`: (sums, geometric inliers, photometric inliers, the level's
        source vertices).  Without `gates` the 28 geometric sums and 0 photometric inliers; with gates = (g_min, rho) the
        joint reduce's 56 sums, geometric then photometric (both intensity pyramids are needed)"""
        return self._step(level, fusion.pose12(pose), float(delta), float(cos_theta), gates)

    def track(self, disp, cal, model_depth, W_prev, W_pred, max_depth=None, left=None, ref_left=None):
        """The pose of the frame of CUDA disparity map `disp`, aligned to `model_depth` (the model rendered at camera-to-world
        W_prev) from the prediction W_pred: (4x4 pose, level-0 inliers, lost).  A lost frame's pose is W_pred.  With the
        photometric term, `left` is the frame's left image and `ref_left` the left image of the frame posed at W_prev;
        both are required then, and refused without it."""
        if self.photometric and (left is None or ref_left is None):
            raise ValueError("the photometric term aligns the frame's left image to the previous frame's: give left and "
                             "ref_left")
        if not self.photometric and (left is not None or ref_left is not None):
            raise ValueError("left and ref_left are the photometric term's images; the tracker's photometric weight is 0")
        Wp, Wq = as4(W_prev), as4(W_pred)
        self.source(disp, cal, max_depth)
        self.model(model_depth, cal)
        gates = None
        if self.photometric:
            self.intensity("source", left)
            self.intensity("reference", ref_left)
            gates = (self.grad_min, self.rho)
        T, inliers, lost = run_icp(lambda *a: self._step(*a, gates), rigid_inv(Wp) @ Wq, self.iters, self.delta, self.theta,
                                   self.photometric)
        return (Wq if lost else Wp @ T), inliers, lost

    def close(self):
        if self._h:
            torch.cuda.synchronize(self.dev)
            adcensus.lib().mccnn_track_destroy(self._h)
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


def write_poses(path, poses):
    """the KITTI odometry format: one line per pose, the 12 numbers of its [R | t] row by row, %.17g (read back bit for
    bit)"""
    with open(path, "w") as f:
        for P in poses:
            f.write(" ".join("%.17g" % v for v in fusion.pose12(P)) + "\n")


def read_poses(path):
    """[4x4 float64] of a KITTI odometry pose file; refuses, naming the file and line, a line without 12 finite numbers"""
    out = []
    with open(path) as f:
        for i, line in enumerate(f, 1):
            if not line.strip():
                continue
            try:
                v = [float(x) for x in line.split()]
            except ValueError:
                v = []
            if len(v) != 12 or not all(math.isfinite(x) for x in v):
                raise ValueError("%s line %d: a pose is 12 finite numbers" % (path, i))
            M = np.eye(4)
            M[:3] = np.reshape(v, (3, 4))
            out.append(M)
    return out


def rotation_angle(R):
    """acos(clamp((tr R - 1) / 2)) in radians"""
    return math.acos(max(-1.0, min(1.0, 0.5 * (R[0, 0] + R[1, 1] + R[2, 2] - 1.0))))


def _relative_error(ea, eb, ga, gb):
    """inv(inv(ea) eb) (inv(ga) gb)"""
    return rigid_inv(rigid_inv(ea) @ eb) @ (rigid_inv(ga) @ gb)


def trajectory_metrics(est, gt):
    """:data:`TrajectoryMetrics` of the estimated poses `est` against the ground truth `gt` (equal-length lists of 4x4 or
    3x4 camera-to-world poses, both starting at the same frame)"""
    est, gt = [as4(P) for P in est], [as4(P) for P in gt]
    if len(est) != len(gt) or not est:
        raise ValueError("trajectories of %d and %d poses: they must be equally long and not empty" % (len(est), len(gt)))
    n = len(gt)
    d = np.array([e[:3, 3] - g[:3, 3] for e, g in zip(est, gt)])
    ate = math.sqrt(float(np.mean(np.sum(d * d, 1))))
    rt, rr = [], []
    for k in range(1, n):
        E = _relative_error(est[k - 1], est[k], gt[k - 1], gt[k])
        rt.append(float(np.linalg.norm(E[:3, 3])))
        rr.append(math.degrees(rotation_angle(E[:3, :3])))
    nan = float("nan")
    # the odometry devkit's segments: first frames every SEGMENT_STEP frames, the last frame the first one whose distance
    # along the ground-truth path exceeds the first's by the segment length
    dist = np.concatenate([[0.0], np.cumsum([np.linalg.norm(gt[k][:3, 3] - gt[k - 1][:3, 3]) for k in range(1, n)])])
    te, re = [], []
    for first in range(0, n, SEGMENT_STEP):
        for length in SEGMENT_LENGTHS:
            beyond = np.nonzero(dist[first:] > dist[first] + length)[0]
            if not len(beyond):
                continue
            last = first + int(beyond[0])
            E = _relative_error(est[first], est[last], gt[first], gt[last])
            te.append(float(np.linalg.norm(E[:3, 3])) / length)
            re.append(rotation_angle(E[:3, :3]) / length)
    return TrajectoryMetrics(ate, float(np.mean(rt)) if rt else nan, float(np.mean(rr)) if rr else nan,
                             100.0 * float(np.mean(te)) if te else nan, math.degrees(float(np.mean(re))) if re else nan,
                             len(te))


def metrics_line(name, m):
    """one printed line of :data:`TrajectoryMetrics`"""
    return "%s ate %.6f rpe_t %.6f rpe_r %.6f t_err %.6f r_err %.6f segments %d" % ((name,) + tuple(m))
