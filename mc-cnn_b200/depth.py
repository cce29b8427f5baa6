"""Metric depth, coloured point clouds and depth metrics of a disparity map, on the GPU (an addition beyond the reference;
DESIGN §20).

    cal = dataio.read_calib("training/calib/000000.txt", "kitti")      # kitti | kitti2015 | mb
    Z = depth(disp, cal, max_depth=None)                                 # CUDA (H, W) fp32, NaN = no depth
    pts = point_cloud(disp, cal, left_u8, conf=None, density=None)      # Cloud(data, n): device bytes, vertex count
    write_ply("scene.ply", pts)
    m = metrics(disp, gt_disp, cal, min_depth=1e-3, max_depth=80.0)     # DepthMetrics
    Zs = velo_depth(scan, raw_cal, H, W)                                  # a LiDAR scan's depth map, 0 = none (DESIGN §21)

A disparity d at pixel (x, y) is valid when it is finite and d + doffs > 0 (fp32 add); then, in fp32 with each operation
rounded once and in this order, Z = fB / (d + doffs), X = ((x - cx) * Z) / f, Y = ((y - cy) * Z) / f, where fB is the
float64 product f * baseline rounded once to fp32 (:func:`fB`).  `max_depth` also makes Z > max_depth invalid.

The point cloud has one vertex (X, Y, Z, r, g, b) per valid pixel in row-major order, its colour the left image's decoded
bytes (a grey image repeated to three channels), packed as binary little-endian PLY records of 15 bytes (float x, y, z,
uchar red, green, blue).  With `conf` and `density` it keeps exactly the pixels :func:`confidence.sparsify` keeps: the map
is made sparse first, and its dropped pixels (NaN) are invalid by the rule above.

The depth metrics (Eigen et al.; KITTI's depth benchmark): S = the pixels whose ground-truth disparity gives a valid depth
Zg in [min_depth, max_depth]; over S and a valid prediction, with the predicted depth clamped to [min_depth, max_depth]:
abs_rel = mean |Z - Zg| / Zg, sq_rel = mean (Z - Zg)^2 / Zg, rmse, rmse_log, a1 / a2 / a3 = the share with max(Z / Zg,
Zg / Z) < 1.25, 1.25^2, 1.25^3, n = the pixel count and coverage = n / |S|.  Sums in float64 in a fixed order; every mean
is NaN when n = 0.
"""
import math
from collections import namedtuple

import numpy as np
import torch

from . import adcensus, confidence

REC = 15                                 # bytes per PLY vertex
PLY_HEADER = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
KITTI_MAX_DEPTH = 80.0
MIN_DEPTH = 1e-3
# the count layout of mccnn_depth_metrics (include/adcensus_b200.h)
GT, N, A1, A2, A3 = range(5)
NCOUNT = 5
NSUM = 4
METRICS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3", "n", "coverage")

Cloud = namedtuple("Cloud", "data n")    # data: (n * 15,) CUDA uint8, the packed PLY records; n: the vertex count
DepthMetrics = namedtuple("DepthMetrics", METRICS)


def fB(cal):
    """f * baseline in float64, rounded once to fp32"""
    return float(np.float32(float(cal.f) * float(cal.baseline)))


def _f32(v):
    return float(np.float32(v))


def _cap(max_depth):
    if max_depth is None:
        return math.inf
    if not max_depth > 0:
        raise ValueError("max_depth must be > 0, got %r" % (max_depth,))
    return float(max_depth)


def _map(t, name, fn):
    """(t as a contiguous (H, W) CUDA float32 tensor, H, W); (1, 1, H, W) is accepted"""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
        raise adcensus.AdcensusError("%s: %s must be a CUDA float32 tensor" % (fn, name))
    if t.dim() < 2 or t.numel() != t.size(-1) * t.size(-2):
        raise adcensus.AdcensusError("%s: %s must be (H, W) or (1, 1, H, W), got %s" % (fn, name, tuple(t.shape)))
    H, W = t.shape[-2:]
    return t.reshape(H, W).contiguous(), H, W


def depth(disp, cal, max_depth=None, xy=False):
    """Z (H, W) of the CUDA disparity map `disp` under calibration `cal` (mccnn_disp_to_depth), NaN where there is no
    depth; with `xy`, (Z, X, Y)."""
    n = "mccnn_disp_to_depth"
    d, H, W = _map(disp, "disp", n)
    Z = torch.empty((H, W), device=d.device, dtype=torch.float32)
    X, Y = (torch.empty_like(Z), torch.empty_like(Z)) if xy else (None, None)
    with torch.cuda.device(d.device):
        adcensus._check(adcensus.lib().mccnn_disp_to_depth(
            d.data_ptr(), H, W, _f32(cal.f), _f32(cal.cx), _f32(cal.cy), fB(cal), _f32(cal.doffs), _cap(max_depth),
            Z.data_ptr(), None if X is None else X.data_ptr(), None if Y is None else Y.data_ptr(), adcensus._stream(d)), n)
    return (Z, X, Y) if xy else Z


def _colour(left, H, W, dev):
    """(left as contiguous CUDA uint8, nch) for a (H, W) grey or (H, W, 3) R, G, B byte image"""
    t = left if isinstance(left, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(left))
    if t.dtype != torch.uint8 or tuple(t.shape[:2]) != (H, W) or not (t.dim() == 2 or (t.dim() == 3 and t.size(2) == 3)):
        raise ValueError("left image: (%d, %d) or (%d, %d, 3) uint8 expected, got %s %s" % (H, W, H, W, t.dtype, tuple(t.shape)))
    return t.to(dev).contiguous(), 1 if t.dim() == 2 else 3


def point_cloud(disp, cal, left, conf=None, density=None, max_depth=None):
    """The :data:`Cloud` of `disp` under `cal`, coloured from the decoded left image `left` ((H, W) or (H, W, 3) uint8,
    host or device): one 15-byte vertex record per valid pixel, row-major (mccnn_point_cloud_count / _fill).  With `conf`
    and `density`, only the pixels confidence.sparsify keeps.  One int64 is read back (the count); the records stay on the
    device."""
    if (conf is None) != (density is None):
        raise ValueError("conf and density go together")
    d, H, W = _map(disp, "disp", "mccnn_point_cloud_fill")
    rgb, nch = _colour(left, H, W, d.device)
    cap = _cap(max_depth)
    with torch.cuda.device(d.device):
        if conf is not None:
            d = confidence.sparsify(d, conf, density)
        lib, s = adcensus.lib(), adcensus._stream(d)
        count = torch.empty(1, dtype=torch.int64, device=d.device)
        adcensus._check(lib.mccnn_point_cloud_count(d.data_ptr(), H, W, fB(cal), _f32(cal.doffs), cap, count.data_ptr(), s),
                        "mccnn_point_cloud_count")
        npts = int(count.item())
        data = torch.empty(max(1, npts) * REC, dtype=torch.uint8, device=d.device)
        adcensus._check(lib.mccnn_point_cloud_fill(d.data_ptr(), rgb.data_ptr(), nch, H, W, _f32(cal.f), _f32(cal.cx),
                                                   _f32(cal.cy), fB(cal), _f32(cal.doffs), cap, data.data_ptr(), npts, s),
                        "mccnn_point_cloud_fill")
    return Cloud(data[:npts * REC], npts)


def ply_bytes(n):
    """the PLY header of an n-vertex cloud"""
    return (PLY_HEADER % n).encode("ascii")


def write_ply(path, pts):
    """`pts` (a :data:`Cloud`) as a binary little-endian PLY file: the header, then the records in one device-to-host copy
    and one write"""
    body = pts.data.cpu().numpy() if isinstance(pts.data, torch.Tensor) else np.asarray(pts.data, np.uint8)
    with open(path, "wb") as f:
        f.write(ply_bytes(pts.n))
        f.write(memoryview(np.ascontiguousarray(body)))


def read_ply(path):
    """(xyz (n, 3) float32, rgb (n, 3) uint8) of a file :func:`write_ply` wrote"""
    with open(path, "rb") as f:
        raw = f.read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    n = int(raw[:end].split(b"element vertex ")[1].split(b"\n")[0])
    if raw[:end] != ply_bytes(n):
        raise ValueError("%s: not a point cloud of this format" % path)
    rec = np.frombuffer(raw, np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]), count=n, offset=end)
    return rec["xyz"].copy(), rec["rgb"].copy()


MESH_HEADER = PLY_HEADER.replace("end_header\n", "element face %d\nproperty list uchar int vertex_indices\nend_header\n")
FACE_REC = np.dtype([("n", "u1"), ("v", "<i4", 3)])     # a face: the count 3, then three int32 vertex indices

Mesh = namedtuple("Mesh", "data n faces")  # data: (n * 15,) CUDA uint8 vertex records; faces: (F, 3) CUDA int32


def mesh_ply_bytes(nv, nf):
    """the PLY header of a mesh of nv vertices and nf triangles"""
    return (MESH_HEADER % (nv, nf)).encode("ascii")


def write_mesh_ply(path, mesh):
    """`mesh` (a :data:`Mesh`) as a binary little-endian PLY file: :func:`write_ply`'s vertex element, then ``element face``
    with ``property list uchar int vertex_indices`` (13 bytes per triangle)"""
    body = mesh.data.cpu().numpy() if hasattr(mesh.data, "cpu") else np.asarray(mesh.data, np.uint8)
    faces = mesh.faces.cpu().numpy() if hasattr(mesh.faces, "cpu") else np.asarray(mesh.faces, np.int32)
    rec = np.zeros(len(faces), FACE_REC)
    rec["n"], rec["v"] = 3, faces.reshape(-1, 3)
    with open(path, "wb") as f:
        f.write(mesh_ply_bytes(mesh.n, len(faces)))
        f.write(memoryview(np.ascontiguousarray(body)))
        f.write(memoryview(rec))


def read_mesh_ply(path):
    """(xyz (n, 3) float32, rgb (n, 3) uint8, faces (F, 3) int32) of a file :func:`write_mesh_ply` wrote"""
    with open(path, "rb") as f:
        raw = f.read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    head = raw[:end]
    try:
        nv = int(head.split(b"element vertex ")[1].split(b"\n")[0])
        nf = int(head.split(b"element face ")[1].split(b"\n")[0])
    except (IndexError, ValueError):
        raise ValueError("%s: not a mesh of this format" % path) from None
    if head != mesh_ply_bytes(nv, nf) or len(raw) != end + REC * nv + FACE_REC.itemsize * nf:
        raise ValueError("%s: not a mesh of this format" % path)
    rec = np.frombuffer(raw, np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]), count=nv, offset=end)
    fr = np.frombuffer(raw, FACE_REC, count=nf, offset=end + REC * nv)
    if nf and not (fr["n"] == 3).all():
        raise ValueError("%s: a face is not a triangle" % path)
    return rec["xyz"].copy(), rec["rgb"].copy(), fr["v"].astype(np.int32)


def counts(disp, gt, cal, min_depth=MIN_DEPTH, max_depth=KITTI_MAX_DEPTH, is_depth=False):
    """(counts (NCOUNT,) int64, sums (NSUM,) float64) CUDA tensors of mccnn_depth_metrics: `disp` and the ground-truth
    disparity `gt` (0 or non-finite = none), CUDA float32 maps of one shape.  max_depth None: no cap.  With `is_depth`,
    `disp` holds depths in metres (valid where finite and > 0), e.g. a depth PNG read back."""
    n = "mccnn_depth_metrics"
    d, H, W = _map(disp, "disp", n)
    g, Hg, Wg = _map(gt, "gt", n)
    if (Hg, Wg) != (H, W):
        raise ValueError("%s: gt is %dx%d, disp %dx%d" % (n, Hg, Wg, H, W))
    if not (min_depth > 0 and (max_depth is None or min_depth <= max_depth)):
        raise ValueError("need 0 < min_depth <= max_depth, got %r, %r" % (min_depth, max_depth))
    c = torch.empty(NCOUNT, dtype=torch.int64, device=d.device)
    s = torch.empty(NSUM, dtype=torch.float64, device=d.device)
    with torch.cuda.device(d.device):
        g = g.to(d.device).contiguous()
        adcensus._check(adcensus.lib().mccnn_depth_metrics(d.data_ptr(), int(is_depth), g.data_ptr(), H, W, fB(cal),
                                                           _f32(cal.doffs), _f32(min_depth), _cap(max_depth), c.data_ptr(),
                                                           s.data_ptr(), adcensus._stream(d)), n)
    return c, s


def metrics_of(c, s):
    """:data:`DepthMetrics` of host counts and sums; every mean is NaN when no pixel is scored"""
    c = [int(v) for v in np.asarray(c).reshape(-1)]
    s = [float(v) for v in np.asarray(s, np.float64).reshape(-1)]
    n, nan = c[N], float("nan")
    q = lambda a: a / n if n else nan
    return DepthMetrics(q(s[0]), q(s[1]), math.sqrt(q(s[2])), math.sqrt(q(s[3])), q(c[A1]), q(c[A2]), q(c[A3]), n,
                        n / c[GT] if c[GT] else nan)


def metrics(disp, gt, cal, min_depth=MIN_DEPTH, max_depth=KITTI_MAX_DEPTH, is_depth=False):
    """:data:`DepthMetrics` of `disp` against the ground-truth disparity `gt` under `cal` (see the module docstring)"""
    c, s = counts(disp, gt, cal, min_depth, max_depth, is_depth)
    return metrics_of(c.cpu(), s.cpu())


def velo_depth(pts, cal, H, W, min_depth=MIN_DEPTH):
    """The (H, W) CUDA float32 depth map of the CUDA LiDAR scan `pts` ((N, 4) float32: x, y, z, reflectance) under
    ``cal.velo`` (a :data:`dataio.RawCalib`, or any 12 numbers of a row-major 3x4 matrix, rounded once to fp32): each pixel
    the smallest camera depth z > min_depth of the points projecting onto it, 0 where none does (mccnn_velo_depth_map,
    DESIGN §21)."""
    n = "mccnn_velo_depth_map"
    if not isinstance(pts, torch.Tensor) or not pts.is_cuda or pts.dtype != torch.float32:
        raise adcensus.AdcensusError("%s: pts must be a CUDA float32 tensor" % n)
    if pts.dim() != 2 or pts.size(1) != 4:
        raise adcensus.AdcensusError("%s: pts must be (N, 4), got %s" % (n, tuple(pts.shape)))
    velo = getattr(cal, "velo", cal)
    P = np.asarray(velo, dtype=np.float64).reshape(-1).astype(np.float32)
    if P.size != 12:
        raise ValueError("%s: a 3x4 matrix expected, got %d numbers" % (n, P.size))
    if not min_depth >= 0:
        raise ValueError("min_depth must be >= 0, got %r" % (min_depth,))
    p = pts.contiguous()
    if p.data_ptr() % 16:
        p = p.clone()
    Z = torch.empty((int(H), int(W)), device=p.device, dtype=torch.float32)
    with torch.cuda.device(p.device):
        adcensus._check(adcensus.lib().mccnn_velo_depth_map(p.data_ptr() if p.numel() else None, p.size(0),
                                                            P.ctypes.data, int(H), int(W), _f32(min_depth), Z.data_ptr(),
                                                            adcensus._stream(p)), n)
    return Z


def disparity_of_depth(Z, cal):
    """the disparity fB / Z (fp32) of a CUDA depth map `Z` with doffs 0, NaN where Z is not > 0: mccnn_disp_to_depth, the
    same map in the other direction.  It turns a scan's depth map into the ground-truth disparity :func:`metrics` takes."""
    if float(cal.doffs) != 0.0:
        raise ValueError("a depth map becomes a disparity this way only when doffs = 0, got %r" % (cal.doffs,))
    return depth(Z, cal)
