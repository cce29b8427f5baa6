"""CPU: the truncated signed distance field (DESIGN §24) -- the numpy restatement (tests/tsdf_oracle.py) against a
brute-force loop, its marching tetrahedra (orientation of every case, a closed sphere, a flat plane), its ray cast of a
plane, the mesh PLY round trip, and every refusal of TSDF, fuse_drive and tools/fuse_raw.py."""
import importlib.util
import os

import numpy as np
import pytest

import mccnn_b200  # noqa: F401
from mccnn_b200 import dataio, depth, fusion, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


to = _load("tsdf_oracle", "tests", "tsdf_oracle.py")
fuse_tool = _load("fuse_raw_tool", "tools", "fuse_raw.py")
CAL = dataio.Calib(50.0, 15.3, 11.7, 0.5, 0.0, None, None)


def _pose(rng, rot=0.1, trans=0.2):
    P = np.eye(4)
    P[:3, :3] = synth._rodrigues(rng.uniform(-1, 1, 3) * rot)
    P[:3, 3] = rng.uniform(-trans, trans, 3)
    return P


def test_integration_is_a_brute_force_loop():
    """every voxel against every pixel: the pixel whose centre lies within half a pixel of the projection"""
    rng = np.random.default_rng(1)
    H, W = 24, 32
    d = rng.uniform(8, 14, (H, W)).astype(np.float32)
    d[rng.random((H, W)) < 0.1] = np.nan
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    P = _pose(rng)
    voxel, mu = 0.07, 0.2
    f = to.Field(voxel, mu)
    fk, pix, out = to.alloc_keys(d, CAL, P, voxel, mu)
    assert pix == int(np.isfinite(d).sum()) and out == 0
    f.allocate(fk)
    f.integrate(d, CAL, img, P)
    Z = to.depth_oracle.depth32(d, CAL)[0]
    c = to.centres(f.keys, voxel).reshape(-1, 3)
    S, n, nc, col = np.zeros(len(c)), np.zeros(len(c), np.int64), np.zeros(len(c), np.int64), np.zeros((len(c), 3), np.int64)
    R, t = P[:3, :3], P[:3, 3]
    fx, cx, cy = float(np.float32(CAL.f)), float(np.float32(CAL.cx)), float(np.float32(CAL.cy))
    for k in range(len(c)):
        q = R.T @ (c[k] - t)
        if q[2] <= 0:
            continue
        u, v = q[0] / q[2] * fx + cx, q[1] / q[2] * fx + cy
        for y in range(H):
            for x in range(W):
                if abs(u - x) <= 0.5 and abs(v - y) <= 0.5 and not np.isnan(Z[y, x]):
                    eta = float(Z[y, x]) - q[2]
                    if eta >= -mu:
                        S[k] += min(eta, mu) / mu
                        n[k] += 1
                        if abs(eta) < mu:
                            col[k] += img[y, x]
                            nc[k] += 1
    assert np.array_equal(f.n.reshape(-1), n) and np.array_equal(f.nc.reshape(-1), nc)
    assert np.array_equal(f.col.reshape(-1, 3), col)
    assert np.allclose(f.S.reshape(-1), S, rtol=0, atol=1e-12)
    assert n.sum() > 1000 and nc.sum() > 100 and (n > 0).sum() < len(n)


def test_every_tetrahedron_case_faces_positive_phi():
    rng = np.random.default_rng(3)
    cube = np.array([[o & 1, (o >> 1) & 1, (o >> 2) & 1] for o in range(8)], np.float64)
    for ti, tet in enumerate(to.TETS):
        P = cube[list(tet)]
        assert (np.linalg.det(P[1:] - P[0]) < 0) == to.TET_ODD[ti]
        for case in range(16):
            neg = [(case >> k) & 1 for k in range(4)]
            tris = to.tet_triangles(neg, to.TET_ODD[ti])
            assert len(tris) == {0: 0, 1: 1, 2: 2, 3: 1, 4: 0}[sum(neg)]
            for _ in range(5):
                phi = np.where(neg, -rng.uniform(0.1, 1, 4), rng.uniform(0.1, 1, 4))
                grad = np.linalg.solve(P[1:] - P[0], phi[1:] - phi[0])     # the linear field's gradient
                for tri in tris:
                    v = [P[a] + phi[a] / (phi[a] - phi[b]) * (P[b] - P[a]) for a, b in tri]
                    nrm = np.cross(v[1] - v[0], v[2] - v[0])
                    assert nrm @ grad > 0, (ti, case, tri)


def _field_of(fn, voxel, lo, hi):
    """a Field whose every voxel in bricks lo .. hi (brick indices) holds phi = fn(centre), observed once"""
    r = np.arange(lo, hi + 1)
    b = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3)
    keys, _ = to.brick_keys(b)
    f = to.Field(voxel)
    f.allocate(np.sort(keys))
    c = to.centres(f.keys, voxel)
    f.S[:] = fn(c)
    f.n[:] = 1
    f.nc[:] = 1
    f.col[:] = 100
    return f


def _edges(faces):
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    return e


def test_sphere_mesh_is_closed_and_on_the_sphere():
    voxel, R = 0.1, 1.23
    centre = np.array([0.013, -0.021, 0.007])
    f = _field_of(lambda c: (np.linalg.norm(c - centre, axis=-1) - R) / 0.4, voxel, -2, 1)
    xyz, rgb, faces = f.mesh()
    used = np.unique(faces)
    assert len(used) == len(xyz) and len(faces) > 1000
    e = _edges(faces)
    directed = {tuple(x) for x in e.tolist()}
    assert len(directed) == len(e)                                   # no directed edge twice: consistent orientation
    assert all((b, a) in directed for a, b in directed)              # every edge shared by two faces, opposite ways
    E = len(e) // 2
    assert len(xyz) - E + len(faces) == 2
    r = np.linalg.norm(xyz.astype(np.float64) - centre, axis=1)
    assert np.abs(r - R).max() < 0.05 * voxel, np.abs(r - R).max()
    assert R >= 10 * voxel
    # outward normals: positive phi outside
    tri = xyz[faces].astype(np.float64)
    nrm = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    assert ((nrm * (tri.mean(1) - centre)).sum(1) > 0).all()
    assert (rgb == 100).all()


def test_plane_mesh_is_flat():
    voxel = 0.05
    n = np.array([0.3, -0.5, 0.8])
    n /= np.linalg.norm(n)
    f = _field_of(lambda c: (c @ n - 0.031) / 0.2, voxel, -1, 0)
    xyz, _, faces = f.mesh()
    assert len(faces) > 200
    assert np.abs(xyz.astype(np.float64) @ n - 0.031).max() < 1e-6
    tri = xyz[faces].astype(np.float64)
    nrm = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    area = np.linalg.norm(nrm, axis=1)
    assert (nrm[area > 1e-9] @ n > 0).all()


def test_render_of_a_plane_is_its_depth():
    """phi = (d - z) / mu of the plane z = d in front of an identity camera: every ray meets it at depth d"""
    voxel, zp = 0.1, 1.537
    f = _field_of(lambda c: (zp - c[..., 2]) / 0.4, voxel, -1, 2)
    cal = dataio.Calib(20.0, 7.5, 5.5, 0.5, 0.0, None, None)
    Z = f.render(cal, np.eye(4), 12, 16)
    assert np.isfinite(Z).all()
    assert np.abs(Z - zp).max() < 1e-5
    assert np.isnan(f.render(cal, np.eye(4), 12, 16, max_depth=1.0)).all()
    assert np.isnan(f.render(cal, np.eye(4), 12, 16, min_frames=2)).all()


def test_mesh_ply_round_trip(tmp_path):
    rng = np.random.default_rng(5)
    xyz = rng.normal(size=(17, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (17, 3), dtype=np.uint8)
    faces = rng.integers(0, 17, (23, 3)).astype(np.int32)
    rec = np.zeros(17, np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))
    rec["xyz"], rec["rgb"] = xyz, rgb
    p = str(tmp_path / "m.ply")
    depth.write_mesh_ply(p, depth.Mesh(np.frombuffer(rec.tobytes(), np.uint8), 17, faces))
    assert open(p, "rb").read() == to.mesh_ply_bytes(xyz, rgb, faces)
    x2, r2, f2 = depth.read_mesh_ply(p)
    assert np.array_equal(x2, xyz) and np.array_equal(r2, rgb) and np.array_equal(f2, faces)
    depth.write_mesh_ply(p, depth.Mesh(np.zeros(0, np.uint8), 0, np.zeros((0, 3), np.int32)))
    x2, r2, f2 = depth.read_mesh_ply(p)
    assert len(x2) == len(f2) == 0
    with open(p, "ab") as fh:
        fh.write(b"x")
    with pytest.raises(ValueError, match="not a mesh"):
        depth.read_mesh_ply(p)
    depth.write_ply(p, depth.Cloud(np.zeros(0, np.uint8), 0))
    with pytest.raises(ValueError, match="not a mesh"):
        depth.read_mesh_ply(p)


def test_trunc_refusals():
    assert fusion.check_trunc(None, 0.1) == pytest.approx(0.4)
    assert fusion.check_trunc(0.1, 0.1) == 0.1
    assert fusion.check_trunc(25.6, 0.1) == 25.6
    for bad in (0.05, 25.7, float("nan"), float("inf"), -1.0, "0.4"):
        with pytest.raises(ValueError, match="trunc must be"):
            fusion.check_trunc(bad, 0.1)


def _base(drive, out):
    return ["kitti", "census", "-drive", drive, "-out", out, "-voxel", "0.1"]


def test_fuse_raw_refusals(tmp_path, monkeypatch):
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    drive, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "raw"), n=2, H=24, W=64)
    out = str(tmp_path / "out")
    for extra, msg in ((["-trunc", "0.4"], "-trunc is the distance field"), (["-score"], "-score renders"),
                       (["-mesh", "-trunc", "0.05"], "-trunc must be"), (["-mesh", "-trunc", "nan"], "-trunc must be"),
                       (["-mesh", "-trunc", "inf"], "-trunc must be"), (["-mesh", "-trunc", "30"], "-trunc must be"), (["-mesh", "-score", "-min_depth", "0"], "-min_depth")):
        with pytest.raises(SystemExit, match=msg):
            fuse_tool.parse_args(_base(drive, out) + extra)
    with pytest.raises(SystemExit):
        fuse_tool.parse_args(_base(drive, out) + ["-mesh", "-score", "-crop", "kitti"])
    args = fuse_tool.parse_args(_base(drive, out) + ["-mesh", "-score", "-crop", "garg", "-trunc", "0.3"])
    assert args.mesh and args.score and args.crop == "garg" and args.trunc == 0.3
    # refused by fuse_drive before any GPU work
    os.makedirs(os.path.join(out, predict_name(drive)))
    open(os.path.join(out, predict_name(drive), "mesh.ply"), "w").close()
    with pytest.raises(ValueError, match="mesh.ply exists"):
        fusion.fuse_drive("kitti", "census", [drive], out=out, mesh=True)
    out2 = str(tmp_path / "out2")
    with pytest.raises(ValueError, match="velodyne_points lacks"):
        fusion.fuse_drive("kitti", "census", [drive], out=out2, mesh=True, score=True)
    for kw, msg in ((dict(trunc=0.4), "need mesh"), (dict(score=True), "need mesh"), (dict(mesh=True, trunc=0.01), "trunc must"),
                    (dict(mesh=True, score=True, crop="x"), "crop must"), (dict(mesh=True, score=True, min_depth=0.0), "min_depth")):
        with pytest.raises(ValueError, match=msg):
            fusion.fuse_drive("kitti", "census", [drive], out=out2, **kw)
    assert not os.path.exists(out2)


def predict_name(drive):
    return os.path.basename(drive)


def test_posed_drive_scans(tmp_path):
    """velodyne=False keeps today's files; with True every frame has a scan of points on the planes"""
    a, _, _, _ = synth.write_kitti_posed_drive(str(tmp_path / "a"), n=2, H=24, W=64)
    b, _, _, poses = synth.write_kitti_posed_drive(str(tmp_path / "b"), n=2, H=24, W=64, velodyne=True)
    assert not os.path.exists(os.path.join(a, "velodyne_points"))
    for sub in ("image_00", "image_01", "oxts"):
        for k in range(2):
            name = dataio.raw_file(a, (sub, "data", "%010d.txt" if sub == "oxts" else "%010d.png"), k)
            assert open(name, "rb").read() == open(name.replace(str(tmp_path / "a"), str(tmp_path / "b")), "rb").read()
    assert dataio.raw_frames(b, velodyne=True) == [0, 1]
    cal = dataio.read_calib(os.path.dirname(b), "kitti_raw")
    for k in range(2):
        scan = dataio.read_velodyne(dataio.raw_file(b, dataio.RAW_SCAN, k)).astype(np.float64)
        assert len(scan) > 100
        # back into the world frame: on one of the planes
        R_rect = synth._rodrigues(synth.POSED_R_RECT_ROT)
        p_rect = scan[:, :3] @ np.asarray(synth.RAW_VELO_R).reshape(3, 3).T @ R_rect.T
        w = p_rect @ poses[k][:3, :3].T + poses[k][:3, 3]
        d = np.min([np.abs(w @ np.asarray(nrm) - off) for nrm, off in synth.POSED_PLANES], axis=0)
        assert d.max() < 1e-4
        assert cal.velo is not None
