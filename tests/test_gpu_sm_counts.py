"""GPU: every launch sized by the SM count gives the same outputs at any SM count.  tests/sm_count_runs.py runs the cases in
a subprocess at ADCENSUS_NUM_SMS = 1, 7 and 114 and once with the variable unset (the device's own count).  At one SM every
capped loop of the small cases wraps, the 1 x 2049-style cases go one element past the cap, and 114 SMs are the other
H100's grids at the full KITTI, raw KITTI and Middlebury sizes.  At every count each output equals the numpy oracle (bit
for bit, or within the tower's and the Lanczos half's documented bars where those have no bit-exact oracle) and the four
runs are byte-identical."""
import importlib.util
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import confidence, depth, frontend, rectify  # noqa: E402
from oracle import kitti_devkit as kd  # noqa: E402
from oracle import preprocess as opp  # noqa: E402
from oracle import preprocess_mb as opm  # noqa: E402
from oracle import render as orr  # noqa: E402
from oracle import tower_head_cases as thc  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


runs_mod = _load("sm_count_runs")
mc = runs_mod.mc
do = _load("depth_oracle")
ro = _load("raw_oracle")
rco = _load("rectify_oracle")
oc = _load("confidence_oracle")
fo = _load("fusion_oracle")
to = _load("tsdf_oracle")

FORCED = (1, 7, 114)
TIMEOUT = 1800                   # seconds per subprocess


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """{label: (SM count the library reported, npz)}: one run per forced count and one with the variable unset"""
    tmp = tmp_path_factory.mktemp("sm_counts")
    out = {}
    for s in FORCED + (None,):
        env = dict(os.environ)
        env.pop("ADCENSUS_NUM_SMS", None)
        if s is not None:
            env["ADCENSUS_NUM_SMS"] = str(s)
        path = str(tmp / ("s%s.npz" % s))
        t0 = time.time()
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "sm_count_runs.py"), path], cwd=ROOT, env=env,
                           capture_output=True, text=True, timeout=TIMEOUT)
        assert r.returncode == 0, "ADCENSUS_NUM_SMS=%s: exit %d\n%s\n%s" % (s, r.returncode, r.stdout, r.stderr[-4000:])
        z = np.load(path)
        print("ADCENSUS_NUM_SMS=%s: the library used %d SMs, %.1f s" % (s, int(z["num_sms"]), time.time() - t0))
        out[s] = (int(z["num_sms"]), z)
    return out


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_the_hook_took_effect(runs):
    assert [runs[s][0] for s in FORCED] == list(FORCED)
    assert runs[None][0] == device_sms()


def bits_equal(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, "%s: %s %s, want %s %s" % (
        what, got.shape, got.dtype, want.shape, want.dtype)
    if got.dtype.kind == "f":
        u = np.dtype("u%d" % got.dtype.itemsize)
        same = (got.view(u) == want.view(u)) | (np.isnan(got) & np.isnan(want))
    else:
        same = got == want
    bad = np.argwhere(~same)
    assert not len(bad), "%s: %d of %d entries differ, first at %s (%r, want %r)" % (
        what, len(bad), same.size, bad[0], got[tuple(bad[0])], want[tuple(bad[0])])


def half_within_bar(img, got, what):
    """the Lanczos half against the float64 oracle: a byte may differ by one only where the oracle is within 1e-3 of a
    half-integer (tests/test_gpu_preprocess_mb.py's bar)"""
    f = opm.half_image_f64(img)
    want = np.clip(np.floor(f + 0.5), 0, 255).astype(np.uint8)
    near = np.abs(f - np.floor(f) - 0.5) < 1e-3
    bad = (got != want) & ~near
    assert not bad.any(), "%s: %d bytes differ away from a half-integer" % (what, int(bad.sum()))
    assert (np.abs(got.astype(int) - want.astype(int)) <= 1).all(), what


def oracle_outputs(c, inp):
    """{name: want} of the outputs that have a bit-exact oracle, and a list of (name, check(got)) of the others"""
    a = c.args
    if c.kind == "depth":
        Z, X, Y = do.depth32(inp["d"], inp["cal"], None)
        return dict(Z=Z, X=X, Y=Y), []
    if c.kind == "velo":
        return dict(depth=ro.velo_depth_map(inp["pts"], inp["P"], a["H"], a["W"], 1e-3)), []
    if c.kind == "render":
        return dict(volume_grey=orr.volume_grey(inp["vol"]), map_grey=orr.map_grey(inp["x"], 70),
                    grey2jet=orr.grey2jet(inp["jet"], 70, mask_blue=True),
                    error_image=orr.error_image(inp["x0"], inp["pred"], inp["gt"], 3.0)), []
    if c.kind == "kitti_eval":
        with np.errstate(invalid="ignore"):
            v = kd.png16_values(inp["disp"])
        counts, sums, ipol = kd.devkit_counts(v, inp["noc"], inp["occ"], inp["obj"])
        gt = inp["noc"].astype(np.float32) / np.float32(256)
        with np.errstate(invalid="ignore"):
            bad = (inp["noc"] != 0) & (np.abs(gt - inp["disp"]) > np.float32(3.0))
        want = dict(ipol=ipol, counts=counts, error_counts=np.array([bad.sum(), (inp["noc"] != 0).sum()], np.int64))
        return want, [("sums", lambda g: np.testing.assert_allclose(g, sums, rtol=1e-12, atol=0))]
    if c.kind == "rectify":
        (Wo, Ho), rect = a["rect"], inp["rect"]
        wl, wv = rco.rectify(inp["left"], rectify.params(rect.left), Ho, Wo)
        wr, _ = rco.rectify(inp["right"], rectify.params(rect.right), Ho, Wo)
        return dict(left=wl, right=wr, valid=wv.astype(np.uint8)), []
    if c.kind == "frontend":
        f = lambda b: b.astype(np.float32) if b.ndim == 2 else np.ascontiguousarray(b.transpose(2, 0, 1).astype(np.float32))
        return dict(x_batch=frontend.make_batch(f(inp["left"]), f(inp["right"]))), []
    if c.kind == "preprocess":
        return dict(nonvisible=opp.remove_nonvisible(inp["y"]), white=opp.remove_white(inp["x0"], inp["y"])), []
    if c.kind == "preprocess_mb":
        return dict(half_disp=opm.half_disp(inp["d"]), mask=opm.mask(inp["d0"], inp["d1"], inp["dy"])), \
            [("half_image", lambda g: half_within_bar(inp["img"], g, c.name))]
    if c.kind == "fill_nan":
        want = {}
        for n in a["ns"]:
            for o in range(4):
                w = np.full(n + 8, 7.0, np.float32)
                w[o:o + n] = np.nan
                want["n%d_offset%d" % (n, o)] = w
        return want, []
    if c.kind == "confidence":
        H, W = a["H"], a["W"]
        want = {"sparsify_%g" % d: oc.sparsify(inp["disp"], inp["conf"], confidence.n_keep(d, H, W), np.nan)
                for d in (0.5, 1e-7, 1.0)}
        M, B, bad = oc.counts(inp["disp"], inp["conf"], inp["gt"], 3.0)
        want["counts"] = np.array([M, B] + bad, np.int64)
        return want, []
    if c.kind == "tower":
        if a["H"] * a["W"] > 10000:
            return {}, []                        # the full-size tower: the runs agree with the device's own grid below
        want = thc.tower_want(inp["x"], inp["layers"], "fast")
        scale = max(1.0, float(np.abs(want).max()))
        return {}, [("nterms3", lambda g: np.testing.assert_array_less(np.abs(g - want).max(), 1e-4 * scale + 1e-30)),
                    ("nterms1", lambda g: np.testing.assert_array_less(np.abs(g - want).max(), 5e-2 * scale + 1e-30))]
    if c.kind == "fusion":
        ref = fo.Table(a["voxel"])
        for d, cal, img, pose in inp["frames"]:
            ref.add(d, cal, img, pose)
        want = dict(keys=ref.keys, n_pix=ref.n_pix, n_frames=ref.n_frames, sums=ref.sums, colours=ref.colours,
                    stats=np.array([ref.pixels, ref.outside, len(ref.keys)], np.int64))
        for m in (1, 2, 3):
            ply = depth.ply_bytes(int((ref.n_frames >= m).sum())) + ref.records(m)
            want["ply_%d" % m] = np.frombuffer(ply, np.uint8)
        return want, []
    if c.kind == "tsdf":
        ref = to.Field(a["voxel"], a["trunc"])
        for d, cal, img, pose in inp["frames"]:
            ref.add(d, cal, img, pose)
        n = len(ref.keys)
        want = dict(keys=ref.keys, S=ref.S.reshape(n * 512), n=ref.n.reshape(n * 512), nc=ref.nc.reshape(n * 512),
                    colours=ref.col.reshape(n * 512, 3), stats=np.array([ref.pixels, ref.outside, n], np.int64))
        for m in (1, 2):
            want["mesh_%d" % m] = np.frombuffer(ref.mesh_ply(m), np.uint8)
        cal, H, W = runs_mod.render_camera(inp["frames"][0][1], a["H"], a["W"])
        for k, (_, _, _, pose) in enumerate(inp["frames"]):
            want["render_%d" % k] = ref.render(cal, pose, H, W, 1)
        want["render_min2"] = ref.render(cal, inp["frames"][-1][3], H, W, 2)
        return want, []
    raise ValueError(c.kind)


@pytest.mark.parametrize("name", [c.name for c in runs_mod.CASES])
def test_outputs_are_the_oracle_at_every_sm_count(runs, name):
    c = runs_mod.case(name)
    inp = runs_mod.inputs(c)
    want, checks = oracle_outputs(c, inp)
    sizes = runs_mod.map_sizes(c, inp) if c.kind in ("fusion", "tsdf") else None
    labels = list(FORCED) + [None]
    keys = sorted(k for k in runs[None][1].files if k.startswith(name + "/"))
    assert keys, name
    for s in labels:
        sms, z = runs[s]
        wrapped = ["%s (%d)" % (launch, mc.sm_passes(cap, n, sms)) for cap, launch, n in runs_mod.loops(c, inp, sizes)
                   if mc.sm_passes(cap, n, sms) > 1]
        print("%s at %d SMs: loops that wrapped (passes): %s" % (name, sms, ", ".join(wrapped) or "none"))
        assert sorted(k for k in z.files if k.startswith(name + "/")) == keys
        for k in keys:
            out = k.split("/", 1)[1]
            got = z[k]
            if out in want:
                w = np.asarray(want[out])
                bits_equal(got, w.reshape(got.shape) if w.size == got.size and w.dtype == got.dtype else w,
                           "%s at %d SMs: %s" % (name, sms, out))
            for o, check in checks:
                if o == out:
                    check(got)
    assert set(want) | {o for o, _ in checks} <= {k.split("/", 1)[1] for k in keys}
    for k in keys:
        ref = runs[None][1][k]
        for s in FORCED:
            assert runs[s][1][k].tobytes() == ref.tobytes(), "%s: %s at %d SMs differs from the device's own count" % (
                name, k, s)
