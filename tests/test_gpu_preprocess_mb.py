"""GPU: the Middlebury kernels of csrc/preprocess_mb.cu against oracle/preprocess_mb.py, and tools/preprocess_mb.py end to end.

mccnn_mb_views and mccnn_mb_half_disp must equal the oracle (numpy's own mean / std, np.sort) bit for bit; the masks and
the lists exactly.  The halving is a restatement of ImageMagick's filter, not pinned against it: a byte may differ from the
float64 oracle only where the oracle's value lies within 1e-3 of a half-integer (fp32 against fp64 rounding)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, dataio, preprocess, synth  # noqa: E402
from oracle import preprocess_mb as opm  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "preprocess_mb")


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def views_of(rgb, color):
    return preprocess.mb_views(cu(np.stack(rgb)), 3 if color == "rgb" else 1).cpu().numpy()


def assert_bits(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, "%s: %s %s, want %s %s" % (
        what, got.shape, got.dtype, want.shape, want.dtype)
    bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
    assert not len(bad), "%s: %d entries differ, first at %s (%r, want %r)" % (
        what, len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])])


def images(seed, shape, n=2):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, shape + (3,)).astype(np.uint8) for _ in range(n)]


@pytest.mark.parametrize("color", ["gray", "rgb"])
@pytest.mark.parametrize("shape", [(1, 1), (1, 2), (1, 7), (1, 8), (2, 21), (1, 43), (1, 128), (1, 129), (3, 43), (16, 16),
                                   (61, 97), (64, 128), (1, 8191), (1, 8193), (997, 1483), (1000, 1500)], ids=str)
def test_views_equal_numpy_bit_for_bit(shape, color):
    rgb = images(shape[0] * 7919 + shape[1], shape, n=3)
    rgb[2][...] = rgb[2][..., :1]                                          # a grey file, replicated
    got = views_of(rgb, color)
    for k, im in enumerate(rgb):
        assert_bits(got[k:k + 1], opm.read_im(im, color), "%s %s view %d" % (shape, color, k))


def test_views_equal_the_scripts_read_im_fixtures(tmp_path):
    g = np.load(os.path.join(GOLDEN, "read_im.npz"))
    for name in sorted({k.split("/")[0] for k in g.files}):
        p = tmp_path / (name + "." + name.split("_")[1])
        p.write_bytes(g[name + "/file"].tobytes())
        rgb = opm.imread_rgb(str(p))
        for color in ("gray", "rgb"):
            assert_bits(views_of([rgb], color), g[name + "/" + color], "%s %s" % (name, color))


def test_half_disp_equals_load_pfm():
    g = np.load(os.path.join(GOLDEN, "pfm.npz"))
    for name in ("special_10x14", "random_36x50"):
        got = preprocess.mb_half_disp(cu(g[name + "/load"][None])).cpu().numpy()[0]
        assert_bits(got, g[name + "/half"], name)
    rng = np.random.default_rng(3)
    d = rng.uniform(0, 300, (3, 1000, 1500)).astype(np.float32)
    d[rng.random(d.shape) < 0.1] = np.inf
    d[rng.random(d.shape) < 0.02] = np.nan
    d[:, ::3] = np.floor(d[:, ::3])                                        # ties
    got = preprocess.mb_half_disp(cu(d)).cpu().numpy()
    for k in range(3):
        assert_bits(got[k], opm.half_disp(d[k]), "1000x1500 map %d" % k)


def maps(seed, H, W, with_dy):
    rng = np.random.default_rng(seed)
    blocks = rng.uniform(0, min(W, 60), (H, W // 16 + 1)).astype(np.float32)
    d0 = (np.repeat(blocks, 16, 1)[:, :W] + rng.uniform(0, 0.5, (H, W))).astype(np.float32)
    d0[rng.random(d0.shape) < 0.1] = np.inf
    d0[rng.random(d0.shape) < 0.02] = np.nan
    d0[:, :3] = np.float32(W + 5)                                           # out of frame on the left
    d1 = synth._mb_right_map(rng, d0)                                       # inf where nothing maps, some off by > 1
    d1[0, :] = np.floor(d0[0, :]) + np.float32(0.5)                         # differences of exactly 1 and ties of x - d0
    d0[0, ::2] = np.floor(d0[0, ::2]) + np.float32(0.5)
    dy = rng.uniform(-1.5, 1.5, (H, W)).astype(np.float32) if with_dy else None
    if with_dy:
        dy[-1, :] = 2                                                       # out of frame at the bottom
        dy[1, 1] = np.nan
    return d0, d1, dy


@pytest.mark.parametrize("with_dy", [False, True], ids=["no_dy", "dy"])
@pytest.mark.parametrize("H,W", [(5, 9), (37, 300), (1000, 1500)], ids=str)
def test_mask_and_lists_equal_the_oracle(H, W, with_dy):
    d0, d1, dy = maps(H * W + with_dy, H, W, with_dy)
    m = preprocess.mb_mask(cu(d0), cu(d1), cu(dy) if with_dy else None)
    want_m = opm.mask(d0, d1, dy)
    assert np.array_equal(m.cpu().numpy(), want_m)
    assert {0, 128, 255} <= set(np.unique(want_m).tolist()) or H * W < 100
    dispnoc, rows = preprocess.mb_nnz(cu(d0), m, 7)
    want_d, want_rows = opm.clean(d0, want_m, 7)
    assert_bits(dispnoc.cpu().numpy(), want_d, "dispnoc")
    assert_bits(rows.cpu().numpy(), want_rows, "rows")


def test_lists_take_a_given_mask_and_may_be_empty():
    d0 = np.arange(12, dtype=np.float32).reshape(3, 4)
    m = np.zeros((3, 4), np.uint8)
    dispnoc, rows = preprocess.mb_nnz(cu(d0), cu(m), 1)
    assert rows.shape == (0, 4) and not dispnoc.cpu().numpy().any()
    m[1, 2] = m[2, 0] = 255
    m[0, 0] = 128
    dispnoc, rows = preprocess.mb_nnz(cu(d0), cu(m), 3)
    assert rows.cpu().numpy().tolist() == [[3, 1, 2, 6], [3, 2, 0, 8]]


def check_half(img, got, what):
    """got (bytes) against the float64 oracle: a differing byte only where the oracle is within 1e-3 of a half-integer"""
    f = opm.half_image_f64(img)
    want = np.clip(np.floor(f + 0.5), 0, 255).astype(np.uint8)
    bad = got != want
    near = np.abs(f - np.floor(f) - 0.5) < 1e-3
    assert not (bad & ~near).any(), "%s: %d bytes differ away from a half-integer, first at %s" % (
        what, int((bad & ~near).sum()), np.argwhere(bad & ~near)[0])
    assert (np.abs(got.astype(int) - want.astype(int)) <= 1).all()
    return int(bad.sum())


@pytest.mark.parametrize("shape", [(1988, 2880), (2008, 2964), (2, 2), (4, 10), (6, 8), (10, 6), (8, 2), (12, 22)], ids=str)
def test_half_image_is_the_lanczos_rule(shape):
    rng = np.random.default_rng(shape[0] + shape[1])
    if shape[0] > 100:
        v = synth.natural_image(rng, shape[0] // 4, shape[1] // 4)
        img = np.clip(np.rint(128 + 60 * v), 0, 255).astype(np.uint8)
        img = np.repeat(np.repeat(img, 4, 0), 4, 1)[..., None] + rng.integers(0, 30, shape + (3,)).astype(np.uint8)
        img[:40, :40] = 255                                                 # a saturated corner: clamping
        img[-40:, -40:] = 0
    else:
        img = rng.integers(0, 256, shape + (3,)).astype(np.uint8)
    got = preprocess.mb_half_image(cu(img[None])).cpu().numpy()[0]
    check_half(img, got, str(shape))


def test_bad_arguments():
    with pytest.raises(adcensus.AdcensusError, match="invalid"):                 # odd sizes
        preprocess.mb_half_image(cu(np.zeros((1, 5, 4, 3), np.uint8)))
    with pytest.raises(adcensus.AdcensusError, match="invalid"):
        preprocess.mb_half_disp(cu(np.zeros((1, 4, 7), np.float32)))
    with pytest.raises(adcensus.AdcensusError, match="uint8"):
        preprocess.mb_views(cu(np.zeros((1, 4, 4, 3), np.float32)), 1)


# ---- end to end -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def raw_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("mb_raw"))
    synth.write_mb_raw(root, seed=5)
    return root


def load_outputs(d):
    out = {}
    for f in sorted(os.listdir(d)):
        if f.endswith(".bin"):
            dim = open(os.path.join(d, f + ".dim")).read()
            out[f] = None if dim.strip() == "0" else dataio.fromfile(os.path.join(d, f))
    return out


def device_half(img):
    got = preprocess.mb_half_image(cu(img[None])).cpu().numpy()[0]
    check_half(img, got, "view")
    return got


@pytest.mark.parametrize("rect,color", [("imperfect", "gray"), ("perfect", "gray"), ("imperfect", "rgb"), ("perfect", "rgb")])
def test_tool_end_to_end_equals_the_oracle(raw_root, rect, color):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "preprocess_mb.py"), rect, color, "-data_root", raw_root,
                        "-gpu", "1"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.split("\n")
    assert lines[:11] == ["Scene%02d" % k for k in range(11)] and lines[12:14] == ["Aloe", "Baby1"]
    want = opm.preprocess_mb(raw_root, rect, color, half=device_half)
    d = preprocess.mb_output_dir(raw_root, rect, color)
    got = load_outputs(d)
    n = len(want["X"])
    names = {"x_%d_%d.bin" % (i + 1, j + 1) for i in range(n) for j in range(len(want["X"][i]))}
    names |= {"dispnoc%d.bin" % (i + 1) for i in range(len(want["dispnoc"]))} | {"meta.bin", "nnz_tr.bin", "nnz_te.bin",
                                                                                   "te.bin"}
    assert set(got) == names
    for i, XX in enumerate(want["X"]):
        for j, x in enumerate(XX):
            f = "x_%d_%d.bin" % (i + 1, j + 1)
            if x is None:
                assert got[f] is None and os.path.getsize(os.path.join(d, f)) == 0
            else:
                assert_bits(got[f], x, f)
    for i, x in enumerate(want["dispnoc"]):
        assert_bits(got["dispnoc%d.bin" % (i + 1)], x, "dispnoc%d" % (i + 1))
    for k in ("meta", "nnz_tr", "nnz_te", "te"):
        assert got[k + ".bin"].dtype == want[k].dtype and np.array_equal(got[k + ".bin"], want[k]), k
    assert open(os.path.join(d, "fname_submit.txt")).read() == want["fname_submit"]
    # scene 3 carries .H caches for every view: its views are the caches' bytes through read_im
    base = os.path.join(raw_root, opm.MB, "scenes2014", "datasets", "Scene02-imperfect")
    cache = opm.imread_rgb(os.path.join(base, "im0.png.H.png"))
    assert_bits(got["x_3_1.bin"][:1], opm.read_im(cache, color), "cached im0")
    assert np.array_equal(got["nnz_te.bin"][:, 0], np.sort(got["nnz_te.bin"][:, 0]))
    assert set(np.unique(got["nnz_te.bin"][:, 0]).tolist()) <= set(range(1, 11))


def test_run_main_reads_the_gray_output(raw_root, tmp_path):
    d = preprocess.mb_output_dir(raw_root, "imperfect", "gray")
    if not os.path.exists(os.path.join(d, "meta.bin")):
        preprocess.preprocess_mb(raw_root, "imperfect", "gray", log=None)
    tool = os.path.join(ROOT, "tools", "run_main.py")
    for action in ("test_te", "submit"):
        r = subprocess.run([sys.executable, tool, "mb", "census", "-a", action, "-data_root", raw_root, "-out",
                            str(tmp_path / "out")], capture_output=True, text=True, timeout=1800, cwd=str(tmp_path))
        assert r.returncode == 0, "%s: %s" % (action, r.stderr[-3000:])
        if action == "test_te":
            assert r.stdout.strip()
    # submit's last 30 images are the MiddEval3 pairs: one disparity map per fname_submit line
    subs = open(os.path.join(d, "fname_submit.txt")).read().split("\n")
    assert len(subs) == 30 and subs[0].startswith("trainingH/") and subs[-1].startswith("testH/")
    for s in subs:
        got = [f for f in os.listdir(str(tmp_path / "out" / s)) if f.startswith("disp0") and f.endswith(".pfm")]
        assert len(got) == 1, s
