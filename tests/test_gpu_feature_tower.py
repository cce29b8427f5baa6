"""GPU parity of the in-library feature tower (csrc/feature_tower.cu) against the CPU oracle (oracle/feature_tower.py, pinned to
the PyTorch restatement of main.lua:726-749 by tests/golden/feature_tower.npz).  Bar: 1e-4, absolute for the unit-norm
features of the fast architecture, scaled by max(1, |want|) for the slow one; plain bf16 operands (nterms = 1): 5e-2."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import adcensus, feature_tower  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import tower_head_cases as cases  # noqa: E402


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to("cuda:0")


def scaled_err(got, want):
    """max |got - want| / max(1, max |want|): the tower's bar is relative to the size of its outputs"""
    return float(np.abs(got - want).max()) / max(1.0, float(np.abs(want).max()))


def check_both_modes(tower, x, want, what):
    """nterms = 3 within 1e-4, nterms = 1 within 5e-2; returns the nterms = 3 error"""
    e3 = scaled_err(tower.forward(cu(x)).cpu().numpy(), want)
    assert e3 <= 1e-4, "%s: nterms 3 off by %.3g" % (what, e3)
    e1 = scaled_err(tower.forward(cu(x), nterms=1).cpu().numpy(), want)
    assert e1 <= 5e-2, "%s: nterms 1 off by %.3g" % (what, e1)
    print("%s: max err %.3g (nterms 3), %.3g (nterms 1)" % (what, e3, e1))
    return e3


def test_golden_fixture():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "feature_tower.npz"))
    layers = [(g["w%d" % i], g["b%d" % i]) for i in range(4)]
    t = feature_tower.FeatureTower(layers, arch="fast")
    got = t.forward(cu(g["x"])).cpu().numpy()
    assert np.abs(got - g["out"]).max() <= 1e-4
    assert np.abs(got - g["out"]).max() <= 2e-5, "the bf16-split path should sit well inside the bar"
    t.close()


@pytest.mark.parametrize("n_in,fm,l1,arch,H,W", [
    (1, 64, 4, "fast", 9, 300),      # kitti fast: three tiles per row, ragged last tile
    (1, 64, 5, "fast", 5, 129),      # mb fast depth
    (1, 112, 4, "slow", 4, 200),     # accurate arch tower: 112 planes (padded to 128), ReLU after the last layer, no Normalize
    (3, 16, 2, "slow", 6, 70),       # colour input, small planes
])
def test_against_oracle(n_in, fm, l1, arch, H, W):
    rng = np.random.default_rng(fm + l1)
    layers = oft.make_weights(rng, l1=l1, fm=fm, n_in=n_in)
    x = rng.standard_normal((2, n_in, H, W)).astype(np.float32)
    want = oft.tower_forward(x, layers, normalize=(arch == "fast"))
    if arch == "slow":
        want = np.maximum(want, 0)                                   # main.lua:684-685: ReLU after every layer
    t = feature_tower.FeatureTower(layers, arch=arch)
    got = t.forward(cu(x)).cpu().numpy()
    scale = max(1.0, float(np.abs(want).max()))
    assert np.abs(got - want).max() <= 1e-4 * scale
    got1 = t.forward(cu(x), nterms=1).cpu().numpy()
    assert np.abs(got1 - want).max() <= 5e-2 * scale                 # plain bf16 operands
    t.close()


@pytest.mark.parametrize("case", cases.TOWER_VARIANTS, ids=lambda c: "fm%d_%s" % (c[2], c[4]))
def test_every_kernel_variant(case):
    """fm 16 .. 128 in steps of 16: every (N, taps per pass) of the ring kernel and the resident kernel at fm = 64"""
    seed, n_in, fm, l1, arch, nimg, H, W = case
    layers, x = cases.tower_case(seed, n_in, fm, l1, nimg, H, W)
    t = feature_tower.FeatureTower(layers, arch=arch)
    check_both_modes(t, x, cases.tower_want(x, layers, arch), "fm %d %s" % (fm, arch))
    t.close()


@pytest.mark.parametrize("case", cases.TOWER_EDGES, ids=lambda c: "seed%d" % c[0])
def test_edges(case):
    """W 1, 2, 127, 128, 129, 257; H 1 .. 3; one to three images; colour input into the resident kernel; l1 = 1 and 8; an
    all-zero image; input scales 1e-3 and 1e3"""
    seed, n_in, fm, l1, arch, nimg, H, W, scale, zero = case
    layers, x = cases.tower_case(seed, n_in, fm, l1, nimg, H, W, scale, zero)
    t = feature_tower.FeatureTower(layers, arch=arch)
    got = t.forward(cu(x))
    assert got.shape == (nimg, fm, H, W)
    check_both_modes(t, x, cases.tower_want(x, layers, arch), "seed %d" % seed)
    t.close()


def test_resident_kernel_loops_over_many_tiles():
    """The resident kernel launches min(#tiles, #SMs) persistent CTAs; at 2 x 48 x 1242 every CTA runs several tiles, so the
    a_full / a_free phases change many times within a CTA"""
    nimg, H, W = 2, 48, 1242
    ntile = nimg * H * math.ceil(W / 128)
    assert ntile >= 4 * torch.cuda.get_device_properties(0).multi_processor_count
    layers, x = cases.tower_case(21, 1, 64, 4, nimg, H, W)
    t = feature_tower.FeatureTower(layers, arch="fast")
    check_both_modes(t, x, cases.tower_want(x, layers, "fast"), "resident, %d tiles" % ntile)
    t.close()


def _free_device_memory():
    import gc

    gc.collect()
    torch.cuda.empty_cache()                                # memory cached by earlier tests counts as used otherwise
    adcensus.lib().adcensus_trim_scratch()
    return torch.cuda.mem_get_info()[0]


@pytest.mark.parametrize("name,seed,fm,l1,arch,H,W,crop,band", [
    ("kitti_fast", 11, 64, 4, "fast", 350, 1242, 64, 4),
    ("mb_fast", 12, 64, 5, "fast", 2000, 3000, 256, 2),
    ("kitti_slow", 13, 112, 4, "slow", 350, 1242, 64, 4),
])
def test_full_size(name, seed, fm, l1, arch, H, W, crop, band):
    """A stereo pair at full size: three full-width row bands (top, middle, bottom) against the oracle, and every row
    bitwise against runs on row crops with l1 rows of margin.  The crops put each tile on another CTA (and, for the
    resident kernel, at another point of a CTA's loop), so a race or a phase error anywhere in the image shows up."""
    nimg = 2
    need = 4 * nimg * fm * W * (3 * H + 3 * (crop + 2 * l1))   # output and two scratch activations, full run and one crop
    if _free_device_memory() < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    layers, x = cases.tower_case(seed, 1, fm, l1, nimg, H, W)
    t = feature_tower.FeatureTower(layers, arch=arch)
    xd = cu(x)
    out = t.forward(xd)
    worst = 0.0
    for y0 in (0, H // 2 - band // 2, H - band):
        got = out[:, :, y0:y0 + band].cpu().numpy()
        e = scaled_err(got, cases.tower_want(x, layers, arch, rows=(y0, y0 + band)))
        assert e <= 1e-4, "%s: rows %d..%d off by %.3g" % (name, y0, y0 + band, e)
        worst = max(worst, e)
    for y0 in range(0, H, crop):
        y1 = min(H, y0 + crop)
        a, b = max(0, y0 - l1), min(H, y1 + l1)
        part = t.forward(xd[:, :, a:b].contiguous())
        assert torch.equal(part[:, :, y0 - a:y1 - a], out[:, :, y0:y1]), "%s: rows %d..%d differ from a crop's" % (name, y0, y1)
        del part
    print("%s: %d x %d, max err %.3g in three bands, every row equal to the crops'" % (name, H, W, worst))
    t.close()
    del out, xd
    _free_device_memory()


def test_side_stream_gives_the_same_bits():
    """a forward on a non-default stream (scratch, launches and the output on that stream) equals the default stream's"""
    for seed, fm, arch in ((41, 64, "fast"), (42, 112, "slow")):
        layers, x = cases.tower_case(seed, 1, fm, 4, 2, 16, 600)
        t = feature_tower.FeatureTower(layers, arch=arch)
        xd = cu(x)
        ref = t.forward(xd)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            got = t.forward(xd)
        torch.cuda.current_stream().wait_stream(s)
        assert torch.equal(got, ref), "fm %d: side stream differs" % fm
        t.close()
