"""CPU: the inputs of the GPU tests of the feature tower and the scorer head have teeth.  With the same seeds and shapes
(oracle/tower_head_cases.py), each of the mistakes a tensor-core port typically makes -- a flipped 3x3 kernel, a dropped
bias, the two halves of the head's first layer swapped, the disparity off by one, the bf16 lo term dropped -- moves the
oracle's output by more than ten times the bar those tests apply (1e-4, scaled by max(1, |want|) for the tower; for the
head's lo term the 2e-5 its nterms = 3 results are held to).  So a kernel that passes them does not carry any of these
mistakes.  Nothing runs on a GPU: the mistakes are made in the oracle.

The head's sweep cases at feature scale 0.01 and 30 test range (tiny activations, a saturated sigmoid), not arithmetic;
they are left out here."""
import numpy as np
import pytest

from oracle import feature_tower as oft
from oracle import scorer_head as osh
from oracle import tower_head_cases as cases

BAR = 1e-4
HEAD_SPLIT_BAR = 2e-5                                                  # the head's nterms = 3 results against the oracle
bf16, tower_bf16, head_volume_bf16 = cases.bf16, cases.tower_bf16, cases.head_volume_bf16


def moved(a, b):
    m = ~np.isnan(a) & ~np.isnan(b)
    return float(np.abs(a[m] - b[m]).max())


@pytest.mark.parametrize("case", cases.TOWER_VARIANTS, ids=lambda c: "fm%d_%s" % (c[2], c[4]))
def test_tower_mistakes_exceed_ten_bars(case):
    seed, n_in, fm, l1, arch, nimg, H, W = case
    layers, x = cases.tower_case(seed, n_in, fm, l1, nimg, H, W)
    want = cases.tower_want(x, layers, arch)
    bar10 = 10 * BAR * max(1.0, float(np.abs(want).max()))
    for l in range(l1):
        flipped = list(layers)
        flipped[l] = (layers[l][0][:, :, ::-1, ::-1].copy(), layers[l][1])
        assert moved(cases.tower_want(x, flipped, arch), want) > bar10, "flipped kernel of layer %d" % l
        nobias = list(layers)
        nobias[l] = (layers[l][0], np.zeros_like(layers[l][1]))
        assert moved(cases.tower_want(x, nobias, arch), want) > bar10, "no bias in layer %d" % l
    assert moved(tower_bf16(x, layers, arch), want) > bar10, "bf16 operands without the lo term"


@pytest.mark.parametrize("case", [c for c in cases.HEAD_SWEEP if c[7] == 1.0], ids=lambda c: "seed%d" % c[0])
def test_head_mistakes_exceed_ten_bars(case):
    seed, fm, nh2, l2, H, W, D, scale = case
    layers, fL, fR = cases.head_case(seed, fm, nh2, l2, H, W, scale)
    want = osh.head_volume(fL, fR, D, layers, -1)
    bar10 = 10 * BAR
    w1, b1 = layers[0]
    swapped = [(np.concatenate([w1[:, fm:], w1[:, :fm]], axis=1), b1)] + layers[1:]
    assert moved(osh.head_volume(fL, fR, D, swapped, -1), want) > bar10, "left and right halves of W1 swapped"
    for l in range(len(layers)):
        nobias = list(layers)
        nobias[l] = (layers[l][0], np.zeros_like(layers[l][1]))
        assert moved(osh.head_volume(fL, fR, D, nobias, -1), want) > bar10, "no bias in layer %d" % l
    if min(D, W) >= 2:                                              # scores of d + 1 stored at d, and of d at d + 1
        assert moved(want[1:], want[:-1]) > bar10, "disparity off by one"
    # A dropped lo term moves the sigmoid by only 3e-4 .. 1e-3 at these shapes: it is the GPU tests' second bar, nterms = 3
    # within 2e-5, that catches it.
    assert moved(head_volume_bf16(fL, fR, D, layers), want) > 10 * HEAD_SPLIT_BAR, "bf16 operands without the lo term"


def test_bf16_rounding():
    x = np.array([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -9, -3.0e-5, 0.0], np.float32)
    got = bf16(x)
    assert got[0] == 1.0 and got[1] == 1.0 and got[2] == 1.0 + 4 * 2.0 ** -8 and got[3] == 1.0   # ties to even
    assert abs(got[4] / x[4] - 1) < 2.0 ** -8 and got[5] == 0.0
