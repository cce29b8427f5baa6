"""Which pixels of a disparity map to trust: the margin confidence, sparse maps kept by it, and the sparsification curve that
scores it (an addition beyond the reference; DESIGN §19).

    disp, conf = margin(vol)                                   # vol (D, H, W) or (1, D, H, W), the final left volume
    sparse = sparsify(disp, conf, 0.5, invalid=0.0)            # the half of the pixels with the largest confidence
    res = sparsification(pred, conf, gt, err_at=3)             # res.curve, res.auc, res.auc_opt

Margin confidence at a pixel: c1 = the cost of the arg-min d1 (main.lua:1049-1050's rule: first strict minimum, NaN skipped,
0 when nothing is below +inf), c2 = the least cost at |d - d1| >= 2 by the same rule, conf = c2 - c1 (float32) when both are
below +inf, else 0.  The ±1 band keeps a smooth cost curve's own neighbours from passing as a rival match.  The confidence
belongs to the integer winner: sub-pixel refinement, median and bilateral filtering move the final disparity, not its
confidence.

Ordering (sparsify and the curve): conf descending, then row-major index ascending.  The sparsification curve of Hu &
Mordohai (TPAMI 2012) over the M pixels of main.lua's mask (gt != 0): e_k = the share of bad pixels (|gt - pred| > err_at)
among the first n_k = ceil(k M / 20), k = 1..20, so e_20 is main.lua's err; AUC = sum_{k=1}^{19} 0.05 (e_k + e_{k+1}) / 2,
and AUC_opt is the same over the ordering that puts every good pixel first.  The counts come from the GPU
(mccnn_sparsification_counts); the curve is computed from them in double on the host.
"""
import math
from collections import namedtuple

import torch

from . import adcensus

POINTS = 20
Sparsification = namedtuple("Sparsification", "M B bad curve auc auc_opt")


def _hw(t, name, n):
    if t.dim() < 2 or t.numel() != t.size(-1) * t.size(-2):
        raise adcensus.AdcensusError("%s: %s must be (H, W) or (1, 1, H, W), got %s" % (n, name, tuple(t.shape)))
    return t.size(-2), t.size(-1)


def margin(vol):
    """(disp, conf), both (H, W): the arg-min and the margin confidence of a (D, H, W) or (1, D, H, W) device volume, from one
    read of it (mccnn_margin_confidence); disp is bit-identical to :func:`adcensus.argmin`."""
    n = "mccnn_margin_confidence"
    if vol.dim() == 4 and vol.size(0) == 1:
        vol = vol[0]
    if vol.dim() != 3:
        raise adcensus.AdcensusError("%s: vol must be (D, H, W), got %s" % (n, tuple(vol.shape)))
    D, H, W = vol.shape
    disp = torch.empty((H, W), device=vol.device, dtype=torch.float32)
    conf = torch.empty_like(disp)
    with torch.cuda.device(vol.device):
        adcensus._check(adcensus.lib().mccnn_margin_confidence(adcensus._t(vol, 1, n), adcensus._t(disp, 2, n),
                                                               adcensus._t(conf, 3, n), D, H, W, adcensus._stream(vol)), n)
    return disp, conf


def n_keep(density, H, W):
    """ceil(density H W), the pixels a map of `density` in (0, 1] keeps"""
    check_density(density)
    return math.ceil(density * H * W)


def check_density(density):
    if not (isinstance(density, (int, float)) and 0 < density <= 1):
        raise ValueError("density must be in (0, 1], got %r" % (density,))


def sparsify(disp, conf, density, invalid=float("nan")):
    """`disp` at the ceil(density H W) pixels of largest `conf` (ties: lower row-major index first), `invalid` elsewhere
    (0 for a KITTI PNG16, +inf for a Middlebury PFM, NaN for a .bin map); device tensors of one (H, W) shape
    (mccnn_sparsify).  Returns a new tensor shaped like `disp`."""
    n = "mccnn_sparsify"
    H, W = _hw(disp, "disp", n)
    if _hw(conf, "conf", n) != (H, W):
        raise adcensus.AdcensusError("%s: conf must be %s like disp, got %s" % (n, (H, W), tuple(conf.shape)))
    keep = n_keep(density, H, W)
    out = torch.empty_like(disp)
    with torch.cuda.device(disp.device):
        adcensus._check(adcensus.lib().mccnn_sparsify(adcensus._t(disp, 1, n), adcensus._t(conf, 2, n), adcensus._t(out, 3, n),
                                                      H, W, keep, float(invalid), adcensus._stream(disp)), n)
    return out


def counts(pred, conf, gt, err_at):
    """(M, B, [bad among the first n_k, k = 1..20]) of `pred` and `conf` against `gt`, device (H, W) tensors
    (mccnn_sparsification_counts)"""
    n = "mccnn_sparsification_counts"
    H, W = _hw(pred, "pred", n)
    for name, t in (("conf", conf), ("gt", gt)):
        if _hw(t, name, n) != (H, W):
            raise adcensus.AdcensusError("%s: %s must be %s like pred, got %s" % (n, name, (H, W), tuple(t.shape)))
    out = torch.empty(2 + POINTS, device=pred.device, dtype=torch.int64)
    with torch.cuda.device(pred.device):
        adcensus._check(adcensus.lib().mccnn_sparsification_counts(adcensus._t(pred, 1, n), adcensus._t(conf, 2, n),
                                                                   adcensus._t(gt, 3, n), H, W, float(err_at),
                                                                   out.data_ptr(), adcensus._stream(pred)), n)
    c = out.cpu().tolist()
    return c[0], c[1], c[2:]


def n_points(M):
    """n_k = ceil(k M / 20), k = 1..20, in integers"""
    return [(k * M + POINTS - 1) // POINTS for k in range(1, POINTS + 1)]


def auc(curve):
    """sum_{k=1}^{19} 0.05 (e_k + e_{k+1}) / 2 of a 20-point curve"""
    return sum(0.05 * (curve[k] + curve[k + 1]) / 2 for k in range(POINTS - 1))


def curve_of_counts(M, B, bad):
    """(curve, AUC, AUC_opt) from the integer counts, in double; NaN everywhere when M = 0 (main.lua's 0 / 0)"""
    if M == 0:
        nan = float("nan")
        return [nan] * POINTS, nan, nan
    ns = n_points(M)
    curve = [b / n for b, n in zip(bad, ns)]
    opt = [max(0, n - (M - B)) / n for n in ns]
    return curve, auc(curve), auc(opt)


def sparsification(pred, conf, gt, err_at):
    """The sparsification curve of `pred` ordered by `conf` against `gt` (device tensors of one (H, W) shape):
    :data:`Sparsification` (M, B, bad counts, curve e_1..e_20, auc, auc_opt)."""
    M, B, bad = counts(pred, conf, gt, err_at)
    curve, a, a_opt = curve_of_counts(M, B, bad)
    return Sparsification(M, B, bad, curve, a, a_opt)
