"""GPU: the MiddEval3 SDK's evaldisp metrics on the device (csrc/mb_eval.cu through mb_eval.evaldisp) against
oracle/mb_evaldisp.py -- every count and every quantile exactly, the float64 sums within 1e-12 and bit-identical across two
runs -- at scales 1, 2 and 4 from 1 x 1 to a full-resolution ground truth; and predict -> score end to end on a synthetic
raw Middlebury tree, with the written maps byte-identical to -a submit's."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import evaluate, mb_eval as me, preprocess, synth, t7  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import mb_evaldisp as od  # noqa: E402

PATTERNS = ["sparse", "unknown", "invalid", "specials", "thresholds"]


def _case(h, w, scale, pattern, seed):
    """(disp (h, w), gt (scale h, scale w), mask or None, maxdisp) with the pattern's special values"""
    rng = np.random.default_rng(seed)
    Hg, Wg = scale * h, scale * w
    maxdisp = int(rng.integers(16, 300))
    disp = rng.uniform(-3, maxdisp * 1.1, (h, w)).astype(np.float32)
    gt = rng.uniform(0, maxdisp * scale, (Hg, Wg)).astype(np.float32)
    gt[rng.random((Hg, Wg)) < 0.05] = np.inf                                       # sparse holes
    if pattern == "unknown":
        gt[:] = np.inf
    elif pattern == "invalid":
        disp[:] = np.inf
    elif pattern in ("sparse", "specials"):
        p = 0.02 if pattern == "sparse" else 0.3
        kind = rng.integers(0, 4, (h, w))
        hit = rng.random((h, w)) < p
        disp[hit & (kind == 0)] = np.nan
        disp[hit & (kind == 1)] = np.inf
        disp[hit & (kind == 2)] = -np.inf
        disp[hit & (kind == 3)] = maxdisp * 4                                       # above maxd
    elif pattern == "thresholds":
        # integer maps against gt = d + one of 0, +-0.5, +-1, +-2, +-4, 4.5: errors on the thresholds and long runs of ties
        disp = rng.integers(0, maxdisp, (h, w)).astype(np.float32)
        up = np.kron(disp, np.ones((scale, scale), np.float32)) * scale
        off = rng.choice(np.array([0, 0.5, -0.5, 1, -1, 2, -2, 4, -4, 4.5], np.float32), (Hg, Wg))
        gt = np.where(np.isinf(gt), np.inf, up + off).astype(np.float32)
    mask = None
    if seed % 3:
        mask = rng.choice(np.array([0, 128, 255], np.uint8), (Hg, Wg), p=[0.1, 0.2, 0.7])
    return disp, gt, mask, maxdisp


SHAPES = [(1, 1, 1), (1, 741, 1), (497, 1, 1), (1, 1, 2), (3, 5, 2), (7, 3, 4), (497, 741, 1), (994, 1482, 1),
          (994, 1482, 2), (300, 450, 4)]


def _bits_or_nan(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    both_nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(both_nan | (a.view(np.uint32) == b.view(np.uint32))))


@pytest.mark.parametrize("h,w,scale", SHAPES)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_evaldisp_equals_the_oracle(h, w, scale, pattern):
    seed = h * 7919 + w * 31 + scale + 1000 * PATTERNS.index(pattern)
    disp, gt, mask, maxdisp = _case(h, w, scale, pattern, seed)
    want_c, want_s, want_q = od.evaldisp(disp, gt, mask, maxdisp)
    dev = torch.device("cuda", 0)
    args = [torch.from_numpy(disp).to(dev), torch.from_numpy(gt).to(dev),
            None if mask is None else torch.from_numpy(mask).to(dev), maxdisp]
    scratch = torch.full((me.scratch_bytes(),), 0x5a, dtype=torch.uint8, device=dev)    # stale contents do not matter
    sums = []
    for run in range(2):
        got = me.evaldisp(*args, scratch=scratch if run else None)
        c, s, q = (t.cpu().numpy() for t in got)
        assert np.array_equal(c, want_c), "counts"
        assert _bits_or_nan(q, want_q), "quantiles %s, want %s" % (q, want_q)
        np.testing.assert_allclose(s, want_s, rtol=1e-12, atol=0)
        sums.append(s.tobytes())
    assert sums[0] == sums[1], "the float64 sums differ between two runs"
    if pattern == "thresholds" and gt.size >= 1000:
        assert (want_c[1, od.BAD05] < want_c[1, od.VALID]) and want_c[1, od.BAD4] > 0


def test_refusals():
    from mccnn_b200.adcensus import AdcensusError

    dev = torch.device("cuda", 0)
    d, g = torch.ones(2, 3, device=dev), torch.ones(6, 9, device=dev)
    with pytest.raises(AdcensusError, match="invalid argument"):
        me.evaldisp(d, g, None, 10)                                       # ratio 3
    with pytest.raises(AdcensusError, match="invalid argument"):
        me.evaldisp(d, torch.ones(4, 7, device=dev), None, 10)
    with pytest.raises(AdcensusError, match="invalid argument"):
        me.evaldisp(d, torch.ones(2, 3, device=dev), None, 0)             # maxdisp < 1
    with pytest.raises(ValueError, match="mask is"):
        me.evaldisp(d, d, torch.ones(2, 4, dtype=torch.uint8, device=dev), 10)
    with pytest.raises(ValueError, match="float32"):
        me.evaldisp(d.double(), d, None, 10)
    with pytest.raises(ValueError, match="uint8"):
        me.evaldisp(d, d, torch.ones(2, 3, device=dev), 10)
    with pytest.raises(ValueError, match="scratch"):
        me.evaldisp(d, d, None, 10, scratch=torch.empty(100, dtype=torch.uint8, device=dev))


# ---- predict -> score end to end ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def world(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("me"))
    unzip = synth.write_mb_raw(root, seed=11)
    synth.write_mb_eval_gt(unzip, seed=12)
    net = os.path.join(root, "fast.t7")
    t7.save_net(net, oft.make_weights(np.random.default_rng(13), l1=5, fm=64))         # the Middlebury fast shape
    return dict(root=root, net=net)


@pytest.mark.parametrize("arch", ["census", "fast"])
def test_predict_then_score_print_the_same_lines(world, capsys, tmp_path, arch):
    out = str(tmp_path / "out")
    net = world["net"] if arch == "fast" else None
    res = me.evaluate_training(arch, net, data_root=world["root"], out=out)
    printed = capsys.readouterr().out
    lines = printed.splitlines()
    scenes = sorted(synth.MB_SUBMIT_NAMES)
    assert res.scenes == scenes and len(lines) == 16
    for i, s in enumerate(scenes):
        assert lines[i] == me.line(s, res.rows[i]) and len(lines[i].split("\t")) == 25
    assert lines[15] == me.line("mean", res.mean)
    method = "MC-CNN-fst" if arch == "fast" else "MC-CNN-acrt"
    for s in scenes:
        assert sorted(os.listdir(os.path.join(out, "trainingH", s))) == ["disp0%s.pfm" % method, "time%s.txt" % method]

    again = me.score_dir(out, data_root=world["root"])
    assert capsys.readouterr().out == printed
    for a, b in zip(again.evals, res.evals):
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))

    # scene 0's counts are the oracle's on the written map, at F (scale 2)
    gt_f, mask_f = me.gt_files(world["root"], scenes[0], "F")
    disp = me._read_topdown(me.find_map(out, scenes[0]))
    c, s, q = od.evaldisp(disp, me._read_topdown(gt_f), preprocess._read_grey(mask_f),
                          preprocess._ndisp(os.path.join(me.scene_dir(world["root"], scenes[0]), "calib.txt")))
    assert np.array_equal(c, res.evals[0].counts) and _bits_or_nan(q, res.evals[0].quantiles)

    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "mb_eval.py"), "score", out, "-data_root",
                        world["root"]], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout == printed
    # res H: the same maps at scale 1, against trainingH's ground truth
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "mb_eval.py"), "score", out, "-data_root",
                        world["root"], "-res", "H", "-alg", method], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    h = me.score_dir(out, data_root=world["root"], res="H", alg=method, verbose=False)
    assert r.stdout.splitlines() == [me.line(s, row) for s, row in zip(h.scenes, h.rows)] + [me.line("mean", h.mean)]
    assert h.evals[0].counts[1, me.N] * 4 != res.evals[0].counts[1, me.N]              # another ground truth

    # the maps are byte-identical to -a submit's trainingH maps on preprocess_mb's output of the same raw tree
    d = preprocess.mb_output_dir(world["root"], "imperfect", "gray")
    if not os.path.exists(os.path.join(d, "meta.bin")):
        preprocess.preprocess_mb(world["root"], "imperfect", "gray")
    ev = evaluate.Evaluator("mb", arch, net_fname=net)
    sub = str(tmp_path / "submit")
    try:
        ev.submit(data_root=world["root"], out=sub)
    finally:
        ev.close()
    for s in scenes:
        name = "disp0%s.pfm" % method
        with open(os.path.join(sub, "trainingH", s, name), "rb") as a, open(os.path.join(out, "trainingH", s, name), "rb") as b:
            assert a.read() == b.read(), s
