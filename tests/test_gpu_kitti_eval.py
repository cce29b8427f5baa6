"""GPU: the devkits' metrics on the device (csrc/kitti_eval.cu through kitti_eval.devkit_counts) against
oracle/kitti_devkit.py -- the interpolated map bit for bit, every count, the float64 error sums -- from float maps and from
stored uint16 values; the 3-pixel count against predict_kitti.error_counts; and predict -> score end to end on synthetic
raw KITTI sets."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, kitti_eval as ke, predict_kitti as pk, synth, t7  # noqa: E402
from oracle import feature_tower as oft  # noqa: E402
from oracle import kitti_devkit as kd  # noqa: E402


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _random_case(H, W, pattern, seed):
    """a float estimate with invalid pixels (0, below 1/256, NaN) in the given pattern, two ground truths and an obj_map"""
    rng = np.random.default_rng(seed)
    disp = rng.uniform(0, 120, (H, W)).astype(np.float32)
    if pattern == "sparse":
        bad = rng.random((H, W)) < 0.1
    elif pattern == "dense":
        bad = rng.random((H, W)) < 0.9
    elif pattern == "runs":                  # long runs, whole invalid rows (first, last, interior) and columns
        bad = np.zeros((H, W), bool)
        for _ in range(max(1, H * W // 200)):
            y, x = rng.integers(0, H), rng.integers(0, W)
            bad[y, x:x + int(rng.integers(1, 80))] = True
        for y in (0, H - 1, H // 2, H // 3):
            bad[y] = rng.random() < 0.7
        bad[:, :min(W, 3)] |= rng.random() < 0.5
        bad[:, -1] |= rng.random() < 0.5
    else:                                    # "none" valid
        bad = np.ones((H, W), bool)
    kind = rng.integers(0, 4, (H, W))
    disp[bad & (kind == 0)] = 0
    disp[bad & (kind == 1)] = rng.uniform(0, 1 / 256, (H, W))[bad & (kind == 1)]
    disp[bad & (kind == 2)] = np.nan
    disp[bad & (kind == 3)] = -rng.uniform(0, 5, (H, W))[bad & (kind == 3)]
    noc = rng.integers(1, 100 * 256, (H, W)).astype(np.uint16)
    noc[rng.random((H, W)) < 0.3] = 0
    occ = np.where(noc == 0, rng.integers(0, 100 * 256, (H, W)), noc).astype(np.uint16)
    # some exact hits of the thresholds: e = 2, 3, 4, 5 and a D1 quotient of exactly 0.05f
    flat, fnoc = disp.reshape(-1), noc.reshape(-1)
    for k, (gt, e) in enumerate([(10, 2), (10, 3), (10, 4), (10, 5), (80, 4), (80, 3)]):
        if k < flat.size and not bad.reshape(-1)[k]:
            fnoc[k], flat[k] = gt * 256, gt + e
    occ = np.where(noc != 0, noc, occ).astype(np.uint16)
    obj = (rng.random((H, W)) < 0.3).astype(np.uint8) * rng.integers(1, 5, (H, W)).astype(np.uint8)
    return disp, noc, occ, obj


SHAPES = [(375, 1242), (375, 1241), (370, 1224), (1, 1), (1, 2), (1, 31), (1, 33), (1, 1242), (7, 1), (375, 1), (3, 65)]
PATTERNS = ["sparse", "dense", "runs", "none"]


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("pattern", PATTERNS)
def test_devkit_counts_equal_the_oracle(H, W, pattern):
    disp, noc, occ, obj = _random_case(H, W, pattern, seed=H * 7919 + W * 31 + PATTERNS.index(pattern))
    with np.errstate(invalid="ignore"):
        v = kd.png16_values(disp)
    with_obj = PATTERNS.index(pattern) % 2 == 0
    want_c, want_s, want_ipol = kd.devkit_counts(v, noc, occ, obj if with_obj else None)
    dev = torch.device("cuda", 0)
    for source in ("float", "uint16"):
        est = torch.from_numpy(disp).to(dev) if source == "float" else v
        sums = []
        for run in range(2):
            ipol = torch.full((H, W), 7.0, device=dev)
            got = ke.devkit_counts(est, noc, occ, obj if with_obj else None, ipol=ipol, device=0)
            torch.cuda.synchronize()
            assert np.array_equal(_bits(ipol.cpu().numpy()), _bits(want_ipol)), "%s %s: interpolated map" % (source, pattern)
            assert np.array_equal(got.counts.cpu().numpy(), want_c), "%s %s: counts" % (source, pattern)
            s = got.sums.cpu().numpy()
            np.testing.assert_allclose(s, want_s, rtol=1e-12, atol=0)
            sums.append(s.tobytes())
        assert sums[0] == sums[1], "the float64 sums differ between two runs"
        got = ke.devkit_counts(est, noc, occ, obj if with_obj else None, device=0)      # no ipol: the same counts
        assert np.array_equal(got.counts.cpu().numpy(), want_c) and got.sums.cpu().numpy().tobytes() == sums[0]


@pytest.mark.parametrize("H,W", [(375, 1242), (370, 1224), (1, 1), (9, 40)])
def test_out_noc_3_equals_error_counts(H, W):
    rng = np.random.default_rng(H + W)
    disp = (rng.integers(1, 120 * 256, (H, W)) / np.float32(256)).astype(np.float32)    # > 0, multiples of 1/256
    noc = rng.integers(0, 120 * 256, (H, W)).astype(np.uint16)
    noc[rng.random((H, W)) < 0.2] = 0
    noc.reshape(-1)[:4] = (disp.reshape(-1)[:4] * 256 + np.array([768, -768, 769, 0])[:min(4, H * W)]).clip(1, 65535)
    d = torch.from_numpy(disp).cuda()
    got = ke.devkit_counts(d, noc, noc).counts.cpu().numpy()
    bad, valid = (int(x) for x in pk.error_counts(d, noc).cpu())
    assert (got[0, ke.OUT3], got[0, ke.GT]) == (bad, valid)
    assert got[0, ke.DENSE] == valid


def test_refusals():
    from mccnn_b200.adcensus import AdcensusError

    noc = np.ones((4, 5), np.uint16)
    with pytest.raises(ValueError, match="gt_occ16 is"):
        ke.devkit_counts(torch.zeros(4, 5, device="cuda"), noc, np.ones((4, 6), np.uint16))
    with pytest.raises(ValueError, match="uint16"):
        ke.devkit_counts(noc, noc.astype(np.int32), noc)
    with pytest.raises(ValueError, match="8-bit"):
        ke.devkit_counts(noc, noc, noc, np.ones((4, 5), np.int16))
    with pytest.raises(ValueError, match="float32"):
        ke.devkit_counts(torch.zeros(4, 5, dtype=torch.float64, device="cuda"), noc, noc)
    with pytest.raises(AdcensusError, match="invalid argument"):
        ke.devkit_counts(np.zeros((0, 5), np.uint16), np.zeros((0, 5), np.uint16), np.zeros((0, 5), np.uint16))


# ---- predict -> score end to end --------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def world(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("ke"))
    for k, ds in enumerate(("kitti", "kitti2015")):
        unzip = synth.write_kitti_raw(root, ds, n_tr=3, n_te=1, seed=50 + k)
        synth.write_kitti_eval_maps(unzip, ds, seed=60 + k)
    net = os.path.join(root, "fast.t7")
    t7.save_net(net, oft.make_weights(np.random.default_rng(70), l1=4, fm=64))
    return dict(root=root, net=net)


@pytest.mark.parametrize("dataset", ["kitti", "kitti2015"])
@pytest.mark.parametrize("arch", ["census", "fast"])
def test_predict_then_score_print_the_same_table(world, capsys, tmp_path, dataset, arch):
    out = str(tmp_path / "out")
    net = world["net"] if arch == "fast" else None
    res = ke.evaluate_training(dataset, net, arch, data_root=world["root"], out=out)
    printed = capsys.readouterr().out
    lines = printed.splitlines()
    n_table = 6 if dataset == "kitti" else 4
    assert len(lines) == 3 + n_table and len(res.pairs) == 3
    assert lines[3:] == ke.table(res.total, dataset)
    for i in range(3):
        assert lines[i] == ke.pair_line(i, res.pairs[i])
        assert len(lines[i].split("\t")) == 1 + len(ke.columns(dataset))
    assert sorted(os.listdir(out if dataset == "kitti" else os.path.join(out, "disp_0"))) == \
        ["%06d_10.png" % i for i in range(3)]

    again = ke.score_dir(dataset, out, data_root=world["root"])
    assert capsys.readouterr().out == printed
    assert np.array_equal(again.counts, res.counts) and again.sums.tobytes() == res.sums.tobytes()

    # pair 0's rates are the oracle's on the written file
    f = ke.training_files(world["root"], dataset)[0]
    est = dataio.read_png16_raw(ke.submission_file(out, dataset, 0))
    obj = ke._read_obj(f[4]) if f[4] else None
    c, s, _ipol = kd.devkit_counts(est, dataio.read_png16_raw(f[2]), dataio.read_png16_raw(f[3]), obj)
    assert ke.rates(c, s, dataset) == pytest.approx(res.pairs[0], rel=1e-12, nan_ok=True)

    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "kitti_eval.py"), "score", dataset, out, "-data_root",
                        world["root"]], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout == printed

