"""CPU: predict_kitti.lua's loop (mccnn_b200/predict_kitti.py, tools/predict_kitti.py) without a GPU -- the command line, the
refusals that come before any GPU work, the printed lines, the sharding over 2 and 3 gloo ranks with an injected compute,
and the claim the front-end kernel rests on: numpy's float64 sum follows the pairwise tree csrc/pairwise.cuh restates."""
import contextlib
import io
import os
import shutil
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import evaluate, predict_kitti as pk, synth  # noqa: E402


# ---- the command line ---------------------------------------------------------------------------------------------------

def _tool():
    import importlib

    return importlib.import_module("predict_kitti")


def test_parse_args_defaults():
    a = _tool().parse_args(["test", "kitti", "-net_fname", "n.t7"])
    assert (a.action, a.dataset, a.arch, a.disp_max, a.gpu, a.data_root, a.out) == ("test", "kitti", "fast", 228, 1, ".", "out")
    a = _tool().parse_args(["submit", "kitti2015", "-arch", "census", "-disp_max", "70", "-gpu", "2", "-out", "o"])
    assert (a.action, a.dataset, a.arch, a.disp_max, a.gpu, a.out) == ("submit", "kitti2015", "census", 70, 2, "o")


@pytest.mark.parametrize("argv", [["test", "kitti"], ["test", "kitti", "-arch", "slow"], ["test", "kitti", "-arch", "census",
                                  "-disp_max", "0"], ["test", "kitti", "-arch", "ad", "-gpu", "0"], ["predict", "kitti"],
                                  ["test", "mb", "-arch", "census"], ["test", "kitti", "-arch", "accurate"]])
def test_parse_args_refusals(argv):
    with pytest.raises(SystemExit):
        _tool().parse_args(argv)


# ---- refusals before any GPU work ---------------------------------------------------------------------------------------

@pytest.fixture
def tree(tmp_path):
    root = str(tmp_path / "data")
    synth.write_kitti_raw(root, "kitti", n_tr=3, n_te=2, H=20, widths=(40, 37), D=8, seed=3)
    return root


def test_pair_files_and_shapes(tree):
    tr, te = pk.pair_files(tree, "kitti", "test"), pk.pair_files(tree, "kitti", "submit")
    assert len(tr) == 3 and len(te) == 2 and all(f[2] is not None for f in tr) and all(f[2] is None for f in te)
    assert [os.path.basename(f[0]) for f in tr] == ["%06d_10.png" % i for i in range(3)]
    assert pk.scan(tr) == [(20, 40), (20, 37), (20, 40)]


def test_missing_disp_noc_refused(tree):
    os.remove(os.path.join(tree, "data.kitti", "unzip", "training", "disp_noc", "000001_10.png"))
    with pytest.raises(FileNotFoundError, match="disp_noc"):
        pk.predict_kitti("test", "kitti", arch="census", data_root=tree)


def test_view_size_mismatch_refused(tree):
    from PIL import Image

    Image.fromarray(np.zeros((20, 41), np.uint8)).save(os.path.join(tree, "data.kitti", "unzip", "training", "image_1",
                                                                    "000002_10.png"))
    with pytest.raises(ValueError, match="20x40.*20x41"):
        pk.predict_kitti("test", "kitti", arch="census", data_root=tree)


def test_grey_with_colour_view_refused(tree):
    from PIL import Image

    Image.fromarray(np.zeros((20, 40, 3), np.uint8)).save(os.path.join(tree, "data.kitti", "unzip", "testing", "image_0",
                                                                       "000000_10.png"))
    with pytest.raises(ValueError, match="grey"):
        pk.predict_kitti("submit", "kitti", arch="census", data_root=tree, out=os.path.join(tree, "out"))


def test_ground_truth_size_mismatch_refused(tree):
    from mccnn_b200 import dataio

    dataio.write_png16(np.ones((19, 40), np.float32), os.path.join(tree, "data.kitti", "unzip", "training", "disp_noc",
                                                                   "000000_10.png"))
    with pytest.raises(ValueError, match="19x40"):
        pk.predict_kitti("test", "kitti", arch="census", data_root=tree)


def test_non_empty_out_refused(tree, tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    (out / ".empty").write_bytes(b"")
    (out / "000000_10.png").write_bytes(b"x")
    with pytest.raises(ValueError, match="not empty"):
        pk.predict_kitti("submit", "kitti", arch="census", data_root=tree, out=str(out))


def test_missing_testing_directory_refused(tree):
    shutil.rmtree(os.path.join(tree, "data.kitti", "unzip", "testing", "image_1"))
    with pytest.raises(FileNotFoundError, match="image_1"):
        pk.predict_kitti("submit", "kitti", arch="census", data_root=tree)


def test_bad_arguments_refused(tree):
    with pytest.raises(ValueError, match="action"):
        pk.predict_kitti("test_te", "kitti", arch="census", data_root=tree)
    with pytest.raises(ValueError, match="dataset"):
        pk.predict_kitti("test", "mb", arch="census", data_root=tree)
    with pytest.raises(ValueError, match="disp_max"):
        pk.predict_kitti("test", "kitti", arch="census", data_root=tree, disp_max=0)


# ---- the printed lines --------------------------------------------------------------------------------------------------

COUNTS = [(7, 100), (0, 3), (1, 3), (5, 0), (2, 9), (123, 4567), (1, 7)]


def _counts(i):
    return torch.tensor(COUNTS[i], dtype=torch.int64)


def _want_test(n):
    errs = [COUNTS[i][0] / COUNTS[i][1] if COUNTS[i][1] else float("nan") for i in range(n)]
    s = 0.0
    for e in errs:
        s = s + e
    return errs, s / n


def test_test_lines(capsys):
    res = pk.report("test", 5, _counts, rank=0, world=1)
    lines = capsys.readouterr().out.splitlines()
    errs, mean = _want_test(5)
    assert lines[:3] == ["0\t0.07", "1\t0", "2\t0.33333333333333"]
    assert lines[3] == "3\tnan"                     # no valid pixel: 0 / 0, as the script's division gives
    assert lines[4] == "4\t%.14g" % (2 / 9) and len(lines) == 6
    assert lines[5] == "nan" and np.isnan(res.mean)
    assert res.errors[:3] == errs[:3]
    res = pk.report("test", 3, _counts, rank=0, world=1, verbose=False)
    assert capsys.readouterr().out == ""
    assert res.mean == (0.07 + 0.0 + 1 / 3) / 3 and evaluate.lua_num(res.mean) == "%.14g" % res.mean


def test_mean_is_accumulated_in_pair_order():
    # Python's sum() of floats is compensated; the script adds in turn
    errs = [0.1, 0.2, 0.3, 1e-17, 0.4]
    counts = [torch.tensor([int(e * 10 ** 17), 10 ** 17]) for e in errs]
    res = pk.report("test", len(errs), lambda i: counts[i], rank=0, world=1, verbose=False)
    s = 0.0
    for e in res.errors:
        s = s + e
    assert res.mean == s / len(errs)


def test_submit_lines(capsys):
    files = pk.report("submit", 3, lambda i: torch.tensor([i]), rank=0, world=1, submission_file=lambda i: "o/%06d_10.png" % i)
    assert capsys.readouterr().out.splitlines() == ["0", "1", "2"]
    assert files == ["o/%06d_10.png" % i for i in range(3)]


# ---- sharding over gloo ranks -------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n, action, outdir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import mccnn_b200  # noqa: F401
    from mccnn_b200 import batch, predict_kitti as pk

    done = []

    def compute(i):
        done.append(i)
        return _counts(i) if action == "test" else torch.tensor([i])

    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        res = pk.report(action, n, compute, submission_file=lambda i: "f%d" % i)
    assert done == batch.shard_indices(n, rank, world)
    if rank == 0:
        with open(os.path.join(outdir, "out.txt"), "w") as f:
            f.write(buf.getvalue())
        np.save(os.path.join(outdir, "res.npy"), np.asarray(res.errors + [res.mean] if action == "test" else res, dtype=object),
                allow_pickle=True)
    else:
        assert res is None and buf.getvalue() == ""
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("action,n", [("test", 7), ("test", 2), ("submit", 5)])
def test_sharded_output_equals_one_process(tmp_path, world, action, n, capsys):
    mp.spawn(_worker, args=(world, _free_port(), n, action, str(tmp_path)), nprocs=world, join=True)
    got_out = open(tmp_path / "out.txt").read()
    got = list(np.load(tmp_path / "res.npy", allow_pickle=True))
    capsys.readouterr()
    one = pk.report(action, n, _counts if action == "test" else (lambda i: torch.tensor([i])), rank=0, world=1,
                    submission_file=lambda i: "f%d" % i)
    assert got_out == capsys.readouterr().out
    want = one.errors + [one.mean] if action == "test" else one
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g == w or (isinstance(w, float) and np.isnan(g) and np.isnan(w))


# ---- numpy's pairwise order -----------------------------------------------------------------------------------------------

def pairwise_sum(a):
    """numpy's pairwise_sum as csrc/pairwise.cuh restates it, in float64"""
    n = len(a)
    if n < 8:
        r = 0.0
        for v in a:
            r = r + v
        return r
    if n <= 128:
        r = [a[j] for j in range(8)]
        body = n - n % 8
        for i in range(8, body, 8):
            for j in range(8):
                r[j] = r[j] + a[i + j]
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(body, n):
            res = res + a[i]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


@pytest.mark.parametrize("shape", [(1, 1, 5), (1, 2, 4), (1, 3, 43), (1, 1, 129), (1, 64, 128), (1, 91, 90), (1, 8193, 1),
                                   (1, 375, 1242), (1, 375, 1241), (1, 370, 1224)])
def test_numpy_float64_sum_is_the_pairwise_tree(shape):
    rng = np.random.default_rng(sum(shape))
    x = (rng.integers(0, 256, shape).astype(np.float32) * np.float32(0.587) - np.float32(97.3)).astype(np.float64)
    assert x.sum() == pairwise_sum(x.reshape(-1).tolist())
    assert ((x - 0.25) ** 2).sum() == pairwise_sum(((x - 0.25) ** 2).reshape(-1).tolist())
