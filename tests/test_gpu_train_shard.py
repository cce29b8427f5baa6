"""GPU: data-parallel training with the ranks as threads of one process on one GPU (tests/rank_threads.py).

* Trainer with R = 2, 4 and 8 ranks against the one-GPU Trainer, at the kitti and mb presets of both architectures and the
  fast and slow edge cases of tests/train_cases.py, for two chunks: parameters, momenta and every loss bit-identical, and
  identical on every rank.
* train.train stopped mid-epoch at R = 2, then resumed at R = 1 and at R = 4: the epoch lines and the .t7 bytes of the
  uninterrupted one-GPU run.
* On two or more GPUs: tools/train.py under torchrun with 2 processes prints and writes what one process does."""
import itertools
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, synth, train  # noqa: E402
from rank_threads import run_ranks  # noqa: E402
from train_cases import FAST_CASES, SLOW_CASES, case_id  # noqa: E402

CHUNK, CHUNKS = 3, 2                     # two chunks, the second one short
N_IMG, H, W = 3, 60, 140


def _images(dev):
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, N_IMG, 1, H, W)).astype(np.float32)
    return [torch.from_numpy(a).to(dev) for a in x]


def _chunks(o):
    """the records of CHUNKS chunks (CHUNK, CHUNK - 1 steps) of the stream's draws over random nnz rows"""
    stream, h = train.Stream(5), o["bs"] // 2
    rng = np.random.default_rng(1)
    out = []
    for n in (CHUNK, CHUNK - 1):
        rows = np.stack([rng.integers(1, N_IMG + 1, n * h), rng.integers(0, H, n * h), rng.integers(0, W, n * h),
                         rng.uniform(0, 40, n * h)], 1).astype(np.float32)
        out.append(train.make_warps(train.draw_params(stream, o, n * h), rows, 1 + 2 * o["l1"]))
    return out


def _run(o, X0, X1, rank=0, world=1, comm=None):
    tower, head = train.init_net(train.Stream(3), o)
    tr = train.Trainer(o, X0, X1, chunk=CHUNK, loss_cap=CHUNK * CHUNKS, rank=rank, world=world, comm=comm)
    try:
        tr.set_layers(tower, head)
        for i, w in enumerate(_chunks(o)):
            tr.run_chunk(w, o["lr"] if i == 0 else o["lr"] / 10)
        params, momenta = tr.state()
        return params, momenta, tr.losses(2 * CHUNK - 1)
    finally:
        tr.close()


def _same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("case", FAST_CASES + SLOW_CASES, ids=case_id)
def test_ranks_match_one_gpu(case):
    from train_cases import options

    o = options(case)
    dev = torch.device("cuda", 0)
    X0, X1 = _images(dev)
    want = _run(o, X0, X1)
    assert np.all(np.isfinite(want[2])) and len(set(want[2].tolist())) > 1
    for R in (2, 4, 8):
        if R > 2 * o["bs"]:
            continue
        got = run_ranks(R, lambda comm: _run(o, X0, X1, comm.rank, comm.world, comm), device=dev, timeout=600)
        for r, g in enumerate(got):
            for name, a, b in zip(("params", "momenta", "losses"), want, g):
                assert _same(a, b), "R = %d, rank %d: %s differ from one GPU" % (R, r, name)


def test_wrong_rank_counts_are_refused_before_gpu_work():
    o = train.options("kitti", "fast", bs=2)
    X0, X1 = _images(torch.device("cuda", 0))
    with pytest.raises(ValueError, match="power of two"):
        train.Trainer(o, X0, X1, rank=0, world=3, comm=object())
    with pytest.raises(ValueError, match="more ranks than the 4 patches"):
        train.Trainer(o, X0, X1, rank=0, world=8, comm=object())
    with pytest.raises(ValueError, match="needs a communicator"):
        train.Trainer(o, X0, X1, rank=0, world=2)
    with pytest.raises(ValueError, match="more ranks than the 4 patches"):
        train.Trainer(train.options("kitti", "slow", bs=2), X0, X1, rank=0, world=8, comm=object())


# ---------------------------------------------------------------------------------------------- stop at R = 2, resume

ROWS, EPOCHS = 1400, 2                   # bs 8: 349 steps, two chunks per epoch
OVER = dict(l1=2, fm=32, bs=8)


@pytest.fixture(scope="module")
def kitti_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    d = synth.write_kitti_set(root, "kitti", n_tr=4, n_te=2, H=48, width=130, widths=(130, 121), seed=1)
    rng = np.random.default_rng(0)
    rows = np.stack([rng.choice(np.arange(1, 5), ROWS), rng.integers(0, 48, ROWS), rng.integers(0, 121, ROWS),
                     rng.uniform(0, 30, ROWS)], 1).astype(np.float32)
    dataio.tofile(os.path.join(d, "nnz_tr.bin"), rows)
    return root


def _fresh(src_root, tmp_path):
    src, dst = os.path.join(src_root, "data.kitti"), os.path.join(str(tmp_path), "data.kitti")
    os.makedirs(dst)
    for f in os.listdir(src):
        os.symlink(os.path.join(src, f), os.path.join(dst, f))
    return str(tmp_path)


_CHECKPOINTS = train.Checkpoints


def _counter_checkpoints(*a, **k):
    """Checkpoints with a clock of its own that advances by one at every reading: each rank has its own"""
    c = itertools.count()
    return _CHECKPOINTS(*a, clock=lambda: next(c), **k)


ARGS = ["-a", "train_tr"] + sum((["-" + k, str(v)] for k, v in OVER.items()), [])


def _train(root, world, **kw):
    """train.train on `world` rank threads (plain on one) -> (rank 0's epoch lines without seconds, net bytes or None,
    (epoch, step) of a stop or None)"""
    o = train.options("kitti", "fast", **OVER)

    def one(comm):
        lines = []
        try:
            fname = train.train("kitti", "train_tr", o, args=ARGS, data_root=root, epochs=EPOCHS, log=lines.append,
                                comm=comm, **kw)
        except train.Stopped as e:
            return lines, None, (e.epoch, e.step)
        return lines, fname, None

    res = one(None) if world == 1 else run_ranks(world, one, device=torch.device("cuda", 0), timeout=900)[0]
    lines, fname, stopped = res
    net = open(fname, "rb").read() if fname else None
    return [l.rsplit("\t", 1)[0] for l in lines if l.count("\t") == 3], net, stopped


@pytest.mark.parametrize("then", [1, 4])
def test_stop_at_two_ranks_resume_at_another_count(then, kitti_root, tmp_path, monkeypatch):
    monkeypatch.setattr(train, "Checkpoints", _counter_checkpoints)
    want_ep, want_net, _ = _train(_fresh(kitti_root, tmp_path / "whole"), 1)
    assert len(want_ep) == EPOCHS and want_net
    root = _fresh(kitti_root, tmp_path / "resumed")
    ep_a, net_a, stop_a = _train(root, 2, stop_after=1, resume=True)
    assert stop_a == (1, 256) and net_a is None and ep_a == []
    assert os.path.exists(train.checkpoint_path(root, "kitti", ARGS))
    ep_b, net_b, stop_b = _train(root, then, resume=True)
    assert stop_b is None and ep_b == want_ep and net_b == want_net
    assert not os.path.exists(train.checkpoint_path(root, "kitti", ARGS))


# ---------------------------------------------------------------------------------------------- torchrun, two GPUs

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_torchrun_two_processes_match_one(kitti_root, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    tool = os.path.join(ROOT, "tools", "train.py")
    args = ["kitti", "fast"] + ARGS
    out = {}
    for name, pre in (("one", [sys.executable]),
                      ("two", [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                               "--master-addr", "127.0.0.1", "--master-port", str(_free_port())])):
        root = _fresh(kitti_root, tmp_path / name)
        r = subprocess.run(pre + [tool] + args + ["-data_root", root], capture_output=True, text=True, cwd=ROOT,
                           timeout=1800)
        assert r.returncode == 0, r.stderr[-3000:]
        lines = [l.rsplit("\t", 1)[0] if l.count("\t") == 3 else l.split("\t")[:-1] if "\t" in l else l
                 for l in r.stdout.splitlines()]
        out[name] = lines, open(train.net_path(root, "kitti", ARGS), "rb").read()
    assert out["two"] == out["one"]
