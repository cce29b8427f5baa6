"""GPU: a training run stopped and resumed from its checkpoint gives the bits of an uninterrupted one -- kitti fast and slow,
mb fast and slow, stopped once mid-epoch and once at an epoch's end before the lr drop -- writing checkpoints changes no
bit, and tools/train_mb.py run in a -resume -stop_after loop ends with the net file and epoch lines of one invocation."""
import functools
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, evaluate, preprocess, synth, train  # noqa: E402

EPOCHS = 13                                              # past the lr drop at epoch 12
ROWS = 1400                                              # bs 8: 349 steps, two chunks per epoch


def _rows(rng, images, H, W, d_max):
    return np.stack([rng.choice(images, ROWS), rng.integers(0, H, ROWS), rng.integers(0, W, ROWS),
                     rng.uniform(0, d_max, ROWS)], 1).astype(np.float32)


@pytest.fixture(scope="module")
def kitti_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    d = synth.write_kitti_set(root, "kitti", n_tr=4, n_te=2, H=48, width=130, widths=(130, 121), seed=1)
    dataio.tofile(os.path.join(d, "nnz_tr.bin"), _rows(np.random.default_rng(0), np.arange(1, 5), 48, 121, 30))
    return root


@pytest.fixture(scope="module")
def mb_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("mb"))
    synth.write_mb_raw(root, seed=7)
    preprocess.preprocess_mb(root, "imperfect", "gray")
    return root


def _fresh(src_root, name, tmp_path, nnz_rows=None):
    """a copy of the set (links to its files) with its own net/ and, with `nnz_rows`, its own nnz_tr.bin"""
    src = os.path.join(src_root, name)
    dst = os.path.join(str(tmp_path), name)
    os.makedirs(dst)
    for f in os.listdir(src):
        if not (nnz_rows is not None and f.startswith("nnz_tr.bin")):
            os.symlink(os.path.join(src, f), os.path.join(dst, f))
    if nnz_rows is not None:
        dataio.tofile(os.path.join(dst, "nnz_tr.bin"), nnz_rows)
    return str(tmp_path)


def _mb_rows(mb_root):
    """ROWS of the set's own nnz_tr rows, seeded"""
    nnz = dataio.fromfile(os.path.join(mb_root, "data.mb.imperfect_gray", "nnz_tr.bin")).reshape(-1, 4)
    assert len(nnz) >= ROWS
    return nnz[np.sort(np.random.default_rng(5).choice(len(nnz), ROWS, replace=False))]


CONFIGS = {
    "kitti_fast": ("kitti", dict(l1=2, fm=32, bs=8)),
    "kitti_slow": ("kitti", dict(l1=2, fm=32, l2=1, nh2=128, bs=8)),
    "mb_fast": ("mb", dict(l1=3, fm=32, bs=8)),
    "mb_slow": ("mb", dict(l1=2, fm=32, l2=1, nh2=128, bs=8, d_exp=0.5, d_light=0.5)),
}


def _counter():
    """a clock that advances by one at every reading: -stop_after m stops at the m-th chunk boundary checked"""
    c = itertools.count()
    return lambda: next(c)


def _train(cfg, root, monkeypatch, capsys, **kw):
    """one train.train call -> (epoch lines without seconds, test_te errors, net bytes, (params, momenta), stopped)"""
    dataset, over = CONFIGS[cfg]
    arch = "slow" if "l2" in over else "fast"
    o = train.options(dataset, arch, **over)
    args = ["-a", "train_tr"] + sum((["-" + k, str(v)] for k, v in over.items()), [])
    final = {}
    close = train.Trainer.close

    def keep_state(tr):
        if getattr(tr, "_h", None):
            final["state"] = tr.state()
        close(tr)

    monkeypatch.setattr(train.Trainer, "close", keep_state)
    monkeypatch.setattr(train, "Checkpoints", functools.partial(train.Checkpoints, clock=_counter()))
    lines = []
    capsys.readouterr()
    stopped = None
    try:
        fname = train.train(dataset, "train_tr", o, args=args, data_root=root, epochs=EPOCHS, log=lines.append, **kw)
    except train.Stopped as e:
        stopped, fname = (e.epoch, e.step), None
    test = [l.split("\t")[-1] for l in capsys.readouterr().out.splitlines()]          # runtime excluded
    net = open(fname, "rb").read() if fname else None
    epochs = [l.rsplit("\t", 1)[0] for l in lines if l.count("\t") == 3]
    assert lines[:len(train.net_lines(o))] == train.net_lines(o)
    return epochs, test, net, final.get("state"), stopped, train.checkpoint_path(root, dataset, args, arch)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_resume_is_bit_identical(cfg, kitti_root, mb_root, tmp_path, monkeypatch, capsys):
    dataset = CONFIGS[cfg][0]
    if dataset == "kitti":
        fresh = lambda sub: _fresh(kitti_root, "data.kitti", tmp_path / sub)                      # noqa: E731
    else:
        rows = _mb_rows(mb_root)
        fresh = lambda sub: _fresh(mb_root, "data.mb.imperfect_gray", tmp_path / sub, rows)       # noqa: E731
    ep, test, net, state, stopped, _ = _train(cfg, fresh("whole"), monkeypatch, capsys)
    assert stopped is None and len(ep) == EPOCHS and len(test) >= 2
    lr = train.options(dataset, "slow" if "l2" in CONFIGS[cfg][1] else "fast")["lr"]
    assert [e.split("\t")[2] for e in ep] == [evaluate.lua_num(lr)] * 11 + [evaluate.lua_num(lr / 10)] * 2
    # checkpointing every chunk changes nothing
    root = fresh("ckpt")
    ep2, test2, net2, state2, stopped2, path = _train(cfg, root, monkeypatch, capsys, checkpoint_steps=256)
    assert stopped2 is None and ep2 == ep and test2 == test and net2 == net
    assert all(_same(x, y) for x, y in zip(state2, state))
    assert not os.path.exists(path)                                                 # deleted after the net file
    # boundaries checked per epoch: the one mid-epoch chunk boundary, then the epoch's end
    root = fresh("resumed")
    ep_a, test_a, _, _, stop_a, path = _train(cfg, root, monkeypatch, capsys, stop_after=3, resume=True)
    assert stop_a == (2, 256) and os.path.exists(path) and test_a == []
    ep_b, _, _, _, stop_b, _ = _train(cfg, root, monkeypatch, capsys, stop_after=19, resume=True, checkpoint_steps=256)
    assert stop_b == (12, 0)
    ep_c, test_c, net_c, state_c, stop_c, _ = _train(cfg, root, monkeypatch, capsys, resume=True)
    assert stop_c is None and not os.path.exists(path)
    assert ep_a + ep_b + ep_c == ep                                                 # every epoch's err, bit for bit
    assert test_c == test and net_c == net
    assert all(_same(x, y) for x, y in zip(state_c, state))


def _tool(args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train_mb.py")] + args, capture_output=True,
                          text=True, cwd=ROOT, timeout=1800)


def _epoch_lines(out):
    return [l.rsplit("\t", 1)[0] for l in out.splitlines() if l.count("\t") == 3]


def _test_errors(out):
    """the lines after the last epoch line (test_te's), runtime excluded"""
    lines = out.splitlines()
    last = max(i for i, l in enumerate(lines) if l.count("\t") == 3)
    return [l.split("\t")[-1] for l in lines[last + 1:]]


def test_tool_stop_and_resume_loop(mb_root, tmp_path):
    rows = _mb_rows(mb_root)
    args = ["mb", "fast", "-a", "train_tr", "-l1", "3", "-fm", "32", "-bs", "8"]
    whole = _fresh(mb_root, "data.mb.imperfect_gray", tmp_path / "whole", rows)
    r = _tool(args + ["-data_root", whole])
    assert r.returncode == 0, r.stderr[-3000:]
    want_lines = _epoch_lines(r.stdout)
    want_test = _test_errors(r.stdout)
    assert len(want_lines) == 14
    seconds = float(r.stdout.splitlines()[[i for i, l in enumerate(r.stdout.splitlines()) if l.count("\t") == 3][-1]]
                    .split("\t")[3])
    root = _fresh(mb_root, "data.mb.imperfect_gray", tmp_path / "loop", rows)
    loop = args + ["-data_root", root, "-resume", "-stop_after", "%.3f" % max(seconds / 4, 1e-3)]
    got_lines, codes = [], []
    for _ in range(40):
        r = _tool(loop)
        codes.append(r.returncode)
        got_lines += _epoch_lines(r.stdout)
        if r.returncode != train.EX_TEMPFAIL:
            break
        assert "stopped: checkpoint" in r.stderr and ".state.npz at epoch" in r.stderr, r.stderr[-2000:]
    assert codes[-1] == 0 and set(codes[:-1]) <= {train.EX_TEMPFAIL} and len(codes) >= 2, (codes, r.stderr[-3000:])
    assert got_lines == want_lines
    assert _test_errors(r.stdout) == want_test and len(want_test) >= 3
    name = os.path.basename(train.net_path(root, "mb", args[2:], "fast"))
    assert open(os.path.join(root, "net", name), "rb").read() == open(os.path.join(whole, "net", name), "rb").read()
    assert os.listdir(os.path.join(root, "net")) == [name]                         # the checkpoint is gone
