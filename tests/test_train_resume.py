"""CPU: checkpointing and resuming a training run without a GPU -- the random stream's state, the host side of the epoch
loop driven through a recording stand-in for the Trainer (KITTI and Middlebury draws, split mid-epoch and at an epoch
end, across the lr drop), the checkpoint file and its refusals, and the tools' options."""
import itertools
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import dataio, synth, train  # noqa: E402

EPOCHS = 13                                             # past the lr drop at epoch 12


def test_stream_round_trip_with_carry():
    a = train.Stream(7)
    a.raw(1000)
    words = a.raw(37)
    a.unread(words[5:])                                  # 32 words handed back, as the mb draws do
    assert len(a.carry) == 32
    key, pos, carry = a.state()
    b = train.Stream(99)
    b.raw(12)
    b.restore(key, pos, carry)
    assert np.array_equal(b.carry, a.carry)
    sizes = [1, 31, 100, 624, 5000, 623, 93621]         # 10^5 words in uneven pieces, through and past the carry
    assert sum(sizes) == 10 ** 5
    got = np.concatenate([b.raw(n) for n in sizes])
    want = a.raw(10 ** 5)
    assert np.array_equal(got, want)


class Recorder:
    """A Trainer without a GPU: records each chunk's warp bytes, step count and lr.  Its parameters, momenta and losses
    are exact functions of the records it has run, so a resumed run that fed different chunks, or lost its state, would
    end elsewhere."""

    P = 1 << 16

    def __init__(self, o):
        self.N = 2 * o["bs"]
        self.chunks = []
        self.params = np.zeros(8, np.float32)
        self.momenta = np.zeros(8, np.float32)
        self._losses = []

    def reset_losses(self):
        self._losses = []

    def run_chunk(self, warps, lr):
        n = len(warps) // self.N
        assert n * self.N == len(warps) and 1 <= n <= train.CHUNK
        self.chunks.append((warps.tobytes(), n, lr))
        for s in range(n):
            c = int(warps[s * self.N:(s + 1) * self.N].view(np.uint8).astype(np.int64).sum() % self.P)
            self.momenta = ((self.momenta.astype(np.int64) * 3 + c) % self.P).astype(np.float32)
            self.params = ((self.params.astype(np.int64) * 7 + self.momenta.astype(np.int64) + np.arange(8)) %
                           self.P).astype(np.float32)
            self._losses.append(np.float32(c / self.P))

    def losses(self, n):
        assert n <= len(self._losses)
        return np.array(self._losses[:n], np.float32)

    def state(self):
        return self.params.copy(), self.momenta.copy()

    def load_state(self, params, momenta):
        self.params, self.momenta = np.array(params, np.float32), np.array(momenta, np.float32)


def _kitti_case():
    o = train.options("kitti", "fast", bs=4)
    rng = np.random.default_rng(1)
    nnz = np.stack([rng.integers(1, 4, 1230), rng.integers(0, 48, 1230), rng.integers(0, 130, 1230),
                    rng.uniform(0, 30, 1230)], 1).astype(np.float32)
    ws = 1 + 2 * o["l1"]
    return o, nnz, lambda stream: (lambda n, rows: train.make_warps(train.draw_params(stream, o, n * 2), rows, ws))


def _mb_case():
    o = train.options("mb", "slow", bs=4, d_exp=0.5, d_light=0.5)
    rng = np.random.default_rng(2)
    counts = {1: (1, 3), 2: (3, 2), 3: (2, 1)}
    nnz = np.stack([rng.integers(1, 4, 1230), rng.integers(0, 40, 1230), rng.integers(0, 90, 1230),
                    rng.uniform(0, 10, 1230)], 1).astype(np.float32)
    ts = train.MbTrainSet.from_counts(nnz, counts)
    ws = 1 + 2 * o["l1"]
    return o, nnz, lambda stream: (lambda n, rows: ts.warps(stream, o, rows, ws))


CASES = {"kitti": _kitti_case, "mb": _mb_case}


def _counter():
    """a clock that advances by one at every reading: -stop_after m stops at the m-th chunk boundary checked"""
    c = itertools.count()
    return lambda: next(c)


def _run(case, ckpt=None, resume_from=None):
    """one invocation of the loop -> (Recorder, epoch lines without the seconds, stopped)"""
    o, nnz, make_build = CASES[case]()
    stream = train.Stream(42)
    perm = train.randperm(stream, len(nnz))
    train.init_net(stream, o)
    tr = Recorder(o)
    start = None
    if resume_from:
        start = train.load_checkpoint(resume_from, ckpt.fp)
        stream.restore(start["mt_key"], start["mt_pos"], start["carry"])
        tr.load_state(start["params"], start["momenta"])
    lines = []
    try:
        train.fit(tr, nnz, perm, make_build(stream), o, stream, epochs=EPOCHS, log=lines.append, ckpt=ckpt, start=start)
        stopped = None
    except train.Stopped as e:
        stopped = (e.epoch, e.step)
    return tr, [l.rsplit("\t", 1)[0] for l in lines], stopped


def _fp(case):
    o, nnz, _ = CASES[case]()
    return train.fingerprint(case, "train_tr", o, 42, train.cmd_str(case, ["-a", "train_tr"], train.arch_of(o)), nnz,
                             [("x0.bin", (3, 1, 48, 130))])


@pytest.mark.parametrize("case", ["kitti", "mb"])
def test_resumed_chunks_equal_uninterrupted(case, tmp_path):
    o, nnz, _ = CASES[case]()
    nsteps = train.steps_per_epoch(len(nnz), o["bs"])
    assert nsteps == 614 and -(-nsteps // train.CHUNK) == 3          # three chunks, the last one partial
    whole, whole_lines, _ = _run(case)
    assert len(whole.chunks) == 3 * EPOCHS and len(whole_lines) == EPOCHS
    assert [c[2] for c in whole.chunks] == [o["lr"]] * 33 + [o["lr"] / 10] * 6
    path = str(tmp_path / "net_x.state.npz")
    fp = _fp(case)
    # boundaries checked per epoch: two mid-epoch ones, then the epoch's end (none after the last epoch)
    a, lines_a, stop_a = _run(case, train.Checkpoints(path, fp, stop_after=2, clock=_counter()))
    assert stop_a == (1, 512)
    b, lines_b, stop_b = _run(case, train.Checkpoints(path, fp, stop_after=31, clock=_counter()), resume_from=path)
    assert stop_b == (12, 0)                                           # at the end of epoch 11, before the lr drop
    st = train.load_checkpoint(path, fp)
    assert (st["epoch"], st["step"], st["lr"], len(st["losses"])) == (12, 0, o["lr"] / 10, 0)
    c, lines_c, stop_c = _run(case, train.Checkpoints(path, fp), resume_from=path)
    assert stop_c is None
    assert a.chunks + b.chunks + c.chunks == whole.chunks
    assert lines_a + lines_b + lines_c == whole_lines
    assert np.array_equal(c.params, whole.params) and np.array_equal(c.momenta, whole.momenta)


@pytest.mark.parametrize("case", ["kitti", "mb"])
def test_checkpointing_changes_nothing(case, tmp_path):
    whole, whole_lines, _ = _run(case)
    path = str(tmp_path / "net_x.state.npz")
    got, lines, stopped = _run(case, train.Checkpoints(path, _fp(case), steps=256))
    assert stopped is None and got.chunks == whole.chunks and lines == whole_lines
    st = train.load_checkpoint(path, _fp(case))                       # the last epoch's end
    assert (st["epoch"], st["step"]) == (EPOCHS + 1, 0)
    assert np.array_equal(st["params"], whole.params)
    assert not os.path.exists(path + ".tmp")


def test_mid_epoch_checkpoint_holds_the_epochs_losses(tmp_path):
    path = str(tmp_path / "s.state.npz")
    tr, _, stopped = _run("mb", train.Checkpoints(path, _fp("mb"), steps=512, stop_after=5, clock=_counter()))
    assert stopped == (2, 512)
    st = train.load_checkpoint(path, _fp("mb"))
    assert np.array_equal(st["losses"], tr.losses(512))                # epoch 2's steps 0 .. 511
    assert len(st["carry"]) > 0                                         # the mb draws handed words back
    assert st["elapsed"] >= 0 and st["lr"] == train.options("mb", "slow")["lr"]


def _state(path, fp, **kw):
    s = train.Stream(3)
    s.raw(100)
    s.unread(np.arange(5, dtype=np.uint32))
    args = dict(epoch=4, step=768, lr=0.002, elapsed=12.5, params=np.arange(10, dtype=np.float32),
                momenta=-np.arange(10, dtype=np.float32), losses=np.linspace(0, 1, 768).astype(np.float32), stream=s)
    args.update(kw)
    train.save_checkpoint(path, fp, **args)
    return s


def test_file_round_trip_and_atomic_replace(tmp_path):
    path = str(tmp_path / "net_kitti_fast_-a_train_tr.state.npz")
    fp = _fp("kitti")
    with open(path + ".tmp", "wb") as f:                               # a stale temporary file of an interrupted write
        f.write(b"not a checkpoint")
    s = _state(path, fp)
    assert not os.path.exists(path + ".tmp")
    st = train.load_checkpoint(path, fp)
    assert (st["epoch"], st["step"], st["lr"], st["elapsed"]) == (4, 768, 0.002, 12.5)
    assert np.array_equal(st["params"], np.arange(10, dtype=np.float32))
    assert np.array_equal(st["momenta"], -np.arange(10, dtype=np.float32))
    assert np.array_equal(st["losses"], np.linspace(0, 1, 768).astype(np.float32))
    assert st["version"] == mccnn_b200.adcensus.version()
    r = train.Stream(0)
    r.restore(st["mt_key"], st["mt_pos"], st["carry"])
    assert np.array_equal(r.raw(2000), s.raw(2000))
    with open(path + ".tmp", "wb") as f:                               # a stale temporary file beside a good checkpoint
        f.write(b"\0" * 100)
    assert train.load_checkpoint(path, fp)["step"] == 768
    _state(path, fp, step=1024)                                        # a later write replaces both
    assert train.load_checkpoint(path, fp)["step"] == 1024 and not os.path.exists(path + ".tmp")


def test_file_refusals(tmp_path):
    path = str(tmp_path / "c.state.npz")
    fp = _fp("kitti")
    _state(path, fp)
    data = open(path, "rb").read()
    bad = str(tmp_path / "bad.state.npz")
    for cut in (0, 100, len(data) // 2, len(data) - 10):
        with open(bad, "wb") as f:
            f.write(data[:cut])
        with pytest.raises(train.CheckpointError, match="truncated"):
            train.load_checkpoint(bad, fp)
    with np.load(path) as z:
        fields = {k: z[k] for k in z.files}
    np.savez(bad, **dict(fields, format=np.int64(2)))
    with pytest.raises(train.CheckpointError, match="format 2, this library reads format 1"):
        train.load_checkpoint(bad, fp)
    np.savez(bad, **{k: v for k, v in fields.items() if k != "carry"})
    with pytest.raises(train.CheckpointError, match="lacks carry"):
        train.load_checkpoint(bad, fp)


def _refused(path, fp, field):
    with pytest.raises(train.CheckpointError, match="another run: %s is" % field):
        train.load_checkpoint(path, fp)


def test_fingerprint_refusals_name_the_field(tmp_path):
    path = str(tmp_path / "c.state.npz")
    o, nnz, _ = _kitti_case()
    shapes = [("x0.bin", (3, 1, 48, 130)), ("x1.bin", (3, 1, 48, 130))]
    fp = lambda **kw: train.fingerprint(*[kw.get(k, v) for k, v in (  # noqa: E731
        ("dataset", "kitti"), ("action", "train_tr"), ("o", o), ("seed", 42), ("cmd", "kitti_fast_-a_train_tr"),
        ("nnz", nnz), ("shapes", shapes), ("rect", None))])
    _state(path, fp())
    train.load_checkpoint(path, fp())
    _refused(path, fp(dataset="kitti2015"), "dataset")
    _refused(path, fp(action="train_all"), "action")
    _refused(path, fp(seed=43), "seed")
    _refused(path, fp(cmd="kitti_fast_-a_train_tr_-bs_4"), "cmd_str")
    _refused(path, fp(rect="perfect"), "rect")
    _refused(path, fp(nnz=nnz[:-1]), "nnz_rows")
    other = nnz.copy()
    other[7, 3] += 1
    _refused(path, fp(nnz=other), "nnz_sha256")
    _refused(path, fp(shapes=[("x0.bin", (3, 1, 48, 131)), shapes[1]]), "shapes")
    _refused(path, fp(o=train.options("kitti", "slow", bs=4)), "arch")
    with pytest.raises(train.CheckpointError, match="option -lr is 0.002 there, 0.003 here"):
        train.load_checkpoint(path, fp(o=dict(o, lr=0.003)))
    with pytest.raises(train.CheckpointError, match="option -hflip"):
        train.load_checkpoint(path, fp(o=dict(o, hflip=1)))


def test_option_refusals():
    for k in (256, 512, 256 * 40):
        train.check_checkpoint_options(k, 1.0)
    for k in (0, -256, 100, 257, 384):
        with pytest.raises(train.CheckpointError, match="-checkpoint_steps %d: must be a positive multiple of the chunk "
                                                        "size 256" % k):
            train.check_checkpoint_options(k)
    for s in (0, -1.5):
        with pytest.raises(train.CheckpointError, match="-stop_after"):
            train.check_checkpoint_options(None, s)
    with pytest.raises(train.CheckpointError, match="-checkpoint_steps 100"):
        train.Checkpoints("x", {}, steps=100)


@pytest.mark.parametrize("argv, msg", [
    (["-checkpoint_steps", "100"], "-checkpoint_steps 100: must be a positive multiple"),
    (["-checkpoint_steps", "0"], "-checkpoint_steps 0: must be a positive multiple"),
    (["-stop_after", "0"], "-stop_after 0.0: must be a positive"),
    (["-stop_after", "-3", "-resume"], "-stop_after -3.0: must be a positive"),
])
def test_cli_refuses_bad_options(argv, msg, tmp_path):
    import train as tool

    with pytest.raises(SystemExit, match=msg):
        tool.main(["kitti", "fast", "-a", "train_tr", "-data_root", str(tmp_path)] + argv)
    assert os.listdir(str(tmp_path)) == []


def test_names_ignore_the_options():
    import train as tool

    base = ["kitti", "fast", "-a", "train_tr", "-lr", "0.01"]
    for extra in (["-checkpoint_steps", "512"], ["-stop_after", "3000"], ["-resume"],
                  ["-resume", "-stop_after", "10", "-checkpoint_steps", "256"], ["-stop_after=5", "-checkpoint_steps=256"]):
        for argv in (base + extra, base[:4] + extra + base[4:]):
            args, _, _ = tool.parse_args(argv)
            assert tool.main_args(args.argv) == ["-a", "train_tr", "-lr", "0.01"], argv
    args, _, _ = tool.parse_args(base + ["-resume", "-stop_after", "10", "-checkpoint_steps", "256"])
    assert (args.resume, args.stop_after, args.checkpoint_steps) == (True, 10.0, 256)
    args, _, _ = tool.parse_args(base)
    assert (args.resume, args.stop_after, args.checkpoint_steps) == (False, None, None)
    assert train.checkpoint_path("/d", "kitti", ["-a", "train_tr"], "fast") == "/d/net/net_kitti_fast_-a_train_tr.state.npz"
    assert train.net_path("/d", "kitti", ["-a", "train_tr"], "fast") == "/d/net/net_kitti_fast_-a_train_tr.t7"


def _kitti_tree(root):
    d = synth.write_kitti_set(str(root), "kitti", n_tr=3, n_te=1, H=24, width=60, widths=(60,), seed=1)
    rng = np.random.default_rng(0)
    nnz = np.stack([rng.integers(1, 4, 300), rng.integers(0, 24, 300), rng.integers(0, 60, 300),
                    rng.uniform(0, 10, 300)], 1).astype(np.float32)
    dataio.tofile(os.path.join(d, "nnz_tr.bin"), nnz)
    return nnz


def test_cli_refuses_a_foreign_checkpoint_before_gpu_work(tmp_path, capsys):
    import train as tool

    nnz = _kitti_tree(tmp_path)
    o = train.options("kitti", "fast")
    cmd = train.cmd_str("kitti", ["-a", "train_tr"], "fast")
    path = train.checkpoint_path(str(tmp_path), "kitti", ["-a", "train_tr"], "fast")
    os.makedirs(os.path.dirname(path))
    shapes = [("x0.bin", (4, 1, 24, 60)), ("x1.bin", (4, 1, 24, 60))]
    _state(path, train.fingerprint("kitti", "train_tr", o, 7, cmd, nnz, shapes))            # another seed
    argv = ["kitti", "fast", "-a", "train_tr", "-data_root", str(tmp_path), "-resume"]
    with pytest.raises(SystemExit, match="another run: seed is 7 there, 42 here"):
        tool.main(argv)
    _state(path, train.fingerprint("kitti", "train_tr", o, 42, cmd, nnz[:-1], shapes))      # other nnz rows
    with pytest.raises(SystemExit, match="nnz_rows is 299 there, 300 here"):
        tool.main(argv)
    with open(path, "wb") as f:
        f.write(b"PK\3\4")
    with pytest.raises(SystemExit, match="truncated"):
        tool.main(argv)
    assert sorted(os.listdir(os.path.dirname(path))) == [os.path.basename(path)]    # no net was written
    net = train.net_path(str(tmp_path), "kitti", ["-a", "train_tr"], "fast")
    open(net, "wb").close()                                                          # an existing net, checkpoint or not
    with pytest.raises(SystemExit, match="already exists; remove it first"):
        tool.main(argv)
