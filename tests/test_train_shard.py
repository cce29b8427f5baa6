"""CPU: data-parallel training -- for arch 'fast' the residue-class split of wgrad_kernel's tree, modelled in float32 numpy,
gives the one-GPU tree's bits; for arch 'slow' every weight-gradient split of every layer has exactly one owner, which
runs the tower on every patch the split reads; each rank's share of a chunk's records puts the chunk back together; and
the training tools refuse a rank count the split cannot reproduce before any GPU work."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import train  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_cases  # noqa: E402

NT = train.WGRAD_THREADS


def _tree(red):
    """wgrad_kernel's shared-memory tree over red (len a power of two), strides len / 2 .. 1, float32 -> the root"""
    red = red.copy()
    s = len(red) // 2
    while s:
        red[:s] = red[:s] + red[s:2 * s]
        s //= 2
    return red[0]


def _thread_sums(v, nt):
    """thread t of nt sums v[t], v[t + nt], ... in order (float32); the threads past len(v) hold 0"""
    acc = np.zeros(nt, np.float32)
    for n0 in range(0, len(v), nt):
        part = v[n0:n0 + nt]
        acc[:len(part)] = acc[:len(part)] + part
    return acc


def one_gpu(v):
    return _tree(_thread_sums(v, NT))


def sharded(v, R):
    """rank r: its patches r, r + R, ... as local patches, NT / R threads, the local tree; then the tree over the ranks"""
    parts = np.array([_tree(_thread_sums(v[r::R], NT // R)) for r in range(R)], np.float32)
    return _tree(parts)


def _values(N, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(N) * 2.0 ** rng.uniform(-12, 12, N)).astype(np.float32)


@pytest.mark.parametrize("N", [4, 256, 260, 512])
@pytest.mark.parametrize("R", [1, 2, 4, 8])
def test_residue_trees_then_rank_tree_equal_one_tree(N, R):
    for seed in range(20):
        v = _values(N, seed)
        want, got = one_gpu(v), sharded(v, R)
        assert want.tobytes() == got.tobytes(), (seed, want, got)


def test_the_model_tells_orders_apart():
    """the values are such that another order of the same sums changes bits: the test above has teeth"""
    differs = 0
    for seed in range(20):
        v = _values(512, seed)
        parts = np.array([_tree(_thread_sums(v[r::4], NT // 4)) for r in range(4)], np.float32)
        seq = np.float32(0)
        for p in parts:                                                           # the ranks' partials in rank order
            seq = np.float32(seq + p)
        contiguous = _tree(np.array([_tree(_thread_sums(v[r * 128:(r + 1) * 128], NT // 4)) for r in range(4)],
                                    np.float32))
        differs += seq.tobytes() != one_gpu(v).tobytes() or contiguous.tobytes() != one_gpu(v).tobytes()
    assert differs >= 10


@pytest.mark.parametrize("N, R", [(4, 4), (6, 4), (256, 8), (260, 8), (512, 2)])
def test_shares(N, R):
    assert sum(train.shard_size(N, r, R) for r in range(R)) == N
    assert [train.shard_size(N, r, R) for r in range(R)] == [len(range(r, N, R)) for r in range(R)]


def _kitti_chunk(o, nsteps, seed):
    stream = train.Stream(seed)
    h = o["bs"] // 2
    rng = np.random.default_rng(seed)
    rows = np.stack([rng.integers(1, 5, nsteps * h), rng.integers(0, 40, nsteps * h), rng.integers(0, 100, nsteps * h),
                     rng.uniform(0, 30, nsteps * h)], 1).astype(np.float32)
    return train.make_warps(train.draw_params(stream, o, nsteps * h), rows, 1 + 2 * o["l1"])


def _mb_chunk(o, nsteps, seed):
    stream = train.Stream(seed)
    h = o["bs"] // 2
    rng = np.random.default_rng(seed)
    rows = np.stack([rng.integers(1, 4, nsteps * h), rng.integers(0, 40, nsteps * h), rng.integers(0, 100, nsteps * h),
                     rng.uniform(0, 30, nsteps * h)], 1).astype(np.float32)
    mb = train.MbTrainSet.from_counts(rows, {1: (2, 3), 2: (1, 4), 3: (3, 1)})
    return mb.warps(stream, o, rows, 1 + 2 * o["l1"])


@pytest.mark.parametrize("case", train_cases.SLOW_CASES + train_cases.FAST_CASES, ids=train_cases.case_id)
def test_slow_splits_have_one_owner_each(case):
    """the plan of csrc/train.cu (mccnn_trainer_slow_shard_plan) for each case's shapes, as if it were arch slow: the
    ranks' patches [b0, b1) cut the batch in order, each split of each layer has one owner, the split starts in its
    owner's patches, and the owner runs the tower on every patch the split reads"""
    N = 2 * case.bs
    splits = train_cases.split_k(case.l1, case.fm, case.bs)
    L = train_cases.layout(case.l1, case.fm, case.bs)
    o = dict(l1=case.l1, fm=case.fm, bs=case.bs)
    for R in (1, 2, 4, 8):
        if R > N:
            continue
        plans = [train.slow_shard_plan(o, r, R) for r in range(R)]
        assert [p[0] for p in plans] == [N * r // R for r in range(R)] and plans[-1][1] == N
        assert all(plans[r][1] == plans[r + 1][0] for r in range(R - 1))
        for k, (K, kchunk, nsplit) in enumerate(splits):
            P = L.sides[k] ** 2
            owners = np.full(nsplit, -1)
            for r, (b0, b1, e, zs) in enumerate(plans):
                z0, z1, ns = zs[k]
                assert ns == nsplit and b0 < b1 <= e <= N
                for z in range(z0, z1):
                    assert owners[z] == -1, (k, z)
                    owners[z] = r
                    k0, k1 = z * kchunk, min(K, (z + 1) * kchunk)
                    assert b0 <= k0 // P < b1                                   # starts in the owner's patches
                    assert b0 <= k0 // P and -(-k1 // P) <= e                   # reads only patches the owner runs
            assert (owners >= 0).all(), (R, k)
            assert (np.diff(owners) >= 0).all()                                 # contiguous, in rank order


@pytest.mark.parametrize("dataset", ["kitti", "mb"])
@pytest.mark.parametrize("arch", ["fast", "slow"])
@pytest.mark.parametrize("bs", [2, 130, 128])
def test_rank_shares_concatenate_to_the_chunk(dataset, arch, bs):
    o = train.options(dataset, arch, bs=bs)
    N, nsteps = 2 * bs, 5
    chunk = (_kitti_chunk if dataset == "kitti" else _mb_chunk)(o, nsteps, 3)
    assert len(chunk) == nsteps * N
    for R in (1, 2, 4, 8):
        if R > N:
            continue
        shares = [train.shard_warps(chunk, o, r, R).reshape(nsteps, -1) for r in range(R)]
        assert [s.shape[1] for s in shares] == [train.shard_patches(o, r, R)[2] for r in range(R)]
        back = np.zeros((nsteps, N), train.WARP_DTYPE)
        for r, s in enumerate(shares):
            first, stride, count = train.shard_patches(o, r, R)
            if arch == "fast":
                assert (first, stride, count) == (r, R, train.shard_size(N, r, R))
                back[:, r::R] = s
            else:
                b0, b1, e, _ = train.slow_shard_plan(o, r, R)
                assert (first, stride, count) == (b0, 1, e - b0)
                assert s.tobytes() == np.ascontiguousarray(chunk.reshape(nsteps, N)[:, b0:e]).tobytes()
                back[:, b0:b1] = s[:, :b1 - b0]
        assert back.tobytes() == chunk.tobytes()


def test_check_world():
    for arch in ("fast", "slow"):
        o = train.options("kitti", arch)
        for w in (1, 2, 4, 8, 256):
            train.check_world(w, o)
        for w, msg in ((3, "power of two"), (6, "power of two"), (512, "more ranks than the 256 patches")):
            with pytest.raises(ValueError, match=msg):
                train.check_world(w, o)
        with pytest.raises(ValueError, match="more ranks than the 4 patches"):
            train.check_world(8, train.options("kitti", arch, bs=2))


@pytest.mark.parametrize("tool, argv, world, msg", [
    ("train", ["kitti", "fast", "-a", "train_tr"], 3, "power of two"),
    ("train", ["kitti2015", "fast", "-a", "train_all", "-bs", "2"], 8, "more ranks than the 4 patches"),
    ("train_slow", ["kitti", "slow", "-a", "train_tr"], 6, "power of two"),
    ("train_slow", ["kitti", "slow", "-a", "train_tr", "-bs", "2"], 8, "more ranks than the 4 patches"),
    ("train_mb", ["mb", "fast", "-a", "train_tr"], 12, "power of two"),
    ("train_mb", ["mb", "slow", "-a", "train_tr", "-bs", "2"], 16, "more ranks than the 4 patches"),
    ("train", ["kitti", "fast", "-a", "train_tr", "-gpu", "2"], 2, "-gpu under torchrun"),
    ("train_mb", ["mb", "slow", "-a", "train_tr", "-gpu", "1"], 4, "-gpu under torchrun"),
])
def test_tools_refuse_rank_counts(tool, argv, world, msg, monkeypatch, tmp_path, capsys):
    """refused before any data is read or a process group is made: the data root does not even exist"""
    import importlib

    monkeypatch.setenv("WORLD_SIZE", str(world))
    monkeypatch.setenv("RANK", "0")
    mod = importlib.import_module(tool)
    with pytest.raises(SystemExit, match=msg):
        mod.main(argv + ["-data_root", str(tmp_path / "missing")])
    assert capsys.readouterr().out == ""
