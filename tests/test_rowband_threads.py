"""CPU: the row-band split of one stereo pair with its ranks as threads of one process (tests/rank_threads.py) and the CPU
oracle standing in for the CUDA operators.  The same driver runs on the CUDA operators in
tests/test_gpu_rowband_threads.py; here it is pinned on the cases of the gloo test and at the edges of its band paths:
1-row bands, column chunks of 1, 7, W and W + 5 (empty chunks skipped), and the second CBCA block's two exchange regimes
(one exchange of n * halo rows, or one of halo rows per iteration).  Every rank's disparity map must equal the
single-process oracle pipeline bit for bit."""
import os
import sys
import threading
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rank_threads import LocalComm, run_ranks  # noqa: E402
from test_rowband_gloo import CASES as GLOO_CASES  # noqa: E402
from test_rowband_gloo import OracleOps  # noqa: E402

import mccnn_b200  # noqa: E402,F401
from mccnn_b200 import pipeline, rowband, synth  # noqa: E402

# name -> ((dataset, arch), overrides, H, W, C, D, world, regime of the second CBCA block)
EDGE_CASES = {
    "kitti_fast_1row_bands": (("kitti", "fast"), {}, 5, 40, 8, 10, 5, None),
    "kitti2015_slow_one_exchange": (("kitti2015", "slow"), {}, 50, 56, 4, 10, 3, "one"),
    "kitti2015_slow_per_iteration": (("kitti2015", "slow"), {}, 47, 56, 4, 10, 3, "per_iteration"),
    "mb_slow_thinnest_band": (("mb", "slow"), {}, 27, 32, 4, 6, 2, "per_iteration"),
    "accurate_cbca4": (("kitti", "accurate_cbca4"), {}, 24, 30, 4, 8, 3, "one"),
}


def _problem(preset, over, H, W, C, D, seed=None):
    opt = pipeline.make_params(*preset, **over)
    return opt, synth.make_pair(H, W, C, D, seed=H + D if seed is None else seed)


def regime(opt, H, world):
    """how band_chain's second CBCA block exchanges halo rows at this split: 'one', 'per_iteration' or None (no exchange)"""
    halo, n = rowband.cbca_halo(opt)[1], int(opt.cbca_i2)
    if halo == 0 or n == 0:
        return None
    band_min = min(b - a for a, b in (rowband.split(H, world, p) for p in range(world)))
    return "one" if n * halo <= band_min else "per_iteration"


def _threaded(orc, opt, p, D, world, chunks=None, comm_type=LocalComm):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))

    def rank(comm):
        return rowband.stereo_predict_rowband(OracleOps(orc), t(p["featL"]), t(p["featR"]), t(p["imgL"]), t(p["imgR"]), D,
                                              opt, comm=comm, chunks=chunks).numpy()

    return run_ranks(world, rank, comm_type=comm_type)


def _want(orc, opt, p, D):
    return orc.stereo_predict(p["featL"], p["featR"], p["imgL"], p["imgR"], D, orc.Params(**opt.as_dict()))


def _assert_all_ranks(outs, want, what):
    for r, got in enumerate(outs):
        assert np.array_equal(got, want, equal_nan=True), "%s: rank %d of %d differs from the single-process pipeline" % (
            what, r, len(outs))


@pytest.mark.parametrize("world,case", [(2, "kitti_slow"), (3, "mb_slow"), (2, "kitti_fast"), (5, "kitti_fast")])
def test_threads_reproduce_the_gloo_cases(oracle, world, case):
    preset, over, H, W, C, D = GLOO_CASES[case]
    opt, p = _problem(preset, over, H, W, C, D)
    _assert_all_ranks(_threaded(oracle, opt, p, D, world), _want(oracle, opt, p, D), case)


@pytest.mark.parametrize("case", sorted(EDGE_CASES))
def test_band_edges(oracle, case):
    preset, over, H, W, C, D, world, want_regime = EDGE_CASES[case]
    opt, p = _problem(preset, over, H, W, C, D, seed=H + 3 * D)
    assert regime(opt, H, world) == want_regime
    _assert_all_ranks(_threaded(oracle, opt, p, D, world), _want(oracle, opt, p, D), case)


@pytest.mark.parametrize("chunks", [1, 7, "W", "W+5"])
def test_column_chunks(oracle, chunks):
    """the SGM wavefront cut into 1, 7, W and W + 5 column chunks (the last: 5 empty chunks, skipped on every rank)"""
    preset, over, H, W, C, D, world, _ = EDGE_CASES["accurate_cbca4"]
    k = {"W": W, "W+5": W + 5}.get(chunks, chunks)
    opt, p = _problem(preset, over, H, W, C, D, seed=H + 3 * D)
    _assert_all_ranks(_threaded(oracle, opt, p, D, world, chunks=k), _want(oracle, opt, p, D), "chunks %s" % chunks)


class HalvedLineStates(LocalComm):
    """a LocalComm that corrupts what arrives through recv: the SGM wavefront's line states"""

    def recv(self, t, peer):
        super().recv(t, peer)
        t.mul_(0.5)


def test_corrupted_line_states_are_seen(oracle):
    """the comparison above sees the line states: halving them on arrival changes the disparity map"""
    preset, over, H, W, C, D = GLOO_CASES["kitti_slow"]
    opt, p = _problem(preset, over, H, W, C, D)
    outs = _threaded(oracle, opt, p, D, 2, comm_type=HalvedLineStates)
    want = _want(oracle, opt, p, D)
    assert not any(np.array_equal(o, want, equal_nan=True) for o in outs)


def _threads_after(before):
    deadline = time.monotonic() + 5.0
    while threading.active_count() > before and time.monotonic() < deadline:
        time.sleep(0.01)
    return threading.active_count()


def test_a_refusal_on_every_rank_is_raised(oracle):
    before = threading.active_count()
    opt, p = _problem(("kitti", "fast"), {"sm_skip": "sgm"}, 8, 16, 4, 4)
    with pytest.raises(ValueError, match="sm_skip"):
        _threaded(oracle, opt, p, 4, 3)
    assert _threads_after(before) == before


def test_a_rank_failing_while_the_others_wait():
    """rank 1 fails before it sends; ranks 0 and 2 wait for it in recv and barrier: its own error comes out, at once"""
    before = threading.active_count()

    def rank(comm):
        if comm.rank == 1:
            raise KeyError("rank 1 fails")
        if comm.rank == 0:
            comm.recv(torch.empty(3), 1)
        comm.barrier()

    t0 = time.monotonic()
    with pytest.raises(KeyError, match="rank 1 fails"):
        run_ranks(3, rank, timeout=60.0)
    assert time.monotonic() - t0 < 10.0
    assert _threads_after(before) == before


def test_a_wait_that_never_ends_times_out():
    def rank(comm):
        if comm.rank == 0:
            comm.recv(torch.empty(3), 1)

    with pytest.raises(TimeoutError):
        run_ranks(2, rank, timeout=0.5)


def test_threads_carry_what_was_sent():
    """exchange, send / recv and barrier deliver each tensor to its peer, in order"""

    def rank(comm):
        n, r = comm.world, comm.rank
        got = {p: torch.empty(2) for p in range(n)}
        comm.exchange({p: torch.tensor([r, p], dtype=torch.float32) for p in range(n)}, got)
        seq = []
        if r == 0:
            for i in range(3):
                comm.send(torch.tensor([float(i)]), n - 1)
        elif r == n - 1:
            for _ in range(3):
                x = torch.empty(1)
                comm.recv(x, 0)
                seq.append(float(x))
        comm.barrier()
        return {p: got[p].tolist() for p in range(n) if p != r}, seq

    out = run_ranks(4, rank)
    for r, (got, seq) in enumerate(out):
        assert got == {p: [float(p), float(r)] for p in range(4) if p != r}
        assert seq == ([0.0, 1.0, 2.0] if r == 3 else [])


class _NoOps:
    def __getattr__(self, name):
        raise AssertionError("operator %s called" % name)


def test_a_band_thinner_than_the_halo_is_refused_before_any_operator():
    """mb slow (L1 14, halo 13) on two bands of 12 and 13 rows"""
    opt = pipeline.make_params("mb", "slow")
    H, W = 25, 32
    with pytest.raises(AssertionError, match="thinner than the CBCA halo"):
        run_ranks(2, lambda comm: rowband.band_chain(_NoOps(), None, True, torch.zeros(H, W), torch.zeros(H, W), 6, opt,
                                                     comm))
