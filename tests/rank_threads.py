"""The ranks of a row-band run as threads of one process (test infrastructure).

rowband.band_chain takes its communicator as an argument and uses four primitives of it: send, recv, exchange and
barrier (halo and all_gather_rows are built on those).  LocalComm implements them over in-process queues, so the band
paths that only run with more than one rank -- halo exchanges, the SGM wavefront's line states, the gathers, write_outputs
from several ranks -- run on the CPU oracle or on ONE GPU without a process group, a port or a second process.

* Only one rank issues library calls at a time: a rank holds the hub's token while it runs and releases it only while
  it blocks in recv or barrier.  The run is deterministic, and what is under test is the band chain, not the library's
  host-thread safety.
* send stages a host copy (``.to("cpu", copy=True)`` waits for the sender's stream) and never blocks, so exchange
  (sends, then receives) cannot deadlock.  Staging through the host also keeps the sender's buffers out of another rank's
  stream: a device tensor handed over directly could be reused by the caching allocator while the receiver still reads it.
* On a GPU every rank runs on a stream of its own, as it would on its own device: an operator that strayed onto the legacy
  default stream would no longer be serialised with the other ranks' work by accident.
* A rank that fails wakes the others (their recv / barrier raise); run_ranks joins every thread with a bound, checks that
  none is left, and re-raises the first failure.  Nothing outlives the call.
"""
import queue
import threading
import time

import torch

import mccnn_b200  # noqa: F401
from mccnn_b200 import rowband


class PeerFailed(RuntimeError):
    """raised in a rank that waits on a rank which has already failed"""


class Hub:
    """What the ranks of one run share: a queue per ordered pair (src, dst), a barrier and the token."""

    def __init__(self, world, timeout=120.0):
        self.world, self.timeout = world, float(timeout)
        self.queues = {(s, d): queue.Queue() for s in range(world) for d in range(world) if s != d}
        self.bar = threading.Barrier(world)
        self.token = threading.Lock()
        self.failed = threading.Event()

    def fail(self):
        self.failed.set()
        self.bar.abort()


class LocalComm(rowband.Comm):
    """rowband.Comm for rank `rank` of a Hub's ranks"""

    def __init__(self, hub, rank):
        self.hub, self.on, self.rank, self.world = hub, True, rank, hub.world

    def _blocked(self, fn):
        """fn() with the token released (another rank may run meanwhile)"""
        self.hub.token.release()
        try:
            return fn()
        finally:
            self.hub.token.acquire()

    def send(self, t, peer):
        self.hub.queues[(self.rank, peer)].put(t.detach().to("cpu", copy=True))

    def _get(self, peer):
        q, deadline = self.hub.queues[(peer, self.rank)], time.monotonic() + self.hub.timeout
        while True:
            try:
                return q.get(timeout=0.05)
            except queue.Empty:
                if self.hub.failed.is_set():
                    raise PeerFailed("rank %d: a peer failed while it waited for rank %d" % (self.rank, peer))
                if time.monotonic() > deadline:
                    raise TimeoutError("rank %d: nothing from rank %d in %.0f s" % (self.rank, peer, self.hub.timeout))

    def _take(self, t, peer):
        x = self._blocked(lambda: self._get(peer))
        if tuple(x.shape) != tuple(t.shape) or x.dtype != t.dtype:
            raise RuntimeError("rank %d: received %s %s from rank %d into %s %s" % (
                self.rank, tuple(x.shape), x.dtype, peer, tuple(t.shape), t.dtype))
        t.copy_(x)

    def recv(self, t, peer):
        """the point-to-point receive; band_chain calls it directly only for the SGM wavefront's line states"""
        self._take(t, peer)

    def exchange(self, sends, recvs):
        for p, t in sends.items():
            if p != self.rank:
                self.send(t.contiguous(), p)
        for p, t in recvs.items():
            if p != self.rank:
                self._take(t, p)

    def barrier(self):
        def wait():
            try:
                self.hub.bar.wait(self.hub.timeout)
            except threading.BrokenBarrierError:
                raise PeerFailed("rank %d: the barrier was broken (a peer failed or timed out)" % self.rank) from None

        self._blocked(wait)


def run_ranks(world, fn, device=None, timeout=120.0, comm_type=LocalComm):
    """fn(comm) on `world` rank threads, each with a LocalComm; returns the per-rank results.  With `device` (a CUDA
    device), every rank runs on that device on a stream of its own and waits for it before returning.  `comm_type`: a
    LocalComm subclass (a test can corrupt what a rank receives).  The first exception of any rank is re-raised after
    every thread has ended."""
    hub = Hub(world, timeout)
    out, errs, lock = [None] * world, [], threading.Lock()

    def body(r):
        with hub.token:
            try:
                comm = comm_type(hub, r)
                if device is None:
                    out[r] = fn(comm)
                else:
                    with torch.cuda.device(device), torch.cuda.stream(torch.cuda.Stream(device)):
                        out[r] = fn(comm)
                        torch.cuda.current_stream().synchronize()
            except BaseException as e:  # noqa: B902 -- re-raised by run_ranks
                with lock:
                    errs.append((r, e))
                hub.fail()

    threads = [threading.Thread(target=body, args=(r,), name="rank%d" % r, daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    deadline = time.monotonic() + timeout + 30.0
    for t in threads:
        t.join(max(0.0, deadline - time.monotonic()))
    alive = [t.name for t in threads if t.is_alive()]
    assert not alive, "rank threads still running after %.0f s: %s" % (timeout + 30.0, alive)
    if errs:
        first = next((e for _, e in errs if not isinstance(e, PeerFailed)), errs[0][1])
        raise first
    return out
