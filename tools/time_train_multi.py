"""Measure data-parallel training (train.Trainer with rank / world / comm) at R = 1 and at every power of two up to the
visible GPUs.

    python tools/time_train_multi.py [-steps 1024] [-repeats 3] [-port 29541] [-json out.json]

The tool runs itself once per rank count R, as a child process: a plain one for R = 1, torch.distributed.run with R
processes (one GPU each, NCCL, rendezvous on 127.0.0.1:-port) for R > 1.  Each run trains kitti fast, mb fast, kitti slow
and mb slow at main.lua's presets (bs 128) on a synthetic device-resident set of 20 images of 350 x 1242, from the same
records on every rank, and reports per preset:

* steps/s:  whole steps, the all-gathers included, chunk after chunk with a device synchronise at the end;
* device:   the same steps with the all-gathers skipped, the segments alone;
* exchange: the difference, in microseconds per step.

A device window leaves each rank's parameters different from the others' (no rank sees the others' gradients), and the
windows after it train on from those parameters.  That changes no launch and no amount of work, so the timings stand, but
the parameters of this tool's runs mean nothing.  Each figure is the median of -repeats windows after a warm-up chunk,
whole and device windows alternated, with the spread (min, max).  The card's name, power limit and maximum SM clock are
printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

PRESETS = (("kitti", "fast"), ("mb", "fast"), ("kitti", "slow"), ("mb", "slow"))
N_IMG, H, W = 20, 350, 1242


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def chunks(o, nsteps, seed=0):
    from mccnn_b200 import train

    stream, h = train.Stream(seed), o["bs"] // 2
    rng = np.random.default_rng(seed)
    out = []
    for s0 in range(0, nsteps, train.CHUNK):
        n = min(train.CHUNK, nsteps - s0)
        rows = np.stack([rng.integers(1, N_IMG + 1, n * h), rng.integers(0, H, n * h), rng.integers(0, W, n * h),
                         rng.uniform(0, 100, n * h)], 1).astype(np.float32)
        out.append(train.make_warps(train.draw_params(stream, o, n * h), rows, 1 + 2 * o["l1"]))
    return out


def measure(dataset, arch, steps, repeats, rank, world, comm, dev):
    import torch

    from mccnn_b200 import train

    o = train.options(dataset, arch)
    g = torch.Generator(device=dev).manual_seed(1)
    X0, X1 = (torch.randn((N_IMG, 1, H, W), device=dev, generator=g) for _ in range(2))
    tr = train.Trainer(o, X0, X1, chunk=train.CHUNK, loss_cap=steps + train.CHUNK, device=dev.index, rank=rank,
                       world=world, comm=comm)
    tr.set_layers(*train.init_net(train.Stream(3), o))
    cs = chunks(o, steps)
    warm = chunks(o, train.CHUNK, seed=1)

    def window(exchange):
        if world > 1 and not exchange:
            tr._all_gather = lambda buf: None
        tr.reset_losses()
        tr.run_chunk(warm[0], o["lr"])
        tr.stream.synchronize()
        if comm is not None:
            comm.barrier()
        t0 = time.perf_counter()
        for c in cs:
            tr.run_chunk(c, o["lr"])
        tr.stream.synchronize()
        dt = time.perf_counter() - t0
        tr.__dict__.pop("_all_gather", None)
        if world > 1:
            t = torch.tensor([dt], dtype=torch.float64, device=dev)
            torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
            dt = float(t.item())
        return steps / dt

    whole, device = [], []
    for _ in range(repeats):                                             # alternated
        whole.append(window(True))
        device.append(window(False))
    tr.close()
    med = lambda v: float(np.median(v))                                  # noqa: E731
    return {"preset": "%s %s" % (dataset, arch), "R": world, "steps_per_s": round(med(whole), 1),
            "steps_per_s_spread": [round(min(whole), 1), round(max(whole), 1)],
            "samples_per_s": round(med(whole) * o["bs"] / 2), "device_steps_per_s": round(med(device), 1),
            "device_spread": [round(min(device), 1), round(max(device), 1)],
            "exchange_us_per_step": round(1e6 * (1 / med(whole) - 1 / med(device)), 1) if world > 1 else 0.0}


def worker(a):
    import torch

    import mccnn_b200  # noqa: F401

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    comm = None
    if world > 1:
        import torch.distributed as dist

        from mccnn_b200 import rowband

        dist.init_process_group("nccl", device_id=dev)
        comm = rowband.Comm()
    try:
        rows = [measure(d, arch, a.steps, a.repeats, rank, world, comm, dev) for d, arch in PRESETS]
    finally:
        if comm is not None:
            torch.distributed.destroy_process_group()
    if rank == 0:
        for r in rows:
            print("RESULT " + json.dumps(r), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("-steps", type=int, default=1024)
    ap.add_argument("-repeats", type=int, default=3)
    ap.add_argument("-port", type=int, default=29541, help="the rendezvous port of the R > 1 runs")
    ap.add_argument("-json", default=None)
    ap.add_argument("-worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    import torch

    n = torch.cuda.device_count()
    if n < 1:
        raise SystemExit("time_train_multi.py: no GPU")
    me = [os.path.abspath(__file__), "-worker", "-steps", str(a.steps), "-repeats", str(a.repeats)]
    rows = []
    R = 1
    while R <= n:
        pre = [sys.executable] if R == 1 else [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                                               "--nproc-per-node", str(R), "--master-addr", "127.0.0.1",
                                               "--master-port", str(a.port)]
        r = subprocess.run(pre + me, capture_output=True, text=True, timeout=3600)
        if r.returncode:
            raise SystemExit("time_train_multi.py: R = %d failed:\n%s" % (R, r.stderr[-3000:]))
        rows += [json.loads(l[len("RESULT "):]) for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        R *= 2
    res = {"card": card(), "visible_gpus": n, "steps": a.steps, "rows": rows}
    print("card: %s, %d visible GPU(s), %d steps per window" % (res["card"], n, a.steps))
    print("%-10s %3s %12s %18s %12s %16s" % ("preset", "R", "steps/s", "spread", "device", "exchange us/step"))
    for r in rows:
        print("%-10s %3d %12.1f %18s %12.1f %16.1f" % (r["preset"], r["R"], r["steps_per_s"], r["steps_per_s_spread"],
                                                       r["device_steps_per_s"], r["exchange_us_per_step"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
