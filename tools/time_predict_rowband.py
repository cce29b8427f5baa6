"""Per-pair time and per-rank peak device memory of the row-band predict (rowband.predict_pair) on N = 1, 2, 4, 8 GPUs.

    python tools/time_predict_rowband.py [--cases kitti_slow,mb_slow,kitti_fast] [--gpus 1,2,4,8] [--iters 3]

For each case and N, runs ``torchrun --nproc-per-node N`` of this script in worker mode.  Every rank builds the same seeded
synthetic pair (standardised on the host, frontend.make_batch) and a random network of the published shapes, then times
predict_pair(want_vols=True) -- the work of main.lua's -a predict, both volumes kept on the device, files not written --
with a device synchronise and a barrier on both sides of each pair, the maximum over the ranks.  Peak memory is
torch.cuda.max_memory_allocated per rank over the timed pairs.  With N = 1 the worker also times the one-GPU path of
frontend.predict (pipeline.stereo_predict with both volumes) on the same inputs.  An N above the visible device count is
reported as not measured.  Prints the card's name and power limit, one JSON line per row and a markdown table.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(1, os.path.dirname(os.path.abspath(__file__)))

# name -> (dataset, arch, H, W, D, tower (l1, fm), head (l2, nh2)): the published shapes of main.lua:70-295
CASES = {
    "kitti_slow": ("kitti", "slow", 350, 1242, 228, (4, 112), (4, 384)),
    "mb_slow": ("mb", "slow", 1000, 1500, 228, (5, 112), (3, 384)),
    "kitti_fast": ("kitti", "fast", 350, 1242, 228, (4, 64), None),
}


def worker(a):
    import numpy as np
    import torch
    import torch.distributed as dist

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import feature_tower, frontend, pipeline, rowband, scorer_head, synth
    from oracle import feature_tower as oft
    from oracle import scorer_head as osh

    dataset, arch, H, W, D, (l1, fm), hd = CASES[a.case]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    comm = rowband.Comm()
    rng = np.random.default_rng(5)
    img = synth.natural_image(rng, H, W + 40)
    x_batch = frontend.make_batch(img[:, 40:], img[:, :W])
    tower = feature_tower.FeatureTower(oft.make_weights(rng, l1=l1, fm=fm), arch=arch, device=dev.index)
    head = scorer_head.ScorerHead(osh.make_weights(rng, fm, hd[1], hd[0]), device=dev.index) if hd else None

    def sync():
        torch.cuda.synchronize(dev)
        comm.barrier()
        torch.cuda.synchronize(dev)

    def timed(fn):
        import time

        fn()                                                   # warm-up
        sync()
        torch.cuda.reset_peak_memory_stats(dev)
        ms = []
        for _ in range(a.iters):
            sync()
            t0 = time.perf_counter()
            out = fn()
            sync()
            ms.append((time.perf_counter() - t0) * 1e3)
            del out
        peak = torch.cuda.max_memory_allocated(dev)
        if world > 1:
            t = torch.tensor(ms, device=dev, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = t.tolist()
            peaks = [torch.zeros(1, device=dev, dtype=torch.int64) for _ in range(world)]
            dist.all_gather(peaks, torch.tensor([peak], device=dev, dtype=torch.int64))
            peak = [int(p.item()) for p in peaks]
        else:
            peak = [peak]
        return ms, peak

    ms, peak = timed(lambda: rowband.predict_pair(x_batch=x_batch, dataset=dataset, arch=arch, disp_max=D, tower=tower,
                                                  head=head, comm=comm, device=dev, want_vols=True))
    res = {"case": a.case, "workload": "%s %s %dx%d D %d" % (dataset, arch, H, W, D), "n_gpus": world,
           "ms_min": round(min(ms), 2), "ms_all": [round(x, 2) for x in ms],
           "peak_gib_per_rank": [round(p / 2 ** 30, 2) for p in peak]}
    if world == 1:
        opt = pipeline.make_params(dataset, arch)

        def one_gpu():
            xb = torch.from_numpy(x_batch).to(dev)
            feats = tower.forward(xb)
            d, vl, vr = pipeline.stereo_predict(xb, feats, opt, D, want_vols=True, arch=arch, head=head)
            return d.cpu(), vl, vr

        ms1, peak1 = timed(one_gpu)
        res.update(frontend_ms_min=round(min(ms1), 2), frontend_ms_all=[round(x, 2) for x in ms1],
                   frontend_peak_gib=round(peak1[0] / 2 ** 30, 2))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print("RESULT " + json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--cases", default="kitti_slow,mb_slow,kitti_fast")
    ap.add_argument("--gpus", default="1,2,4,8")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--case", default=None)
    ap.add_argument("--port", type=int, default=29581)
    a = ap.parse_args()
    if a.worker:
        return worker(a)

    import torch
    from time_preprocess_mb import card

    if not torch.cuda.is_available():
        raise SystemExit("time_predict_rowband.py: no CUDA device")
    ndev = torch.cuda.device_count()
    print("card: %s (%d visible)" % (card(), ndev), flush=True)
    rows = []
    for case in a.cases.split(","):
        for n in [int(x) for x in a.gpus.split(",")]:
            if n > ndev:
                rows.append({"case": case, "n_gpus": n, "not_measured": "only %d device(s) visible" % ndev})
                print(json.dumps(rows[-1]), flush=True)
                continue
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
                   "--master-addr", "127.0.0.1", "--master-port", str(a.port + len(rows)), os.path.abspath(__file__),
                   "--worker", "--case", case, "--iters", str(a.iters)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            lines = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
            if r.returncode != 0 or not lines:
                sys.stderr.write(r.stderr[-3000:])
                rows.append({"case": case, "n_gpus": n, "failed": r.returncode})
            else:
                rows.append(json.loads(lines[-1][len("RESULT "):]))
            print(json.dumps(rows[-1]), flush=True)
    print("\n| case | N | ms / pair (min) | peak GiB per rank | one-GPU frontend.predict path |")
    print("|---|---|---|---|---|")
    for row in rows:
        if "ms_min" not in row:
            print("| %s | %d | not measured | | |" % (row["case"], row["n_gpus"]))
            continue
        ref = "%.1f ms, %.2f GiB" % (row["frontend_ms_min"], row["frontend_peak_gib"]) if "frontend_ms_min" in row else ""
        print("| %s | %d | %.1f | %s | %s |" % (row["workload"], row["n_gpus"], row["ms_min"],
                                               " / ".join("%.2f" % p for p in row["peak_gib_per_rank"]), ref))
    return 1 if any("failed" in row for row in rows) else 0


if __name__ == "__main__":
    sys.exit(main())
