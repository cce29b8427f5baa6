"""Throughput of the test_te parameter search (mc-cnn_b200/search.py) on a synthetic KITTI-size validation set.

    python tools/time_search.py [-n_te 40] [-archs fast,slow,census] [-evals 3] [-out time_search.json]

Workload: synth.write_kitti_set at 350 x 1242, D = 228 (main.lua's KITTI crop), -n_te test_te images (fewer for arch 'slow'
when the host has less than 0.8 GB of available memory per image for the pinned volume cache); random nets with the
published shapes (fast: 4 x 64-plane layers; slow: 4 x 112-plane layers, head 4 x 384), written with t7.save_net.  Per arch:

* cache_fill_s: Searcher construction for 'slow' -- the scorer head's volumes of every image into pinned memory (0 otherwise);
* evals_per_s: Searcher.score calls per second over -evals random grid points (after one untimed warm-up evaluation);
* h2d_share (slow): the share of one evaluation's wall time the cache's host-to-device copies take when timed alone
  (CUDA events around the staging copies of all images);
* evaluator_s: one Evaluator(...).test('test_te') per candidate -- what hs.py pays per evaluation minus process start-up.

Prints one JSON object with the card's name and power limit, read in the same run.  Needs a GPU; nothing falls back.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W, D = 350, 1242, 228
SLOW_IMAGE_BYTES = 2 * D * H * W * 4


def parser():
    ap = argparse.ArgumentParser(prog="time_search.py", description=__doc__.splitlines()[0])
    ap.add_argument("-n_te", type=int, default=40, help="test_te images (default 40)")
    ap.add_argument("-archs", default="fast,slow,census")
    ap.add_argument("-evals", type=int, default=3, help="timed evaluations per arch")
    ap.add_argument("-seed", type=int, default=0)
    ap.add_argument("-out", default="", help="also write the JSON here")
    return ap


def parse_args(argv=None):
    a = parser().parse_args(argv)
    a.archs = [s for s in a.archs.split(",") if s]
    bad = [s for s in a.archs if s not in ("fast", "slow", "ad", "census")]
    if bad:
        raise SystemExit("time_search.py: unknown arch %s" % ", ".join(bad))
    if a.n_te < 1 or a.evals < 1:
        raise SystemExit("time_search.py: -n_te and -evals must be >= 1")
    return a


def available_host_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0), "power_limit": "not measured"}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60)
        if q.returncode == 0 and q.stdout.strip():
            pl, clk = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
            out.update(power_limit=pl, max_sm_clock=clk)
    except (OSError, subprocess.SubprocessError):
        pass
    return out


def write_world(root, n_te, seed):
    """the synthetic set (test_te = n_te rows: write_kitti_set validates on a third of its training rows) and the two nets"""
    import numpy as np

    from mccnn_b200 import synth, t7
    from oracle import feature_tower as oft
    from oracle import scorer_head as osh

    synth.write_kitti_set(root, "kitti", n_tr=3 * n_te, n_te=1, H=H, width=W, widths=(W,), seed=seed)
    rng = np.random.default_rng(seed + 1)
    nets = {"fast": os.path.join(root, "net_fast.t7"), "slow": os.path.join(root, "net_slow.t7")}
    t7.save_net(nets["fast"], oft.make_weights(rng, l1=4, fm=64))
    t7.save_net(nets["slow"], oft.make_weights(rng, l1=4, fm=112), osh.make_weights(rng, 112, 384, 4))
    return nets


def h2d_share(s, eval_s):
    """time the staging copies of one evaluation alone (CUDA events on the copy stream)"""
    import torch

    n = len(s.examples)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record(s.copy_stream)
    for i in range(n):
        k = i % 2
        with torch.cuda.stream(s.copy_stream):
            s.slots[k][:s.cache[i].numel()].copy_(s.cache[i], non_blocking=True)
    t1.record(s.copy_stream)
    torch.cuda.synchronize()
    h2d = t0.elapsed_time(t1) / 1e3
    return {"h2d_s": h2d, "h2d_share": h2d / eval_s, "h2d_bytes": s.cache_bytes,
            "h2d_GBps": s.cache_bytes / h2d / 1e9}


def time_arch(arch, root, nets, n_avail, n_evals, seed):
    import random

    import torch

    from mccnn_b200 import evaluate, search

    net = nets.get(arch)
    t = time.perf_counter()
    s = search.Searcher("kitti", arch, net_fname=net, data_root=root)
    torch.cuda.synchronize()
    res = {"images": len(s.examples), "construct_s": time.perf_counter() - t, "cache_fill_s": s.cache_fill_seconds}
    rng = random.Random(seed)
    pts = []
    while len(pts) < n_evals + 1:
        ps = dict(search.point(s.params, search.propose("random", s.params, rng)))
        if search.valid(ps):
            pts.append(ps)
    s.score(pts[0])                                                   # warm-up: first launches, tensor-map encoding
    torch.cuda.synchronize()
    t = time.perf_counter()
    scores = [s.score(p)[0] for p in pts[1:]]
    dt = (time.perf_counter() - t) / n_evals
    res.update(eval_s=dt, evals_per_s=1.0 / dt, scores=scores)
    if arch == "slow":
        res.update(h2d_share(s, dt))
    s.close()
    del s
    torch.cuda.empty_cache()
    ev = evaluate.Evaluator("kitti", arch, net_fname=net, **pts[1])
    t = time.perf_counter()
    r = ev.test("test_te", data_root=root, verbose=False)
    res["evaluator_s"] = time.perf_counter() - t
    ev.close()
    res["evaluator_score"] = float("%.14g" % r.mean)
    res["evaluator_matches_search"] = res["evaluator_score"] == scores[0]
    torch.cuda.empty_cache()
    return res


def main(argv=None):
    a = parse_args(argv)
    import torch

    import mccnn_b200  # noqa: F401

    if not torch.cuda.is_available():
        raise SystemExit("time_search.py: no GPU")
    out = {"workload": {"H": H, "W": W, "D": D, "n_te": a.n_te, "evals": a.evals}, "card": card()}
    avail = available_host_bytes()
    with tempfile.TemporaryDirectory() as tmp:
        t = time.perf_counter()
        n_slow = max(1, min(a.n_te, int(0.8 * avail) // SLOW_IMAGE_BYTES))
        roots = {}
        for n in sorted({a.n_te, n_slow if "slow" in a.archs else a.n_te}):
            roots[n] = os.path.join(tmp, "n%d" % n)
            os.makedirs(roots[n])
            write_world(roots[n], n, a.seed)
        out["data_s"] = time.perf_counter() - t
        for arch in a.archs:
            n = n_slow if arch == "slow" else a.n_te
            nets = {k: os.path.join(roots[n], "net_%s.t7" % k) for k in ("fast", "slow")}
            out[arch] = time_arch(arch, roots[n], nets, n, a.evals, a.seed)
            print(json.dumps({arch: out[arch]}), flush=True)
    if n_slow < a.n_te and "slow" in a.archs:
        out["slow_note"] = "slow on %d images: %d bytes of host memory available, %d per image" % (n_slow, avail,
                                                                                                  SLOW_IMAGE_BYTES)
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
