"""Time the devkit scoring (mc-cnn_b200/kitti_eval.py) against predict_kitti.py test on synthetic full-size KITTI trees.

    python tools/time_kitti_eval.py [--pairs 20]

For 2012 (grey) and 2015 (RGB): synth.write_kitti_raw trees of --pairs training pairs of 375x1242 / 1241 / 1224 with
synth.write_kitti_eval_maps' disp_occ and obj_map, and a random net of the published KITTI 'fast' shape written by
t7.save_net.  Reports, with the card's name and power limit read in the same run:

1. the whole loop, predict_kitti `test` against kitti_eval `predict` (the printed lines muted), alternated three times after
   one untimed warm-up run of each: seconds per pair, and the difference per pair;
2. the scoring alone: kitti_eval.devkit_counts of one device map (the float map, the ground truths uploaded from the host as
   the loop does), timed with CUDA events around 50 calls per pair after a warm-up, median over the pairs; and the kernels
   alone with the ground truths already on the device.
"""
import argparse
import os
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from time_preprocess_mb import card  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=20)
    args = ap.parse_args(argv)

    import numpy as np
    import torch

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import evaluate, frontend, kitti_eval as ke, predict_kitti as pk, synth, t7
    from oracle import feature_tower as oft

    print("card: %s" % card(), flush=True)
    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as root:
        net = os.path.join(root, "fast.t7")
        t7.save_net(net, oft.make_weights(np.random.default_rng(0), l1=4, fm=64))
        for k, ds in enumerate(("kitti", "kitti2015")):
            unzip = synth.write_kitti_raw(root, ds, n_tr=args.pairs, n_te=0, seed=k)
            synth.write_kitti_eval_maps(unzip, ds, seed=k)
            files = ke.training_files(root, ds)
            n = len(files)
            what = "%s, %d pairs of 375x1242/1241/1224, arch fast, disp_max 228" % (ds, n)
            runs = {"predict_kitti test": lambda: pk.predict_kitti("test", ds, net_fname=net, data_root=root, verbose=False),
                    "kitti_eval predict": lambda: ke.evaluate_training(ds, net, "fast", data_root=root, verbose=False)}
            for f in runs.values():
                f()                                                  # warm-up
            per_pair = {name: [] for name in runs}
            for _ in range(3):
                for name, f in runs.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    f()
                    torch.cuda.synchronize()
                    per_pair[name].append((time.perf_counter() - t0) / n * 1e3)
            for name, ts in per_pair.items():
                print("%s: %s, whole loop: %s ms per pair" % (what, name, " / ".join("%.2f" % t for t in ts)), flush=True)
            diffs = [b - a for a, b in zip(*per_pair.values())]
            print("%s: kitti_eval predict - predict_kitti test: %s ms per pair" % (what, " / ".join("%+.2f" % d for d in diffs)),
                  flush=True)

            ev = evaluate.Evaluator(ds, "fast", net_fname=net)
            ev.prepare([(375, 1242, 228)])
            decoded = [pk.decode(f[:3]) + ke._decode_maps(f[3:]) for f in files[:6]]
            maps = [ev.stereo_predict(frontend.make_batch_cuda(p[0], p[1], dev), 228).clone() for p in decoded]
            torch.cuda.synchronize()
            ev.close()
            on_dev = [tuple(torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).to(dev) if a is not None else None
                            for a in p[2:]) for p in decoded]
            reps = 50
            for label, gts in (("ground truths from the host", [p[2:] for p in decoded]), ("kernels alone", on_dev)):
                ts = []
                for m, g in zip(maps, gts):
                    ke.devkit_counts(m, *g)                          # warm-up
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(reps):
                        ke.devkit_counts(m, *g)
                    b.record()
                    b.synchronize()
                    ts.append(a.elapsed_time(b) / reps)
                print("%s: devkit_counts per pair, %s: %.3f ms (median over %d pairs)" % (what, label, statistics.median(ts),
                                                                                           len(ts)), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
