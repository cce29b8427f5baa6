"""Time predict_kitti.lua's loop (mc-cnn_b200/predict_kitti.py) and its parts on synthetic full-size KITTI trees.

    python tools/time_predict_kitti.py [--pairs 40]

For 2012 (grey) and 2015 (RGB): synth.write_kitti_raw trees of --pairs training pairs of 375x1242 / 1241 / 1224, and a random
net of the published KITTI 'fast' shape (4 layers of 64 3x3 maps) written by t7.save_net.  Reports, each with the card's name
and power limit read in the same run:

1. the whole `test` loop (net load, pipeline creation, every pair, the printed lines muted): pairs/s, with the decode
   prefetch thread and without it, alternated twice after one untimed warm-up run;
2. the image front end alone, per pair from the decoded bytes: frontend.make_batch (numpy) plus the upload of its float
   batch, which is what frontend.predict does, against frontend.make_batch_cuda (upload of the bytes, the kernels, the
   statistics read back); median over the pairs after one warm-up pair;
3. for scale: the PNG decode of one pair on the host, and Evaluator.stereo_predict of one pair on the GPU (medians).
"""
import argparse
import os
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from time_preprocess_mb import card  # noqa: E402


def _median_ms(f, items):
    f(items[0])                                                     # warm-up
    ts = []
    for it in items:
        t0 = time.perf_counter()
        f(it)
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=40)
    args = ap.parse_args(argv)

    import numpy as np
    import torch

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import evaluate, frontend, predict_kitti as pk, synth, t7
    from oracle import feature_tower as oft

    print("card: %s" % card(), flush=True)
    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as root:
        net = os.path.join(root, "fast.t7")
        t7.save_net(net, oft.make_weights(np.random.default_rng(0), l1=4, fm=64))
        for k, ds in enumerate(("kitti", "kitti2015")):
            synth.write_kitti_raw(root, ds, n_tr=args.pairs, n_te=0, seed=k)
            files = pk.pair_files(root, ds, "test")
            what = "%s (%s), %d pairs of 375x1242/1241/1224, arch fast, disp_max 228" % (ds, "grey" if ds == "kitti" else "RGB",
                                                                                         len(files))
            run = lambda prefetch: pk.predict_kitti("test", ds, net_fname=net, data_root=root, prefetch=prefetch, verbose=False)
            run(True)                                                # warm-up: module loads, first launches
            rates = {True: [], False: []}
            for prefetch in (True, False, True, False):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run(prefetch)
                torch.cuda.synchronize()
                rates[prefetch].append(len(files) / (time.perf_counter() - t0))
            for prefetch in (True, False):
                print("%s: whole test loop, prefetch %s: %s pairs/s" % (what, "on " if prefetch else "off",
                                                                       " / ".join("%.2f" % r for r in rates[prefetch])), flush=True)

            decoded = [pk.decode(f) for f in files]

            def host(p):
                f = lambda b: b.astype(np.float32) if b.ndim == 2 else np.ascontiguousarray(b.transpose(2, 0, 1).astype(np.float32))
                torch.from_numpy(frontend.make_batch(f(p[0]), f(p[1]))).to(dev)
                torch.cuda.synchronize()

            def device(p):
                frontend.make_batch_cuda(p[0], p[1], dev)
                torch.cuda.synchronize()

            print("%s: front end per pair: numpy make_batch + upload %.2f ms, make_batch_cuda %.2f ms (medians)"
                  % (what, _median_ms(host, decoded), _median_ms(device, decoded)), flush=True)
            ev = evaluate.Evaluator(ds, "fast", net_fname=net)
            ev.prepare([(375, 1242, 228)])
            xs = [frontend.make_batch_cuda(p[0], p[1], dev) for p in decoded[:6]]
            gpu = _median_ms(lambda x: ev.timed(x, 228), xs)
            ev.close()
            print("%s: PNG decode of one pair (two views and the ground truth) %.2f ms, stereo_predict of one pair %.2f ms "
                  "(medians)" % (what, _median_ms(pk.decode, files), gpu), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
