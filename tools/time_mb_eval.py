"""Time the MiddEval3 scoring (mc-cnn_b200/mb_eval.py) on synthetic scenes of MiddEval3 sizes.

    python tools/time_mb_eval.py [--height 994 --width 1482 --ndisp 290]

On a synth.write_mb_raw tree whose 15 trainingH pairs are --height x --width (ndisp --ndisp) with synth.write_mb_eval_gt's
ground truth (the F one is twice the size), and a random net of the published Middlebury 'fast' shape (l1 5, fm 64)
written by t7.save_net.  Reports, with the card's name and power limit read in the same run:

1. mb_eval.evaldisp alone, timed with CUDA events around 50 calls per scene after a warm-up, median over the scenes: at H
   (the ground truth at the map's size, scale 1) and at F (twice the size, scale 2), inputs already on the device;
2. the whole `predict` loop (mb_eval.evaluate_training at res F, the lines muted) after one untimed warm-up run, three
   runs: seconds per scene.
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
    ap.add_argument("--height", type=int, default=994)
    ap.add_argument("--width", type=int, default=1482)
    ap.add_argument("--ndisp", type=int, default=290)
    args = ap.parse_args(argv)

    import numpy as np
    import torch

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import mb_eval as me, preprocess, synth, t7
    from oracle import feature_tower as oft

    print("card: %s" % card(), flush=True)
    dev = torch.device("cuda", 0)
    h, w = args.height, args.width
    with tempfile.TemporaryDirectory() as root:
        unzip = synth.write_mb_raw(root, n2014=0, half_size=(h, w), D=2 * args.ndisp)
        synth.write_mb_eval_gt(unzip)
        net = os.path.join(root, "fast.t7")
        t7.save_net(net, oft.make_weights(np.random.default_rng(0), l1=5, fm=64))
        scenes = me.training_scenes(root)
        rng = np.random.default_rng(1)
        reps = 50
        for res in ("H", "F"):
            ts = []
            for s in scenes:
                gt_path, mask_path = me.gt_files(root, s, res)
                gt = torch.from_numpy(me._read_topdown(gt_path)).to(dev)
                mask = torch.from_numpy(preprocess._read_grey(mask_path)).to(dev)
                disp = torch.from_numpy(rng.uniform(0, args.ndisp, (h, w)).astype(np.float32)).to(dev)
                scratch = torch.empty(me.scratch_bytes(), dtype=torch.uint8, device=dev)
                me.evaldisp(disp, gt, mask, args.ndisp, scratch)              # warm-up
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(reps):
                    me.evaldisp(disp, gt, mask, args.ndisp, scratch)
                b.record()
                b.synchronize()
                ts.append(a.elapsed_time(b) / reps)
            Hg, Wg = gt.shape
            print("evaldisp at %s, map %dx%d, ground truth %dx%d: %.3f ms per scene (median over %d scenes)"
                  % (res, h, w, Hg, Wg, statistics.median(ts), len(ts)), flush=True)

        run = lambda: me.evaluate_training("fast", net, data_root=root, res="F", verbose=False)
        run()                                                                   # warm-up
        per_scene = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run()
            torch.cuda.synchronize()
            per_scene.append((time.perf_counter() - t0) / len(scenes) * 1e3)
        print("mb_eval predict fast, res F, %d scenes of %dx%d, ndisp %d: %s ms per scene"
              % (len(scenes), h, w, args.ndisp, " / ".join("%.1f" % t for t in per_scene)), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
