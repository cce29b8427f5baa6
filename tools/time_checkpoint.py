"""Measure training checkpoints (-checkpoint_steps / -stop_after / -resume) on a synthetic KITTI-sized set.

    python tools/time_checkpoint.py [-steps 2048] [-rounds 3] [-gpu 1] [-json out.json]

Reported, with the card's name and power limit:

* save:     the time and bytes of one checkpoint (stream drained, parameters, momenta and half an epoch's losses read
            back, written, fsynced and renamed) at the kitti slow and mb slow presets, median of five;
* overhead: steps/s of one epoch of -steps steps at the kitti fast preset (the shortest step, so the largest relative
            cost) without checkpoints and with -checkpoint_steps 256, alternated -rounds times in one process;
* resume:   the time to resume at 2^20 nnz rows: Stream -> randperm -> init_net replayed, the fingerprint (SHA-256 of the
            rows), the file loaded and checked, and the state uploaded, at the kitti slow preset.
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

ROWS = 1 << 20


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("-steps", type=int, default=2048)
    ap.add_argument("-rounds", type=int, default=3)
    ap.add_argument("-gpu", type=int, default=1)
    ap.add_argument("-json", default="")
    args = ap.parse_args(argv)

    import torch

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import train
    from time_train import card

    dev = torch.device("cuda", args.gpu - 1)
    rng = np.random.default_rng(0)
    n_img, H, W = 8, 350, 1242
    X0, X1 = (torch.from_numpy(rng.standard_normal((n_img, 1, H, W)).astype(np.float32)).to(dev) for _ in range(2))

    def rows(n):
        return np.stack([rng.integers(1, n_img + 1, n), rng.integers(0, H, n), rng.integers(0, W, n),
                         rng.uniform(0, 200, n)], 1).astype(np.float32)

    nnz = rows(ROWS)
    out = {"card": card(), "rows": ROWS}
    tmp = tempfile.mkdtemp(prefix="mccnn_ckpt_")
    path = os.path.join(tmp, "net.state.npz")
    fp = lambda o: train.fingerprint("kitti", "train_tr", o, 42, "kitti", nnz, [("x0.bin", X0.shape)])  # noqa: E731

    # one checkpoint at the slow presets
    out["save"] = {}
    for name, o in (("kitti_slow", train.options("kitti", "slow")), ("mb_slow", train.options("mb", "slow"))):
        tr = train.Trainer(o, X0, X1, device=dev.index, loss_cap=train.steps_per_epoch(ROWS, o["bs"]))
        s = train.Stream(1)
        tr.set_layers(*train.init_net(s, o))
        tr.run_chunk(train.make_warps(train.draw_params(s, o, 64 * 16), rows(64 * 16), tr.ws), o["lr"])
        half = train.steps_per_epoch(ROWS, o["bs"]) // 2
        ck = train.Checkpoints(path, fp(o), steps=256)
        times = []
        for _ in range(5):
            torch.cuda.synchronize(dev)
            t = time.perf_counter()
            ck.save(tr, s, 1, half, o["lr"], 1.0, np.zeros(half, np.float32))
            times.append(time.perf_counter() - t)
        out["save"][name] = dict(ms=1e3 * float(np.median(times)), ms_all=[1e3 * v for v in times],
                                 bytes=os.path.getsize(path), params=tr.size(train.TRAIN_PARAMS))
        # resume at 2^20 rows: replay, fingerprint, load and check, upload
        torch.cuda.synchronize(dev)
        t = time.perf_counter()
        s2 = train.Stream(42)
        train.randperm(s2, ROWS)
        train.init_net(s2, o)
        st = train.load_checkpoint(path, fp(o))
        s2.restore(st["mt_key"], st["mt_pos"], st["carry"])
        tr.load_state(st["params"], st["momenta"])
        out["save"][name]["resume_ms"] = 1e3 * (time.perf_counter() - t)
        tr.close()

    # steps/s with and without -checkpoint_steps 256, alternated
    o = train.options("kitti", "fast")
    h = o["bs"] // 2
    sub = nnz[:args.steps * h + h]
    assert train.steps_per_epoch(len(sub), o["bs"]) == args.steps
    rates = {"none": [], "256": []}
    for r in range(args.rounds + 1):                                  # round 0 warms up
        for mode in ("none", "256"):
            tr = train.Trainer(o, X0, X1, device=dev.index, loss_cap=args.steps)
            s = train.Stream(42)
            perm = train.randperm(s, len(sub))
            tr.set_layers(*train.init_net(s, o))
            build = lambda n, rw: train.make_warps(train.draw_params(s, o, n * h), rw, tr.ws)  # noqa: E731
            ck = train.Checkpoints(path, fp(o), steps=256) if mode == "256" else None
            torch.cuda.synchronize(dev)
            t = time.perf_counter()
            train.fit(tr, sub, perm, build, o, s, epochs=1, log=lambda line: None, ckpt=ck)
            torch.cuda.synchronize(dev)
            dt = time.perf_counter() - t
            if r:
                rates[mode].append(args.steps / dt)
            tr.close()
    out["overhead"] = dict(steps=args.steps, preset="kitti fast", steps_per_s=rates,
                           median=dict((k, float(np.median(v))) for k, v in rates.items()))
    os.remove(path)
    os.rmdir(tmp)
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
