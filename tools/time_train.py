"""Measure the training step of the fast or slow architecture (csrc/train.cu) on a synthetic full-size KITTI 2012 set.

    python tools/time_train.py [-arch fast|slow] [-dataset kitti|mb] [-steps 2000] [-gpu 1] [-json out.json]

With -dataset mb the presets are main.lua's mb ones (l1 5; fm 64 'fast', 112 'slow') and the set is a synthetic ragged
Middlebury set on the device (see mb_shapes: 50 images, one pair per image, light and exposure, 1,048,576 nnz rows); the
host build is the mb draw builder (MbTrainSet.warps), and the pair count and the bytes of the planes are reported.

The set is 389 views of 350 x 1242 per side on the device and 1,048,576 nnz rows, at main.lua's kitti presets (l1 4, fm 64,
bs 128).  Reported, each after a warm-up:

* device:   the captured step alone, warp parameters already on the device (steps/s, samples/s = steps/s * bs / 2);
* driver:   as train.train runs it: the host draws and builds each chunk of parameters while the GPU runs the previous one;
* baseline: the same step written with torch autograd / cuDNN in fp32 (conv2d, the Normalize2 / StereoJoin1 / Margin2 formulas,
  the momentum update as main.lua:871-874) on patches from the same sampler, TF32 off.

With -arch slow (l1 4, fm 112, l2 4, nh2 384, bs 128) the baseline is net_tr + BCECriterion2 + the update in autograd, and
the device and baseline runs alternate three times in the one call (each round is reported, then the medians).
The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def mb_shapes(rng):
    """a synthetic Middlebury training set of realistic size: 20 scenes of about 1000 x 1450 with 3 to 6 lights of 3
    exposures (the 2014 half-size scenes) and 30 of about 550 x 690 with 3 x 3 (2006 / 2005 HalfSize and smaller)
    -> ([(H, W)] per image, {image: (lights, exposures)})"""
    sizes, counts = [], {}
    for k in range(50):
        big = k < 20
        sizes.append((int(rng.integers(950, 1050)), int(rng.integers(1350, 1500))) if big else
                     (int(rng.integers(500, 600)), int(rng.integers(640, 740))))
        counts[k + 1] = (int(rng.integers(3, 7)) if big else 3, 3)
    return sizes, counts


def baseline_step(x, params, vel, o, lr):
    import torch

    F = torch.nn.functional
    h = x
    for i in range(o["l1"]):
        h = F.conv2d(h, params[2 * i], params[2 * i + 1])
        if i < o["l1"] - 1:
            h = torch.relu(h)
    h = h / ((h * h).sum(1, keepdim=True) + 1e-5).sqrt()
    s = (h[0::2] * h[1::2]).sum(1).reshape(-1)
    f = torch.clamp(s[1::2] - s[0::2] + o["m"], min=0)
    loss = f.mean() if o["pow"] == 1 else (0.5 * f * f).mean()
    grads = torch.autograd.grad(loss, params)
    with torch.no_grad():
        for p, v, g in zip(params, vel, grads):
            v.mul_(o["mom"]).add_(g, alpha=-lr)
            p.add_(v)
    return loss


def baseline_step_slow(x, params, vel, o, lr):
    import torch

    F = torch.nn.functional
    h = x
    for i in range(o["l1"]):
        h = torch.relu(F.conv2d(h, params[2 * i], params[2 * i + 1]))
    h = h.reshape(o["bs"], -1)
    k = 2 * o["l1"]
    for j in range(o["l2"] + 1):
        h = F.linear(h, params[k + 2 * j], params[k + 2 * j + 1])
        if j < o["l2"]:
            h = torch.relu(h)
    y = torch.sigmoid(h).reshape(-1)
    t = torch.arange(o["bs"], device=x.device).remainder(2).float()
    loss = -((torch.log(y + 1e-12) * t + torch.log(1 - y + 1e-12) * (1 - t)) / o["bs"]).sum()
    grads = torch.autograd.grad(loss, params)
    with torch.no_grad():
        for p, v, g in zip(params, vel, grads):
            v.mul_(o["mom"]).add_(g, alpha=-lr)
            p.add_(v)
    return loss


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("-steps", type=int, default=2000)
    ap.add_argument("-gpu", type=int, default=1)
    ap.add_argument("-json", default="")
    ap.add_argument("-arch", choices=("fast", "slow"), default="fast")
    ap.add_argument("-dataset", choices=("kitti", "mb"), default="kitti")
    args = ap.parse_args(argv)
    import torch

    import mccnn_b200  # noqa: F401
    from mccnn_b200 import train

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", args.gpu - 1)
    torch.cuda.set_device(dev)
    o = train.options(args.dataset, args.arch)
    rows = 1 << 20
    g = torch.Generator(device=dev).manual_seed(0)
    rng = np.random.default_rng(0)
    extra = {}
    if args.dataset == "mb":
        sizes, counts = mb_shapes(rng)
        img = rng.integers(1, len(sizes) + 1, rows)
        hw = np.array(sizes)[img - 1]
        nnz = np.stack([img, rng.integers(0, hw[:, 0]), rng.integers(0, hw[:, 1]), rng.uniform(1, 140, rows)],
                       1).astype(np.float32)
        mb = train.MbTrainSet.from_counts(nnz, counts)
        planes = []
        for i, (hh, ww) in enumerate(sizes, 1):                   # MbTrainSet.upload's order: image, light, exposure
            for _ in range(counts[i][0]):
                grp = torch.randn((counts[i][1], 2, hh, ww), device=dev, generator=g)
                planes += [(grp[e, 0], grp[e, 1]) for e in range(counts[i][1])]
        extra = dict(pairs=len(planes), images=len(sizes),
                     plane_bytes=sum(2 * a.numel() * 4 for a, _ in planes))
        X0 = X1 = None
    else:
        n_img, H, W = 389, 350, 1242
        X0 = torch.randn((n_img, 1, H, W), device=dev, generator=g)
        X1 = torch.randn((n_img, 1, H, W), device=dev, generator=g)
        nnz = np.stack([rng.integers(1, n_img + 1, rows), rng.integers(0, H, rows), rng.integers(0, W, rows),
                        rng.uniform(1, 200, rows)], 1).astype(np.float32)
        planes = None
    s = train.Stream(42)
    perm = train.randperm(s, rows)
    chunk = train.CHUNK
    tr = train.Trainer(o, X0, X1, chunk=chunk, loss_cap=args.steps + 4 * chunk, device=dev.index, planes=planes)
    tr.set_layers(*train.init_net(s, o))
    h = o["bs"] // 2
    res = dict(card=card(), launches_per_step=tr.launches_per_step, steps=args.steps)
    if args.arch == "slow":
        res["arch"] = "slow"
    if args.dataset == "mb":
        res.update(dataset="mb", **extra)

    def warps_for(s0, n):
        r = nnz[perm[(s0 * h) % (rows - n * h):][:n * h] - 1]
        if args.dataset == "mb":
            return mb.warps(s, o, r, tr.ws)
        return train.make_warps(train.draw_params(s, o, n * h), r, tr.ws)

    # device: parameters already on the device
    dw = torch.from_numpy(warps_for(0, chunk).view(np.uint8)).to(dev)
    tr.run(dw, o["lr"])
    torch.cuda.synchronize()

    def device_rate():
        n = 0
        t0 = time.perf_counter()
        while n < args.steps:
            tr.run(dw, o["lr"])
            n += chunk
        torch.cuda.synchronize()
        return n / (time.perf_counter() - t0)

    res["device_steps_per_s"] = device_rate()
    res["device_samples_per_s"] = res["device_steps_per_s"] * h

    # driver: host-built chunks through two pinned buffers, as train.train does
    rec = train.WARP_DTYPE.itemsize * tr.N
    pinned = [torch.empty(chunk * rec, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    ev = [None, None]
    n = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    k = 0
    while n < args.steps:
        w = warps_for(n, chunk)
        b = k % 2
        if ev[b] is not None:
            ev[b].synchronize()
        pinned[b].numpy()[:] = w.view(np.uint8)
        tr.run(pinned[b], o["lr"])
        ev[b] = torch.cuda.Event()
        ev[b].record(tr.stream)
        n += chunk
        k += 1
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    res["driver_steps_per_s"] = n / dt
    res["driver_samples_per_s"] = n * h / dt
    t = time.perf_counter()
    warps_for(0, chunk)
    res["host_build_s_per_step"] = (time.perf_counter() - t) / chunk

    # baseline: torch autograd / cuDNN on the sampler's patches
    tower, head = tr.net()
    params = []
    for w, b_ in tower + (head or []):
        params += [torch.from_numpy(w).to(dev).requires_grad_(), torch.from_numpy(b_).to(dev).requires_grad_()]
    vel = [torch.zeros_like(p) for p in params]
    x = tr.get(train.TRAIN_PATCHES).reshape(tr.N, 1, tr.ws, tr.ws)
    step = baseline_step_slow if args.arch == "slow" else baseline_step
    for _ in range(50):
        step(x, params, vel, o, o["lr"])
    torch.cuda.synchronize()
    nb = max(200, args.steps // 4)

    def baseline_rate():
        t0 = time.perf_counter()
        for _ in range(nb):
            step(x, params, vel, o, o["lr"])
        torch.cuda.synchronize()
        return nb / (time.perf_counter() - t0)

    res["baseline_steps_per_s"] = baseline_rate()
    res["baseline_samples_per_s"] = res["baseline_steps_per_s"] * h
    if args.arch == "slow":                                     # alternate the two in this one call
        rounds = [(res["device_steps_per_s"], res["baseline_steps_per_s"])]
        for _ in range(2):
            rounds.append((device_rate(), baseline_rate()))
        res["rounds_device_baseline_steps_per_s"] = rounds
        res["device_steps_per_s"] = float(np.median([r[0] for r in rounds]))
        res["baseline_steps_per_s"] = float(np.median([r[1] for r in rounds]))
        res["device_samples_per_s"] = res["device_steps_per_s"] * h
        res["baseline_samples_per_s"] = res["baseline_steps_per_s"] * h
        res["device_ms_per_step"] = 1e3 / res["device_steps_per_s"]
    tr.close()
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
