"""Generate tests/golden/preprocess/*.npz: what THE REFERENCE'S OWN label cleaning kernels and make_dataset2 compute.

Needs a GPU and oracle/_ref/libadcensus_ref.so (`make -C oracle ref`).  Run once; the fixtures are committed:

    python oracle/make_preprocess_golden.py [OUT_DIR]

Each case holds a stack y (n, 1, H, W) of maps in readPNG16's domain (multiples of 1/256 in [0, 256)), left images x0 of the
same shape (with some entries exactly 255, so that remove_white fires), per-image te flags, and the reference's outputs:
remove_nonvisible(y), remove_occluded(y), remove_occluded(remove_nonvisible(y)), remove_white(x0, y), and the sample lists of
preprocess_kitti.lua:93-116 (nonvisible -> occluded -> white -> make_dataset2 per map) as nnz_tr / nnz_te.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def png16(rng, shape, dmax=64.0, p_zero=0.1):
    """seeded maps in readPNG16's domain: piecewise-constant runs of random disparities (occlusions at every jump to a
    larger value) with random 1/256 fractions and zero pixels"""
    v = np.floor(rng.uniform(0, dmax * 256, size=shape)) / 256
    runs = np.repeat(rng.uniform(0, dmax, size=shape[:-1] + (shape[-1] // 7 + 1,)), 7, axis=-1)[..., :shape[-1]]
    v = np.where(rng.random(shape) < 0.5, np.floor(runs * 256) / 256, v)
    v[rng.random(shape) < p_zero] = 0
    return v.astype(np.float32)


def tie_rows(W):
    """hand-made rows: exact ties a_j == a_x (must NOT occlude), strict occluders one 1/256 beyond a tie, a row with no
    valid pixel, a row where every entry is at or past the left border, fractions straddling 0.5"""
    x = np.arange(W, dtype=np.float32)
    rows = []
    r = np.zeros(W, np.float32)
    r[10], r[14] = 3.0, 7.0                 # a_10 = 7, a_14 = 7: tie
    r[20], r[23] = 2.5, 5.5                 # a_20 = 17.5, a_23 = 17.5: tie
    r[30], r[33] = 2.5, 5.5 + 1 / 256       # a_33 = a_30 - 1/256: occludes
    r[40], r[41], r[42] = 0.5, 0.5 + 1 / 256, 0.25
    rows.append(r)
    rows.append(np.zeros(W, np.float32))                            # no valid pixel
    rows.append(x + np.float32(1 / 256))                            # every entry >= x: all nonvisible
    r = np.minimum(np.float32(255.99609375), np.float32(0.75) * x)  # a slope: a_j increases, nothing occluded
    rows.append(r)
    r = np.maximum(np.float32(0), np.float32(60) - np.float32(0.5) * x)  # decreasing disparity: many ties and occlusions
    rows.append(np.floor(r * 256) / 256)
    return np.stack(rows).astype(np.float32)


def cases():
    rng = np.random.default_rng(2024)
    out = {}
    W = 77
    y = tie_rows(W)[None, None]
    out["ties_w77"] = (y, np.zeros_like(y), np.array([0], np.int32))
    y = png16(rng, (5, 1, 6, 131), dmax=40)
    x0 = rng.standard_normal(y.shape).astype(np.float32)
    x0[rng.random(y.shape) < 0.05] = 255
    out["random_5x6x131"] = (y, x0, np.array([0, 1, 0, 0, 1], np.int32))
    y = png16(rng, (2, 1, 3, 1242), dmax=200)
    y[0, 0, 0] = np.concatenate([tie_rows(64).reshape(-1), np.zeros(1242 - 5 * 64, np.float32)])[:1242]
    x0 = rng.standard_normal(y.shape).astype(np.float32)
    x0[0, 0, 1, ::17] = 255
    out["wide_2x3x1242"] = (y, x0, np.array([1, 0], np.int32))
    return out


def reference_outputs(shim, y, x0, is_te):
    """the reference's kernels through the shim on cuda:0"""
    import torch

    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    res = {}

    def run(name, *ops):
        t = cu(y)
        for op in ops:
            shim.call(op, *((cu(x0), t) if op == "remove_white" else (t,)))
        torch.cuda.synchronize()
        res[name] = t.cpu().numpy()

    run("nonvisible", "remove_nonvisible")
    run("occluded", "remove_occluded")
    run("nonvisible_occluded", "remove_nonvisible", "remove_occluded")
    run("white", "remove_white")
    lists = {0: [], 1: []}
    n, _, H, W = y.shape
    for i in range(n):                                      # preprocess_kitti.lua:94-111
        t = cu(y[i:i + 1])
        shim.call("remove_nonvisible", t)
        shim.call("remove_occluded", t)
        shim.call("remove_white", cu(x0[i:i + 1]), t)
        d = t.cpu().contiguous()
        nnz = torch.zeros((H * W, 4), dtype=torch.float32)
        cnt = int(shim.call("make_dataset2", d, nnz, i + 1, 0)[0])
        lists[int(is_te[i])].append(nnz[:cnt].numpy().copy())
    for k, name in ((0, "nnz_tr"), (1, "nnz_te")):
        res[name] = np.concatenate(lists[k]) if lists[k] else np.zeros((0, 4), np.float32)
    return res


def main(out_dir):
    from oracle import refdriver

    os.makedirs(out_dir, exist_ok=True)
    shim = refdriver.ShimLibrary(refdriver.REF_LIB)
    for name, (y, x0, is_te) in cases().items():
        res = reference_outputs(shim, y, x0, is_te)
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), y=y, x0=x0, is_te=is_te, **res)
        print("wrote", name, {k: v.shape for k, v in res.items()}, flush=True)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "preprocess"))
