"""CPU restatement of preprocess_kitti.lua's label cleaning and sample lists -- TEST INFRASTRUCTURE.

The three cleaning kernels (adcensus.cu:1723-1796) and make_dataset2 (:1900-1929) written as the reference's own loops, NOT
as the suffix minimum of csrc/preprocess.cu: remove_occluded tests ``i - y[x+i] < -y[x]`` in fp32 for every i, deciding each
pixel on the values before the call (what a loop over x in ascending order, or the reference's racing threads, sees: a pixel
only reads pixels to its right).  The loop over x runs vectorised, one numpy operation per offset i; offsets past
max(y) - min(y) + 1 cannot satisfy the test and are skipped.  ``preprocess_kitti`` restates the whole script for small
frames on top of them.
"""
import os

import numpy as np


def remove_nonvisible(y):
    """adcensus.cu:1723-1734 on a copy: y[id] >= id % W -> 0"""
    y = np.array(y, dtype=np.float32)
    x = np.arange(y.shape[-1], dtype=np.float32)
    y[y >= x] = 0
    return y


def remove_occluded(y):
    """adcensus.cu:1747-1760 on a copy: y[x] -> 0 if some i >= 1, x + i < W, has i - y[x+i] < -y[x] (fp32)"""
    y0 = np.array(y, dtype=np.float32)
    W = y0.shape[-1]
    occ = np.zeros(y0.shape, bool)
    if y0.size == 0:
        return y0
    span = float(y0.max()) - float(y0.min())
    for i in range(1, min(W - 1, int(np.ceil(span)) + 2) + 1):
        occ[..., :W - i] |= (np.float32(i) - y0[..., i:]) < -y0[..., :W - i]
    out = y0.copy()
    out[occ] = 0
    return out


def remove_white(x, y):
    """adcensus.cu:1773-1783 on a copy: y -> 0 where x == 255"""
    y = np.array(y, dtype=np.float32)
    y[np.asarray(x, dtype=np.float32).reshape(y.shape) == 255] = 0
    return y


def make_dataset2(disp, img):
    """adcensus.cu:1900-1929 for one (H, W) map: the (img, i, j, disp) float32 rows of the entries > 0.5, rows then columns
    (np.nonzero walks a C-ordered array in exactly that order)"""
    d = np.asarray(disp, dtype=np.float32).reshape(disp.shape[-2], disp.shape[-1])
    i, j = np.nonzero(d > np.float32(0.5))
    return np.stack([np.full(i.shape, img, np.float32), i.astype(np.float32), j.astype(np.float32), d[i, j]], axis=1)


def clean(disp, x0):
    """preprocess_kitti.lua:96-99 for one map: nonvisible, occluded, white"""
    return remove_white(x0, remove_occluded(remove_nonvisible(disp)))


def nnz_lists(dispnoc, x0, te):
    """preprocess_kitti.lua:93-116: (nnz_tr, nnz_te) from the (n_tr, 1, H, W) maps, their left images and the 1-based te"""
    te = set(int(v) for v in np.asarray(te).reshape(-1))
    out = {True: [np.zeros((0, 4), np.float32)], False: [np.zeros((0, 4), np.float32)]}
    for i in range(1, len(dispnoc) + 1):
        out[i in te].append(make_dataset2(clean(dispnoc[i - 1], x0[i - 1]), i))
    return np.concatenate(out[False]), np.concatenate(out[True])


def preprocess_kitti(data_root, dataset, height=350, width=1242):
    """The whole of preprocess_kitti.lua for one dataset, on the CPU: dict name -> array of the eight outputs.  Image
    decoding, rgb2y and standardisation are frontend's; the split is mccnn_b200.preprocess.split (pinned on its own)."""
    from mccnn_b200 import dataio, frontend
    from mccnn_b200 import preprocess as pp

    lay = pp.LAYOUT[dataset]
    unzip = os.path.join(data_root, lay["path"], "unzip")
    count = lambda sub: len([f for f in os.listdir(os.path.join(unzip, sub, lay["image_0"])) if f.endswith("_10.png")])
    n_tr, n_te = count("training"), count("testing")
    examples = [("training", i) for i in range(1, n_tr + 1)] + [("testing", i) for i in range(1, n_te + 1)]
    x0 = np.zeros((n_tr + n_te, 1, height, width), np.float32)
    x1 = np.zeros_like(x0)
    dispnoc = np.zeros((n_tr, 1, height, width), np.float32)
    metadata = np.zeros((n_tr + n_te, 3), np.int32)
    for i, (sub, cnt) in enumerate(examples, 1):
        path = lambda d: os.path.join(unzip, sub, d, "%06d_10.png" % (cnt - 1))
        img_0 = frontend.load_image(path(lay["image_0"]))
        img_1 = frontend.load_image(path(lay["image_1"]))
        if dataset == "kitti2015":
            img_0, img_1 = frontend.rgb2y(img_0), frontend.rgb2y(img_1)
        img_height, img_width = img_0.shape[1], img_0.shape[2]
        img_0 = img_0[:, img_height - height:]
        img_1 = img_1[:, img_height - height:]
        x0[i - 1, :, :, :img_width] = frontend.standardise(img_0)
        x1[i - 1, :, :, :img_width] = frontend.standardise(img_1)
        if sub == "training":
            d = dataio.read_png16(path(lay["disp_noc"]))
            dispnoc[i - 1, 0, :, :img_width] = d[img_height - height:]
        metadata[i - 1] = (img_height, img_width, cnt - 1)
    tr, te = pp.split(n_tr)
    nnz_tr, nnz_te = nnz_lists(dispnoc, x0, te)
    return dict(x0=x0, x1=x1, dispnoc=dispnoc, metadata=metadata, tr=tr, te=te, nnz_tr=nnz_tr, nnz_te=nnz_te)
