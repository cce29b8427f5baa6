"""preprocess_kitti.lua for KITTI 2012 and 2015: raw ``unzip/`` tree in, main.lua's data layout out.

    preprocess_kitti(".", "kitti")        # data.kitti/unzip/... -> data.kitti/{x0,x1,dispnoc,metadata,tr,te,nnz_tr,nnz_te}.bin

Per image (preprocess_kitti.lua:41-86): the two views are loaded as bytes (grey for 2012; RGB through ``image.rgb2y`` for
2015, :frontend.rgb2y), the bottom `height` rows are kept, each view is standardised (:frontend.standardise) and stored
zero-padded to `width` columns; a training image's ``disp_noc`` map (:dataio.read_png16) is cropped and padded the same way,
and ``metadata`` holds (uncropped height, width, index in its directory).  Then (:88-116) the Torch7 split of the training
images -- ``torch.manualSeed(42); torch.randperm(n_tr)``, the first 40 to ``te``, the rest to ``tr`` -- and the per-pixel
training-sample lists ``nnz_tr`` / ``nnz_te``: each map cleaned by remove_nonvisible, remove_occluded and remove_white, then
every entry > 0.5 as a float row (image, row, column, disparity), image 1-based, row and column 0-based in the padded frame.
That last stage runs on the GPU (csrc/preprocess.cu, one count pass and one fill pass); there is no CPU fallback.

The split restates ``THTensor_(randperm)``: swap element i with element i + (THRandom_random() % (n - i)) for i = 0 .. n-2,
THRandom_random being MT19937's tempered 32-bit output after ``init_genrand(42)``, then add 1.  Torch7 is not available to
compare against, so this is **parity unpinned** against Torch itself; the generator is pinned against C++'s
``std::mt19937(42)`` in the tests.

Deliberate deviations from preprocess_kitti.lua:

* n_tr and n_te are the numbers of ``%06d_10.png`` files in the left-image directories of ``training/`` and ``testing/``
  (194 / 195 for 2012, 200 / 200 for 2015 on the published archives) instead of constants;
* a set with n_tr <= 40 (no training rows left after the split) is refused, as are images shorter than the crop or wider
  than `width`, views of different sizes, and missing files -- all before any output is written;
* existing outputs are refused (the script runs ``rm -f``), as ``evaluate.Evaluator.submit`` refuses a non-empty directory;
* the sample lists are sized by a count pass instead of preallocating 23e6 rows.
"""
import os
import re

import numpy as np

from . import dataio, frontend

LAYOUT = {
    "kitti": dict(year=2012, path="data.kitti", image_0="image_0", image_1="image_1", disp_noc="disp_noc", nchannel=1),
    "kitti2015": dict(year=2015, path="data.kitti2015", image_0="image_2", image_1="image_3", disp_noc="disp_noc_0",
                      nchannel=3),
}
OUTPUTS = ("x0.bin", "x1.bin", "dispnoc.bin", "metadata.bin", "tr.bin", "te.bin", "nnz_tr.bin", "nnz_te.bin")
N_VAL = 40            # preprocess_kitti.lua:90
SEED = 42             # :11
HEIGHT, WIDTH = 350, 1242
_PNG = re.compile(r"^(\d{6})_10\.png$")


class MT19937:
    """The Mersenne Twister of Torch7's THRandom.c (Matsumoto and Nishimura's mt19937ar): ``init_genrand(seed)``, then
    ``random()`` returns the tempered 32-bit outputs, the same stream as C++'s ``std::mt19937(seed)``."""

    N, M = 624, 397

    def __init__(self, seed):
        mt = [seed & 0xFFFFFFFF]
        for j in range(1, self.N):
            mt.append((1812433253 * (mt[-1] ^ (mt[-1] >> 30)) + j) & 0xFFFFFFFF)
        self.mt, self.i = mt, self.N

    def _twist(self):
        mt, N, M = self.mt, self.N, self.M
        for k in range(N):
            y = (mt[k] & 0x80000000) | (mt[(k + 1) % N] & 0x7FFFFFFF)
            mt[k] = mt[(k + M) % N] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
        self.i = 0

    def random(self):
        if self.i >= self.N:
            self._twist()
        y = self.mt[self.i]
        self.i += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        return y & 0xFFFFFFFF


def randperm(n, seed=SEED):
    """``torch.manualSeed(seed); torch.randperm(n)`` as int64, 1-based (THTensor_(randperm) + 1)"""
    g = MT19937(seed)
    p = list(range(n))
    for i in range(n - 1):
        z = g.random() % (n - i)
        p[i], p[i + z] = p[i + z], p[i]
    return np.asarray(p, dtype=np.int64) + 1


def split(n_tr, seed=SEED):
    """preprocess_kitti.lua:88-91: (tr, te), 1-based int64; te = the first 40 entries of the permutation"""
    if n_tr <= N_VAL:
        raise ValueError("%d training images: the split keeps %d for validation and needs at least one more" % (n_tr, N_VAL))
    perm = randperm(n_tr, seed)
    return perm[N_VAL:].copy(), perm[:N_VAL].copy()


def count_images(d):
    """the number of ``%06d_10.png`` files in directory `d`; they must be 000000 .. n-1 (the script reads them in turn)"""
    if not os.path.isdir(d):
        raise FileNotFoundError("missing image directory %s" % d)
    ids = sorted(int(m.group(1)) for m in map(_PNG.match, os.listdir(d)) if m)
    if ids != list(range(len(ids))):
        missing = sorted(set(range(len(ids))) - set(ids))[0]
        raise FileNotFoundError("%s: %06d_10.png is missing (the files must be numbered from 000000 on)" % (d, missing))
    return len(ids)


def input_files(data_root, dataset):
    """preprocess_kitti.lua:37-58: [(dir, cnt, left, right, disp_noc or None)] for cnt = 1 .. n, training first; every
    file must exist"""
    lay = LAYOUT[dataset]
    unzip = os.path.join(data_root, lay["path"], "unzip")
    out = []
    for sub in ("training", "testing"):
        n = count_images(os.path.join(unzip, sub, lay["image_0"]))
        for cnt in range(1, n + 1):
            name = "%06d_10.png" % (cnt - 1)
            f = (os.path.join(unzip, sub, lay["image_0"], name), os.path.join(unzip, sub, lay["image_1"], name),
                 os.path.join(unzip, sub, lay["disp_noc"], name) if sub == "training" else None)
            for p in f:
                if p is not None and not os.path.exists(p):
                    raise FileNotFoundError("missing input file %s" % p)
            out.append((sub, cnt) + f)
    return out


def _load_view(path, dataset, nchannel):
    img = frontend.load_image(path)                                            # image.loadPNG(.., nchannel, 'byte'):float()
    if img.shape[0] != nchannel:
        raise ValueError("%s: %d channel(s), %s expects %d" % (path, img.shape[0], dataset, nchannel))
    return frontend.rgb2y(img) if nchannel == 3 else img                       # :53-56


def load_host(data_root, dataset, height=HEIGHT, width=WIDTH, log=None):
    """The host half of the script (preprocess_kitti.lua:33-86): dict(x0, x1 (n, 1, height, width), dispnoc (n_tr, 1,
    height, width), metadata (n, 3) int32, n_tr, n_te).  dispnoc holds the maps as read (uncleaned)."""
    lay = LAYOUT[dataset]
    files = input_files(data_root, dataset)
    n = len(files)
    n_tr = sum(1 for f in files if f[0] == "training")
    if n_tr <= N_VAL:
        raise ValueError("%s: %d training images; the split keeps %d for validation and needs at least one more"
                         % (dataset, n_tr, N_VAL))
    x0 = np.zeros((n, 1, height, width), np.float32)
    x1 = np.zeros((n, 1, height, width), np.float32)
    dispnoc = np.zeros((n_tr, 1, height, width), np.float32)
    metadata = np.zeros((n, 3), np.int32)
    for i, (sub, cnt, f0, f1, fd) in enumerate(files):
        img_0, img_1 = _load_view(f0, dataset, lay["nchannel"]), _load_view(f1, dataset, lay["nchannel"])
        img_height, img_width = img_0.shape[1], img_0.shape[2]
        if img_1.shape != img_0.shape:
            raise ValueError("%s is %dx%d, %s is %dx%d" % (f0, img_height, img_width, f1, img_1.shape[1], img_1.shape[2]))
        if img_height < height:
            raise ValueError("%s: %d rows, fewer than the %d the crop keeps" % (f0, img_height, height))
        if img_width > width:
            raise ValueError("%s: %d columns, more than the %d of the padded frame" % (f0, img_width, width))
        if log:
            log(str(i + 1))                                                    # :63
        x0[i, :, :, :img_width] = frontend.standardise(img_0[:, img_height - height:])     # :59-60, 65-69
        x1[i, :, :, :img_width] = frontend.standardise(img_1[:, img_height - height:])
        if fd is not None:                                                     # :71-75
            d = dataio.read_png16(fd)
            if d.shape != (img_height, img_width):
                raise ValueError("%s is %dx%d, the image is %dx%d" % (fd, d.shape[0], d.shape[1], img_height, img_width))
            dispnoc[i, 0, :, :img_width] = d[img_height - height:]
        metadata[i] = (img_height, img_width, cnt - 1)                         # :77-79
    return dict(x0=x0, x1=x1, dispnoc=dispnoc, metadata=metadata, n_tr=n_tr, n_te=n - n_tr)


def kitti_nnz(disp, x0, is_te):
    """preprocess_kitti.lua:93-116 on the GPU: disp (n, 1, H, W) and x0 (>= n, 1, H, W) CUDA float32 on one device, is_te
    (n) booleans -> (nnz_tr, nnz_te), (rows, 4) CUDA float32 tensors.  disp is not modified."""
    import ctypes

    import torch

    from .adcensus import AdcensusError, _check, _stream, _t, lib

    name = "kitti_nnz"
    if disp.dim() != 4 or x0.dim() != 4 or x0.shape[1:] != disp.shape[1:] or x0.size(0) < disp.size(0):
        raise AdcensusError("%s: disp (n,1,H,W) and x0 (>= n,1,H,W) expected, got %s and %s"
                            % (name, tuple(disp.shape), tuple(x0.shape)))
    if x0.device != disp.device:
        raise AdcensusError("%s: x0 on %s, disp on %s" % (name, x0.device, disp.device))
    n, _, H, W = disp.shape
    if len(is_te) != n:
        raise AdcensusError("%s: %d te flags for %d maps" % (name, len(is_te), n))
    pd, px = _t(disp, 1, name), _t(x0, 2, name)
    dev = disp.device
    with torch.cuda.device(dev):
        flags = torch.as_tensor(np.asarray(is_te, dtype=np.int32)).to(dev)
        counts = torch.zeros(2, dtype=torch.int64, device=dev)
        l, s = lib(), _stream(disp)
        pf = ctypes.c_void_p(flags.data_ptr())
        _check(l.mccnn_kitti_nnz_count(pd, px, pf, n, H, W, ctypes.c_void_p(counts.data_ptr()), s), name)
        n_tr_rows, n_te_rows = (int(v) for v in counts.cpu())
        nnz_tr = torch.empty((n_tr_rows, 4), dtype=torch.float32, device=dev)
        nnz_te = torch.empty((n_te_rows, 4), dtype=torch.float32, device=dev)
        ptr = lambda t: ctypes.c_void_p(t.data_ptr() if t.numel() else None)
        _check(l.mccnn_kitti_nnz_fill(pd, px, pf, n, H, W, ptr(nnz_tr), ctypes.c_longlong(n_tr_rows), ptr(nnz_te),
                                      ctypes.c_longlong(n_te_rows), s), name)
    return nnz_tr, nnz_te


def output_dir(data_root, dataset):
    return os.path.join(data_root, LAYOUT[dataset]["path"])


def check_outputs_absent(d):
    """refuse to overwrite: the first of the eight outputs (or its .dim / .type) that exists in `d` is named"""
    for f in OUTPUTS:
        for p in (f, f + ".dim", f + ".type"):
            if os.path.exists(os.path.join(d, p)):
                raise FileExistsError("%s already exists; remove the old outputs first (nothing was written)"
                                      % os.path.join(d, p))


def preprocess_kitti(data_root, dataset, device=0, height=HEIGHT, width=WIDTH, log=None):
    """preprocess_kitti.lua for one dataset ('kitti' or 'kitti2015'): reads ``data_root/<path>/unzip``, writes the eight
    outputs to ``data_root/<path>`` (path = data.kitti / data.kitti2015) and returns that directory.  The sample lists
    are computed on CUDA device `device` (0-based).  `log` receives the lines the script prints.  `height` and `width`
    exist so that tests can use small frames."""
    import torch

    if dataset not in LAYOUT:
        raise ValueError("dataset must be 'kitti' or 'kitti2015', got %r" % (dataset,))
    d = output_dir(data_root, dataset)
    check_outputs_absent(d)
    if log:
        log("dataset %d" % LAYOUT[dataset]["year"])                           # :9
    host = load_host(data_root, dataset, height, width, log)
    tr, te = split(host["n_tr"])                                               # :88-91
    is_te = np.zeros(host["n_tr"], bool)
    is_te[te - 1] = True
    dev = torch.device("cuda", device)
    disp = torch.from_numpy(host["dispnoc"]).to(dev)
    x0 = torch.from_numpy(host["x0"][:host["n_tr"]]).to(dev)
    nnz_tr, nnz_te = kitti_nnz(disp, x0, is_te)                               # :93-116
    nnz_tr, nnz_te = nnz_tr.cpu().numpy(), nnz_te.cpu().numpy()
    del disp, x0
    write_outputs(d, dict(x0=host["x0"], x1=host["x1"], dispnoc=host["dispnoc"], metadata=host["metadata"], tr=tr, te=te,
                          nnz_tr=nnz_tr, nnz_te=nnz_te))
    return d


def write_outputs(d, out):
    """preprocess_kitti.lua:136-144: the eight arrays of `out` (keyed by name without .bin) through dataio.tofile, in the
    script's order; refuses if any output exists already"""
    check_outputs_absent(d)
    os.makedirs(d, exist_ok=True)
    for f in OUTPUTS:
        dataio.tofile(os.path.join(d, f), out[f[:-len(".bin")]])
