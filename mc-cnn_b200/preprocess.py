"""preprocess_kitti.lua and preprocess_mb.py: raw KITTI 2012 / 2015 and Middlebury trees in, main.lua's data layout out.

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

preprocess_mb.py for one (rect, color): the raw Middlebury tree in, ``data.mb.<rect>_<color>/`` out.

    preprocess_mb(".", "imperfect", "gray")     # data.mb/unzip/... -> data.mb.imperfect_gray/{x_<i>_<j>,dispnoc<i>,meta,...}

Images, in the script's order: the 2014 scenes (``scenes2014/datasets/*-imperfect``, sorted; views im0, im1, im1E, im1L and
the ambient lights, every view halved), the 2006 and 2005 ``HalfSize`` scenes that have ``disp1.png``, the 2003 conesH and
teddyH, the 2001 scenes with ground truth, and the MiddEval3 ``trainingH`` then ``testH`` pairs.  ``x_<i>_<j>.bin`` holds
image i's view group j (2014: (4, C, H, W), then one (n_exp, 2, C, H, W) group per light; 2006 / 2005: an empty group 1,
then (3, 2, C, H, W) per light; 2003 / 2001: an empty group 1, then (1, 2, C, H, W); MiddEval3: (2, C, H, W)).  Each
view is read_im: grey (cv2's BGR2GRAY) or the R, G, B planes, standardised as numpy does in float32.  ``dispnoc<i>.bin``
is the left map with every pixel the mask does not accept set to 0, ``nnz_tr`` / ``nnz_te`` list the accepted pixels as
(image, row, column, disparity) -- only 2014 scenes 1 to 10 (``te.bin``) feed ``nnz_te``.  ``meta.bin`` is (H, W, ndisp).

The per-pixel work runs on the GPU (csrc/preprocess_mb.cu); there is no CPU fallback.  Two of the script's steps call tools
this project does not ship, and are restated rather than pinned:

* ``convert X -resize 50%`` (ImageMagick) -> mccnn_mb_half_image, a Lanczos-3 filter renormalised at the border.  Cached
  ``<file>.H.png`` / ``.H.pfm`` next to the inputs are read when present, as the script does, so a tree the script has
  already processed gives the script's own views; they are never written;
* ``computemask`` (MiddEval3 SDK) -> mccnn_mb_mask (the rule is in include/adcensus_b200.h and DESIGN.md).

Deliberate deviations from preprocess_mb.py:

* existing outputs (``*.bin``, ``*.dim``, ``*.type``, ``*.txt`` in the output directory) are refused, where the script runs
  ``rm -f``; the output directory is created; no ``tmp/`` files are written;
* every input is found and its header checked before anything is written;
* exposures are counted only from names matching ``im[01]e<k>.png``; an exposure count missing from the script's table is
  refused (the script raises a KeyError);
* fewer than 10 2014 scenes are refused (``te.bin`` would name images outside the 2014 set); odd full-size 2014 views or
  maps are refused (the script's halving loop crashes on them);
* 16-bit images, and disparity or mask images that are not 8-bit grey, are refused; maps must have their images' size.
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
        _check(l.mccnn_kitti_nnz_count(pd, px, flags.data_ptr(), n, H, W, counts.data_ptr(), s), name)
        n_tr_rows, n_te_rows = (int(v) for v in counts.cpu())
        nnz_tr = torch.empty((n_tr_rows, 4), dtype=torch.float32, device=dev)
        nnz_te = torch.empty((n_te_rows, 4), dtype=torch.float32, device=dev)
        _check(l.mccnn_kitti_nnz_fill(pd, px, flags.data_ptr(), n, H, W, nnz_tr.data_ptr(), n_tr_rows, nnz_te.data_ptr(),
                                      n_te_rows, s), name)
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


# ---- Middlebury: preprocess_mb.py ---------------------------------------------------------------------------------------
MB_DATA = os.path.join("data.mb", "unzip", "vision.middlebury.edu", "stereo", "data")
MB_EVAL = os.path.join("data.mb", "unzip", "MiddEval3")
MB_EXPOSURES = {8: (1, 3, 5), 7: (1, 3, 5), 6: (0, 2, 4), 5: (0, 2, 4), 3: (0, 1, 2), 2: (0, 1)}   # preprocess_mb.py:148-155
MB_TE = tuple(range(1, 11))                                                                       # :121
_MB_EXP = re.compile(r"^im([01])e(\d)\.png$")
_MB_OUT = re.compile(r"\.(bin|dim|txt|type)$")


def mb_output_dir(data_root, rect, color):
    return os.path.join(data_root, "data.mb.%s_%s" % (rect, color))


def _image_size(path):
    """(H, W) of an 8-bit image from its header; 16-bit and float images are refused"""
    from PIL import Image

    if not os.path.isfile(path):
        raise FileNotFoundError("missing input file %s" % path)
    with Image.open(path) as im:
        if im.mode in ("I;16", "I;16B", "I;16L", "I", "F"):
            raise ValueError("%s: %s image; 8-bit images expected" % (path, im.mode))
        return im.size[1], im.size[0]


def _grey_size(path):
    from PIL import Image

    if not os.path.isfile(path):
        raise FileNotFoundError("missing input file %s" % path)
    with Image.open(path) as im:
        if im.mode != "L":
            raise ValueError("%s: %s image; an 8-bit grey map expected" % (path, im.mode))
        return im.size[1], im.size[0]


def _pfm_size(path):
    if not os.path.isfile(path):
        raise FileNotFoundError("missing input file %s" % path)
    with open(path, "rb") as f:
        kind = f.readline().strip()
        dims = f.readline().split()
    if kind != b"Pf":
        raise ValueError("%s: %s; a single-channel PFM (Pf) expected" % (path, kind[:8]))
    if len(dims) != 2:
        raise ValueError("%s: malformed PFM header" % path)
    return int(dims[1]), int(dims[0])


def _half_size(path, header):
    """the size of `path` after the script's halving: its .H cache's if present, else half the full size (even only)"""
    cache = path + (".H.pfm" if path.endswith(".pfm") else ".H.png")
    if os.path.isfile(cache):
        return header(cache)
    h, w = header(path)
    if h % 2 or w % 2:
        raise ValueError("%s is %dx%d: halving needs even sizes" % (path, h, w))
    return h // 2, w // 2


def _ndisp(calib):
    if not os.path.isfile(calib):
        raise FileNotFoundError("missing input file %s" % calib)
    with open(calib) as f:
        m = re.search("ndisp=(.*)", f.read())
    if not m:
        raise ValueError("%s: no ndisp= line" % calib)
    return int(m.group(1))


def _listdir(d):
    if not os.path.isdir(d):
        raise FileNotFoundError("missing input directory %s" % d)
    return sorted(os.listdir(d))


def _same_size(scene, sizes):
    sizes = list(sizes)
    for p, s in sizes:
        if s != sizes[0][1]:
            raise ValueError("%s: %s is %dx%d, %s is %dx%d" % (scene, p, s[0], s[1], sizes[0][0], *sizes[0][1]))
    return sizes[0][1]


def mb_scenes(data_root, rect):
    """Every image of preprocess_mb.py in the script's order, found and checked from file headers only: a list of dicts
    (log = the line the script prints, groups = [None or (files, shape)], half = whether the views are halved, disp =
    how the maps are read, ndisp, size = (H, W), submit = the fname_submit line or None)."""
    if rect not in ("perfect", "imperfect"):
        raise ValueError("rect must be 'perfect' or 'imperfect', got %r" % (rect,))
    out = []
    base1 = os.path.join(data_root, MB_DATA, "scenes2014", "datasets")
    for d in _listdir(base1):                                                  # :125-184
        if not d.endswith("imperfect"):
            continue
        imp = os.path.join(base1, d)
        perf = imp.replace("imperfect", "perfect")
        ndisp = _ndisp(os.path.join(imp, "calib.txt")) // 2                    # Python 2's int / 2
        groups = [([os.path.join(imp, f) for f in ("im0.png", "im1.png", "im1E.png", "im1L.png")], (4,))]
        base3 = os.path.join(perf if rect == "perfect" else imp, "ambient")
        lights = _listdir(base3)
        cams = ([], [])
        for f in _listdir(os.path.join(base3, "L1")):
            m = _MB_EXP.match(f)
            if m:
                cams[int(m.group(1))].append(int(m.group(2)) + 1)
        if not cams[0] or not cams[1]:
            raise ValueError("%s: no im0e<k>.png / im1e<k>.png exposures" % os.path.join(base3, "L1"))
        num_exp = min(max(cams[0]), max(cams[1]))
        if num_exp not in MB_EXPOSURES:
            raise ValueError("%s: %d exposures, which preprocess_mb.py's table (%s) does not cover"
                             % (os.path.join(base3, "L1"), num_exp, sorted(MB_EXPOSURES)))
        for light in range(len(lights)):
            b4 = os.path.join(base3, "L%d" % (light + 1))
            files = [os.path.join(b4, "im%de%d.png" % (cam, e)) for e in MB_EXPOSURES[num_exp] for cam in range(2)]
            groups.append((files, (len(files) // 2, 2)))
        disp = [os.path.join(imp, f) for f in ("disp0.pfm", "disp1.pfm", "disp0y.pfm")]
        size = _same_size(d, [(p, _half_size(p, _image_size)) for g in groups for p in g[0]]
                          + [(p, _half_size(p, _pfm_size)) for p in disp])
        out.append(dict(log=d.split("-")[0], groups=groups, half=True, disp=("pfm",) + tuple(disp), ndisp=ndisp,
                        size=size, submit=None, year=2014))
    n2014 = len(out)
    if n2014 < len(MB_TE):
        raise ValueError("%d 2014 scenes under %s; te.bin names images 1-%d, so at least %d are needed"
                         % (n2014, base1, len(MB_TE), len(MB_TE)))

    def pair_scene(log, base, views, d0, d1, div, ndisp, year, light_groups=None, tsukuba=False):
        groups = [None] + (light_groups or [([os.path.join(base, v) for v in views], (1, 2))])
        sizes = [(p, _image_size(p)) for g in groups[1:] for p in g[0]]
        maps = [os.path.join(base, d0)] + ([os.path.join(base, "nonocc.png")] if tsukuba else [os.path.join(base, d1)])
        size = _same_size(log, sizes + [(p, _grey_size(p)) for p in maps])
        return dict(log=log, groups=groups, half=False, disp=("tsukuba" if tsukuba else "grey", div) + tuple(maps),
                    ndisp=ndisp, size=size, submit=None, year=year)

    for year in (2006, 2005):                                                  # :189-231
        base1 = os.path.join(data_root, MB_DATA, "scenes%d" % year, "HalfSize")
        for d in _listdir(base1):
            base2 = os.path.join(base1, d)
            if not os.path.isfile(os.path.join(base2, "disp1.png")):
                continue
            lg = [([os.path.join(base2, "Illum%d" % (light + 1), "Exp%d" % e, v) for e in (0, 1, 2)
                    for v in ("view1.png", "view5.png")], (3, 2)) for light in range(3)]
            out.append(pair_scene(d, base2, None, "disp1.png", "disp5.png", 2, "ceil", year, light_groups=lg))
    for d in ("conesH", "teddyH"):                                             # :234-264
        base1 = os.path.join(data_root, MB_DATA, "scenes2003", d)
        out.append(pair_scene(d, base1, ("im2.ppm", "im6.ppm"), "disp2.pgm", "disp6.pgm", 2, "ceil", 2003))
    base1 = os.path.join(data_root, MB_DATA, "scenes2001", "data")
    for d in _listdir(base1):                                                  # :269-308
        if d == "tsukuba":
            f = ("scene1.row3.col3.ppm", "scene1.row3.col4.ppm"), "truedisp.row3.col3.pgm", None, 16
        elif d == "map":
            f = ("im0.pgm", "im1.pgm"), "disp0.pgm", "disp1.pgm", 8
        else:
            f = ("im2.ppm", "im6.ppm"), "disp2.pgm", "disp6.pgm", 8
        base2 = os.path.join(base1, d)
        if os.path.isfile(os.path.join(base2, f[1])):
            out.append(pair_scene(d, base2, *f, -1, 2001, tsukuba=d == "tsukuba"))
    for d1 in ("trainingH", "testH"):                                          # :313-328
        base2 = os.path.join(data_root, MB_EVAL, d1)
        for d2 in _listdir(base2):
            base3 = os.path.join(base2, d2)
            files = [os.path.join(base3, "im0.png"), os.path.join(base3, "im1.png")]
            size = _same_size(d2, [(p, _image_size(p)) for p in files])
            out.append(dict(log=os.path.join(d1, d2), groups=[(files, (2,))], half=False, disp=None,
                            ndisp=_ndisp(os.path.join(base3, "calib.txt")), size=size, submit=os.path.join(d1, d2),
                            year=None))
    return out


def _u8(x, narg, name):
    import torch

    from .adcensus import AdcensusError

    if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.uint8 or not x.is_contiguous():
        raise AdcensusError("bad argument #%d to '%s' (contiguous CUDA uint8 tensor expected)" % (narg, name))
    return x.data_ptr()


def _rgb_stack(x, name):
    from .adcensus import AdcensusError

    if x.dim() != 4 or x.size(3) != 3:
        raise AdcensusError("%s: (n, H, W, 3) bytes expected, got %s" % (name, tuple(x.shape)))
    return x.shape[:3]


def mb_views(rgb, nchannel):
    """read_im on the GPU: rgb (n, H, W, 3) CUDA uint8 (R, G, B) -> (n, nchannel, H, W) CUDA float32"""
    import torch

    from .adcensus import _check, _stream, lib

    name = "mb_views"
    p = _u8(rgb, 1, name)
    n, H, W = _rgb_stack(rgb, name)
    with torch.cuda.device(rgb.device):
        out = torch.empty((n, nchannel, H, W), dtype=torch.float32, device=rgb.device)
        _check(lib().mccnn_mb_views(p, out.data_ptr(), n, H, W, nchannel, _stream(rgb)), name)
    return out


def mb_half_image(rgb):
    """`convert -resize 50%` restated on the GPU: (n, H, W, 3) CUDA uint8 -> (n, H/2, W/2, 3)"""
    import torch

    from .adcensus import _check, _stream, lib

    name = "mb_half_image"
    p = _u8(rgb, 1, name)
    n, H, W = _rgb_stack(rgb, name)
    with torch.cuda.device(rgb.device):
        out = torch.empty((n, H // 2, W // 2, 3), dtype=torch.uint8, device=rgb.device)
        _check(lib().mccnn_mb_half_image(p, out.data_ptr(), n, H, W, _stream(rgb)), name)
    return out


def mb_half_disp(d):
    """load_pfm(.., True) on the GPU: (n, H, W) CUDA float32 top-down maps -> (n, H/2, W/2)"""
    import torch

    from .adcensus import AdcensusError, _check, _stream, _t, lib

    name = "mb_half_disp"
    p = _t(d, 1, name)
    if d.dim() != 3:
        raise AdcensusError("%s: (n, H, W) maps expected, got %s" % (name, tuple(d.shape)))
    n, H, W = d.shape
    with torch.cuda.device(d.device):
        out = torch.empty((n, H // 2, W // 2), dtype=torch.float32, device=d.device)
        _check(lib().mccnn_mb_half_disp(p, out.data_ptr(), n, H, W, _stream(d)), name)
    return out


def mb_mask(d0, d1, d0y=None):
    """the computemask rule on the GPU: (H, W) CUDA float32 maps -> (H, W) CUDA uint8 mask (0, 128, 255)"""
    import torch

    from .adcensus import AdcensusError, _check, _stream, _t, lib

    name = "mb_mask"
    maps = [d0, d1] + ([d0y] if d0y is not None else [])
    ps = [_t(m, k + 1, name) for k, m in enumerate(maps)]
    if d0.dim() != 2 or any(m.shape != d0.shape or m.device != d0.device for m in maps):
        raise AdcensusError("%s: (H, W) maps of one size on one device expected, got %s"
                            % (name, [tuple(m.shape) for m in maps]))
    H, W = d0.shape
    with torch.cuda.device(d0.device):
        out = torch.empty((H, W), dtype=torch.uint8, device=d0.device)
        _check(lib().mccnn_mb_mask(ps[0], ps[2] if d0y is not None else None, ps[1], H, W, out.data_ptr(), _stream(d0)), name)
    return out


def mb_nnz(d0, mask, image):
    """dispnoc and the training rows of one map on the GPU: d0 (H, W) CUDA float32, mask (H, W) CUDA uint8, image 1-based
    -> (dispnoc (H, W), rows (n, 4) float32 (image, y, x, d0) for mask == 255 in row-major order)"""
    import torch

    from .adcensus import AdcensusError, _check, _stream, _t, lib

    name = "mb_nnz"
    pd, pm = _t(d0, 1, name), _u8(mask, 2, name)
    if d0.dim() != 2 or mask.shape != d0.shape or mask.device != d0.device:
        raise AdcensusError("%s: d0 and mask (H, W) on one device expected, got %s and %s"
                            % (name, tuple(d0.shape), tuple(mask.shape)))
    H, W = d0.shape
    dev = d0.device
    with torch.cuda.device(dev):
        count = torch.zeros(1, dtype=torch.int64, device=dev)
        s = _stream(d0)
        _check(lib().mccnn_mb_nnz_count(pm, H, W, count.data_ptr(), s), name)
        n = int(count.item())
        dispnoc = torch.empty((H, W), dtype=torch.float32, device=dev)
        rows = torch.empty((n, 4), dtype=torch.float32, device=dev)
        _check(lib().mccnn_mb_nnz_fill(pd, pm, H, W, int(image), dispnoc.data_ptr(), rows.data_ptr(), n, s), name)
    return dispnoc, rows


def check_mb_outputs_absent(d):
    """refuse to overwrite: the first file the script's ``rm -f <dir>/*.{bin,dim,txt,type}`` would remove is named"""
    if os.path.isdir(d):
        for f in sorted(os.listdir(d)):
            if _MB_OUT.search(f):
                raise FileExistsError("%s already exists; remove the old outputs first (nothing was written)"
                                      % os.path.join(d, f))


def _read_rgb(path):
    """cv2.imread(path): (H, W, 3) R, G, B bytes, a grey file replicated, alpha dropped"""
    from PIL import Image

    with Image.open(path) as im:
        return np.asarray(im.convert("RGB"), dtype=np.uint8)


def _read_grey(path):
    from PIL import Image

    with Image.open(path) as im:
        return np.array(im, dtype=np.uint8)


def _read_pfm_topdown(path):
    return np.ascontiguousarray(np.flipud(dataio.read_pfm(path)))


def _mb_views(scene, color, dev):
    """every view of the scene through read_im, halved first for 2014: [None or (shape + (C, H, W)) float32 array]"""
    import torch

    files = [p for g in scene["groups"] if g for p in g[0]]
    imgs = [None] * len(files)
    full = []
    for k, p in enumerate(files):
        if scene["half"] and os.path.isfile(p + ".H.png"):
            imgs[k] = _read_rgb(p + ".H.png")
        elif scene["half"]:
            full.append(k)
        else:
            imgs[k] = _read_rgb(p)
    if full:
        big = torch.from_numpy(np.stack([_read_rgb(files[k]) for k in full])).to(dev)
        half = mb_half_image(big).cpu().numpy()
        del big
        for j, k in enumerate(full):
            imgs[k] = half[j]
    C = 3 if color == "rgb" else 1
    x = mb_views(torch.from_numpy(np.stack(imgs)).to(dev), C).cpu().numpy()
    out, k = [], 0
    for g in scene["groups"]:
        if g is None:
            out.append(None)
            continue
        n = len(g[0])
        out.append(x[k:k + n].reshape(g[1] + x.shape[1:]))
        k += n
    return out


def _mb_maps(scene, dev):
    """(d0, mask, ndisp) on the device for a scene with ground truth"""
    import torch

    kind = scene["disp"][0]
    if kind == "pfm":
        maps = [None] * 3
        todo = []
        for k, p in enumerate(scene["disp"][1:]):
            if os.path.isfile(p + ".H.pfm"):
                maps[k] = torch.from_numpy(_read_pfm_topdown(p + ".H.pfm")).to(dev)
            else:
                todo.append(k)
        if todo:
            full = torch.from_numpy(np.stack([_read_pfm_topdown(scene["disp"][1 + k]) for k in todo])).to(dev)
            half = mb_half_disp(full)
            for j, k in enumerate(todo):
                maps[k] = half[j].contiguous()
        d0, d1, dy = maps
        return d0, mb_mask(d0, d1, dy), scene["ndisp"]
    div = np.float32(scene["disp"][1])
    d0 = _read_grey(scene["disp"][2]).astype(np.float32) / div
    if kind == "tsukuba":                                                       # :290-292
        return torch.from_numpy(d0).to(dev), torch.from_numpy(_read_grey(scene["disp"][3])).to(dev), scene["ndisp"]
    d1 = _read_grey(scene["disp"][3]).astype(np.float32) / div
    ndisp = scene["ndisp"]
    if ndisp == "ceil":                                                         # 2006, 2005, 2003: before 0 -> inf
        ndisp = int(np.ceil(d0.max()))
        d0[d0 == 0] = np.inf
        d1[d1 == 0] = np.inf
    d0, d1 = torch.from_numpy(d0).to(dev), torch.from_numpy(d1).to(dev)
    return d0, mb_mask(d0, d1), ndisp


def _tofile_mb(fname, x):
    """preprocess_mb.py:99-106: an empty group is the .dim file ``0`` AND an empty data file"""
    if x is None:
        dataio.tofile(fname, None)
        open(fname, "wb").close()
    else:
        dataio.tofile(fname, x)


def preprocess_mb(data_root, rect, color, device=0, log=None):
    """preprocess_mb.py for one (rect, color): reads ``data_root/data.mb/unzip``, writes ``data_root/data.mb.<rect>_<color>``
    and returns that directory.  The per-pixel work runs on CUDA device `device` (0-based); `log` receives the lines the
    script prints."""
    import torch

    if color not in ("gray", "rgb"):
        raise ValueError("color must be 'gray' or 'rgb', got %r" % (color,))
    d = mb_output_dir(data_root, rect, color)
    check_mb_outputs_absent(d)
    scenes = mb_scenes(data_root, rect)
    os.makedirs(d, exist_ok=True)
    dev = torch.device("cuda", device)
    meta, nnz_tr, nnz_te, submit = [], [], [], []
    say = log or (lambda s: None)
    shape = lambda rows: "(%d, 4)" % sum(len(r) for r in rows)
    order = (2014, 2006, 2005, 2003)                                           # the script prints nnz_tr's shape after
    marks = [sum(1 for sc in scenes if sc["year"] in order[:k + 1]) for k in range(len(order))]   # each of these years

    def mark(done):
        while marks and marks[0] == done:
            say(shape(nnz_tr))
            marks.pop(0)

    for i, sc in enumerate(scenes, 1):
        say(sc["log"])
        views = _mb_views(sc, color, dev)
        for j, x in enumerate(views, 1):
            _tofile_mb(os.path.join(d, "x_%d_%d.bin" % (i, j)), x)
        ndisp = sc["ndisp"]
        if sc["disp"] is not None:
            d0, mask, ndisp = _mb_maps(sc, dev)
            dispnoc, rows = mb_nnz(d0, mask, i)
            dataio.tofile(os.path.join(d, "dispnoc%d.bin" % i), dispnoc.cpu().numpy())
            (nnz_te if sc["year"] == 2014 and i in MB_TE else nnz_tr).append(rows.cpu().numpy())
        meta.append((sc["size"][0], sc["size"][1], ndisp))
        if sc["submit"]:
            submit.append(sc["submit"])
        mark(i)
    cat = lambda rows: np.concatenate(rows) if rows else np.zeros((0, 4), np.float32)
    dataio.tofile(os.path.join(d, "meta.bin"), np.array(meta, dtype=np.int32))
    dataio.tofile(os.path.join(d, "nnz_tr.bin"), cat(nnz_tr))
    dataio.tofile(os.path.join(d, "nnz_te.bin"), cat(nnz_te))
    dataio.tofile(os.path.join(d, "te.bin"), np.array(MB_TE, dtype=np.int64))
    with open(os.path.join(d, "fname_submit.txt"), "w") as f:
        f.write("\n".join(submit))
    return d
