"""stereo_predict for the 'fast' architecture, from the tower output onwards.

Two faces over the same kernels:

* :func:`stereo_predict` chains the ``adcensus.*`` operator calls exactly as
  main.lua:929-1082 does (same order, same tensors, same Lua-side fill / copy /
  transpose / argmin steps), so it reads like the reference's own driver;
* :class:`StereoPipeline` is the native fused object behind
  ``mccnn_pipeline_*`` (include/adcensus_b200.h): buffers allocated once, one
  stream, no host sync -- what bench.py and a batch driver use.

Hyper-parameter presets are main.lua:70-295 copied as data.
"""
import ctypes

import torch

from . import adcensus


class Params(ctypes.Structure):
    """mccnn_params; field names are main.lua's option names."""

    _fields_ = [
        ("L1", ctypes.c_int),
        ("tau1", ctypes.c_float),
        ("cbca_i1", ctypes.c_int),
        ("cbca_i2", ctypes.c_int),
        ("pi1", ctypes.c_float),
        ("pi2", ctypes.c_float),
        ("sgm_q1", ctypes.c_float),
        ("sgm_q2", ctypes.c_float),
        ("alpha1", ctypes.c_float),
        ("tau_so", ctypes.c_float),
        ("sgm_i", ctypes.c_int),
        ("blur_sigma", ctypes.c_double),
        ("blur_t", ctypes.c_float),
        ("border", ctypes.c_int),
        ("lr_check", ctypes.c_int),
        ("sm_terminate", ctypes.c_int),   # a SM_TERMINATE code (main.lua's -sm_terminate), 0 = the full chain
        ("sm_skip", ctypes.c_int),        # a SM_SKIP code (-sm_skip), 0 = none
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# main.lua's -sm_terminate / -sm_skip values (main.lua:953-1082) -> the MCCNN_SM_* codes of include/adcensus_b200.h.
# "" means neither option.  main.lua accepts any string and ignores the ones it does not test; these tables refuse them, so
# that a misspelt step cannot silently give the full chain.
SM_TERMINATE = {"": 0, "cnn": 1, "cbca1": 2, "sgm": 3, "cbca2": 4, "occlusion": 5, "mismatch": 6,
                "subpixel_enchancement": 7, "median": 8}
SM_SKIP = {"": 0, "cbca": 10, "sgm": 3, "occlusion": 5, "subpixel_enchancement": 7, "median": 8, "bilateral": 9}


def stage_code(option, name):
    """the code of main.lua's ``-sm_terminate`` / ``-sm_skip`` value `name` (option "sm_terminate" or "sm_skip")"""
    table = SM_TERMINATE if option == "sm_terminate" else SM_SKIP
    if not isinstance(name, str) or name not in table:
        raise ValueError("-%s %r is not a step (valid: %s)" % (option, name, " ".join(n for n in table if n)))
    return table[name]


def idle_steps(opt):
    """The -sm_skip / -sm_terminate names whose step does no work under `opt`'s parameters: skipping or stopping after such a
    step gives the result of another variant (skip cbca without CBCA iterations is the full chain, terminate cbca1 with
    cbca_i1 = 0 is terminate cnn, ...).  The LR-check steps do no work without the LR check (mb)."""
    idle = set()
    if opt.cbca_i1 + opt.cbca_i2 == 0:
        idle.add("cbca")
    if opt.cbca_i1 == 0:
        idle.add("cbca1")
    if opt.cbca_i2 == 0:
        idle.add("cbca2")
    if opt.sgm_i == 0:
        idle.add("sgm")
    if not opt.lr_check:
        idle |= {"occlusion", "mismatch"}
    return idle


def stages(opt):
    """Which steps of main.lua:953-1082 run for the stage fields of `opt`: a dict step -> bool over cbca1 (the cross arms and
    the first CBCA block), sgm, cbca2, occlusion, mismatch, subpixel, median, bilateral.  csrc/pipeline.cu's stages_of is the
    same table."""
    T, S = opt.sm_terminate, opt.sm_skip
    lr = bool(opt.lr_check)
    st = {}
    active = T != SM_TERMINATE["cnn"]                                              # :988
    st["cbca1"] = active and S != SM_SKIP["cbca"]                                  # :992
    active = active and T != SM_TERMINATE["cbca1"]                                 # :1005
    st["sgm"] = active and S != SM_SKIP["sgm"]                                     # :1007
    active = active and T != SM_TERMINATE["sgm"]                                   # :1031
    st["cbca2"] = active and S != SM_SKIP["cbca"]                                  # :1033
    active = active and T != SM_TERMINATE["cbca2"]                                 # :1040
    st["occlusion"] = lr and active and S != SM_SKIP["occlusion"]                  # :1057
    active = active and not (lr and T == SM_TERMINATE["occlusion"])                # :1060
    st["mismatch"] = lr and active and S != SM_SKIP["occlusion"]                   # :1062
    active = active and not (lr and T == SM_TERMINATE["mismatch"])                 # :1065
    st["subpixel"] = active and S != SM_SKIP["subpixel_enchancement"]             # :1067
    active = active and T != SM_TERMINATE["subpixel_enchancement"]                 # :1071
    st["median"] = active and S != SM_SKIP["median"]                               # :1072
    active = active and T != SM_TERMINATE["median"]                                # :1076
    st["bilateral"] = active and S != SM_SKIP["bilateral"]                         # :1077
    return st


# (dataset, arch) -> stereo-method options, main.lua:70-295.  `border` = (window-1)/2 of the
# feature tower (main.lua:382-391, 923): 4 conv3x3 layers -> 4 (mb: 5 layers -> 5).
PRESETS = {
    ("kitti", "slow"): dict(L1=5, tau1=0.13, cbca_i1=2, cbca_i2=0, pi1=1.32, pi2=24.25, sgm_q1=3, sgm_q2=2,
                            alpha1=2, tau_so=0.08, blur_sigma=5.99, blur_t=6, border=4, lr_check=1),
    ("kitti2015", "slow"): dict(L1=5, tau1=0.03, cbca_i1=2, cbca_i2=4, pi1=2.3, pi2=24.25, sgm_q1=3, sgm_q2=2,
                                alpha1=1.75, tau_so=0.08, blur_sigma=5.99, blur_t=5, border=4, lr_check=1),
    ("mb", "slow"): dict(L1=14, tau1=0.02, cbca_i1=2, cbca_i2=16, pi1=1.3, pi2=13.9, sgm_q1=4.5, sgm_q2=2,
                         alpha1=2.75, tau_so=0.13, blur_sigma=1.67, blur_t=2, border=5, lr_check=0),
    ("kitti", "fast"): dict(L1=0, tau1=0, cbca_i1=0, cbca_i2=0, pi1=4, pi2=55.72, sgm_q1=3, sgm_q2=2.5,
                            alpha1=1.5, tau_so=0.02, blur_sigma=7.74, blur_t=5, border=4, lr_check=1),
    ("kitti2015", "fast"): dict(L1=0, tau1=0, cbca_i1=0, cbca_i2=0, pi1=2.3, pi2=18.38, sgm_q1=3, sgm_q2=2,
                                alpha1=1.25, tau_so=0.08, blur_sigma=4.64, blur_t=5, border=4, lr_check=1),
    ("mb", "fast"): dict(L1=0, tau1=0, cbca_i1=0, cbca_i2=0, pi1=2.3, pi2=24.3, sgm_q1=4, sgm_q2=2,
                         alpha1=1.5, tau_so=0.08, blur_sigma=6, blur_t=2, border=5, lr_check=0),
    # net-free cost volumes (main.lua:146-204): no feature tower, hence no fix_border (border = 0)
    ("kitti", "census"): dict(L1=0, tau1=0.01, cbca_i1=4, cbca_i2=8, pi1=4, pi2=128.0, sgm_q1=3, sgm_q2=3.5,
                              alpha1=1.25, tau_so=1.0, blur_sigma=7.74, blur_t=6, border=0, lr_check=1),
    ("mb", "census"): dict(L1=5, tau1=0.22, cbca_i1=8, cbca_i2=8, pi1=4.0, pi2=32.0, sgm_q1=4, sgm_q2=3,
                           alpha1=1.5, tau_so=1.0, blur_sigma=2.78, blur_t=3, border=0, lr_check=0),
    ("kitti", "ad"): dict(L1=3, tau1=0.03, cbca_i1=0, cbca_i2=4, pi1=0.76, pi2=13.93, sgm_q1=3.5, sgm_q2=2,
                          alpha1=2.5, tau_so=0.01, blur_sigma=7.74, blur_t=6, border=0, lr_check=1),
    ("mb", "ad"): dict(L1=5, tau1=0.36, cbca_i1=0, cbca_i2=4, pi1=0.4, pi2=8.0, sgm_q1=3, sgm_q2=4,
                       alpha1=2.5, tau_so=0.08, blur_sigma=7.74, blur_t=1, border=0, lr_check=0),
    # BASELINE.json config 3 ("KITTI accurate: CBCA x4 + SGM"): kitti slow post-processing with
    # cbca_i1 = cbca_i2 = 2
    ("kitti", "accurate_cbca4"): dict(L1=5, tau1=0.13, cbca_i1=2, cbca_i2=2, pi1=1.32, pi2=24.25, sgm_q1=3,
                                      sgm_q2=2, alpha1=2, tau_so=0.08, blur_sigma=5.99, blur_t=6, border=4,
                                      lr_check=1),
}


ARCHS = ("fast", "slow", "ad", "census")


def check_arch(arch):
    """refuse an architecture main.lua does not have"""
    if arch not in ARCHS:
        raise ValueError("arch must be %s or %r" % (", ".join(map(repr, ARCHS[:-1])), ARCHS[-1]))


def make_params(dataset="kitti", arch="fast", **overrides):
    """The preset of (dataset, arch) with `overrides`; ``sm_terminate`` / ``sm_skip`` take main.lua's step names.  kitti2015
    shares kitti's 'ad' and 'census' presets (main.lua:146-204)."""
    if dataset == "kitti2015" and arch in ("ad", "census"):
        dataset = "kitti"
    d = dict(PRESETS[(dataset, arch)])
    d.setdefault("sgm_i", 1)
    for k in ("sm_terminate", "sm_skip"):
        if k in overrides:
            overrides[k] = stage_code(k, overrides[k])
    d.update(overrides)
    return Params(**d)


def stereo_predict(x_batch, features, opt, disp_max, want_vols=False, arch="fast", head=None, conf=None, lr=None):
    """main.lua:929-1082 through the adcensus.* operators.

    x_batch  (2,1,H,W) standardised images (left, right); arch 'fast': features (2,C,H,W) the tower
    output (unit-norm); arch 'ad' / 'census': the matching cost comes from the images themselves
    (main.lua:932-942), `features` is ignored; arch 'slow' (main.lua:956-981): features (2,fm,H,W) = the accurate
    architecture's tower output and `head` a :class:`mccnn_b200.scorer_head.ScorerHead` (net_te2), which scores every
    disparity into both volumes.  opt a :class:`Params`.
    `conf` / `lr` (H, W) device tensors or None (an addition beyond the reference, DESIGN §19): receive the margin
    confidence of the final left volume (:func:`confidence.margin`) and main.lua:1056's outlier map (0 consistent,
    1 mismatch, 2 occlusion; only with the LR check, computed even when -sm_terminate / -sm_skip leave it unused).
    Returns disp (1,1,H,W) [, left vol, right vol].
    """
    assert x_batch.is_cuda
    check_arch(arch)
    if lr is not None and not opt.lr_check:
        raise adcensus.AdcensusError("stereo_predict: lr needs the LR check (kitti / kitti2015); main.lua has none for mb")
    H, W = x_batch.size(2), x_batch.size(3)
    dev = x_batch.device
    vols = torch.empty((2, disp_max, H, W), device=dev, dtype=torch.float32)
    adcensus.fill_nan(vols)                                                       # :933 / :939 / :946
    if arch == "ad":
        adcensus.ad(x_batch[0:1], x_batch[1:2], vols[0:1], -1)                    # :934
        adcensus.ad(x_batch[1:2], x_batch[0:1], vols[1:2], 1)                     # :935
    elif arch == "census":
        adcensus.census(x_batch[0:1], x_batch[1:2], vols[0:1], -1)                # :940
        adcensus.census(x_batch[1:2], x_batch[0:1], vols[1:2], 1)                 # :941
    elif arch == "fast":
        assert features is not None and features.is_cuda
        adcensus.StereoJoin(features[0:1], features[1:2], vols[0:1], vols[1:2])   # :947
        adcensus.fix_border(vols[0:1], opt.border, -1)                            # :948
        adcensus.fix_border(vols[1:2], opt.border, 1)                             # :949
    elif arch == "slow":
        assert features is not None and features.is_cuda and head is not None, "arch 'slow' needs the tower output and a ScorerHead"
        vl, vr = head.volumes(features[0].contiguous(), features[1].contiguous(), disp_max)   # :962-979 (both directions at once)
        vols[0:1].copy_(vl)
        vols[1:2].copy_(vr)
        adcensus.fix_border(vols[0:1], opt.border, -1)                            # :981
        adcensus.fix_border(vols[1:2], opt.border, 1)

    st = stages(opt)                                                              # -sm_terminate / -sm_skip
    disp = {}
    out_vols = {}
    vol = None
    for direction in (1, -1):                                                     # :955
        vol = vols[0:1] if direction == -1 else vols[1:2]                         # :986
        if st["cbca1"]:                                                           # :992
            x0c = torch.empty((1, 4, H, W), device=dev, dtype=torch.float32)      # :993-996
            x1c = torch.empty((1, 4, H, W), device=dev, dtype=torch.float32)
            adcensus.cross(x_batch[0], x0c, opt.L1, opt.tau1)
            adcensus.cross(x_batch[1], x1c, opt.L1, opt.tau1)
            tmp_cbca = torch.empty_like(vol)
            for _ in range(opt.cbca_i1):                                          # :998-1001
                adcensus.cbca(x0c, x1c, vol, tmp_cbca, direction)
                vol.copy_(tmp_cbca)
        if st["sgm"]:                                                             # :1007
            volt = adcensus.transpose_dhw_to_hwd(vol)                             # :1008
            out = torch.empty_like(volt)
            tmp = torch.empty((W, disp_max), device=dev, dtype=torch.float32)     # :1012
            for _ in range(opt.sgm_i):
                out.zero_()                                                       # :1014
                adcensus.sgm2(x_batch[0], x_batch[1], volt, out, tmp, opt.pi1, opt.pi2, opt.tau_so, opt.alpha1,
                              opt.sgm_q1, opt.sgm_q2, direction)                  # :1015
                volt.copy_(out).div_(4)                                           # :1017
            vol.copy_(adcensus.transpose_hwd_to_dhw_div4(out))                    # :1019-1020
        if st["cbca2"]:                                                           # :1033
            for _ in range(opt.cbca_i2):                                          # :1035-1038
                adcensus.cbca(x0c, x1c, vol, tmp_cbca, direction)
                vol.copy_(tmp_cbca)
        if want_vols:
            out_vols[direction] = vol.clone()                                     # :1042-1047
        disp[1 if direction == 1 else 2] = adcensus.argmin(vol)                   # :1049-1050

    if conf is not None:
        from . import confidence

        conf.view(H, W).copy_(confidence.margin(vol)[1].view(H, W))
    d = disp[2]
    if opt.lr_check:                                                              # :1054-1066
        outlier = torch.zeros_like(d)
        adcensus.outlier_detection(disp[2], disp[1], outlier, disp_max)
        if lr is not None:
            lr.view(H, W).copy_(outlier.view(H, W))
        if st["occlusion"]:
            d = adcensus.interpolate_occlusion(d, outlier)
        if st["mismatch"]:
            d = adcensus.interpolate_mismatch(d, outlier)
    if st["subpixel"]:
        d = adcensus.subpixel_enchancement(d, vol, disp_max)                      # :1068 (left volume)
    if st["median"]:
        d = adcensus.median2d(d, 5)                                               # :1073
    if st["bilateral"]:
        d = adcensus.mean2d(d, adcensus.gaussian(opt.blur_sigma).to(dev), opt.blur_t)  # :1078
    if want_vols:
        return d, out_vols[-1], out_vols[1]
    return d


class StereoPipeline:
    """Native fused stereo_predict (mccnn_pipeline_*): buffers allocated once per (C,D,H,W); :meth:`run` runs at that
    shape, :meth:`run_shape` at any (H, W, D) that fits inside it."""

    def __init__(self, C, D, H, W, params, device=0, cbca_mode=None):
        """``cbca_mode``: "fast" (library default) = constant-work aggregation inside the north star's 1e-4 contract
        for float aggregation; "exact" = tap-by-tap sums, volumes bit-identical to the reference."""
        self.C, self.D, self.H, self.W = C, D, H, W
        self.params = params
        self.device = int(device)
        self._h = ctypes.c_void_p()
        rc = adcensus.lib().mccnn_pipeline_create(ctypes.byref(self._h), C, D, H, W, ctypes.byref(params), self.device)
        adcensus._check(rc, "mccnn_pipeline_create")
        if cbca_mode is not None:
            self.set_cbca_mode(cbca_mode)

    def close(self):
        if self._h:
            adcensus.lib().mccnn_pipeline_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_overlap(self, mode=2):
        """1 or 2 (the default): run the two directions concurrently on two streams; 0: sequentially on one stream, with
        less device memory (mccnn_pipeline_set_overlap).  Results are unchanged."""
        adcensus._check(adcensus.lib().mccnn_pipeline_set_overlap(self._h, int(mode)), "mccnn_pipeline_set_overlap")

    def set_cbca_mode(self, mode):
        """"fast" / 1: constant-work CBCA (csrc/cbca_tma.cu, ~1e-6 relative to the tap-by-tap sums, bar 1e-4);
        "exact" / 0: bit-identical to the reference (mccnn_pipeline_set_cbca_mode)."""
        m = {"fast": 1, "exact": 0}.get(mode, mode)
        adcensus.lib().mccnn_pipeline_set_cbca_mode(self._h, int(bool(m)))

    @property
    def cbca_mode(self):
        return "fast" if adcensus.lib().mccnn_pipeline_get_cbca_mode(self._h) else "exact"

    def set_params(self, params):
        """Re-target the pipeline to another :class:`Params` (mccnn_pipeline_set_params): later runs give the bits of a
        pipeline created with them.  Waits for the work enqueued on the pipeline's device."""
        if not isinstance(params, Params):
            raise adcensus.AdcensusError("mccnn_pipeline_set_params: a pipeline.Params expected, got %s" % type(params).__name__)
        adcensus._check(adcensus.lib().mccnn_pipeline_set_params(self._h, ctypes.byref(params)), "mccnn_pipeline_set_params")
        self.params = params

    @property
    def device_bytes(self):
        return adcensus.lib().mccnn_pipeline_device_bytes(self._h)

    @property
    def launches_per_run(self):
        return adcensus.lib().mccnn_pipeline_launches_per_run(self._h)

    def run(self, featL, featR, imgL, imgR, disp=None, volL=None, volR=None):
        """Device tensors in, device disparity map out; asynchronous on torch's current stream."""
        n = "mccnn_pipeline_run"
        if disp is None:
            disp = torch.empty((self.H, self.W), device=featL.device, dtype=torch.float32)
        with torch.cuda.device(featL.device):
            rc = adcensus.lib().mccnn_pipeline_run(self._h, adcensus._t(featL, 1, n), adcensus._t(featR, 2, n),
                                                   adcensus._t(imgL, 3, n), adcensus._t(imgR, 4, n),
                                                   adcensus._t(disp, 5, n), adcensus._t(volL, 0, n, optional=True),
                                                   adcensus._t(volR, 0, n, optional=True), adcensus._stream(featL))
        adcensus._check(rc, n)
        return disp

    def run_shape(self, featL, featR, imgL, imgR, disp_max=None, disp=None, volL=None, volR=None, conf=None, lr=None):
        """:meth:`run` at a smaller shape than the created one (mccnn_pipeline_run_shape): H, W from ``imgL``, D =
        ``disp_max`` (default: the created D); every tensor must be contiguous at that shape.  Same results, bit for bit,
        as a pipeline created at this shape, without allocating: one pipeline created at the largest (H, W, D) of a dataset
        serves all of its images.  ``conf`` / ``lr`` (H, W) receive the margin confidence and the LR check's outlier map
        (mccnn_pipeline_run_shape_conf; ``lr`` only with the LR check); ``disp`` is the same with or without them.
        Asynchronous on torch's current stream."""
        n = "mccnn_pipeline_run_shape"
        if imgL.dim() != 2:
            raise adcensus.AdcensusError("%s: imgL must be (H, W), got %s" % (n, tuple(imgL.shape)))
        H, W = imgL.shape
        D = self.D if disp_max is None else int(disp_max)
        if disp is None:
            disp = torch.empty((H, W), device=imgL.device, dtype=torch.float32)
        want = [("featL", featL, (self.C, H, W)), ("featR", featR, (self.C, H, W)), ("imgR", imgR, (H, W)),
                ("disp", disp, (H, W)), ("volL", volL, (D, H, W)), ("volR", volR, (D, H, W)), ("conf", conf, (H, W)),
                ("lr", lr, (H, W))]
        for name, t, shape in want:
            if t is not None and tuple(t.shape) != shape:
                raise adcensus.AdcensusError("%s: %s must be %s, got %s" % (n, name, shape, tuple(t.shape)))
        self._check_lr(lr, n)
        with torch.cuda.device(imgL.device):
            ptrs = (adcensus._t(featL, 1, n), adcensus._t(featR, 2, n), adcensus._t(imgL, 3, n), adcensus._t(imgR, 4, n),
                    adcensus._t(disp, 5, n))
            vols = (adcensus._t(volL, 6, n, optional=True), adcensus._t(volR, 7, n, optional=True))
            if conf is None and lr is None:
                rc = adcensus.lib().mccnn_pipeline_run_shape(self._h, H, W, D, *ptrs, *vols, adcensus._stream(imgL))
            else:
                rc = adcensus.lib().mccnn_pipeline_run_shape_conf(self._h, H, W, D, *ptrs, adcensus._t(conf, 8, n, optional=True),
                                                                  adcensus._t(lr, 9, n, optional=True), *vols,
                                                                  adcensus._stream(imgL))
        adcensus._check(rc, n)
        return disp

    def _check_lr(self, lr, n):
        if lr is not None and not self.params.lr_check:
            raise adcensus.AdcensusError("%s: lr needs the LR check (kitti / kitti2015); main.lua has none for mb" % n)

    def run_volumes(self, volL, volR, imgL, imgR, disp_max=None, disp=None, outL=None, outR=None, conf=None, lr=None):
        """The chain of :meth:`run_shape` from given cost volumes (mccnn_pipeline_run_volumes): volL / volR (D, H, W) or
        (1, D, H, W) device tensors as main.lua holds them at :986 (NaN fill, fix_border applied); they are not modified.
        ``volR`` may be None when the parameters have no LR check and ``outR`` is None.  H, W from ``imgL``, D = ``disp_max``
        (default: the created D).  ``conf`` / ``lr`` as in :meth:`run_shape`.  Asynchronous on torch's current stream."""
        n = "mccnn_pipeline_run_volumes"
        if imgL.dim() != 2:
            raise adcensus.AdcensusError("%s: imgL must be (H, W), got %s" % (n, tuple(imgL.shape)))
        H, W = imgL.shape
        D = self.D if disp_max is None else int(disp_max)
        if disp is None:
            disp = torch.empty((H, W), device=imgL.device, dtype=torch.float32)
        vol = lambda t: t[0] if t is not None and t.dim() == 4 and t.shape[0] == 1 else t
        volL, volR = vol(volL), vol(volR)
        want = [("volL", volL, (D, H, W)), ("volR", volR, (D, H, W)), ("imgR", imgR, (H, W)), ("disp", disp, (H, W)),
                ("outL", outL, (D, H, W)), ("outR", outR, (D, H, W)), ("conf", conf, (H, W)), ("lr", lr, (H, W))]
        for name, t, shape in want:
            if t is not None and tuple(t.shape) != shape:
                raise adcensus.AdcensusError("%s: %s must be %s, got %s" % (n, name, shape, tuple(t.shape)))
        if volR is None and (self.params.lr_check or outR is not None):
            raise adcensus.AdcensusError("%s: volR is needed (LR check or outR)" % n)
        self._check_lr(lr, n)
        ptrs = (adcensus._t(volL, 1, n), adcensus._t(volR, 2, n, optional=True), adcensus._t(imgL, 3, n),
                adcensus._t(imgR, 4, n), adcensus._t(disp, 5, n))
        outs = (adcensus._t(outL, 6, n, optional=True), adcensus._t(outR, 7, n, optional=True))
        with torch.cuda.device(imgL.device):
            if conf is None and lr is None:
                rc = adcensus.lib().mccnn_pipeline_run_volumes(self._h, H, W, D, *ptrs, *outs, adcensus._stream(imgL))
            else:
                rc = adcensus.lib().mccnn_pipeline_run_volumes_conf(self._h, H, W, D, *ptrs, adcensus._t(conf, 8, n, optional=True),
                                                                    adcensus._t(lr, 9, n, optional=True), *outs,
                                                                    adcensus._stream(imgL))
        adcensus._check(rc, n)
        return disp

    def run_batch(self, pairs, disps=None):
        """``pairs``: list of (featL, featR, imgL, imgR) DEVICE tensors.  One call for the whole list, ordered on torch's
        current stream as a whole; pairs alternate between two internal lanes (mccnn_pipeline_run_batch) so that the
        post-processing tail of one pair overlaps the volume kernels of the next.  Returns the list of device disparity maps."""
        n = "mccnn_pipeline_run_batch"
        k = len(pairs)
        if disps is None:
            disps = [torch.empty((self.H, self.W), device=pairs[0][0].device, dtype=torch.float32) for _ in range(k)]
        arr = lambda ts, i: (ctypes.c_void_p * k)(*[adcensus._t(t, i, n) for t in ts])
        with torch.cuda.device(pairs[0][0].device):
            rc = adcensus.lib().mccnn_pipeline_run_batch(
                self._h, k, arr([p[0] for p in pairs], 1), arr([p[1] for p in pairs], 2), arr([p[2] for p in pairs], 3),
                arr([p[3] for p in pairs], 4), arr(disps, 5), adcensus._stream(pairs[0][0]))
        adcensus._check(rc, n)
        return disps

    def run_host(self, featL, featR, imgL, imgR, disp=None):
        """Host (CPU, ideally pinned) float32 tensors in and out; synchronous.  This is the call
        a non-CUDA host (the Lua/FFI side) makes: H2D + pipeline + D2H inside."""
        n = "mccnn_pipeline_run_host"
        for t in (featL, featR, imgL, imgR):
            if t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
                raise adcensus.AdcensusError("%s: contiguous host float tensors expected" % n)
        if disp is None:
            disp = torch.empty((self.H, self.W), dtype=torch.float32)
        rc = adcensus.lib().mccnn_pipeline_run_host(self._h, featL.data_ptr(), featR.data_ptr(), imgL.data_ptr(),
                                                    imgR.data_ptr(), disp.data_ptr())
        adcensus._check(rc, n)
        return disp

    def run_host_batch(self, pairs, disps=None):
        """``pairs``: list of (featL, featR, imgL, imgR) host float32 tensors (pinned for overlap).
        H2D of pair i+1 and D2H of pair i-1 overlap the kernels of pair i.  Returns the list of
        host disparity maps (synchronous)."""
        n = "mccnn_pipeline_run_host_batch"
        k = len(pairs)
        for pr in pairs:
            for t in pr:
                if t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
                    raise adcensus.AdcensusError("%s: contiguous host float tensors expected" % n)
        if disps is None:
            disps = [torch.empty((self.H, self.W), dtype=torch.float32).pin_memory() for _ in range(k)]
        arr = lambda ts: (ctypes.c_void_p * k)(*[t.data_ptr() for t in ts])
        rc = adcensus.lib().mccnn_pipeline_run_host_batch(
            self._h, k, arr([p[0] for p in pairs]), arr([p[1] for p in pairs]), arr([p[2] for p in pairs]),
            arr([p[3] for p in pairs]), arr(disps))
        adcensus._check(rc, n)
        return disps
