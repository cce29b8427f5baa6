"""main.lua:929-1082 with -sm_terminate / -sm_skip (main.lua:953-1082), restated for the stage tests on two independent
operator sets: the CPU oracle's per-operator functions (oracle/oracle.py) and the reference's own kernels through the shim
(oracle/refdriver.py).  Both follow main.lua's sm_active logic line by line on the option NAMES, so they share nothing with
the product's name table (mccnn_b200.pipeline.SM_*) or its stage plan (pipeline.stages, csrc/pipeline.cu's stages_of).

The oracle's own stereo_predict / stereo_predict_chain run the full chain only: oracle.Params(**opt.as_dict()) keeps the
stage fields as plain attributes that nothing reads, so they must never be handed a variant.  `full_chain_params` turns a
pipeline.Params into oracle.Params and refuses a non-default stage field.
"""
import numpy as np

SKIP = ("cbca", "sgm", "occlusion", "subpixel_enchancement", "median", "bilateral")
TERMINATE = ("cnn", "cbca1", "sgm", "cbca2", "occlusion", "mismatch", "subpixel_enchancement", "median")
VARIANTS = [("", "")] + [("", s) for s in SKIP] + [(t, "") for t in TERMINATE]     # (sm_terminate, sm_skip)


def variant_id(v):
    t, s = v
    return "full" if not (t or s) else ("skip_" + s if s else "terminate_" + t)


def full_chain_params(orc, opt):
    if getattr(opt, "sm_terminate", 0) or getattr(opt, "sm_skip", 0):
        raise AssertionError("the oracle's one-call chains run the full chain only; use stage_chain for a variant")
    d = opt.as_dict()
    d.pop("sm_terminate", None)
    d.pop("sm_skip", None)
    return orc.Params(**d)


def oracle_chain(orc, imgL, imgR, D, opt, sm_terminate="", sm_skip="", arch="fast", featL=None, featR=None, volL=None,
                 volR=None, want_vols=False):
    """the oracle's operators in main.lua's order.  arch 'fast': StereoJoin of featL / featR + fix_border; 'census' / 'ad':
    the image volumes; 'volumes': volL / volR given (NaN fill and fix_border already applied, as main.lua holds them at
    :986).  Returns disp (H, W) [, left volume, right volume after the steps that ran]."""
    imgL = np.ascontiguousarray(imgL, np.float32)
    imgR = np.ascontiguousarray(imgR, np.float32)
    if arch == "fast":
        volL, volR = orc.stereo_join(featL, featR, D)                                  # :946-947
        orc.fix_border(volL, opt.border, -1)                                           # :948
        orc.fix_border(volR, opt.border, 1)                                            # :949
    elif arch == "census":
        volL, volR = orc.census(imgL, imgR, D, -1), orc.census(imgR, imgL, D, 1)       # :940-941
    elif arch == "ad":
        volL, volR = orc.ad(imgL, imgR, D, -1), orc.ad(imgR, imgL, D, 1)               # :934-935
    elif arch == "volumes":
        volL, volR = np.array(volL, np.float32), np.array(volR, np.float32)
    else:
        raise ValueError(arch)
    disp, vols = {}, {}
    sm_active = True
    for direction in (1, -1):                                                          # :955
        sm_active = True                                                               # :956
        vol = volL if direction == -1 else volR                                        # :986
        sm_active = sm_active and sm_terminate != "cnn"                                # :988
        if sm_active and sm_skip != "cbca":                                            # :992-1004
            x0c, x1c = orc.cross(imgL, opt.L1, opt.tau1), orc.cross(imgR, opt.L1, opt.tau1)
            for _ in range(opt.cbca_i1):
                vol = orc.cbca(x0c, x1c, vol, direction)
        sm_active = sm_active and sm_terminate != "cbca1"                              # :1005
        if sm_active and sm_skip != "sgm":                                             # :1007-1030
            for _ in range(opt.sgm_i):
                out = orc.sgm2(imgL, imgR, orc.transpose_dhw_to_hwd(vol), opt.pi1, opt.pi2, opt.tau_so, opt.alpha1,
                               opt.sgm_q1, opt.sgm_q2, direction)
                vol = orc.transpose_hwd_to_dhw_div4(out)
        sm_active = sm_active and sm_terminate != "sgm"                                # :1031
        if sm_active and sm_skip != "cbca":                                            # :1033-1039
            for _ in range(opt.cbca_i2):
                vol = orc.cbca(x0c, x1c, vol, direction)
        sm_active = sm_active and sm_terminate != "cbca2"                              # :1040
        vols[direction] = vol                                                          # :1042-1047
        disp[direction] = orc.spatial_argmin(vol) - 1                                  # :1049-1050
    d = disp[-1]
    if opt.lr_check:                                                                   # :1054-1066
        outlier = orc.outlier_detection(disp[-1], disp[1], D)
        if sm_active and sm_skip != "occlusion":
            d = orc.interpolate_occlusion(d, outlier)
        sm_active = sm_active and sm_terminate != "occlusion"
        if sm_active and sm_skip != "occlusion":
            d = orc.interpolate_mismatch(d, outlier)
        sm_active = sm_active and sm_terminate != "mismatch"
    if sm_active and sm_skip != "subpixel_enchancement":                               # :1067-1070
        d = orc.subpixel_enchancement(d, vols[-1], D)
    sm_active = sm_active and sm_terminate != "subpixel_enchancement"
    if sm_active and sm_skip != "median":                                              # :1072-1075
        d = orc.median2d(d, 5)
    sm_active = sm_active and sm_terminate != "median"
    if sm_active and sm_skip != "bilateral":                                           # :1077-1079
        d = orc.mean2d(d, orc.gaussian(opt.blur_sigma), opt.blur_t)
    return (d, vols[-1], vols[1]) if want_vols else d


def reference_chain(shim, x_batch, features, opt, disp_max, sm_terminate="", sm_skip="", want_vols=False,
                    directions=(1, -1)):
    """oracle/refdriver.stereo_predict (arch 'fast', the reference's kernels through `shim`) with the stage options"""
    import torch

    from oracle import refdriver

    call = shim.call
    H, W = x_batch.size(2), x_batch.size(3)
    dev = x_batch.device
    vols = torch.full((2, disp_max, H, W), float("nan"), device=dev, dtype=torch.float32)   # :946
    call("StereoJoin", features[0:1], features[1:2], vols[0:1], vols[1:2])                  # :947
    refdriver.fix_border(vols[0:1], opt.border, -1)                                         # :948
    refdriver.fix_border(vols[1:2], opt.border, 1)                                          # :949
    disp, out_vols = {}, {}
    vol = None
    sm_active = True
    for direction in directions:                                                            # :954-955
        sm_active = True
        vol = vols[0:1] if direction == -1 else vols[1:2]                                   # :986
        sm_active = sm_active and sm_terminate != "cnn"
        if sm_active and sm_skip != "cbca":
            x0c = torch.empty((1, 4, H, W), device=dev, dtype=torch.float32)
            x1c = torch.empty((1, 4, H, W), device=dev, dtype=torch.float32)
            call("cross", x_batch[0], x0c, opt.L1, opt.tau1)                                # :995
            call("cross", x_batch[1], x1c, opt.L1, opt.tau1)                                # :996
            tmp_cbca = torch.empty_like(vol)
            for _ in range(opt.cbca_i1):                                                    # :998-1001
                call("cbca", x0c, x1c, vol, tmp_cbca, direction)
                vol.copy_(tmp_cbca)
        sm_active = sm_active and sm_terminate != "cbca1"
        if sm_active and sm_skip != "sgm":
            volt = vol.transpose(1, 2).transpose(2, 3).clone(memory_format=torch.contiguous_format)   # :1008
            out = torch.empty_like(volt)
            tmp = torch.empty((volt.size(2), volt.size(3)), device=dev, dtype=torch.float32)
            for _ in range(opt.sgm_i):
                out.zero_()
                call("sgm2", x_batch[0], x_batch[1], volt, out, tmp, opt.pi1, opt.pi2, opt.tau_so,
                     opt.alpha1, opt.sgm_q1, opt.sgm_q2, direction)                         # :1015
                volt.copy_(out).div_(4)
            vol.copy_(out.transpose(2, 3).transpose(1, 2)).div_(4)                          # :1019-1020
        sm_active = sm_active and sm_terminate != "sgm"
        if sm_active and sm_skip != "cbca":
            for _ in range(opt.cbca_i2):                                                    # :1035-1038
                call("cbca", x0c, x1c, vol, tmp_cbca, direction)
                vol.copy_(tmp_cbca)
        sm_active = sm_active and sm_terminate != "cbca2"
        out_vols[direction] = vol.clone()
        d = torch.empty((1, 1, H, W), device=dev, dtype=torch.float32)
        call("spatial_argmin", vol, d)                                                      # :1049
        disp[1 if direction == 1 else 2] = d.add_(-1)                                       # :1050
    d = disp[2]
    if opt.lr_check:                                                                        # :1054-1066
        outlier = torch.zeros_like(d)
        call("outlier_detection", disp[2], disp[1], outlier, disp_max)
        if sm_active and sm_skip != "occlusion":
            d = call("interpolate_occlusion", d, outlier)[0]
        sm_active = sm_active and sm_terminate != "occlusion"
        if sm_active and sm_skip != "occlusion":
            d = call("interpolate_mismatch", d, outlier)[0]
        sm_active = sm_active and sm_terminate != "mismatch"
    if sm_active and sm_skip != "subpixel_enchancement":
        d = call("subpixel_enchancement", d, out_vols[-1], disp_max)[0]                     # :1068
    sm_active = sm_active and sm_terminate != "subpixel_enchancement"
    if sm_active and sm_skip != "median":
        d = call("median2d", d, 5)[0]                                                       # :1073
    sm_active = sm_active and sm_terminate != "median"
    if sm_active and sm_skip != "bilateral":
        d = call("mean2d", d, refdriver.gaussian(opt.blur_sigma).to(dev), opt.blur_t)[0]    # :1078
    if want_vols:
        return d, out_vols[-1], out_vols.get(1)
    return d
