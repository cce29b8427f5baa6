"""Host-side mirror of the reference's Lua table ``adcensus`` for the stereo hot path.

Same function names, positional arguments, in-place/returned-tensor behaviour and
error style as the lua_CFunctions registered by luaopen_libadcensus
(adcensus.cu:2061-2105); each call goes through the C ABI of
libadcensus_b200.so (include/adcensus_b200.h) with the tensors' raw device
pointers on torch's current CUDA stream.  torch is plumbing only (device memory
and streams); there is no CPU or eager fallback: if the CUDA library is missing
or a tensor is not a CUDA float tensor the call raises.

Shapes are read from the tensors exactly where the reference reads them,
e.g. StereoJoin takes C from input_L:size(2), D from
output_L:size(2).  Tensors must be contiguous (the reference silently assumes
it: raw THCudaTensor_data + sizes, strides never read).
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libadcensus_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "adcensus_b200.h")
_lib = None

# the C types include/adcensus_b200.h uses; every pointer (and adcensus_stream_t) is c_void_p
_C_TYPES = {"int": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double, "long long": ctypes.c_longlong,
            "size_t": ctypes.c_size_t, "adcensus_stream_t": ctypes.c_void_p, "void": None}


class AdcensusError(RuntimeError):
    """What luaL_error raises in the reference (adcensus.cu:31-36)."""


def _ctype(t, fn):
    """the ctypes type of C type `t`: a return type, or a parameter with its name (a pointer parameter may keep it)"""
    t = " ".join(t.replace("*", " * ").split())
    if t == "const char *":                       # adcensus_version's string
        return ctypes.c_char_p
    if "*" in t:
        return ctypes.c_void_p
    if t not in _C_TYPES:
        raise AdcensusError("%s: unsupported C type '%s' in %s" % (fn, t, os.path.basename(HEADER_PATH)))
    return _C_TYPES[t]


def prototypes(src):
    """{name: (restype, argtypes)} of every adcensus_* / mccnn_* function declared in the C header text `src`"""
    out = {}
    for decl in re.sub(r"/\*.*?\*/|^\s*#[^\n]*", " ", src, flags=re.S | re.M).split(";"):
        m = re.fullmatch(r"(.*?)\b((?:adcensus|mccnn)_\w+)\s*\((.*)\)", decl.strip(), re.S)
        if m:
            ret, fn, params = m.groups()
            params = [] if params.strip() == "void" else params.split(",")
            out[fn] = (_ctype(ret, fn), [_ctype(p if "*" in p else p.rsplit(None, 1)[0], fn) for p in params])
    return out


def lib():
    """Load libadcensus_b200.so (fails loudly if it has not been built) and type every function include/adcensus_b200.h
    declares, so that each call converts its arguments as the C prototype says."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise AdcensusError(
                "libadcensus_b200.so not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                "there is no fallback path"
            )
        if not os.path.exists(HEADER_PATH):
            raise AdcensusError("%s not found: the library's prototypes are read from it" % HEADER_PATH)
        with open(HEADER_PATH) as f:
            protos = prototypes(f.read())
        l = ctypes.CDLL(LIB_PATH)
        for fn, (restype, argtypes) in protos.items():
            getattr(l, fn).restype, getattr(l, fn).argtypes = restype, argtypes
        _lib = l
    return _lib


def version():
    return lib().adcensus_version().decode()


def num_sms():
    """the SM count the launches sized by it use on the current device (ADCENSUS_NUM_SMS when set, DESIGN §4)"""
    return lib().adcensus_num_sms()


def _check(rc, what):
    if rc == 0:
        return
    if rc > 0:
        raise AdcensusError("%s: CUDA error %d" % (what, rc))
    raise AdcensusError("%s: %s" % (what, {-1: "invalid argument", -2: "size limit exceeded", -3: "value out of range",
                                           -4: "file cannot be read"}.get(rc, "error %d" % rc)))


def _t(x, narg, name, optional=False):
    # luaT_checkudata(L, narg, "torch.CudaTensor"); optional: None passes as NULL
    if optional and x is None:
        return None
    if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.float32:
        raise AdcensusError("bad argument #%d to '%s' (torch.CudaTensor expected)" % (narg, name))
    if not x.is_contiguous():
        raise AdcensusError("bad argument #%d to '%s' (contiguous tensor expected)" % (narg, name))
    return x.data_ptr()


def _stream(x):
    return torch.cuda.current_stream(x.device).cuda_stream


def StereoJoin(input_L, input_R, output_L, output_R):
    """adcensus.StereoJoin(input_L, input_R, output_L, output_R)  adcensus.cu:1479-1498"""
    n = "StereoJoin"
    pL, pR, oL, oR = _t(input_L, 1, n), _t(input_R, 2, n), _t(output_L, 3, n), _t(output_R, 4, n)
    C, D = input_L.size(1), output_L.size(1)
    H, W = output_L.size(2), output_L.size(3)
    with torch.cuda.device(input_L.device):
        _check(lib().adcensus_StereoJoin(pL, pR, oL, oR, C, D, H, W, _stream(input_L)), n)


def cross(x0, out, L1, tau1):
    """adcensus.cross(x0, out, L1, tau1)  adcensus.cu:324-341"""
    n = "cross"
    p0, po = _t(x0, 1, n), _t(out, 2, n)
    H, W = out.size(2), out.size(3)
    with torch.cuda.device(out.device):
        _check(lib().adcensus_cross(p0, po, H, W, int(L1), tau1, _stream(out)), n)


def cbca(x0c, x1c, vol_in, vol_out, direction, max_arm=None):
    """adcensus.cbca(x0c, x1c, vol_in, vol_out, direction)  adcensus.cu:379-400

    ``max_arm`` (extension): the longest arm cross() can have produced, max(L1, 2); when given the
    call is fully asynchronous (adcensus_cbca_ex), otherwise the library reads it back once."""
    n = "cbca"
    a, b, vi, vo = _t(x0c, 1, n), _t(x1c, 2, n), _t(vol_in, 3, n), _t(vol_out, 4, n)
    D, H, W = vol_out.size(1), vol_out.size(2), vol_out.size(3)
    with torch.cuda.device(vol_out.device):
        if max_arm is None:
            _check(lib().adcensus_cbca(a, b, vi, vo, D, H, W, int(direction), _stream(vol_out)), n)
        else:
            _check(lib().adcensus_cbca_ex(a, b, vi, vo, D, H, W, int(direction), int(max_arm), _stream(vol_out)), n)


def sgm2(x0, x1, input, output, tmp, pi1, pi2, tau_so, alpha1, sgm_q1, sgm_q2, direction):
    """adcensus.sgm2(...)  adcensus.cu:620-697; input/output are (1,H,W,D)"""
    n = "sgm2"
    p0, p1, pi, po = _t(x0, 1, n), _t(x1, 2, n), _t(input, 3, n), _t(output, 4, n)
    pt = _t(tmp, 5, n, optional=True)
    H, W, D = input.size(1), input.size(2), input.size(3)
    with torch.cuda.device(input.device):
        _check(lib().adcensus_sgm2(p0, p1, pi, po, pt, H, W, D, pi1, pi2, tau_so, alpha1,
                                   sgm_q1, sgm_q2, int(direction), _stream(input)), n)


def outlier_detection(d0, d1, outlier, disp_max):
    """adcensus.outlier_detection(d0, d1, outlier, disp_max)  adcensus.cu:901-918"""
    n = "outlier_detection"
    a, b, o = _t(d0, 1, n), _t(d1, 2, n), _t(outlier, 3, n)
    H, W = d0.size(-2), d0.size(-1)
    with torch.cuda.device(d0.device):
        _check(lib().adcensus_outlier_detection(a, b, o, H, W, int(disp_max), _stream(d0)), n)


def interpolate_occlusion(d0, outlier):
    """adcensus.interpolate_occlusion(d0, outlier) -> new tensor  adcensus.cu:1107-1125"""
    n = "interpolate_occlusion"
    a, b = _t(d0, 1, n), _t(outlier, 2, n)
    out = torch.empty_like(d0)  # new_tensor_like, adcensus.cu:40-45
    with torch.cuda.device(d0.device):
        _check(lib().adcensus_interpolate_occlusion(a, b, _t(out, 0, n), d0.size(-2), d0.size(-1), _stream(d0)), n)
    return out


def interpolate_mismatch(d0, outlier):
    """adcensus.interpolate_mismatch(d0, outlier) -> new tensor  adcensus.cu:1060-1077"""
    n = "interpolate_mismatch"
    a, b = _t(d0, 1, n), _t(outlier, 2, n)
    out = torch.empty_like(d0)
    with torch.cuda.device(d0.device):
        _check(lib().adcensus_interpolate_mismatch(a, b, _t(out, 0, n), d0.size(-2), d0.size(-1), _stream(d0)), n)
    return out


def subpixel_enchancement(d0, c2, disp_max):
    """adcensus.subpixel_enchancement(d0, c2, disp_max) -> new tensor  adcensus.cu:1222-1239"""
    n = "subpixel_enchancement"
    a, b = _t(d0, 1, n), _t(c2, 2, n)
    out = torch.empty_like(d0)
    with torch.cuda.device(d0.device):
        _check(lib().adcensus_subpixel_enchancement(a, b, _t(out, 0, n), d0.size(-2), d0.size(-1), int(disp_max),
                                                    _stream(d0)), n)
    return out


def median2d(img, kernel_size):
    """adcensus.median2d(img, kernel_size) -> new tensor  adcensus.cu:1596-1613"""
    n = "median2d"
    a = _t(img, 1, n)
    out = torch.empty_like(img)
    with torch.cuda.device(img.device):
        _check(lib().adcensus_median2d(a, _t(out, 0, n), img.size(-2), img.size(-1), int(kernel_size), _stream(img)), n)
    return out


def mean2d(img, kernel, alpha2):
    """adcensus.mean2d(img, kernel, alpha2) -> new tensor  adcensus.cu:1263-1282"""
    n = "mean2d"
    a, k = _t(img, 1, n), _t(kernel, 2, n)
    out = torch.empty_like(img)
    with torch.cuda.device(img.device):
        _check(lib().adcensus_mean2d(a, k, _t(out, 0, n), img.size(-2), img.size(-1), kernel.size(0), alpha2,
                                     _stream(img)), n)
    return out


def Normalize_forward(input, norm, output):
    """adcensus.Normalize_forward(input, norm, output)  adcensus.cu:1310-1333"""
    n = "Normalize_forward"
    a, b, c = _t(input, 1, n), _t(norm, 2, n), _t(output, 3, n)
    N, C, H, W = input.shape
    with torch.cuda.device(input.device):
        _check(lib().adcensus_Normalize_forward(a, b, c, N, C, H, W, _stream(input)), n)


def spatial_argmin(input, output):
    """adcensus.spatial_argmin(input, output)  adcensus.cu:264-278 (1-based)"""
    n = "spatial_argmin"
    a, b = _t(input, 1, n), _t(output, 2, n)
    N, D = input.size(0), input.size(1)
    HW = input.size(2) * input.size(3)
    with torch.cuda.device(input.device):
        _check(lib().adcensus_spatial_argmin(a, b, N, D, HW, _stream(input)), n)


def ad(x0, x1, out, direction):
    """adcensus.ad(x0, x1, out, direction)  adcensus.cu:95-114"""
    n = "ad"
    a, b, o = _t(x0, 1, n), _t(x1, 2, n), _t(out, 3, n)
    with torch.cuda.device(out.device):
        _check(lib().adcensus_ad(a, b, o, out.size(1), out.size(2), out.size(3), int(direction), _stream(out)), n)


def census(x0, x1, out, direction):
    """adcensus.census(x0, x1, out, direction)  adcensus.cu:155-175"""
    n = "census"
    a, b, o = _t(x0, 1, n), _t(x1, 2, n), _t(out, 3, n)
    with torch.cuda.device(out.device):
        _check(lib().adcensus_census(a, b, o, out.size(1), x0.size(1), out.size(2), out.size(3), int(direction),
                                     _stream(out)), n)


# ---- label cleaning of preprocess_kitti.lua (not in the Lua face yet) --------

def _stack_shape(y):
    """(N, H, W) of a disparity stack: W = the last size (the reference's size(3) of an (n,1,H,W) tensor), H the one before"""
    W = y.size(-1) if y.dim() else 1
    H = y.size(-2) if y.dim() >= 2 else 1
    return y.numel() // max(1, H * W), H, W


def remove_nonvisible(y):
    """adcensus.remove_nonvisible(y)  adcensus.cu:1735-1745: in place, y >= x (the column index) -> 0"""
    n = "remove_nonvisible"
    p = _t(y, 1, n)
    if y.numel():
        with torch.cuda.device(y.device):
            _check(lib().adcensus_remove_nonvisible(p, *_stack_shape(y), _stream(y)), n)


def remove_occluded(y):
    """adcensus.remove_occluded(y)  adcensus.cu:1761-1771: in place; bit-identical to the reference for maps in readPNG16's
    domain (see adcensus_remove_occluded in include/adcensus_b200.h)"""
    n = "remove_occluded"
    p = _t(y, 1, n)
    if y.numel():
        with torch.cuda.device(y.device):
            _check(lib().adcensus_remove_occluded(p, *_stack_shape(y), _stream(y)), n)


def remove_white(x, y):
    """adcensus.remove_white(x, y)  adcensus.cu:1784-1796: in place, y -> 0 where x == 255"""
    n = "remove_white"
    px, py = _t(x, 1, n), _t(y, 2, n)
    if x.numel() != y.numel():
        raise AdcensusError("bad argument #1 to '%s' (%d elements, y has %d)" % (n, x.numel(), y.numel()))
    if x.device != y.device:
        raise AdcensusError("bad argument #1 to '%s' (on %s, y on %s)" % (n, x.device, y.device))
    if y.numel():
        with torch.cuda.device(y.device):
            _check(lib().adcensus_remove_white(px, py, *_stack_shape(y), _stream(y)), n)


# ---- the Lua-side tensor ops of stereo_predict ------------------------------

def fill_nan(t):
    """vols:fill(0/0)  main.lua:946"""
    with torch.cuda.device(t.device):
        _check(lib().mccnn_fill_nan(_t(t, 1, "fill_nan"), t.numel(), _stream(t)), "fill_nan")


def fix_border(vol, n, direction):
    """fix_border(net, vol, direction)  main.lua:922-927 with n = (window-1)/2"""
    with torch.cuda.device(vol.device):
        _check(lib().mccnn_fix_border(_t(vol, 1, "fix_border"), vol.size(1), vol.size(2), vol.size(3), int(n),
                                      int(direction), _stream(vol)), "fix_border")


def transpose_dhw_to_hwd(vol):
    """vol:transpose(2,3):transpose(3,4):clone()  main.lua:1008"""
    _, D, H, W = vol.shape
    out = torch.empty((1, H, W, D), device=vol.device, dtype=torch.float32)
    with torch.cuda.device(vol.device):
        _check(lib().mccnn_transpose_dhw_to_hwd(_t(vol, 1, "transpose"), _t(out, 0, "transpose"), D, H, W, _stream(vol)),
               "transpose_dhw_to_hwd")
    return out


def transpose_hwd_to_dhw_div4(out_hwd):
    """vol:copy(out:transpose(3,4):transpose(2,3)):div(4)  main.lua:1020"""
    _, H, W, D = out_hwd.shape
    vol = torch.empty((1, D, H, W), device=out_hwd.device, dtype=torch.float32)
    with torch.cuda.device(vol.device):
        _check(lib().mccnn_transpose_hwd_to_dhw_div4(_t(out_hwd, 1, "transpose"), _t(vol, 0, "transpose"), D, H, W,
                                                     _stream(vol)), "transpose_hwd_to_dhw_div4")
    return vol


def argmin(vol):
    """_, d = torch.min(vol, 2); d:cuda():add(-1)  main.lua:1049-1050"""
    _, D, H, W = vol.shape
    out = torch.empty((1, 1, H, W), device=vol.device, dtype=torch.float32)
    with torch.cuda.device(vol.device):
        _check(lib().mccnn_argmin(_t(vol, 1, "argmin"), _t(out, 0, "argmin"), D, H * W, _stream(vol)), "argmin")
    return out


def gaussian(sigma):
    """gaussian(sigma)  main.lua:528-540 (host tensor, float32)"""
    l = lib()
    ks = l.mccnn_gaussian(sigma, None)
    out = torch.empty((ks, ks), dtype=torch.float32)
    l.mccnn_gaussian(sigma, out.data_ptr())
    return out
