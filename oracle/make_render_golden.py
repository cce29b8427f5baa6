"""Build tests/golden/render.npz: the reference's own adcensus.grey2jet (adcensus.cu:2001-2053, through the shim build
oracle/_ref/libadcensus_ref.so) on the grey values the colour map is most sensitive to -- TEST INFRASTRUCTURE.

    python oracle/make_render_golden.py

Inputs (float64 grey, the values grey2jet multiplies by 4):
* every band boundary hit exactly, val = -0.1, 0.5, 1.5, 2.5, 3.5, 4.1, and the two float64 neighbours of each;
* a dense ramp over the whole accepted range;
* main.lua's grey of every disparity, (d + 1) / disp_max for d = 0 .. disp_max - 1, with disp_max 70 and 228.

The file holds ``grey`` (N,) and ``rgb`` (3, N), the reference's double colours.  Only in-range values are passed: the
reference asserts on the others (compiled out under -DNDEBUG, where it prints and returns black).
"""
import ctypes
import os
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))

from oracle import refdriver  # noqa: E402

OUT = os.path.join(os.path.dirname(_HERE), "tests", "golden", "render.npz")
BOUNDS = (-0.1, 0.5, 1.5, 2.5, 3.5, 4.1)


class _Tensor(ctypes.Structure):
    """the shim's tensor header (REFSHIM_TENSOR_FIELDS in oracle/refshim/refshim.h)"""
    _fields_ = [("size", ctypes.c_long * 8), ("nDimension", ctypes.c_int), ("storage", ctypes.c_void_p),
                ("refcount", ctypes.c_int), ("owns", ctypes.c_int), ("on_device", ctypes.c_int), ("elsize", ctypes.c_int)]


def _double_tensor(a):
    t = _Tensor()
    for i, n in enumerate(a.shape):
        t.size[i] = n
    t.nDimension, t.storage, t.refcount, t.owns, t.on_device, t.elsize = a.ndim, a.ctypes.data, 1, 0, 0, 8
    return t


def reference_grey2jet(grey, path=refdriver.REF_LIB):
    """adcensus.grey2jet(grey_img, col_img) of the reference on a float64 (H, W) or (N,) grey image: (3, ...) float64"""
    grey = np.ascontiguousarray(grey, dtype=np.float64)
    g2 = grey.reshape(1, -1) if grey.ndim == 1 else grey
    col = np.zeros((3,) + g2.shape, np.float64)
    shim = refdriver.ShimLibrary(path)
    l, L = shim.lib, shim.L
    l.luaT_pushudata.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_char_p]
    tg, tc = _double_tensor(g2), _double_tensor(col)
    l.shim_reset(L)
    l.luaT_pushudata(L, ctypes.addressof(tg), b"torch.DoubleTensor")
    l.luaT_pushudata(L, ctypes.addressof(tc), b"torch.DoubleTensor")
    if l.shim_call(L, b"adcensus", b"grey2jet") < 0:
        msg = l.shim_last_error(L).decode()
        l.shim_reset(L)
        raise refdriver.ShimError(msg)
    l.shim_reset(L)
    return col.reshape((3,) + grey.shape)


def inputs():
    """the float64 grey values of the fixture, in order"""
    parts = []
    for b in BOUNDS:
        v = np.array([np.nextafter(b, -np.inf), b, np.nextafter(b, np.inf)])
        v = v[(v >= -0.1) & (v <= 4.1)]
        parts.append(v / 4)                  # exact: grey * 4 gives v back
    parts.append(np.linspace(-0.1, 4.1, 4201) / 4)
    for disp_max in (70, 228):
        parts.append((np.arange(disp_max, dtype=np.float64) + 1) / disp_max)
    return np.concatenate(parts)


def main():
    grey = inputs()
    assert np.all(grey * 4 >= -0.1) and np.all(grey * 4 <= 4.1)
    rgb = reference_grey2jet(grey)
    np.savez_compressed(OUT, grey=grey, rgb=rgb)
    print("wrote %s: %d grey values" % (OUT, grey.size))


if __name__ == "__main__":
    main()
