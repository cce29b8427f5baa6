"""Generate tests/golden/preprocess_mb/*.npz: what preprocess_mb.py's OWN read_im, load_pfm and save_pfm compute, under
OpenCV and numpy.

Needs the reference tree (for preprocess_mb.py) and OpenCV (cv2).  Run once where both exist; the fixtures are committed:

    python oracle/make_mb_golden.py REFERENCE_DIR [OUT_DIR]

The three functions are taken out of preprocess_mb.py with ``ast`` at generation time and run unmodified, with the Python 3
shims described in tests/golden/preprocess_mb/README.md.  Inputs: seeded RGB PNG, PPM and grey PGM / PNG files (the grey
one holds every byte value), and little-endian PFMs with inf, -inf, NaN and exact ties inside 2x2 blocks.  Outputs:
read_im(.., False) for color = gray and rgb, load_pfm(.., False), load_pfm(.., True) and the .H.pfm file save_pfm wrote.
"""
import ast
import io
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Py2Reader(io.BufferedReader):
    """open(fname) of Python 2: readline returns str; the data stays binary for np.fromfile"""

    def readline(self, *a):
        return super().readline(*a).decode("latin-1")


class _Py2Writer(io.BufferedWriter):
    def write(self, s):
        return super().write(s.encode("latin-1") if isinstance(s, str) else s)


def _py2_open(fname, mode="r"):
    if "w" in mode:
        return _Py2Writer(io.FileIO(fname, "w"))
    return _Py2Reader(io.FileIO(fname, "r"))


def script_functions(reference_dir):
    """read_im, load_pfm and save_pfm of preprocess_mb.py, compiled from its source, in a namespace whose global `color`
    the caller sets"""
    import cv2

    path = os.path.join(reference_dir, "preprocess_mb.py")
    tree = ast.parse(open(path).read(), path)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("read_im", "load_pfm", "save_pfm")]
    assert len(keep) == 3, "preprocess_mb.py: read_im, load_pfm and save_pfm not all found"
    ns = dict(os=os, re=re, sys=sys, np=np, cv2=cv2, subprocess=subprocess, open=_py2_open, color="gray")
    exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
    return ns


def image_cases(rng):
    """name -> (file suffix, array for PIL): shapes cross numpy's pairwise block edges (128 elements and the splits)"""
    from mccnn_b200 import synth

    v = synth.natural_image(rng, 61, 97)
    smooth = np.clip(np.rint(128 + 50 * v), 0, 255)
    rgb = np.stack([smooth * t for t in (0.9, 1.0, 1.1)], 2) + rng.integers(-20, 21, (61, 97, 3))
    grey = rng.permutation(np.arange(256).repeat(3))[:43 * 17].reshape(43, 17)
    return {
        "rgb_png_61x97": (".png", np.clip(rgb, 0, 255).astype(np.uint8)),
        "rgb_ppm_13x11": (".ppm", rng.integers(0, 256, (13, 11, 3)).astype(np.uint8)),
        "rgb_png_2x3": (".png", rng.integers(0, 256, (2, 3, 3)).astype(np.uint8)),
        "grey_pgm_43x17": (".pgm", grey.astype(np.uint8)),
        "grey_png_16x16": (".png", np.arange(256).reshape(16, 16).astype(np.uint8)),
    }


def pfm_cases(rng):
    a = rng.uniform(0, 60, (10, 14)).astype(np.float32)
    a[0, 0:2] = a[1, 0:2] = np.float32(7.25)                        # a block of four ties
    a[2, 2], a[3, 3] = np.float32(3.5), np.float32(3.5)             # ties on the diagonal
    a[0, 4], a[1, 5] = np.inf, np.inf
    a[2, 4] = np.nan
    a[0, 6], a[0, 7], a[1, 6] = np.nan, np.nan, np.inf
    a[2, 6:8] = a[3, 6:8] = np.inf
    a[4, 0], a[5, 1] = -np.inf, np.nan
    a[4, 2:4] = a[5, 2:4] = np.nan
    a[6, 0] = np.float32(1e-45)                                     # a subnormal: x / 2 rounds
    b = rng.uniform(0, 200, (36, 50)).astype(np.float32)
    b[rng.random(b.shape) < 0.2] = np.inf
    return {"special_10x14": a, "random_36x50": b}


def main(reference_dir, out_dir):
    from PIL import Image

    from mccnn_b200 import dataio

    rng = np.random.default_rng(2025)
    ns = script_functions(reference_dir)
    os.makedirs(out_dir, exist_ok=True)
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, (suffix, arr) in image_cases(rng).items():
            p = os.path.join(tmp, name + suffix)
            Image.fromarray(arr).save(p)
            res[name + "/file"] = np.frombuffer(open(p, "rb").read(), np.uint8)
            for color in ("gray", "rgb"):
                ns["color"] = color
                res[name + "/" + color] = ns["read_im"](p, False)
        np.savez_compressed(os.path.join(out_dir, "read_im.npz"), **res)
        res = {}
        for name, a in pfm_cases(rng).items():
            p = os.path.join(tmp, name + ".pfm")
            dataio.write_pfm(a, p)                                  # file order: rows as given
            res[name + "/file"] = np.frombuffer(open(p, "rb").read(), np.uint8)
            res[name + "/load"] = ns["load_pfm"](p, False)[0]
            res[name + "/half"] = ns["load_pfm"](p, True)[0]
            res[name + "/half_file"] = np.frombuffer(open(p + ".H.pfm", "rb").read(), np.uint8)
            res[name + "/half_cached"] = ns["load_pfm"](p, True)[0]
        np.savez_compressed(os.path.join(out_dir, "pfm.npz"), **res)
    print("wrote", out_dir)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    import mccnn_b200  # noqa: F401

    if len(sys.argv) < 2:
        raise SystemExit("usage: make_mb_golden.py REFERENCE_DIR [OUT_DIR]")
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "tests", "golden", "preprocess_mb"))
