"""CPU: the C-ABI shared library builds, loads, and exports every symbol that
include/adcensus_b200.h declares; the host-side mirror exposes every hot-path name of the
reference's funcs[] table (adcensus.cu:2061-2096).  No compute calls (no GPU here)."""
import ctypes
import os
import re

import pytest

import mccnn_b200
from mccnn_b200 import adcensus, pipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    mccnn_b200.build()
    return adcensus.lib()


def declared_functions():
    src = open(os.path.join(ROOT, "include", "adcensus_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b((?:adcensus|mccnn)_[A-Za-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(lib):
    names = declared_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), "libadcensus_b200.so does not export %s" % n


C_TYPES = {"int": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double, "long long": ctypes.c_longlong,
           "size_t": ctypes.c_size_t, "adcensus_stream_t": ctypes.c_void_p, "void": None, "const char *": ctypes.c_char_p}


def test_loader_types_every_declared_function(lib):
    """the loader types exactly the functions the header declares, each as the header's prototype reads"""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "adcensus_b200.h")).read(), flags=re.S)
    names = declared_functions()
    assert sorted(adcensus.prototypes(src)) == names
    for n in names:
        ret, params = re.search(r"([\w ]+?\s*\**)\s*\b%s\s*\(([^)]*)\)" % n, src).groups()
        want = [ctypes.c_void_p if "*" in q else C_TYPES[q.rsplit(None, 1)[0].strip()]
                for q in params.split(",") if q.strip() != "void"]
        fn = getattr(lib, n)
        assert fn.restype is C_TYPES[ret.strip()], n
        assert fn.argtypes == want, n


def test_loader_prototypes_pinned(lib):
    """a few prototypes written out, so that a parser bug cannot pass by agreeing with itself"""
    f, i, p = ctypes.c_float, ctypes.c_int, ctypes.c_void_p
    assert lib.adcensus_sgm2.argtypes == [p] * 5 + [i] * 3 + [f] * 6 + [i, p]
    assert lib.adcensus_sgm2.restype is i
    assert lib.mccnn_trainer_run.argtypes == [p, p, i, ctypes.c_double, p]
    assert lib.mccnn_trainer_size.restype is ctypes.c_longlong
    assert lib.mccnn_packed_hv_bytes.restype is ctypes.c_size_t
    assert lib.mccnn_sgm_tables_bytes.restype is ctypes.c_size_t
    assert lib.mccnn_fill_nan.argtypes == [p, ctypes.c_size_t, p]
    assert lib.mccnn_pipeline_destroy.restype is None
    assert lib.adcensus_version.restype is ctypes.c_char_p and lib.adcensus_version.argtypes == []
    assert lib.adcensus_num_sms.restype is i and lib.adcensus_num_sms.argtypes == []
    assert lib.mccnn_mb_sample_starts.argtypes == [p, ctypes.c_longlong, i, ctypes.c_double, p, ctypes.c_longlong, p, p]


def test_loader_refuses_unsupported_types():
    with pytest.raises(adcensus.AdcensusError, match="mccnn_x: unsupported C type 'short'"):
        adcensus.prototypes("/* int mccnn_y(int a); */\nint mccnn_x(int a,\n            short b);\n")
    with pytest.raises(adcensus.AdcensusError, match="adcensus_u: unsupported C type 'unsigned'"):
        adcensus.prototypes("unsigned adcensus_u(void);")
    got = adcensus.prototypes("/* int mccnn_y(float a); */\n#define X(a) a\nvoid mccnn_z(const float *const *a,\n  long long n);")
    assert got == {"mccnn_z": (None, [ctypes.c_void_p, ctypes.c_longlong])}


def test_version(lib):
    assert "sm_90a" in adcensus.version()


HOT_PATH_LUA_NAMES = ["StereoJoin", "cross", "cbca", "sgm2", "outlier_detection", "interpolate_occlusion",
                      "interpolate_mismatch", "subpixel_enchancement", "median2d", "mean2d", "Normalize_forward",
                      "spatial_argmin", "ad", "census"]


def test_python_mirror_has_reference_names():
    for n in HOT_PATH_LUA_NAMES:
        assert callable(getattr(adcensus, n)), n


def test_bad_arguments_are_rejected_without_a_gpu(lib):
    # null pointers / bad sizes return ADCENSUS_EINVAL before any CUDA call
    assert lib.adcensus_StereoJoin(None, None, None, None, 64, 16, 64, 128, None) == -1
    assert lib.adcensus_cross(None, None, 4, 4, 5, ctypes.c_float(0.1), None) == -1
    one = ctypes.c_void_p(16)
    assert lib.adcensus_StereoJoin(one, one, one, one, 129, 16, 64, 128, None) == -2      # C > 128
    assert lib.adcensus_sgm2(one, one, one, ctypes.c_void_p(32), None, 4, 8, 513, ctypes.c_float(1), ctypes.c_float(1),
                             ctypes.c_float(1), ctypes.c_float(1), ctypes.c_float(1), ctypes.c_float(1), 1, None) == -2
    assert lib.adcensus_median2d(one, one, 4, 4, 13, None) == -2
    assert lib.adcensus_median2d(one, one, 4, 4, 4, None) == -1                            # even kernel
    assert lib.adcensus_cbca(one, one, one, one, 4, 4, 4, 1, None) == -1                   # in aliases out


def test_round2_entry_points_reject_bad_arguments_without_a_gpu(lib):
    """scorer head / feature tower / batch call: EINVAL (-1) for null or nonsensical arguments, ELIMIT (-2) for shapes the
    kernels are not built for -- all decided before the first CUDA call"""
    h = ctypes.c_void_p()
    arr = (ctypes.c_void_p * 5)(*[16] * 5)
    sh = lambda fm, nh2, l2, W=arr, b=arr: lib.mccnn_scorer_head_create(ctypes.byref(h), fm, nh2, l2, W, b, 0, None)
    assert sh(112, 384, 3, None) == -1 and sh(112, 384, 3, arr, None) == -1
    assert lib.mccnn_scorer_head_create(None, 112, 384, 3, arr, arr, 0, None) == -1
    assert sh(112, 384, 0) == -1 and sh(4, 384, 3) == -1 and sh(112, 64, 3) == -1
    assert sh(112, 200, 3) == -2                                   # nh2 must be a multiple of 128
    assert sh(108, 384, 3) == -2                                   # fm must be a multiple of 8
    assert sh(112, 384, 9) == -2                                   # more hidden layers than the kernel unrolls
    assert h.value is None
    ft = lambda n_in, fm, l1, W=arr, b=arr: lib.mccnn_feature_tower_create(ctypes.byref(h), n_in, fm, l1, 0, 1, W, b, 0, None)
    assert ft(1, 64, 4, None) == -1 and ft(2, 64, 4) == -1 and ft(1, 64, 0) == -1 and ft(1, 4, 4) == -1
    assert ft(1, 72, 4) == -2                                      # fm must be a multiple of 16
    assert ft(1, 64, 40) == -2
    assert h.value is None
    assert lib.mccnn_scorer_head_forward(None, arr, arr, arr, arr, 4, 4, 4, 3, None) == -1
    assert lib.mccnn_feature_tower_forward(None, arr, arr, 2, 4, 4, 3, None) == -1
    assert lib.mccnn_pipeline_run_batch(None, 1, arr, arr, arr, arr, arr, None) == -1


def test_trainer_create_checks_every_limit_without_a_gpu(lib):
    """mccnn_trainer_create: EINVAL (-1) for the scalars, then the pair table, then ELIMIT (-2), one rule at a time -- all
    decided before the first CUDA call, with *h NULL after the refusal"""
    import numpy as np

    from mccnn_b200 import train

    fast = dict(slow=0, l1=4, fm=64, bs=128, mom=0.9, margin=0.2, pow=1, chunk=256, loss_cap=1, rank=0, world=1)
    slow = dict(slow=1, l1=4, fm=112, bs=128, mom=0.9, l2=4, nh2=384, chunk=256, loss_cap=1, rank=0, world=1)
    good = np.zeros(2, train.PAIR_DTYPE)
    good["x0"], good["x1"], good["H"], good["W"] = 1 << 20, 1 << 21, 350, 1242

    def create(base, table=good, n=None, **kw):
        h = ctypes.c_void_p(16)
        cfg = train.TrainerConfig(**dict(base, **kw))
        rc = lib.mccnn_trainer_create(ctypes.byref(h), ctypes.byref(cfg), table.ctypes.data_as(ctypes.c_void_p),
                                      len(table) if n is None else n, -1, None)
        assert h.value is None, (base["slow"], kw)
        return rc

    def pairs(**kw):
        t = good.copy()
        for k, v in kw.items():
            t[k][1] = v
        return t

    # the valid ones pass every check and reach CUDA, which refuses device -1
    for base in (fast, slow):
        assert create(base) > 0 and create(base, rank=1, world=2) > 0 and create(base, world=256) > 0
    cfg = train.TrainerConfig(**fast)
    assert lib.mccnn_trainer_create(None, ctypes.byref(cfg), good.ctypes.data_as(ctypes.c_void_p), 2, -1, None) == -1
    h = ctypes.c_void_p(16)
    assert lib.mccnn_trainer_create(ctypes.byref(h), None, good.ctypes.data_as(ctypes.c_void_p), 2, -1, None) == -1
    assert h.value is None
    for base in (fast, slow):
        for kw in (dict(slow=2), dict(l1=0), dict(fm=0), dict(bs=0), dict(bs=1), dict(bs=3), dict(chunk=0),
                   dict(loss_cap=0), dict(world=0), dict(world=3), dict(world=6, rank=1), dict(rank=-1),
                   dict(rank=1), dict(world=4, rank=4)):
            assert create(base, **kw) == -1, kw
        assert create(base, n=0) == -1
        for t in (pairs(x0=0), pairs(x1=0), pairs(H=0), pairs(W=0)):
            assert create(base, t) == -1
        assert create(base, pairs(H=40000)) == -2 and create(base, pairs(W=40000)) == -2
        for kw in (dict(l1=9), dict(fm=129), dict(world=512, bs=512), dict(world=8, bs=2)):
            assert create(base, **kw) == -2, kw
        assert create(base, pairs(W=40000), fm=0) == -1                   # the scalars before the table
        assert create(base, pairs(H=0), l1=9) == -1                       # the table before the limits
    for kw in (dict(pow=0), dict(pow=3)):
        assert create(fast, **kw) == -1, kw
        assert create(slow, **kw) > 0, kw                                 # read only for 'fast'
    for kw in (dict(l2=0), dict(nh2=0)):
        assert create(slow, **kw) == -1, kw
        assert create(fast, **kw) > 0, kw                                 # read only for 'slow'
    for kw in (dict(fm=120), dict(l2=5), dict(nh2=200), dict(fm=128, l1=8, bs=29028)):
        assert create(slow, **kw) == -2, kw
        assert create(fast, **kw) > 0, kw
    assert create(slow, fm=128, l1=8, bs=29026) > 0                       # 2 bs fm ws^2 just under 2^31


def test_trainer_config_mirrors_the_header():
    from mccnn_b200 import train

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "adcensus_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\} mccnn_trainer_config;", src).group(1)
    want = []
    for decl in body.split(";"):
        if decl.strip():
            ctype, names = decl.split(None, 1)
            want += [(n.strip(), {"int": ctypes.c_int, "float": ctypes.c_float}[ctype]) for n in names.split(",")]
    assert train.TrainerConfig._fields_ == want


def test_python_mirror_type_errors():
    import torch

    with pytest.raises(adcensus.AdcensusError, match="torch.CudaTensor expected"):
        adcensus.StereoJoin(torch.zeros(1, 2, 3, 4), torch.zeros(1, 2, 3, 4), torch.zeros(1, 2, 3, 4), torch.zeros(1, 2, 3, 4))


def test_presets_match_main_lua():
    p = pipeline.make_params("kitti", "fast")
    assert (p.L1, p.cbca_i1, p.cbca_i2, p.sgm_i) == (0, 0, 0, 1)
    assert abs(p.pi2 - 55.72) < 1e-5 and abs(p.blur_sigma - 7.74) < 1e-12
    p = pipeline.make_params("mb", "slow")
    assert (p.L1, p.cbca_i2, p.lr_check, p.border) == (14, 16, 0, 5)


def test_gaussian_host_helper(lib):
    from oracle import oracle as orc

    import numpy as np

    for s in (0.5, 1.67, 5.99, 7.74):
        assert np.array_equal(adcensus.gaussian(s).numpy(), orc.gaussian(s))
