"""CPU: the cases of tests/test_gpu_map_edges.py land on the edges they claim and reach every edge between them, and the
tracker's sums are order-sensitive on the cases' data.  The size rules are tests/map_edge_cases.py's restatement of
csrc/tsdf.cu, csrc/keysort.cuh and csrc/track.cu; the data edges (unique keys, table sizes) and the sums come from the
numpy oracles, so a kernel that reordered a sum or dropped a run of a grid-stride loop would not pass the GPU test."""
import importlib.util
import math
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tests", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mc = _load("map_edge_cases")
to = _load("tsdf_oracle")
po = _load("track_photometric_oracle")
tro = po.track_oracle
COS30 = math.cos(math.radians(30.0))


# ------------------------------------------------------------------------------------------------------------ the rules

def test_size_rules():
    assert [mc.nblk(mc.points(H, W, K)) for H, W, K in ((32, 64, 1), (32, 65, 1), (1, 1, 1), (375, 1242, 2), (96, 320, 64))] \
        == [3, 4, 1, 1138, 1935]
    assert [mc.scan_per(n) for n in (1, 1024, 1025, 1138, 1935, 2048, 2049)] == [1, 1, 2, 2, 2, 2, 3]
    assert [mc.grid_cap(s) for s in mc.H100_SMS] == [270336, 233472]
    for s in mc.H100_SMS:
        cap = mc.grid_cap(s)
        assert mc.grid_for(cap, s) == s * 8 and not mc.wraps(cap, s) and mc.wraps(cap + 1, s)
        assert mc.grid_for(1, s) == 1 and mc.grid_for(0, s) == 1
    assert [mc.hash_bits(n) for n in (0, 1, 512, 513, 1024, 1025)] == [10, 10, 10, 11, 11, 12]
    assert mc.K_of(0.125, 32.0) == 64 and mc.K_of(*mc.K65) == 65 and mc.K65[1] > 32.0
    assert mc.K_of(*mc.K65) == to.K_of(*mc.K65)
    # the tracker's levels at KITTI size: chunks 455/115/29, padded to 512/128/32, last chunks of 854, 12 and 562 pixels
    H, W = mc.KITTI_H, mc.KITTI_W
    assert [mc.level_shape(H, W, l) for l in range(3)] == [(375, 1242), (188, 621), (94, 311)]
    assert [mc.chunks(H, W, l) for l in range(3)] == [455, 115, 29]
    assert [mc.pad(mc.chunks(H, W, l)) for l in range(3)] == [512, 128, 32]
    assert [mc.last_chunk(H, W, l) for l in range(3)] == [854, 12, 562]
    assert [mc.normal_sites(3, 7, l) for l in range(3)] == [12, 3, 0]
    assert [mc.photo_sites(40, 12, l) for l in range(3)] == [333, 51, 0]


# ------------------------------------------------------------------------------------------------------------- coverage

def _tsdf_data(case):
    """(largest unique-key count of one frame, [table bricks before frame 2 .., after the last]) by the oracle's allocation"""
    keys, U, table = np.zeros(0, np.uint64), [], []
    for d, cal, _, P in mc.tsdf_frames(case):
        if len(keys):
            table.append(len(keys))
        fk, _, _ = to.alloc_keys(d, cal, P, case.voxel, case.trunc)
        U.append(len(fk))
        keys = np.union1d(keys, fk)
    return max(U), table + [len(keys)]


_DATA = {}


def tsdf_edges(case, sms):
    if case.name not in _DATA:
        _DATA[case.name] = _tsdf_data(case)
    U, table = _DATA[case.name]
    return mc.tsdf_size_edges(case) | mc.tsdf_data_edges(U, table, sms)


@pytest.mark.parametrize("sms", mc.H100_SMS)
@pytest.mark.parametrize("case", mc.TSDF_CASES, ids=mc.case_id)
def test_tsdf_case_hits_its_edges(case, sms):
    e = tsdf_edges(case, sms)
    print("%s on %d SMs: %s" % (case.name, sms, sorted(e)))
    assert set(case.edges) <= e, "%s misses %s" % (case.name, set(case.edges) - e)
    assert case.H * case.W * (2 * mc.K_of(case.voxel, case.trunc) + 1) < 1 << 31 and mc.K_of(case.voxel, case.trunc) <= mc.MAX_K


@pytest.mark.parametrize("sms", mc.H100_SMS)
def test_tsdf_cases_reach_every_edge(sms):
    reached = set().union(*(tsdf_edges(c, sms) for c in mc.TSDF_CASES))
    assert mc.TSDF_EDGES <= reached, mc.TSDF_EDGES - reached


@pytest.mark.parametrize("case", mc.TRACK_CASES, ids=mc.case_id)
def test_track_case_hits_its_edges(case):
    e = mc.track_edges(case)
    print("%s: %s" % (case.name, sorted(e)))
    assert set(case.edges) <= e, "%s misses %s" % (case.name, set(case.edges) - e)


def test_track_cases_reach_every_edge():
    reached = set().union(*(mc.track_edges(c) for c in mc.TRACK_CASES))
    assert mc.TRACK_EDGES <= reached, mc.TRACK_EDGES - reached


# ------------------------------------------------------------------------------------------------------------ the teeth

def _halve(a):
    return tro.halve(a)


def seq_chunks(t):
    """each chunk summed in pixel order, the chunk sums by the tree"""
    n = len(t)
    nch = max(1, -(-n // tro.CHUNK))
    a = np.zeros((nch * tro.CHUNK, t.shape[1]))
    a[:n] = t
    a = a.reshape(nch, tro.CHUNK, -1)
    s = np.zeros((nch, t.shape[1]))
    for i in range(tro.CHUNK):
        s = s + a[:, i]
    b = np.zeros((mc.pad(nch), t.shape[1]))
    b[:nch] = s
    return _halve(b[None])[0]


def _chunk_sums(t, chunk=tro.CHUNK):
    n = len(t)
    nch = max(1, -(-n // chunk))
    a = np.zeros((nch * chunk, t.shape[1]))
    a[:n] = t
    return _halve(a.reshape(nch, chunk, -1))


def seq_chunk_sums(t):
    """the tree inside each chunk, the chunk sums added in chunk order"""
    c = _chunk_sums(t)
    s = np.zeros(t.shape[1])
    for row in c:
        s = s + row
    return s


def pad_to_n(t):
    """the chunk sums halved without padding: a[i] += a[i + ceil(k / 2)] over the k left"""
    a = _chunk_sums(t)
    while len(a) > 1:
        h = -(-len(a) // 2)
        b = a[:h].copy()
        b[:len(a) - h] += a[h:]
        a = b
    return a[0]


def chunks_of(size):
    return lambda t: tro.tree_sum(t) if size == tro.CHUNK else _halve(np.concatenate(
        [_chunk_sums(t, size), np.zeros((mc.pad(len(_chunk_sums(t, size))) - len(_chunk_sums(t, size)), t.shape[1]))])[None])[0]


def _differs(a, b):
    return bool((np.asarray(a).view(np.uint64) != np.asarray(b).view(np.uint64)).any())


SUM_CASES = [c for c in mc.TRACK_CASES if c.H * c.W >= 1024]


@pytest.mark.parametrize("case", SUM_CASES, ids=mc.case_id)
def test_sums_are_order_sensitive(case):
    """on the case's data at the true pose, each other order of the sums gives other bits than the oracle's tree, geometric
    and photometric, at every level where that order is a different tree"""
    cal, disp, Zm, img, ref_img, T = mc.track_frame(case)
    src, mod = tro.source_pyramid(disp, cal), tro.model_pyramid(Zm, cal)
    isrc, iref = po.pyramid(img), po.pyramid(ref_img)
    p12 = T[:3].reshape(12)
    for level in range(mc.LEVELS):
        tg, okg = tro.terms(src, mod, cal, level, p12, 0.5, COS30)
        tp, okp = po.photometric_terms(src, mod, isrc, iref, cal, level, p12, 0.5, 2.0, 30.0)
        n = mc.chunks(case.H, case.W, level)
        for kind, t, ok in (("geometric", tg, okg), ("photometric", tp, okp)):
            if ok.sum() < 3:
                continue
            want = tro.tree_sum(t)
            what = "%s level %d %s (%d terms)" % (case.name, level, kind, int(ok.sum()))
            assert _differs(seq_chunks(t), want), what + ": sequential inside a chunk"
            if np.prod(mc.level_shape(case.H, case.W, level)) > 512:      # else the first halving only adds +0.0
                assert _differs(chunks_of(512)(t), want), what + ": chunks of 512"
            if n > 4:                          # with 3 or 4 chunk sums another order can round alike
                assert _differs(seq_chunk_sums(t), want), what + ": chunk sums in order"
            if n != mc.pad(n) and n > 4:
                assert _differs(pad_to_n(t), want), what + ": chunk sums padded to n"
