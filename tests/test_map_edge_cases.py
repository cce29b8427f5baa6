"""CPU: the cases of tests/test_gpu_map_edges.py land on the edges they claim and reach every edge between them, and the
tracker's sums are order-sensitive on the cases' data.  The size rules are tests/map_edge_cases.py's restatement of
csrc/tsdf.cu, csrc/keysort.cuh and csrc/track.cu; the data edges (unique keys, table sizes) and the sums come from the
numpy oracles, so a kernel that reordered a sum or dropped a run of a grid-stride loop would not pass the GPU test."""
import importlib.util
import math
import os
import re

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


# ------------------------------------------------------------------------------------------ launches sized by the SM count

CSRC = os.path.join(ROOT, "mc-cnn_b200", "csrc")
# the name a file launches its SM-capped grids by: its helper, or the variable its use of adc_num_sms sets
CAPPED_GRID = {"keysort.cuh": r"grid_for\(", "fusion.cu": r"grid_for\(", "tsdf.cu": r"grid_for\(",
               "depth.cu": r"grid_for\(", "render.cu": r"grid_for\(", "kitti_eval.cu": r"grid_for\(",
               "preprocess.cu": r"elementwise_grid\(", "preprocess_mb.cu": r"elementwise_grid\(",
               "rectify.cu": r"dim3\(grid, 2\)$", "frontend.cu": r"grid$", "post.cu": r"blocks$",
               "confidence.cu": r"(sel_blocks\(|blocks$)", "feature_tower.cu": r"nb$"}


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _launches(src):
    """[(kernel, grid expression)] of every <<<...>>> launch in a source"""
    out = []
    for m in re.finditer(r"(\w+)(?:<[^<>;]*>)?\s*<<<", src):
        depth, i = 0, m.end()
        while depth or src[i] != ",":
            depth += {"(": 1, ")": -1}.get(src[i], 0)
            i += 1
        out.append((m.group(1), src[m.end():i].strip()))
    return out


def test_sm_caps_are_every_use_of_adc_num_sms():
    """each line of csrc/ that uses adc_num_sms is one site of one row of the table, and each site is such a line"""
    lines = []
    for name in sorted(os.listdir(CSRC)):
        if name in ("common.cu", "common.cuh"):                    # the definition and its declaration
            continue
        lines += [(name, l.strip()) for l in _src(name).splitlines() if "adc_num_sms" in l]
    sites = [(f, rx, c.name) for c in mc.SM_CAPS for f, rx in c.sites]
    for f, l in lines:
        hit = [s for s in sites if s[0] == f and re.search(s[1], l)]
        assert len(hit) == 1, "%s: '%s' is not one row's site of map_edge_cases.SM_CAPS" % (f, l)
    for f, rx, cap in sites:
        assert sum(1 for g, l in lines if g == f and re.search(rx, l)) == 1, "%s site %s of %s is not in csrc" % (cap, rx, f)
    assert len(lines) == len(sites)


def test_sm_caps_list_every_capped_launch():
    """the launches a file sizes by its capped grid are the ones its rows list, and the SM-free files use no SM count"""
    listed = {}
    for c in mc.SM_CAPS:
        for f, k in c.launches:
            listed.setdefault(f, set()).add(k)
    assert set(listed) | {"keysort.cuh"} == set(CAPPED_GRID)
    for f, rx in CAPPED_GRID.items():
        got = {k for k, g in _launches(_src(f)) if re.search(rx, g)}
        assert got == listed.get(f, set()), "%s: capped launches %s, the table lists %s" % (f, sorted(got), sorted(listed.get(f, ())))
    for f in sorted(os.listdir(CSRC)):
        if "grid_for(" in _src(f) and f != "keysort.cuh":
            assert f in CAPPED_GRID, "%s launches on a grid_for grid the table does not list" % f
    for f in mc.SM_FREE:
        src = _src(f)
        assert "adc_num_sms" not in src and "keysort.cuh" not in src, f
        assert _launches(src), f


def test_sm_cap_rules():
    """the issue's table: the elements each cap's largest grid takes before the cap binds, at s SMs"""
    s = 132
    assert [mc.sm_cap_elements(c, s) for c in ("grid8", "grid16", "fill_nan", "sel", "resident")] == \
        [2048 * s, 4096 * s, 16384 * s, 8192 * s, s]
    for c in mc.SM_CAPS:
        for s in (1, 7, 114, 132):
            e = mc.sm_cap_elements(c.name, s)
            assert c.blocks(e, s) == -(-e // c.uncapped) and c.blocks(e + 1, s) < -(-(e + 1) // c.uncapped)
            assert mc.sm_passes(c.name, e + 1, s) > mc.sm_passes(c.name, e, s) or c.name == "sel"
    assert mc.sel_blocks(1, 1) == 1 and mc.sel_blocks(2049, 1) == 2 and mc.sel_blocks(8193, 1) == 4
    assert mc.sm_passes("sel", 2048, 132) == 8 and mc.sm_passes("sel", 8193, 1) == 9
    assert mc.fill_nan_blocks(3, 1) == 1 and mc.fill_nan_blocks(16388, 1) == 16
    assert mc.resident_ctas(7500, 114) == 114 and mc.resident_ctas(24, 114) == 24


smr = _load("sm_count_runs")


def test_sm_count_cases_wrap_every_cap():
    """at one SM every row's loop wraps at least twice in some case and goes one block's elements past its cap in another;
    the fusion merges wrap at 1 and 7 SMs, the TSDF merges and the render's hash build at 1; 114 SMs run the full sizes"""
    passes = {}                                       # (cap, launch) -> [(case, passes at 1, 7, 114 SMs, elements)]
    for c in smr.CASES:
        inp = smr.inputs(c)
        sizes = smr.map_sizes(c, inp) if c.kind in ("fusion", "tsdf") else None
        for cap, launch, n in smr.loops(c, inp, sizes):
            passes.setdefault(cap, []).append((c.name, launch, [mc.sm_passes(cap, n, s) for s in (1, 7, 114)], n))
    assert set(passes) == {c.name for c in mc.SM_CAPS}
    for cap, rows in passes.items():
        assert any(p[0] >= 3 for _, _, p, _ in rows), cap
        past = mc.sm_cap_elements(cap, 1)
        assert any(past < n <= past + mc.sm_cap(cap).uncapped for _, _, _, n in rows), "%s: no case one past the cap" % cap
    p = {launch: ps for rows in passes.values() for _, launch, ps, _ in rows}
    assert p["fusion merge_frame"][1] >= 2 and p["fusion merge_table"][1] >= 2
    assert min(p["tsdf merge_frame"][0], p["tsdf merge_table"][0], p["tsdf hash_build"][0]) >= 3
    names = {c.name for c in smr.CASES}
    assert {"frontend_kitti_grey", "frontend_kitti_rgb", "rectify_raw_grey", "rectify_raw_rgb", "render_mb", "confidence_mb",
            "depth_mb", "tower_kitti"} <= names
