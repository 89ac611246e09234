"""GPU parity of clustering and box fitting in the size regimes where their kernels switch paths.

The segment-offset scan of the counting sort picks 8 / 4 / 2 / 1 lanes per cluster and runs one round per 1,024 lanes, with a
second loop for more than 16 tiles per lane; tile_hist / scatter keep one int per cluster id in shared memory (above 48 KB from
max_clusters = 12,288 on); box_fit_kernel fits several clusters per CTA once K exceeds its grid, reads a cluster's points in
batches of 4 x NT, and its last CTA compacts the accepted boxes in rounds of NT clusters, cut at max_boxes; the CCL kernel falls
back from its 4,096-entry pair list to re-deriving every adjacency.  Every test drives one of the far sides with the scenes of
detect_scenes.py, compares with the reference compiled from its own sources at the bars of test_cluster_box_gpu.py (label grid
and numCluster bit-exact, boxes bit-exact as uint32, markers to 1e-4), and asserts and prints the regime it reached, proven from
the REFERENCE's outputs.
"""
import ctypes as C

import numpy as np
import pytest

import detect_scenes as S

pytestmark = pytest.mark.gpu

MB = 4096           # max_boxes of the contexts here: a full lattice is 3,844 accepted boxes


def _params(pkg, mode="o2", **kw):
    p = pkg.default_params()
    p.rule_filter = pkg.RULE_GCC13_O2_COMPAT if mode == "o2" else pkg.RULE_INTENDED
    p.max_boxes = MB
    p.pipeline_depth = 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _ctx(pkg, mode="o2", **kw):
    return pkg.Lmot(_params(pkg, mode, **kw))


@pytest.fixture(scope="module")
def contexts(pkg):
    """rule mode -> context at the default max_clusters, and a context at the ABI's bound of 50,000 clusters"""
    made = {"o2": _ctx(pkg, "o2"), "intended": _ctx(pkg, "intended"), "o2_50k": _ctx(pkg, "o2", max_clusters=50000)}
    yield made
    for c in made.values():
        c.close()


def _refs(ref_intended, ref_o2):
    return {"intended": ref_intended, "o2": ref_o2}


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _check(ctx, ref, e, what):
    """componentClustering then boxFitting on the reference's grid -> (K, boxes) of the reference"""
    g_ref, k_ref = ref.component_clustering(e)
    g, k = ctx.component_cluster(e)
    assert k == k_ref, (what, k, k_ref)
    assert np.array_equal(g, g_ref), what
    b_ref, m_ref = ref.box_fitting(e, g_ref, k_ref, MB)
    b, m = ctx.box_fit(e, g_ref, k_ref, max_boxes=MB)
    assert b.shape == b_ref.shape, (what, b.shape, b_ref.shape)
    assert np.array_equal(_bits(b), _bits(b_ref)), what
    np.testing.assert_allclose(m, m_ref, rtol=1e-4, atol=1e-4, err_msg=what)
    return k_ref, g_ref, b_ref


# ------------------------------------------------------------------------------------------------ cluster counts
@pytest.mark.parametrize("which", ["o2", "o2_50k"])
def test_cluster_count_sweep(contexts, ref_o2, which):
    """K at every lanes-per-cluster switch, two and four scan rounds, a full grid -- every box accepted, so the compaction runs its
    rounds of 512 clusters with a carry.  o2_50k: the same on a context at max_clusters = 50,000 (200 KB of shared memory in
    tile_hist / scatter)."""
    ctx = contexts[which]
    for K in S.K_SWEEP:
        k, _, b = _check(ctx, ref_o2, S.k_sweep(K), (which, K))
        print(f"{which}: K={k} lanes/cluster={S.seg_lanes(k)} clusters per CTA (264 CTAs)={-(-k // 264)} accepted={len(b)}")
        assert k == K and len(b) == K


def test_many_tiles_per_lane(contexts, ref_o2, ref_intended):
    refs = _refs(ref_intended, ref_o2)
    for e in (S.tiles_few_clusters(), S.tiles_many_clusters()):
        for mode in ("o2", "intended"):
            k, _, b = _check(contexts[mode], refs[mode], e, ("tiles", mode, len(e)))
            per = S.tiles_per_lane(len(e), k)
            print(f"{mode}: n={len(e)} K={k} tiles/lane={per} boxes={len(b)}")
            assert per > 16


def test_default_fit_ctas_mixed(contexts, ref_o2, ref_intended):
    """more clusters than the 264 CTAs of a frame's box-fit grid, of every kind, at the default grid"""
    refs = _refs(ref_intended, ref_o2)
    for seed in (0, 1):
        e = S.mixed(seed)
        for mode in ("o2", "intended"):
            k, g, b = _check(contexts[mode], refs[mode], e, ("mixed", seed, mode))
            sz = S.cluster_sizes(e, g, k)
            print(f"mixed {seed} {mode}: K={k} rejected early={int((sz < 30).sum())} largest={sz.max()} boxes={len(b)}")
            assert k > 264


@pytest.mark.parametrize("mode", ["o2", "intended"])
def test_grid_stride_eight_ctas(pkg, ref_o2, ref_intended, monkeypatch, mode):
    """LMOT_FIT_CTAS = 8: every box-fit CTA fits hundreds of clusters in a row and must reset all of its per-cluster state"""
    ref = _refs(ref_intended, ref_o2)[mode]
    monkeypatch.setenv("LMOT_FIT_CTAS", "8")
    ctx = _ctx(pkg, mode)
    try:
        for name, e in (("lattice", S.k_sweep(3844)), ("mixed0", S.mixed(0)), ("mixed1", S.mixed(1)), ("degenerate", S.interleave(S.degenerate_set()))):
            k, g, b = _check(ctx, ref, e, (name, mode))
            print(f"8 CTAs {mode} {name}: K={k} clusters per CTA={-(-k // 8)} boxes={len(b)}")
            assert k > 8                                     # some CTA fits two clusters or more
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ big and degenerate clusters
def test_big_clusters(contexts, ref_o2, ref_intended):
    """clusters around one 4 x 512-point batch of the per-point pass, far above it, 200,000 points in one cluster (both branches) and a
    ring whose pixel hull has over 100 vertices"""
    refs = _refs(ref_intended, ref_o2)
    scenes = [("big", S.big_clusters()), ("huge MAR", S.huge_cluster(False)), ("huge L", S.huge_cluster(True)), ("ring", S.ring(60000))]
    for name, e in scenes:
        for mode in ("o2", "intended"):
            k, g, b = _check(contexts[mode], refs[mode], e, (name, mode))
            cid = S.cluster_ids(e, g)
            reached = [(int((cid == c).sum()), S.takes_l_shape(e[cid == c])) for c in range(1, k + 1)]
            print(f"{name} {mode}: (size, L-shape) {reached} boxes={len(b)}")
    assert S.hull_size(S.ring(60000)) > 100


@pytest.mark.parametrize("mode", ["o2", "intended"])
def test_degenerate_hulls_and_slope_edges(contexts, ref_o2, ref_intended, mode):
    """a one-pixel cluster (hull m = 1), one pixel column and a pixel diagonal (m = 2), duplicated points, distinct points tied at the
    smallest slope on one ray from the origin and at +-0 slopes, +-inf slopes at x = +-0, NaN slopes at the origin -- each alone and
    all interleaved"""
    ref = _refs(ref_intended, ref_o2)[mode]
    parts = S.degenerate_set()
    for i, p in enumerate(parts):
        k, _, b = _check(contexts[mode], ref, p, ("degenerate", i, mode))
        assert k == 1
    for seed in (0, 3):
        k, _, b = _check(contexts[mode], ref, S.interleave(S.degenerate_set(seed), seed), ("degenerate set", seed, mode))
        print(f"degenerate set {seed} {mode}: K={k} boxes={len(b)} hulls one/column/diagonal="
              f"{[S.hull_size(p) for p in parts[:3]]} ray ties={S.slope_ties(parts[4])}")
        assert k == len(parts)


# ------------------------------------------------------------------------------------------------ capacities
def _frame_raw(pkg, ctx, raw, ts=1e6):
    """lmot_frame through the raw call, so that an error status keeps its outputs -> (status, result dict)"""
    p, n, s = pkg._pts(raw)
    fo, bufs = ctx._frame_out(ctx.params.max_tracks)
    st = ctx.lib.lmot_frame(ctx.h, pkg._fp(p), n, s, C.c_double(ts), C.c_double(0.0), C.c_double(0.0), C.byref(fo))
    return st, ctx._frame_result(fo, bufs)


def _ref_detect(ref, raw):
    e, _ = ref.ground_remove(raw)
    g, k = ref.component_clustering(e)
    return e, g, k


@pytest.mark.parametrize("max_boxes,K", [(100, 300), (700, 1100)])
def test_capacity_compaction_cut(pkg, ref_o2, max_boxes, K):
    """more accepted boxes than max_boxes: LMOT_ERR_CAPACITY and the reference's first max_boxes boxes (700 of 1,100: the cut falls in
    the compaction's second round)"""
    ctx = _ctx(pkg, "o2", max_boxes=max_boxes)
    try:
        raw = S.frame(S.lattice(K, 30, seed=K, keep=S.sensor_range()))
        e, g, k = _ref_detect(ref_o2, raw)
        b_ref, _ = ref_o2.box_fitting(e, g, k, MB)
        st, r = _frame_raw(pkg, ctx, raw)
        print(f"compaction cut: K={k} accepted={len(b_ref)} max_boxes={max_boxes} status={st}")
        assert len(b_ref) == K > max_boxes
        assert st == pkg.ERR_CAPACITY
        assert r["num_cluster"] == k and r["n_elevated"] == len(e)
        assert r["boxes"].shape == (max_boxes, 8, 3) and np.array_equal(_bits(r["boxes"]), _bits(b_ref[:max_boxes]))
    finally:
        ctx.close()


@pytest.mark.parametrize("max_clusters", [1000, 200])
def test_capacity_too_many_clusters(pkg, ref_o2, max_clusters):
    """more components than max_clusters: LMOT_ERR_CAPACITY, num_cluster = the reference's K, and the boxes of the clusters
    1..max_clusters -- the reference's boxFitting on its grid with the higher ids cleared (it skips label 0, box_fitting.cpp:63)"""
    ctx = _ctx(pkg, "o2", max_clusters=max_clusters)
    try:
        raw = S.frame(S.lattice(1100, 30, seed=5, keep=S.sensor_range()))
        e, g, k = _ref_detect(ref_o2, raw)
        cut = np.where(g > max_clusters, 0, g).astype(np.int32)
        b_ref, _ = ref_o2.box_fitting(e, cut, max_clusters, MB)
        st, r = _frame_raw(pkg, ctx, raw)
        print(f"too many clusters: K={k} max_clusters={max_clusters} boxes={len(r['boxes'])} status={st}")
        assert k == 1100 > max_clusters and len(b_ref) == max_clusters
        assert st == pkg.ERR_CAPACITY
        assert r["num_cluster"] == k
        assert r["boxes"].shape == b_ref.shape and np.array_equal(_bits(r["boxes"]), _bits(b_ref))
        with pytest.raises(pkg.LmotError) as err:
            ctx.box_fit(e, g, k, max_boxes=MB)
        assert err.value.status == pkg.ERR_CAPACITY
        # the context still works at its capacity
        b, _ = ctx.box_fit(e, cut, max_clusters, max_boxes=MB)
        assert np.array_equal(_bits(b), _bits(b_ref))
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ batched ticks (NT = 256)
def _ref_frame(ref, raw):
    e, gr = ref.ground_remove(raw)
    g, k = ref.component_clustering(e)
    b, _ = ref.box_fitting(e, g, k, MB)
    return (len(e), len(gr), k, len(b)), b


@pytest.mark.parametrize("mode", ["o2", "intended"])
def test_batch_tick_in_every_regime(pkg, ref_o2, ref_intended, mode):
    """one 8-frame lmot_batch tick whose frames sit in different regimes of the batched kernels: K > 256, K > 1024, clusters of 1,023 to
    3,000 points, an empty frame.  Every lattice point stays elevated on the reference (ground disc beneath)."""
    ref = _refs(ref_intended, ref_o2)[mode]
    scenes = S.batch_scenes()
    raws = [S.frame(el) for el in scenes]
    want = [_ref_frame(ref, raw) for raw in raws]
    ctx = _ctx(pkg, mode, max_boxes=8192)
    try:
        r = ctx.batch(raws, 1e6)
        got = list(zip(r["n_elevated"], r["n_ground"], r["num_cluster"], r["n_boxes"]))
        print(f"batch {mode}: (n_elev, n_ground, K, boxes) per frame {[w for w, _ in want]}")
        assert got == [w for w, _ in want]
        allb = np.concatenate([b for _, b in want])
        assert r["boxes"].shape == allb.shape and np.array_equal(_bits(r["boxes"]), _bits(allb))
        ks = [w[2] for w, _ in want]
        assert ks[0] > 256 and ks[1] > 1024 and ks[5] == 0
        for i in range(7):
            assert want[i][0][0] == len(scenes[i]), i           # the reference kept every scene point elevated
    finally:
        ctx.close()


def test_sequence_tick_with_own_detect_params(pkg, ref_o2, ref_intended):
    """eight sequences, each with its own detection values (rule mode alternating): box_fit_frame_kernel<256> on the same regimes"""
    raws = [S.frame(el) for el in S.batch_scenes()]
    ctx = _ctx(pkg, "intended")
    try:
        ctx.seq_open(8, ring=2)
        modes = ["o2" if k % 2 == 0 else "intended" for k in range(8)]
        for k, m in enumerate(modes):
            ctx.seq_set_detect_params(k, rule_filter=pkg.RULE_GCC13_O2_COMPAT if m == "o2" else pkg.RULE_INTENDED)
        out = ctx.seq(raws, [1e6] * 8)
        refs = _refs(ref_intended, ref_o2)
        for k, (raw, m) in enumerate(zip(raws, modes)):
            w, b = _ref_frame(refs[m], raw)
            got = out[k]
            assert (got["n_elevated"], got["n_ground"], got["num_cluster"], len(got["boxes"])) == w, (k, m)
            assert np.array_equal(_bits(got["boxes"]), _bits(b)), (k, m)
            print(f"sequence {k} ({m}): (n_elev, n_ground, K, boxes) {w}")
    finally:
        ctx.close()


_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
import detect_scenes as S
frames = [S.frame(S.lattice(300, 30, seed=1, keep=S.sensor_range())), S.frame(S.lattice(40, 1100, seed=2, keep=S.sensor_range()))]
out = {}
p = pkg.default_params(); p.max_boxes = 4096; p.pipeline_depth = 1
ctx = pkg.Lmot(p)
ctx.batch(frames, 1e6); torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    ctx.batch(frames, 1.1e6); torch.cuda.synchronize()
out["batch"] = [e.name for e in prof.events() if "box_fit" in e.name]
ctx.seq_open(2, ring=2)
for k in range(2):
    ctx.seq_set_detect_params(k, rule_filter=k)
ctx.seq(frames, [1e6] * 2); torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    ctx.seq(frames, [1.1e6] * 2); torch.cuda.synchronize()
out["seq"] = [e.name for e in prof.events() if "box_fit" in e.name]
ctx.close()
print(json.dumps(out))
"""


def test_batched_kernels_are_the_256_thread_variants():
    """the batched tick runs box_fit_kernel<256, .>, the sequence tick with own values box_fit_frame_kernel<256> (torch.profiler, in a
    process of its own: profiler sessions in the test process disturb later tests' sessions)"""
    import json
    import os
    import re
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    print("box-fit kernels:", {k: sorted(set(v)) for k, v in names.items()})
    nt256 = lambda kernel, n: re.search(kernel + r"(<256\b|ILi256E)", n) is not None
    assert names["batch"] and all(nt256("box_fit_kernel", n) for n in names["batch"]), names
    assert names["seq"] and all(nt256("box_fit_frame_kernel", n) for n in names["seq"]), names


# ------------------------------------------------------------------------------------------------ CCL
@pytest.mark.parametrize("side", sorted(S.PAIR_SIDES))
def test_ccl_pair_list_both_sides(pkg, contexts, ref_o2, side):
    """pair-list scenes at 4,096 pairs and above, through lmot_component_cluster, the fused ground-tail clustering of lmot_frame and
    the batched ccl_dense_kernel of lmot_batch"""
    ref = ref_o2
    e = S.pair_scene(S.PAIR_SIDES[side], rows=195)
    k, g, b = _check(contexts["o2"], ref, e, ("pairs", side))
    print(f"component_cluster {side}: K={k} pairs={S.ccl_pairs(g != 0)}")
    raw = S.frame(S.pair_scene(*S.PAIR_FRAME_SIDES[side]))
    ef, gf, kf = _ref_detect(ref, raw)
    bf, _ = ref.box_fitting(ef, gf, kf, MB)
    ctx = contexts["o2"]
    st, r = _frame_raw(pkg, ctx, raw)
    assert st >= 0 and r["num_cluster"] == kf and np.array_equal(_bits(r["boxes"]), _bits(bf))
    grid, nc = ctx.debug_label_grid()
    assert nc == kf and np.array_equal(grid, gf)
    print(f"lmot_frame {side}: K={kf} pairs={S.ccl_pairs(gf != 0)}")
    other = S.frame(S.k_sweep(300))
    eo, go, ko = _ref_detect(ref, other)
    bo, _ = ref.box_fitting(eo, go, ko, MB)
    rb = ctx.batch([raw, other, raw], 2e6)
    assert list(rb["num_cluster"]) == [kf, ko, kf] and list(rb["n_boxes"]) == [len(bf), len(bo), len(bf)]
    assert np.array_equal(_bits(rb["boxes"]), _bits(np.concatenate([bf, bo, bf])))
    ctx.tracker_reset()


def test_ccl_sparse_label_grid_across_frames(pkg, ref_o2):
    """the label grid is updated sparsely from the previous frame's occupancy: a full grid, one cluster, nothing, the lattice shifted by
    a cell; then lmot_box_fit uploads a foreign grid, and clustering must start from a clean slate again"""
    ref = ref_o2
    ctx = _ctx(pkg, "o2")
    try:
        seq = S.grid_sequence()
        ks = []
        for i, e in enumerate(seq + seq[:1]):
            g_ref, k_ref = ref.component_clustering(e)
            g, k = ctx.component_cluster(e)
            assert k == k_ref and np.array_equal(g, g_ref), i
            ks.append(k)
        foreign_e = S.mixed(0)
        foreign_g, foreign_k = ref.component_clustering(foreign_e)
        b_ref, _ = ref.box_fitting(foreign_e, foreign_g, foreign_k, MB)
        b, _ = ctx.box_fit(foreign_e, foreign_g, foreign_k, max_boxes=MB)
        assert np.array_equal(_bits(b), _bits(b_ref))
        for i, e in enumerate([seq[1], seq[0], seq[3], seq[2]]):
            g_ref, k_ref = ref.component_clustering(e)
            g, k = ctx.component_cluster(e)
            assert k == k_ref and np.array_equal(g, g_ref), ("after foreign grid", i)
            ks.append(k)
        print("label grid sequence K:", ks)
        assert ks[:4] == [3844, 1, 0, 3844]
    finally:
        ctx.close()
