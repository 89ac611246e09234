"""Every scene of the detection regime suite (test_detect_regimes_gpu.py) reaches its regime on the REFERENCE, without a GPU.

Scene drift -- a builder change that moves a scene back to the near side of a switch -- is caught here; each test prints the
witness it reached.  The witnesses come from the reference's outputs only (detect_scenes.py).
"""
import numpy as np
import pytest

import detect_scenes as S


@pytest.fixture(scope="module")
def ref(ref_o2):
    return ref_o2


def _sizes(ref, e):
    g, k = ref.component_clustering(e)
    return g, k, S.cluster_sizes(e, g, k)


@pytest.mark.parametrize("K", S.K_SWEEP)
def test_k_sweep_reaches_its_lane_count(ref, K):
    e = S.k_sweep(K)
    g, k, sz = _sizes(ref, e)
    b, _ = ref.box_fitting(e, g, k)
    print(f"K={k} lanes/cluster={S.seg_lanes(k)} scan rounds={-(-k * S.seg_lanes(k) // 1024)} accepted(o2)={len(b)}")
    assert k == K and np.all(sz == 30) and len(b) == K
    assert S.ccl_pairs(g != 0) == 0


def test_many_tiles_per_lane(ref):
    for e, lo in ((S.tiles_few_clusters(), 0), (S.tiles_many_clusters(), 512)):
        g, k, sz = _sizes(ref, e)
        per = S.tiles_per_lane(len(e), k)
        print(f"n={len(e)} K={k} tiles={S.n_tiles(len(e))} lanes={S.seg_lanes(k)} tiles/lane={per}")
        assert per > 16 and sz.sum() == len(e)
        assert (k <= 128 and len(e) >= 131073) if lo == 0 else (k > 512 and len(e) > 16384)


def test_big_clusters_sizes_and_branches(ref):
    e = S.big_clusters()
    g, k, sz = _sizes(ref, e)
    cid = S.cluster_ids(e, g)
    got = sorted((int(sz[c - 1]), S.takes_l_shape(e[cid == c])) for c in range(1, k + 1))
    print("big clusters (size, L-shape):", got)
    assert got == sorted((n, l) for n in S.BIG_SIZES for l in (False, True))
    for l_shape in (False, True):
        h = S.huge_cluster(l_shape)
        g, k, sz = _sizes(ref, h)
        print(f"huge: K={k} n={sz.tolist()} L-shape={S.takes_l_shape(h)} tiles/lane={S.tiles_per_lane(len(h), k)}")
        assert k == 1 and sz[0] == S.HUGE and S.takes_l_shape(h) == l_shape


def test_ring_hull_has_hundreds_of_vertices(ref):
    r = S.ring(60000)
    g, k, sz = _sizes(ref, r)
    m = S.hull_size(r)
    print(f"ring: K={k} n={sz.tolist()} hull vertices={m} columns={S.pixel_columns(r)} L-shape={S.takes_l_shape(r)}")
    assert k == 1 and m > 100 and not S.takes_l_shape(r)


def test_degenerate_hulls_and_slope_edges(ref):
    parts = S.degenerate_set()
    e = S.interleave(parts)
    g, k = ref.component_clustering(e)
    assert k == len(parts)
    for p in parts:
        gp, kp = ref.component_clustering(p)
        assert kp == 1 and len(p) >= 30
    one, col, diag, dup, ray, arm, ax_a, ax_b, ax_c, ax_d, nan = parts
    w = [(S.pixel_columns(p), S.hull_size(p)) for p in (one, col, diag)]
    print("(columns, hull) of one pixel / one column / diagonal:", w)
    assert w[0] == (1, 1) and w[1] == (1, 2) and w[2][0] > 1 and w[2][1] == 2
    ties = {name: (S.slope_ties(p), S.takes_l_shape(p)) for name, p in
            (("ray", ray), ("+-0 arm", arm), ("x=+0,y=10", ax_a), ("x=-0,y=13", ax_b), ("x=+0,y=-10", ax_c), ("x=-0,y=-13", ax_d))}
    print("(distinct points tied at min / max slope), L-shape:", ties)
    assert ties["ray"][0][0] >= 2 and ties["ray"][1]
    assert ties["+-0 arm"][0][0] >= 2 and ties["+-0 arm"][1]
    assert np.any(np.signbit(arm[:, 1]) & (arm[:, 1] == 0)) and np.any(~np.signbit(arm[:, 1]) & (arm[:, 1] == 0))
    for name in ("x=+0,y=10", "x=-0,y=13", "x=+0,y=-10", "x=-0,y=-13"):
        (lo, hi), l_shape = ties[name]
        assert max(lo, hi) >= 2 and l_shape, name
    assert np.sum((nan[:, 0] == 0) & (nan[:, 1] == 0)) == 4


def test_mixed_scene(ref):
    e = S.mixed()
    g, k, sz = _sizes(ref, e)
    cid = S.cluster_ids(e, g)
    n_l = sum(S.takes_l_shape(e[cid == c]) for c in range(1, k + 1) if sz[c - 1] >= 30)
    early = int(np.sum(sz < 30))
    print(f"mixed: K={k} largest={sz.max()} rejected early={early} L-shape={n_l} tiles={S.n_tiles(len(e))}")
    assert k > 1024 and early > 100 and n_l >= 8 and sz.max() >= 20000
    # rejected, L-shape and big clusters interleave in cluster-id order
    ids_early = np.where(sz < 30)[0]
    assert ids_early.min() < k // 4 and ids_early.max() > 3 * k // 4


@pytest.mark.parametrize("side", sorted(S.PAIR_SIDES))
def test_pair_scenes_straddle_the_pair_list(ref, side):
    e = S.pair_scene(S.PAIR_SIDES[side], rows=195)
    g, k = ref.component_clustering(e)
    pairs = S.ccl_pairs(g != 0)
    print(f"pair scene {side}: K={k} pairs={pairs} (list holds {S.PAIR_CAP})")
    assert k > 100
    assert (pairs == S.PAIR_CAP) if side == "at_cap" else (pairs > S.PAIR_CAP)
    e, _ = ref.ground_remove(S.frame(S.pair_scene(*S.PAIR_FRAME_SIDES[side])))
    g, k = ref.component_clustering(e)
    pairs = S.ccl_pairs(g != 0)
    print(f"pair frame {side}: K={k} pairs={pairs}")
    assert k > 100
    assert (S.PAIR_CAP - 8 <= pairs <= S.PAIR_CAP) if side == "at_cap" else (pairs > S.PAIR_CAP)


def test_grid_sequence(ref):
    ks = [ref.component_clustering(f)[1] for f in S.grid_sequence()]
    print("grid sequence K:", ks)
    assert ks[0] == 3844 and ks[1] == 1 and ks[2] == 0 and ks[3] >= 3700


def test_batch_frames_stay_elevated(ref):
    """the ground disc under every scene makes the reference's groundRemove keep all scene points beyond 3.4 m elevated"""
    reached = []
    for i, el in enumerate(S.batch_scenes()):
        raw = S.frame(el)
        e, gr = ref.ground_remove(raw)
        far = np.hypot(el[:, 0], el[:, 1]) > 3.5
        assert int(far.sum()) <= len(e) <= len(el), i
        if i != 7:                                    # the lattices and discs lie beyond 4 m whole; the ring passes the sensor
            assert len(e) == len(el) and far.all(), i
        g, k, sz = _sizes(ref, e)
        reached.append((k, int(sz.max()) if k else 0))
    print("batch frames (K, largest cluster):", reached)
    ks = [k for k, _ in reached]
    sizes = [s for _, s in reached]
    assert ks[0] > 256 and ks[1] > 1024 and ks[4] > 512 and ks[5] == 0 and max(sizes) > 1024 and ks[3] == 128
