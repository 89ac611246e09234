"""Every scene of the ground-removal regime suite (test_ground_regimes_gpu.py) reaches its regime, without a GPU.

The launch geometry is ground_scenes.launch at 132 and 114 SMs (H100 SXM / PCIe); the probes' sides and ties come from the
REFERENCE's outputs.  A builder change that moves a scene back to the near side of a switch, or a probe off its tie, fails here; each
test prints the witness it reached.
"""
import numpy as np
import pytest

import ground_scenes as S
from oracle.ref import labels_from_clouds

SMS = (132, 114)


@pytest.fixture(scope="module")
def ref(ref_intended):
    return ref_intended


@pytest.fixture(scope="module")
def ref_dt():
    from oracle import ref_detect_tunable
    if not ref_detect_tunable.have_ref("detect_tunable"):
        pytest.skip("oracle/_ref/libref_detect_tunable.so not built")
    return ref_detect_tunable.RefDetectTunable()


@pytest.fixture(scope="module")
def pool(ref):
    return S.checker_probe_pool(ref.cell_index, n=24000, seed=1)


def _labels(ref, pts):
    e, g = ref.ground_remove(pts)
    return labels_from_clouds(pts, e, g)


def test_geometry_restates_the_switches():
    for sms in SMS:
        g = S.launch([sms * 16384], sms, ppc=16384)
        assert g["G"] == sms and g["frames"][0]["chunk"] == 16384 and not g["capacity"]
        assert S.launch([sms * 16384 + 1], sms, ppc=16384)["capacity"]
        half = max(sms // 2, 8) * 8192
        on, off = S.launch([half], sms, entry="frame"), S.launch([half + 1], sms, entry="frame")
        print(f"{sms} SMs: half-SM cap at n={half}: {S.describe(on)} | n={half + 1}: {S.describe(off)}")
        assert on["half"] and on["G"] == sms // 2 and not off["half"] and off["G"] == sms
        org = S.launch([128 * 2048], sms, entry="frame")
        print(f"{sms} SMs: organized 128 x 2048 frame: {S.describe(org)}")
        assert org["half"] and org["frames"][0]["chunk"] > S.PEND_CAP
        rag = S.launch([0, 9, (sms // 3) * 16384], sms, entry="batch")
        assert rag["G"] == sms // 3 and rag["frames"][2]["chunk"] == 16384 and rag["frames"][1]["chunk"] == 1
        assert sum(c["cnt"] for c in rag["frames"][1]["ctas"]) == 9 and rag["frames"][0]["ctas"][0]["cnt"] == 0
        for G in (8, 9, 13, 33, sms // 2, 79, 80, 81, sms):
            n = max(12000, 300 * G)
            ppc = S.ppc_for(G, n)
            assert ppc is not None and S.launch([n], sms, ppc=ppc)["G"] == G, G
    # the switches by chunk
    for chunk, T, stage, res in ((2048, 2, False, 2), (2049, 3, True, 3), (8192, 8, True, 8), (8193, 9, True, 8), (16384, 16, True, 8)):
        g = S.launch([8 * chunk], 132, ppc=chunk)
        f = g["frames"][0]
        assert g["G"] == 8 and f["chunk"] == chunk and f["ctas"][0]["T"] == T and f["stage_lim"] == stage and f["res_tiles"] == res
    assert S.launch([3000], 132, ppc=256)["frames"][0]["ctas"][0]["full_pairs"] == 0
    assert S.launch([8 * 5000], 132, ppc=5000)["frames"][0]["ctas"][0]["full_pairs"] == 2
    assert S.launch([8 * 5000], 132, ppc=5000, prefilter=True)["frames"][0]["ctas"][0]["full_pairs"] == 0


def test_checkerboard_probes_are_queued_and_one_sided(ref, pool):
    floor = S.full_floor(S.checker_heights())
    grid = ref.polar_grid(floor)
    assert grid["isground"].all() and np.all(S.certainly_fast(floor))
    pts = np.concatenate([floor, pool])
    lab = _labels(ref, pts)
    assert np.all(lab[len(floor):] == 2) and np.all(lab[: len(floor)] == 1)
    g2 = ref.polar_grid(pts)
    assert all(np.array_equal(g2[k].view(np.uint32), grid[k].view(np.uint32)) for k in ("minz", "height", "hground"))
    # across the nearest boundary the probe is ground: the high cell's limit is above -1.4
    assert S.label_limit(S.HIGH, 0.25) > S.PROBE_Z > S.label_limit(S.LOW, 0.25)
    assert S.label_limit(S.HIGH, 0.3) > S.PROBE_Z > S.label_limit(S.LOW, 0.3)
    assert S.label_limit(S.HIGH, 0.1) > S.PROBE_Z > S.label_limit(S.LOW, 0.1)
    print(f"checkerboard: {len(pool)} probes, all certainly queued, all elevated on the reference")


@pytest.mark.parametrize("sms", SMS)
def test_overflow_scenes_queue_above_the_cap(ref, pool, sms):
    floor = S.full_floor(S.checker_heights())
    for name, n, ppc, q in (("stage T=4", 8 * 4096, 4096, [1500, 2048, 2049, 4096] * 2),
                            ("stage T=16", sms * 16384, 16384, [4000] * sms)):
        g = S.launch([n], sms, ppc=ppc)
        pts = S.layout(g, q, pool, floor, seed=3)
        per = S.queued_per_cta(pts, g)
        print(f"{sms} SMs {name}: {S.describe(g)} certainly queued per CTA {sorted(set(per[:, 0].tolist()))}")
        assert np.array_equal(per[:, 0], np.minimum(q, [c["cnt"] for c in g["frames"][0]["ctas"]]))
        assert np.all(per.sum(1) == [c["cnt"] for c in g["frames"][0]["ctas"]])        # exact: every other point certainly fast
        assert per[:, 0].max() > S.PEND_CAP
        if n < 100000:
            lab = _labels(ref, pts)
            assert np.all(lab[S.certainly_queued(pts)] == 2)


@pytest.mark.parametrize("sms", SMS)
def test_organized_frame_overflows_with_in_range_points(ref, sms):
    pts = S.organized(ref.cell_index)
    g = S.launch([len(pts)], sms, entry="frame")
    q = S.certainly_queued(pts)
    ch, b = S.coords(pts)
    with np.errstate(invalid="ignore"):
        in_range = np.isfinite(b) & (b > 0) & (b < S.NUM_BIN)
    per_in = [int((q & in_range)[c["beg"]: c["beg"] + c["cnt"]].sum()) for c in g["frames"][0]["ctas"]]
    per = S.queued_per_cta(pts, g)[:, 0]
    print(f"{sms} SMs organized: {S.describe(g)} queued per CTA max {per.max()} in-range queued max {max(per_in)} "
          f"CTAs over the cap: {(per > S.PEND_CAP).sum()} / with in-range overflow: {(np.array(per_in) > S.PEND_CAP).sum()}")
    assert g["half"] and max(per_in) > S.PEND_CAP
    lab = _labels(ref, pts)
    assert np.all(lab[q & in_range] == 2) and np.all(lab[~in_range] == 0)


def _tie_case(ref_dt, values, heights, zero=False):
    base = S.full_floor(heights)
    tol = values.get("ground_tolerance", 0.25)
    with ref_dt.detect_params(values):
        g0 = ref_dt.polar_grid(base)
        probes, want = S.tie_probes(g0["hground"], g0["isground"], tol, zero)
        pts = np.concatenate([base, probes])
        g1 = ref_dt.polar_grid(pts)
        e, gr = ref_dt.ground_remove(pts)
    lab = labels_from_clouds(pts, e, gr)
    return g0, g1, lab[len(base):], want


TIE_CASES = {
    "tol0.25": (dict(), dict(centre=-1.6)),
    "tol0.3": (dict(ground_tolerance=0.3), dict(centre=-1.6)),
    "tol0.1": (dict(ground_tolerance=0.1), dict(centre=-1.6)),
    "thr0": (dict(t_hmax=-0.1), dict(centre=-0.3, amp=0.05, exact=(-0.25, 0.3))),
    "h>0 (0.8 m mount)": (dict(t_hmin=-0.8, t_hmax=0.8, h_sensor=0.8), dict(centre=0.3)),
}


@pytest.mark.parametrize("case", sorted(TIE_CASES))
def test_tie_probes_sit_on_the_reference_tie(ref_dt, case):
    values, hk = TIE_CASES[case]
    g0, g1, lab, want = _tie_case(ref_dt, values, S.smooth_heights(**hk), zero=case == "thr0")
    for k in ("minz", "height", "smoothed", "hdiff", "hground", "isground"):
        assert np.array_equal(np.asarray(g0[k]).view(np.uint8), np.asarray(g1[k]).view(np.uint8)), k
    assert g0["isground"].all()
    h = g0["hground"][g0["isground"].astype(bool)]
    tol = values.get("ground_tolerance", 0.25)
    thr = h.astype(np.float64) + tol
    representable = np.mean(thr.astype(np.float32).astype(np.float64) == thr)
    print(f"{case}: {len(lab)} tie probes, h + tol a float in {representable:.0%} of cells, h > 0 in {np.mean(h > 0):.0%}, "
          f"limit -denormal in {int(np.sum(S.label_limit(h, tol) == -np.finfo(np.float32).smallest_subnormal))} cells")
    assert np.array_equal(lab, want)
    if case == "tol0.25":
        assert representable == 1.0
    if case in ("tol0.3", "tol0.1"):
        assert representable < 0.05
    if case == "thr0":
        assert np.any(S.label_limit(h, tol) == -np.finfo(np.float32).smallest_subnormal)
    if case.startswith("h>0"):
        assert np.mean(h > 0) > 0.5 and 0.0 < representable < 1.0


@pytest.mark.parametrize("gc", [8, 9, 13, 33, 57, 66, 79, 80])
def test_seam_patterns_rewrite_the_seam_cells(ref, gc):
    pts, marks = S.seam_scene(gc)
    grid = ref.polar_grid(pts)
    lab = _labels(ref, pts)
    done = [(k, ch, b) for k, ch, b in marks if S.rewritten(grid, ch, b) and grid["isground"][ch, b]]
    print(f"gc={gc}: seam channels {S.seam_channels(gc)[:6]}... {len(done)} / {len(marks)} seam cells rewritten by the reference")
    assert done == marks
    # the rewrite is what makes the cells' probes ground
    ch, b = S.coords(pts)
    cells = np.floor(ch).astype(int) * S.NUM_BIN + np.floor(b).astype(int)
    for _, c, bb in marks:
        sel = cells == c * S.NUM_BIN + bb
        assert np.all(lab[sel] == 1), (c, bb)


def test_tie_probes_on_filter_rewrites(ref):
    base, marks = S.seam_scene(8)
    g0 = ref.polar_grid(base)
    probes, want = S.tie_probes(g0["hground"], g0["isground"], 0.25, minz=g0["minz"])
    pts = np.concatenate([base, probes])
    g1 = ref.polar_grid(pts)
    assert all(np.array_equal(np.asarray(g0[k]).view(np.uint8), np.asarray(g1[k]).view(np.uint8)) for k in g0)
    lab = _labels(ref, pts)[len(base):]
    ch, b = S.coords(probes)
    cells = set(zip(np.floor(ch).astype(int).tolist(), np.floor(b).astype(int).tolist()))
    probed = [(c, bb) for _, c, bb in marks if (c, bb) in cells]
    print(f"filter rewrites: {len(want)} tie probes, {len(probed)} / {len(marks)} rewritten seam cells probed")
    assert np.array_equal(lab, want) and len(probed) == len(marks)
