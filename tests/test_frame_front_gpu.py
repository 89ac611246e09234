"""A single-stream frame is a one-frame run of the detection front end (csrc/api.cu, detect_front), so every per-stream setting must
give the same outputs through lmot_frame_submit as through lmot_batch_submit with one frame: counts, boxes, every track field, the
obstacle footprints and the accumulation info, bit for bit, across combinations of the settings and with global_frame off and on."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
f32 = np.float32

SETTINGS = {
    "deskew": lambda ctx: ctx.set_deskew(on=1),
    "area": lambda ctx: ctx.set_detect_area([np.array([[-20.0, -20.0], [20.0, -20.0], [20.0, 20.0], [-20.0, 20.0]])]),
    "acc": lambda ctx: ctx.set_accumulate(sweeps=3),
    "search": lambda ctx: ctx.set_box_search(on=1, n_angles=30),
    "lines": lambda ctx: ctx.set_ground_lines(on=1),
    "layers": lambda ctx: ctx.set_layers(on=1),
    "obs": lambda ctx: ctx.set_obstacles(on=1),
}
# every setting alone, every setting with each other one at least once, and all of them
COMBOS = [(), *((s,) for s in SETTINGS), ("deskew", "area", "layers"), ("acc", "search", "obs"), ("lines", "layers", "obs"),
          ("deskew", "acc", "lines"), ("area", "search", "lines"), ("deskew", "search", "obs"), ("area", "acc", "layers"),
          ("deskew", "obs", "area", "acc"), ("search", "layers"), tuple(SETTINGS)]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(f"u{a.dtype.itemsize}") if a.dtype.kind == "f" else a


def _frames(synth, n):
    """the bench-style scene, every point's time (a 100 ms sweep, column order) in its fourth float"""
    cfg = synth.SceneConfig(rings=32, azimuths=900, n_objects=30, seed=23)
    tau = (-0.1 + (np.arange(900) + 0.5) / 900 * 0.1).astype(f32)
    out = []
    for ts, p in synth.frames(cfg, n):
        p = np.ascontiguousarray(p, f32).copy()
        p[:, 3] = np.tile(tau, len(p) // 900)
        out.append((ts, p))
    return out


@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("combo", COMBOS, ids=lambda c: "+".join(c) or "plain")
def test_frame_equals_one_frame_batch(pkg, synth, combo, gf):
    ctxs = []
    for _ in range(2):
        p = pkg.default_params()
        p.max_points = 1 << 17
        p.global_frame = gf
        ctxs.append(pkg.Lmot(p))
    fr, bt = ctxs
    try:
        for ctx in ctxs:
            for s in combo:
                SETTINGS[s](ctx)
        for i, (ts, pts) in enumerate(_frames(synth, 5)):
            v, yaw = 8.0, 0.02 * i
            fr.frame_submit(pts, ts, v, yaw)
            a = fr.frame_collect()
            bt.batch_submit([pts], ts, v, yaw)
            b = bt.batch_collect()
            assert (a["n_elevated"], a["n_ground"], a["num_cluster"], len(a["boxes"])) == \
                (b["n_elevated"][0], b["n_ground"][0], b["num_cluster"][0], b["n_boxes"][0]), i
            for k in ("boxes", "targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb"):
                assert np.array_equal(_bits(a[k]), _bits(b[k])), (i, k)
            if "obs" in combo:
                oa, ob = fr.obstacles_result(0), bt.obstacles_result(0)
                assert (oa["status"], oa["n_units"], oa["n_vertices"]) == (ob["status"], ob["n_units"], ob["n_vertices"]), i
                assert oa["obstacles"].tobytes() == ob["obstacles"].tobytes(), i
                assert np.array_equal(_bits(oa["vertices"]), _bits(ob["vertices"])), i
            ia, ib = fr.accumulate_info(), bt.accumulate_info()
            assert len(ia) == len(ib) == (1 if "acc" in combo else 0), i
            for ua, ub in zip(ia, ib):
                assert ua["sweeps_used"] == ub["sweeps_used"] and ua["n_points"] == ub["n_points"], i
                assert np.array_equal(_bits(np.asarray(ua["stamp_us"])), _bits(np.asarray(ub["stamp_us"])))
                assert np.array_equal(_bits(np.asarray(ua["pose"], f32)), _bits(np.asarray(ub["pose"], f32)))
    finally:
        for ctx in ctxs:
            ctx.close()
