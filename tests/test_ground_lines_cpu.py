"""Ground lines on the host (include/lmot.h, lmot_ground_lines_grid): the library's grid against the restatement in
tests/ground_lines_scenes.py bit for bit, the setting's validation, and the quality of the reference's chain on sloped scenes."""
import math

import numpy as np
import pytest

import ground_lines_scenes as gls

f32 = np.float32
EMPTY = f32(1000.0)


def _pkg():
    import importlib
    return importlib.import_module("3d-lidar-multi-object-tracking_b200")


def _bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def _grid(slope_x=0.0, slope_y=0.0, pitch=0.0, roll=0.0, h=1.73, r_min=3.4, r_max=120.0, noise=0.02, fill=1.0, seed=0):
    """min z of a ground plane seen from the sensor: channel ch looks along azimuth a_ch, cell b at range r_b"""
    rng = np.random.default_rng(seed)
    ch = (np.arange(80) + 0.5) / 80 * 2 * math.pi - math.pi
    r = r_min + (np.arange(120) + 0.5) * (r_max - r_min) / 120
    x = np.cos(ch)[:, None] * r[None, :]
    y = np.sin(ch)[:, None] * r[None, :]
    z = -h + slope_x * x + slope_y * y + math.tan(math.radians(pitch)) * x + math.tan(math.radians(roll)) * y
    z = z + rng.normal(0, noise, z.shape)
    z = np.where(rng.random(z.shape) < fill, z, EMPTY)
    return z.astype(f32)


def _check(minz, r_min=3.4, r_max=120.0, h=2.0, **kw):
    got = _pkg().ground_lines_grid(minz, r_min, r_max, h, **kw)
    want = gls.lines_grid(minz, r_min, r_max, h, **kw)
    assert np.array_equal(_bits(got), _bits(want))
    return got


@pytest.mark.parametrize("name,kw", [
    ("flat", {}),
    ("grade4", dict(slope_x=0.04)),
    ("grade8", dict(slope_x=0.08, slope_y=-0.03)),
    ("pitch3", dict(pitch=3.0)),
    ("roll2", dict(roll=2.0)),
    ("steep", dict(slope_x=0.5)),            # steeper than max_slope: seeds fail, lines break up
    ("sparse", dict(fill=0.3, slope_x=0.06)),
    ("noisy", dict(noise=0.2)),
])
def test_grid_matches_restatement(name, kw):
    minz = _grid(**kw, seed=sum(map(ord, name)))
    gz = _check(minz)
    if name in ("flat", "grade4", "pitch3", "roll2"):
        assert np.isfinite(gz).all()


def test_object_steps_and_gaps():
    minz = _grid(slope_x=0.05, seed=3)
    minz[5, 40:48] = minz[5, 40:48] + f32(1.5)         # a car's roof over the ground
    minz[6, 40:42] = minz[6, 40:42] + f32(0.25)        # a kerb inside max_step
    minz[7, 30:90] = EMPTY                             # a gap
    minz[8, ::3] = EMPTY
    minz[9, 60] = f32(-10.0)                           # a lone low outlier
    gz = _check(minz)
    L = gls.channel_lines(minz[5], 3.4, 120.0, 2.0)
    assert len(L) >= 2                                 # the roof ended the first line; the ground after it started a new one
    for b in range(40, 48):                            # the roof is not ground
        assert minz[5, b] > gz[5, b] + 0.25


def test_empty_channels_and_grid():
    minz = _grid(seed=4)
    minz[10:12] = EMPTY
    minz[11, 0] = f32(-1.9)                            # one prototype: no line
    gz = _check(minz)
    assert np.all(gz[10] == f32(-2.0)) and np.all(gz[11] == f32(-2.0))
    empty = np.full((80, 120), EMPTY, f32)
    assert np.all(_check(empty) == f32(-2.0))
    assert np.all(_check(empty, h=1.73) == f32(-1.73))


@pytest.mark.parametrize("r_min,r_max", [(3.4, 120.0), (1.0, 60.0), (5.25, 80.5)])
def test_moved_window(r_min, r_max):
    minz = _grid(slope_x=0.03, r_min=r_min, r_max=r_max, seed=7)
    _check(minz, r_min=r_min, r_max=r_max)


@pytest.mark.parametrize("kw", [dict(max_slope=0.1), dict(max_rmse=0.02), dict(max_step=0.1), dict(max_slope=1.0, max_rmse=0.5)])
def test_other_values(kw):
    _check(_grid(slope_x=0.07, noise=0.05, seed=9), **kw)


def test_validation():
    pkg = _pkg()
    minz = _grid(seed=1)
    assert pkg.default_ground_lines() == {"on": 0, "max_slope": 0.3, "max_rmse": 0.08, "max_step": 0.3}
    for bad in (dict(max_slope=0.0), dict(max_rmse=-1.0), dict(max_step=0.0), dict(max_slope=math.inf), dict(max_rmse=math.nan),
                dict(on=2)):
        with pytest.raises(pkg.LmotError):
            pkg.ground_lines_grid(minz, 3.4, 120.0, 2.0, **bad)
    for r_min, r_max, h in ((3.4, 3.4, 2.0), (3.4, math.nan, 2.0), (3.4, 120.0, math.inf)):
        with pytest.raises(pkg.LmotError):
            pkg.ground_lines_grid(minz, r_min, r_max, h)
    with pytest.raises(KeyError):
        pkg.ground_lines_grid(minz, 3.4, 120.0, 2.0, slope=0.1)


# ------------------------------------------------------------------------------------------------ quality on sloped scenes
# Objects found (a box centre within 2 m) out of 40 by the reference's chain (groundRemove, componentClustering, boxFitting) and by the
# same chain with ground lines at the default values (ground_lines_scenes.ref_lines_detect), with the renderer of ground_lines_scenes.py.
# The reference's column is within one object of the table that motivated the feature except roll2 (25 there); the lines' column
# is at least as good as that table's prototype on every scene.
QUALITY = {
    "flat": (28, 29),
    "grade4": (22, 27),
    "grade8": (15, 23),
    "pitch3": (19, 26),
    "roll2": (23, 28),
}


def _tunable():
    from oracle import ref_detect_tunable as rdt
    if not rdt.have_ref("detect_tunable"):
        pytest.skip("oracle/_ref/libref_detect_tunable.so not built")
    return rdt.RefDetectTunable()


@pytest.mark.parametrize("name", sorted(QUALITY))
def test_quality_reference_chain(name):
    rt = _tunable()
    pts, obj = gls.render(name)
    e, g = rt.ground_remove(pts)
    grid, k = rt.component_clustering(e)
    b, _ = rt.box_fitting(e, grid, k)
    ref = gls.objects_found(b, obj)
    lin = gls.objects_found(gls.ref_lines_detect(rt, pts)["boxes"], obj)
    assert (ref, lin) == QUALITY[name]
