"""Sweep accumulation without a device: lmot_accumulate_pose against the NumPy restatement of the definition's step 2, bit for bit, and
the defaults and argument checks of the settings."""
import math

import numpy as np
import pytest

from accumulate_scenes import e_acc, pose_ref, rig_apply

f32 = np.float32


def _mount(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return np.concatenate([q, rng.uniform(-3.0, 3.0, (3, 1))], 1).astype(f32)


def test_pose_bit_exact(pkg):
    """random folds, yaw differences across (-pi, pi] and beyond, with and without random orthonormal mounts"""
    rng = np.random.default_rng(7)
    for i in range(400):
        fs = np.array([rng.uniform(-200, 200), rng.uniform(-200, 200), rng.uniform(-4.0, 4.0)])
        dy = rng.uniform(-math.pi, math.pi) if i % 4 else rng.choice([0.0, math.pi, -math.pi, 2 * math.pi, 1e-9])
        ft = np.array([fs[0] + rng.normal(0, 3), fs[1] + rng.normal(0, 3), fs[2] + dy])
        mount = None if i % 2 else _mount(rng)
        got = pkg.accumulate_pose(fs, ft, mount)
        assert np.array_equal(got.view(np.uint32), pose_ref(fs, ft, mount).view(np.uint32)), (i, fs, ft)


def test_pose_is_relative_motion(pkg):
    """the same fold twice is the identity; a point fixed in the global frame maps from sensor s to sensor t"""
    f = np.array([3.0, -2.0, 0.7])
    assert np.array_equal(pkg.accumulate_pose(f, f), np.eye(3, 4, dtype=f32))
    fs, ft = np.array([1.0, 2.0, -1.5707963267948966]), np.array([-0.5, 4.0, -1.2])
    g = np.array([7.0, -3.0])

    def to_sensor(fold, p):
        c, s = math.cos(fold[2]), math.sin(fold[2])
        return np.array([c * p[0] - s * p[1] + fold[0], s * p[0] + c * p[1] + fold[1]])

    ps, pt = to_sensor(fs, g), to_sensor(ft, g)
    moved = rig_apply(pkg.accumulate_pose(fs, ft), np.array([[ps[0], ps[1], 0.5, 0.0]], f32))[0]
    assert np.allclose(moved[:2], pt, atol=1e-5) and moved[2] == f32(0.5) and moved[3] == f32(1)


def test_pose_rejects_bad_mount(pkg):
    bad = np.eye(3, 4, dtype=f32)
    bad[0, 0] = np.nan
    with pytest.raises(pkg.LmotError):
        pkg.accumulate_pose([0, 0, 0], [1, 0, 0], bad)


def test_defaults_and_fields(pkg):
    d = pkg.default_accumulate()
    assert d == dict(sweeps=1, max_age_s=0.5)
    assert pkg.MAX_SWEEPS == 8
    with pytest.raises(KeyError):
        pkg._accumulate(dict(sweep=2))


def test_e_acc_cuts():
    """the restatement's prefix rule: a sweep too old, a stamp not before t, or one that does not fit whole ends the prefix"""
    e = lambda n: np.zeros((n, 4), f32)
    f = np.zeros(3)
    hist = [(e(5), 9e5, f), (e(5), 8e5, f), (e(5), 1e5, f)]
    acc, used = e_acc(e(3), 1e6, f, hist, 0.5, 100)
    assert len(acc) == 13 and [u[0] for u in used] == [9e5, 8e5]
    acc, used = e_acc(e(3), 1e6, f, hist, 0.5, 12)
    assert len(acc) == 8 and len(used) == 1
    acc, used = e_acc(e(3), 1e6, f, [(e(5), 1e6, f)] + hist, 0.5, 100)
    assert len(acc) == 3 and used == []
