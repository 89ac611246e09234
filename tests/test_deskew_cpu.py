"""Sweep deskew on the host (no device): the defaults, and lmot_deskew_table against a Python restatement of include/lmot.h's definition.

The restatement uses math.sin / math.cos (the same libm the library calls) and evaluates every product and sum in the order the
header gives, so the tables must agree bit for bit.
"""
import ctypes as C
import math

import numpy as np
import pytest

SLICES = 256
# a mount rotated about z by 30 degrees and tilted, offset from the vehicle origin (a rotation that is orthonormal in float32)
_A, _B = math.radians(30.0), math.radians(-4.0)
_RZ = np.array([[math.cos(_A), -math.sin(_A), 0], [math.sin(_A), math.cos(_A), 0], [0, 0, 1]])
_RY = np.array([[math.cos(_B), 0, math.sin(_B)], [0, 1, 0], [-math.sin(_B), 0, math.cos(_B)]])
MOUNT = np.concatenate([(_RZ @ _RY), [[1.35], [-0.42], [1.9]]], 1).astype(np.float32)


def table_ref(v, omega, mount=None, t_min=-0.1, t_max=0.0, **_):
    """include/lmot.h, sweep deskew: D_s = M^-1 T(tau_s) M in double, rounded to float once per entry"""
    M = [[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0]]
    if mount is not None:
        m = np.asarray(mount, np.float32).reshape(3, 4)
        M = [[float(m[i, j]) for j in range(4)] for i in range(3)]
    Mi = [[M[j][i] for j in range(3)] + [-((M[0][i] * M[0][3] + M[1][i] * M[1][3]) + M[2][i] * M[2][3])] for i in range(3)]

    def mul(L, R):
        out = []
        for i in range(3):
            row = []
            for j in range(4):
                acc = (L[i][0] * R[0][j] + L[i][1] * R[1][j]) + L[i][2] * R[2][j]
                if j == 3:
                    acc = acc + L[i][3]
                row.append(acc)
            out.append(row)
        return out

    h = (t_max - t_min) / SLICES
    out = np.zeros((SLICES, 3, 4), np.float32)
    for s in range(SLICES):
        tau = t_min + (s + 0.5) * h
        th = omega * tau
        if abs(omega) < 1e-9:
            tx, ty = v * tau, 0.0
        else:
            tx, ty = v * math.sin(th) / omega, v * (1.0 - math.cos(th)) / omega
        c, sn = math.cos(th), math.sin(th)
        T = [[c, -sn, 0.0, tx], [sn, c, 0.0, ty], [0.0, 0.0, 1.0, 0.0]]
        out[s] = np.array(mul(Mi, mul(T, M)), np.float64).astype(np.float32)
    return out


def test_defaults(pkg):
    assert pkg.default_deskew() == dict(on=0, time_field=3, time_scale=1.0, time_offset=0.0, t_min=-0.1, t_max=0.0)
    assert C.sizeof(pkg.Deskew) == 40 and pkg.DESKEW_SLICES == SLICES


@pytest.mark.parametrize("mount", [None, MOUNT], ids=["identity", "mounted"])
@pytest.mark.parametrize("omega", [0.0, 3e-10, 2e-8, 0.5, -0.5])
def test_table_equals_restatement(pkg, mount, omega):
    """Catches a changed evaluation order, a missed mount (or a mount applied as M T M^-1), the small-omega branch taken at the wrong
    threshold, and slices centred at the wrong time."""
    for v, win in ((15.0, {}), (-3.25, dict(t_min=-0.05, t_max=0.05)), (20.0, dict(t_min=-0.2, t_max=0.3))):
        got = pkg.deskew_table(v, omega, mount, **win)
        want = table_ref(v, omega, mount, **win)
        assert got.shape == (SLICES, 3, 4) and got.dtype == np.float32
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (v, omega, win)


def test_table_is_a_rigid_motion(pkg):
    """Sanity of the definition itself: at the window's end the identity-mount table has moved the vehicle by ~v * tau along x."""
    t = pkg.deskew_table(10.0, 0.0)
    tau0 = -0.1 + 0.5 * 0.1 / SLICES
    assert abs(t[0, 0, 3] - 10.0 * tau0) < 1e-6 and t[0, 1, 3] == 0.0
    R = t[:, :, :3].astype(np.float64)
    assert np.abs(np.einsum("sij,sik->sjk", R, R) - np.eye(3)).max() < 1e-6
    tm = pkg.deskew_table(10.0, 0.5, MOUNT)
    R = tm[:, :, :3].astype(np.float64)
    assert np.abs(np.einsum("sij,sik->sjk", R, R) - np.eye(3)).max() < 1e-6


@pytest.mark.parametrize("bad", [dict(t_min=0.0, t_max=0.0), dict(t_min=0.1, t_max=0.0), dict(t_min=-0.6, t_max=0.5),
                                 dict(t_min=float("nan")), dict(t_max=float("inf")), dict(time_scale=float("nan")),
                                 dict(time_offset=float("-inf")), dict(time_field=2), dict(time_field=-1)])
def test_table_validation(pkg, bad):
    with pytest.raises(pkg.LmotError) as e:
        pkg.deskew_table(1.0, 0.1, **bad)
    assert e.value.status == pkg.ERR_INVALID


def test_table_validation_motion_and_mount(pkg):
    for v, w in ((float("nan"), 0.0), (1.0, float("inf")), (float("-inf"), 0.2)):
        with pytest.raises(pkg.LmotError):
            pkg.deskew_table(v, w)
    skewed = MOUNT.copy()
    skewed[0, 0] *= 1.01                         # not orthonormal
    with pytest.raises(pkg.LmotError):
        pkg.deskew_table(1.0, 0.1, skewed)
    pkg.deskew_table(1.0, 0.1, t_min=-0.5, t_max=0.5)      # a window of exactly 1 s is allowed
    lib = pkg.load_library()
    out = np.zeros((SLICES, 12), np.float32)
    assert lib.lmot_deskew_table(None, C.c_double(0), C.c_double(0), None, out.ctypes.data_as(C.c_void_p)) == pkg.ERR_INVALID
    d = pkg.Deskew()
    assert lib.lmot_default_deskew(C.byref(d)) == pkg.OK
    assert lib.lmot_deskew_table(C.byref(d), C.c_double(0), C.c_double(0), None, None) == pkg.ERR_INVALID
    assert lib.lmot_default_deskew(None) == pkg.ERR_INVALID
