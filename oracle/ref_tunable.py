"""TEST INFRASTRUCTURE ONLY -- ctypes binding to oracle/_ref/libref_tunable.so (oracle/tunable.mk).

RefTunable() is RefOracle("intended") with the tracker's constants in globals: set_tracker_params(dict) writes them through ctypes
in_dll, with lmot_tracker_params' field names.  The reference fixes std_a, std_yawdd, the lidar noise, the transition matrix, the
initial mode probabilities and P_merge_ when a track's UKF is constructed (ukf.cpp:20-322): new values reach existing tracks only
through tracker_load, which constructs them again.
"""
from __future__ import annotations

import ctypes as C

from oracle.ref import _OracleBase, ref_lib_path, have_ref  # noqa: F401  (have_ref: callers test have_ref("tunable"))

# field -> (symbol, ctype, number of elements; 0 = scalar, (symbol, index) for one element of a shared array)
GLOBALS = {
    "gamma_g": ("gammaG_", C.c_double, 0), "p_g": ("pG_", C.c_double, 0), "p_d": ("pD_", C.c_double, 0),
    "distance_thres": ("distanceThres_", C.c_double, 0), "lifetime_thres": ("lifeTimeThres_", C.c_int, 0),
    "bb_yaw_change_thres": ("bbYawChangeThres_", C.c_double, 0), "second_init_v": ("lmot_tp_second_init_v", C.c_double, 0),
    "static_lifetime": ("lmot_tp_static_lifetime", C.c_int, 0), "static_dist": ("lmot_tp_static_dist", C.c_double, 0),
    "std_a": ("lmot_tp_std_a", C.c_double, 3), "std_yawdd": ("lmot_tp_std_yawdd", C.c_double, 3),
    "std_las_x": (("lmot_tp_std_las", 0), C.c_double, 0), "std_las_y": (("lmot_tp_std_las", 1), C.c_double, 0),
    "trans": ("lmot_tp_trans", C.c_double, 9), "mode_prob0": ("lmot_tp_mode_prob0", C.c_double, 3),
    "p0_diag": ("lmot_tp_p0_diag", C.c_double, 5),
}


class RefTunable(_OracleBase):
    def __init__(self):
        super().__init__(ref_lib_path("tunable"), "ref_")
        self.mode = "tunable"
        self.defaults = self.get_tracker_params()

    def _var(self, field):
        sym, ct, n = GLOBALS[field]
        if isinstance(sym, tuple):
            return (ct * 2).in_dll(self.lib, sym[0]), sym[1]
        return (ct * n if n else ct).in_dll(self.lib, sym), None

    def get_tracker_params(self) -> dict:
        out = {}
        for f, (_, _, n) in GLOBALS.items():
            v, i = self._var(f)
            if i is not None:
                out[f] = v[i]
            elif n == 9:
                out[f] = [list(v[3 * r: 3 * r + 3]) for r in range(3)]
            elif n:
                out[f] = list(v)
            else:
                out[f] = v.value
        return out

    def set_tracker_params(self, params: dict | None = None):
        """every field of `params` (the defaults for the others; None: all defaults)"""
        full = dict(self.defaults)
        full.update(params or {})
        for f, val in full.items():
            v, i = self._var(f)
            n = GLOBALS[f][2]
            if i is not None:
                v[i] = float(val)
            elif n == 9:
                flat = [float(x) for row in val for x in row]
                for j in range(9):
                    v[j] = flat[j]
            elif n:
                for j in range(n):
                    v[j] = float(val[j])
            else:
                v.value = val
