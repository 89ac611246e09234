"""TEST INFRASTRUCTURE ONLY -- the oracle of track prediction (lmot_predict_tracks).

predictor(oracle) -> a callable predict(t_us, cap=None) -> dict with the layout of Lmot.predict_tracks (without ids: the reference
numbers nothing), computed on copies of the rows of the reference table `oracle` steps (RefOracle("intended") or RefTunable()) by
the reference's own ProcessIMMUKF / findMaxZandS / PostProcessIMMUKF, through oracle/_ref/libref_predict_<mode>.so
(oracle/predict.mk, oracle/ref_predict.cpp).  The table is not written.  Only tests/ and scripts may import this.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _mode(oracle) -> str:
    name = os.path.basename(oracle.lib._name)          # libref_<mode>.so
    if not (name.startswith("libref_") and name.endswith(".so")):
        raise ValueError(f"{name}: not a reference library (prediction needs the reference's own table)")
    return name[len("libref_"):-len(".so")]


def predict_lib_path(mode: str) -> str:
    return os.path.join(HERE, "_ref", f"libref_predict_{mode}.so")


def have_predict(mode: str = "intended") -> bool:
    return os.path.exists(predict_lib_path(mode))


def predictor(oracle):
    """ref_tracker_predict on `oracle`'s table (the library must already be loaded: the helper binds to that instance)"""
    lib = C.CDLL(predict_lib_path(_mode(oracle)))
    fn = lib.ref_tracker_predict
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 7
    fn.restype = C.c_int

    def predict(t_us, cap: int | None = None) -> dict:
        t = np.ascontiguousarray(np.atleast_1d(np.asarray(t_us, np.float64)))
        n_t = int(t.shape[0])
        if cap is None:
            cap = oracle.tracker_num_tracks()
        r = {"track_manage": np.zeros(cap, np.int32), "flags": np.zeros((n_t, cap), np.uint8),
             "x": np.zeros((n_t, cap, 5)), "P": np.zeros((n_t, cap, 5, 5)), "mode_prob": np.zeros((n_t, cap, 3)),
             "gate_z": np.zeros((n_t, cap, 2)), "gate_S": np.zeros((n_t, cap, 4))}
        n = fn(t.ctypes.data, n_t, cap, *(r[k].ctypes.data for k in ("track_manage", "flags", "x", "P", "mode_prob", "gate_z", "gate_S")))
        m = min(n, cap)
        return {k: (a[:m] if k == "track_manage" else a[:, :m]) for k, a in r.items()}

    return predict
