"""TEST INFRASTRUCTURE ONLY -- the oracle of track retirement (lmot_set_track_retirement).

retirer(oracle) -> a callable that stably erases the tracks with trackNumVec_ == 0 from the reference table `oracle` steps
(RefOracle("intended") or RefTunable()), through oracle/_ref/libref_retire_<mode>.so (oracle/retire.mk, oracle/ref_retire.cpp).
The ego state is not touched.  Only tests/ and scripts may import this.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def _mode(oracle) -> str:
    name = os.path.basename(oracle.lib._name)          # libref_<mode>.so
    if not (name.startswith("libref_") and name.endswith(".so")):
        raise ValueError(f"{name}: not a reference library (retirement needs the reference's own table)")
    return name[len("libref_"):-len(".so")]


def retire_lib_path(mode: str) -> str:
    return os.path.join(HERE, "_ref", f"libref_retire_{mode}.so")


def have_retire(mode: str = "intended") -> bool:
    return os.path.exists(retire_lib_path(mode))


def retirer(oracle):
    """ref_tracker_retire on `oracle`'s table (the library must already be loaded: the helper binds to that instance)"""
    lib = C.CDLL(retire_lib_path(_mode(oracle)))
    fn = lib.ref_tracker_retire
    fn.argtypes = []
    fn.restype = None
    return fn
