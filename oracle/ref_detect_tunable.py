"""TEST INFRASTRUCTURE ONLY -- ctypes binding to oracle/_ref/libref_detect_tunable.so (oracle/detect_tunable.mk).

RefDetectTunable() is RefOracle("intended") with the two detection literals (ground_removal.cpp:239 `+ 0.25`, box_fitting.cpp:100
`< 30`) in globals.  detect_params(values) sets lmot_detect_params fields -- by their lmot names -- in the reference's globals for the
duration of a `with` block: the reference's own mutable globals (rMin, roiM, ramPoints, ...; picScale, a dynamic initialiser of roiM,
follows roiM) and the two globals of this build.  The previous values come back afterwards.
"""
from __future__ import annotations

import contextlib
import ctypes as C

import numpy as np

from oracle.ref import _OracleBase, ref_lib_path, have_ref  # noqa: F401  (have_ref: callers test have_ref("detect_tunable"))

# lmot_detect_params field -> (global, ctype)
GLOBALS = {
    "r_min": ("rMin", C.c_float), "r_max": ("rMax", C.c_float), "t_hmin": ("tHmin", C.c_float), "t_hmax": ("tHmax", C.c_float),
    "t_hdiff": ("tHDiff", C.c_float), "h_sensor": ("hSeonsor", C.c_float), "roi_m": ("roiM", C.c_float),
    "ram_points": ("ramPoints", C.c_int), "l_slope_dist": ("lSlopeDist", C.c_int), "l_num_points": ("lnumPoints", C.c_int),
    "sensor_height": ("sensorHeight", C.c_float), "t_height_min": ("tHeightMin", C.c_float), "t_height_max": ("tHeightMax", C.c_float),
    "t_width_min": ("tWidthMin", C.c_float), "t_width_max": ("tWidthMax", C.c_float), "t_len_min": ("tLenMin", C.c_float),
    "t_len_max": ("tLenMax", C.c_float), "t_area_max": ("tAreaMax", C.c_float), "t_ratio_min": ("tRatioMin", C.c_float),
    "t_ratio_max": ("tRatioMax", C.c_float), "min_len_ratio": ("minLenRatio", C.c_float), "t_pt_per_m3": ("tPtPerM3", C.c_float),
    "ground_tolerance": ("lmot_dp_ground_tolerance", C.c_double), "min_cluster_points": ("lmot_dp_min_cluster_points", C.c_int),
}


class RefDetectTunable(_OracleBase):
    def __init__(self):
        super().__init__(ref_lib_path("detect_tunable"), "ref_")
        self.mode = "detect_tunable"

    def var(self, field):
        name, ct = GLOBALS[field]
        return ct.in_dll(self.lib, name)

    @contextlib.contextmanager
    def detect_params(self, values: dict):
        unknown = set(values) - set(GLOBALS)
        if unknown:
            raise ValueError(f"no reference global for {sorted(unknown)}")
        g = {k: self.var(k) for k in values}
        pic = C.c_float.in_dll(self.lib, "picScale")
        saved = {k: v.value for k, v in g.items()}
        saved_pic = pic.value
        for k, v in values.items():
            g[k].value = v
        if "roi_m" in values:
            pic.value = float(np.float32(900) / np.float32(values["roi_m"]))     # float picScale = 900/roiM, box_fitting.cpp:18
        try:
            yield self
        finally:
            for k, v in saved.items():
                g[k].value = v
            pic.value = saved_pic
