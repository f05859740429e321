"""Configurations at the limits of every GroundGridConfig field (cfg/GroundGrid.cfg:8-21) and at the values a caller can
set beyond them: each double field at both ends of its cfg range and at 0, -0.0, -1, NaN, +inf and -inf; the int fields
at their cfg ends and at -7, INT_MIN and INT_MAX (max_ring also at 65535 and 65536, around the ring field's uint16 range);
every field at its cfg minimum and every field at its cfg maximum at once; and occupied_cells_decrease_factor at 0.5 and
on both sides of the switch of decay_confidence's floor shortcut (CfgConst::decay_floor_ok).

Every case keeps thread_count = 1: the reference's answer is defined there (more threads race, 0 divides by zero).
The fields come from capi.Config, so a field added later without a range here fails test_config_limits.py.

CPU only.
"""
import math

import numpy as np

from groundgrid_b200 import capi

INT_MIN, INT_MAX = -2**31, 2**31 - 1
# (min, max) of each field in cfg/GroundGrid.cfg:8-21
RANGES = {
    "point_count_cell_variance_threshold": (0, 30),
    "max_ring": (0, 1024),
    "groundpatch_detection_minimum_threshold": (0.0, 1.0),
    "distance_factor": (0.0, 0.01),
    "minimum_distance_factor": (0.0, 0.01),
    "miminum_point_height_threshold": (0.0, 1.0),
    "minimum_point_height_obstacle_threshold": (0.0, 0.2),
    "outlier_tolerance": (-0.5, 0.5),
    "ground_patch_detection_minimum_point_count_threshold": (0.01, 1.0),
    "patch_size_change_distance": (0.0, 50.0),
    "occupied_cells_decrease_factor": (1.0, 100.0),
    "occupied_cells_point_count_factor": (1.0, 50.0),
    "min_outlier_detection_ground_confidence": (0.0, 5.0),
    "thread_count": (1, 64),
}
FIELDS = [name for name, _ in capi.Config._fields_]
DOUBLES = [name for name, t in capi.Config._fields_ if t is capi.C.c_double]
INTS = [name for name, t in capi.Config._fields_ if t is capi.C.c_int and name != "thread_count"]
DOUBLE_VALUES = (0.0, -0.0, -1.0, math.nan, math.inf, -math.inf)
INT_VALUES = (-7, INT_MIN, INT_MAX)
DECAY = "occupied_cells_decrease_factor"
FLOOR = float(np.float32(0.001))


def decay_floor_ok(factor):
    """CfgConst::decay_floor_ok as derive_config computes it (gg_internal.h), in the same correctly rounded fp64 steps."""
    return factor >= 1.0 and (FLOOR - FLOOR / factor) < 0.000999


def decay_switch():
    """(below, above): the largest decrease factor that takes the floor shortcut and the next double, which does not.
    FLOOR - FLOOR / F rises with F, so the switch is found by bisection over the doubles between 1 and 10^4."""
    lo, hi = int(np.float64(1.0).view(np.int64)), int(np.float64(1e4).view(np.int64))
    assert decay_floor_ok(1.0) and not decay_floor_ok(1e4)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if decay_floor_ok(float(np.int64(mid).view(np.float64))):
            lo = mid
        else:
            hi = mid
    return float(np.int64(lo).view(np.float64)), float(np.int64(hi).view(np.float64))


def _name(cfg):
    return ",".join(f"{k}={v!r}" for k, v in cfg.items() if k != "thread_count")


def cases():
    """name -> {field: value} (thread_count = 1 in every case), in a fixed order."""
    out = []
    for f in DOUBLES:
        lo, hi = RANGES[f]
        for v in (lo, hi) + DOUBLE_VALUES:
            out.append({f: v})
    for f in INTS:
        lo, hi = RANGES[f]
        for v in (lo, hi) + INT_VALUES + ((65535, 65536) if f == "max_ring" else ()):
            out.append({f: v})
    out.append({f: RANGES[f][0] for f in FIELDS if f != "thread_count"})
    out.append({f: RANGES[f][1] for f in FIELDS if f != "thread_count"})
    below, above = decay_switch()
    out += [{DECAY: 0.5}, {DECAY: below}, {DECAY: above}]
    named = {}
    for c in out:
        key = _name(c) if len(c) == 1 else ("all at the cfg minimum" if c[DECAY] == RANGES[DECAY][0] else "all at the cfg maximum")
        # -0.0 == 0.0 and NaN != NaN: compare the names, which repr keeps apart
        named.setdefault(key, dict(c, thread_count=1))
    return named


CASES = cases()


def decay_factors():
    """Every decrease factor the cases set (the spiral paths run each of them)."""
    seen = {}
    for c in CASES.values():
        if len(c) == 2 and DECAY in c:
            seen.setdefault(repr(c[DECAY]), c[DECAY])
    return list(seen.values())
