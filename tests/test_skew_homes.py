"""The skewed-layout slots patch detection stores each cell to (gg_internal.h:skew_home).

k_detect derives a cell's slot from (x, y) in closed form and reads the per-cell homes table only for the cells the
layout marks as exceptions (ring corners, lane ends, the centre and the border ring).  Whatever path it takes, the slots
must be exactly those build_spiral_skew placed the cell at, for every map size that runs the skewed spiral.
"""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi
from test_host_logic import host_spiral_skew
from test_spiral_layouts import LAYOUTS


def skew_homes(n):
    fn = capi.load().gg_host_skew_homes
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    homes = np.full(n * n * 4, -7, np.int32)
    n_table = C.c_int(-1)
    ok = fn(n, homes.ctypes.data, C.byref(n_table))
    return (homes.reshape(n * n, 4), n_table.value) if ok else (None, 0)


def regular_home(n, t, x, y):
    """The closed form, written out once more: ring k = Chebyshev distance from the centre minus one; the side and the
    position j along it as the sequential sweep walks the ring; level 3 k + (0, 2, 3, 5)[side] + j."""
    c = n // 2 - 1
    k = max(abs(x - c), abs(y - c)) - 1
    if k < 0 or k > t["K"]:
        return -1
    p, q = c - 1 - k, c + 1 + k
    if x == p and y < q:
        s, j = 0, y - p
    elif y == p and x < q:
        s, j = 1, x - p
    elif x == q:
        s, j = 2, q - y
    else:
        s, j = 3, q - x
    return (s * t["rows"] + 3 * k + (0, 2, 3, 5)[s] + j + t["row0"]) * t["KP"] + k + 1


SKEW_SIZES = sorted({n for lo, hi, kind, *_ in LAYOUTS if kind == "skew" for n in (lo, hi)})


@pytest.mark.parametrize("n", SKEW_SIZES)
def test_derived_homes_match_the_homes_table(n):
    t = host_spiral_skew(n)
    assert t is not None
    homes, n_table = skew_homes(n)
    assert homes is not None
    assert np.array_equal(homes, t["home"])
    # the table path is the exception: about six cells per ring (two corners, the last cells of side 3) and the border
    assert 0 < n_table <= 8 * n


@pytest.mark.parametrize("n", [14, 15, 100, 101, 300, 301, 364, 600])
def test_closed_form_covers_every_single_home_cell_off_the_lane_ends(n):
    """Away from the innermost rings, the ring corners and the ends of the lanes, every cell has one home, and it is
    the closed-form slot."""
    t = host_spiral_skew(n)
    home = t["home"]
    c = n // 2 - 1
    checked = 0
    for y in range(n):
        for x in range(n):
            k = max(abs(x - c), abs(y - c)) - 1
            if k < 4 or k >= t["K"]:   # the innermost rings start irregularly
                continue
            p, q = c - 1 - k, c + 1 + k
            along = y - p if x in (p, q) else x - p
            if along < 6 or along > q - p - 6:   # near a corner: lane ends and double visits
                continue
            assert tuple(home[x + y * n]) == (regular_home(n, t, x, y), -1, -1, -1), (n, x, y)
            checked += 1
    assert checked > n * n // 2 or n < 20


def test_maps_without_a_skewed_layout_have_no_homes():
    for n in (3, 8, 13):
        assert skew_homes(n)[0] is None
