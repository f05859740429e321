"""The cell-shift resolve of gg_update_poses_from_device (gg_internal.h:resolve_move, run by k_pose_resolve on the
device and exported for the host as gg_host_resolve_move), against the host roll's own arithmetic (gg_host_move_map),
bit for bit; and the ctypes image of gg_scan_desc against the C header.  No GPU needed."""
import os
import subprocess

import numpy as np
import pytest

from groundgrid_b200 import capi

RES = float(np.float32(0.33))
FAR = (0.0, 1.0e5, -3.4e5, 1.2e6, 5.6e6, -6.0e6)


def neighbours(x, steps=3):
    """x and its `steps` nextafter neighbours on either side."""
    out = [x]
    lo = hi = x
    for _ in range(steps):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        out += [lo, hi]
    return out


def same_as_host(res, pos, target):
    status, p_dev, s_dev = capi.host_resolve_move(res, pos, target)
    moved, p_host, s_host = capi.host_move_map(res, pos, target)
    assert status == int(moved), f"{pos} -> {target}: status {status}, host moved {moved}"
    assert p_dev.view(np.uint64).tolist() == p_host.view(np.uint64).tolist(), f"{pos} -> {target}: position bits"
    assert s_dev == s_host, f"{pos} -> {target}: shift {s_dev} != {s_host}"
    return status, s_dev


@pytest.mark.parametrize("res", [RES, 0.2, 1.0])
@pytest.mark.parametrize("far", FAR)
def test_half_cell_boundaries_match_the_host_roll(res, far):
    """Targets at the nextafter neighbours of every half-cell boundary in [-12.5, 12.5] cells, around map positions up to
    6e6 m from the origin (where one ulp of a position is a large share of a cell)."""
    rng = np.random.default_rng(int(abs(far)) + int(res * 100))
    pos = np.array([far + rng.uniform(-1, 1), -far + rng.uniform(-1, 1)])
    rounded = {-1: 0, 0: 0, 1: 0}
    for m in range(-13, 13):
        edge_x = pos[0] + (m + 0.5) * res
        edge_y = pos[1] + (-m - 0.5) * res
        for nx in neighbours(edge_x):
            for ny in (pos[1], edge_y):
                status, shift = same_as_host(res, pos, (nx, ny))
                rounded[int(np.sign(shift[0]))] += 1
        for ny in neighbours(edge_y):
            same_as_host(res, pos, (pos[0], ny))
    assert rounded[-1] and rounded[1] and rounded[0], "targets on both sides of the map position and at it"


@pytest.mark.parametrize("far", FAR)
def test_whole_map_jumps_and_random_targets_match_the_host_roll(far):
    rng = np.random.default_rng(77)
    N = capi.host_cells_per_side(120.0, 0.33)
    pos = np.array([far, far * 0.5])
    for k in (1, 2, 3, 10, 1000):
        for sx, sy in ((1, 0), (0, -1), (-1, 1), (1, 1)):
            status, shift = same_as_host(RES, pos, (pos[0] + sx * k * N * RES, pos[1] + sy * k * N * RES))
            assert status == 1 and abs(shift[0]) + abs(shift[1]) >= k * N - 1
    for _ in range(500):
        target = pos + rng.uniform(-40, 40, 2) * rng.choice([0.01, 1.0, 100.0])
        same_as_host(RES, pos, target)
    assert same_as_host(RES, pos, pos) == (0, (0, 0)), "no move: status 0"


@pytest.mark.parametrize("target", [(np.nan, 0.0), (0.0, np.nan), (np.inf, 0.0), (0.0, -np.inf), (np.inf, np.nan),
                                    (1.0e9, 0.0), (0.0, -1.0e9), (1.0e300, 1.0e300), (-2147483648.0 * RES, 0.0)])
def test_invalid_poses_report_minus_one_and_change_nothing(target):
    pos = np.array([12.25, -7.5])
    status, p, shift = capi.host_resolve_move(RES, pos, (pos[0] + target[0], pos[1] + target[1]))
    assert status == -1
    assert p.view(np.uint64).tolist() == pos.view(np.uint64).tolist() and shift == (0, 0)


def test_largest_int32_shift_is_valid_and_one_more_is_not():
    """With res = 1 the quotient is exact: a rounded shift of 2^31 - 1 cells resolves, 2^31 does not (its negation, the
    buffer shift, would not fit either)."""
    for t, valid in ((2147483647.4, True), (2147483647.6, False), (-2147483647.4, True), (-2147483647.6, False)):
        status, _, shift = capi.host_resolve_move(1.0, (0.0, 0.0), (t, 0.0))
        assert (status != -1) == valid, t
        if valid:
            assert same_as_host(1.0, np.zeros(2), (t, 0.0))[1] == shift


HEADER_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "groundgrid_b200.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu %d\n", sizeof(gg_scan_desc), offsetof(gg_scan_desc, slot), offsetof(gg_scan_desc, flags),
           offsetof(gg_scan_desc, n_points), offsetof(gg_scan_desc, origin), offsetof(gg_scan_desc, base_z), GG_SCAN_DEVICE_POSE);
    return 0;
}
"""


def test_scan_desc_binding_matches_the_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(HEADER_PROBE)
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)], check=True)
    size, o_slot, o_flags, o_n, o_origin, o_base_z, flag = map(int, subprocess.run([str(exe)], check=True, capture_output=True,
                                                                                    text=True).stdout.split())
    S = capi.ScanDesc
    assert capi.C.sizeof(S) == size == capi.SCAN_DESC_DTYPE.itemsize
    assert (S.slot.offset, S.flags.offset, S.n_points.offset, S.origin.offset, S.base_z.offset) == (o_slot, o_flags, o_n, o_origin, o_base_z)
    f = capi.SCAN_DESC_DTYPE.fields
    assert (f["slot"][1], f["flags"][1], f["n_points"][1], f["origin"][1], f["base_z"][1]) == (o_slot, o_flags, o_n, o_origin, o_base_z)
    assert capi.SCAN_DEVICE_POSE == flag
    descs = capi.GroundGridB200._device_descs([3, 1], [10, 20], "device", None)
    assert descs["flags"].tolist() == [flag, flag] and descs["origin"].tolist() == [[0.0] * 3] * 2
