"""The ctypes image of gg_step_parts (capi.StepParts) against the C header: size, every field offset and the field order,
compiled with the host C compiler; and the new scan flag's value.  No GPU needed."""
import os
import subprocess

from groundgrid_b200 import capi

FIELDS = ("n_parts", "parts", "dev_T_map_from_part", "dev_part_counts", "parts_per_slot")

HEADER_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "groundgrid_b200.h"
#define OFF(f) printf(" %zu", offsetof(gg_step_parts, f))
int main(void) {
    printf("%zu %d %d", sizeof(gg_step_parts), GG_SCAN_DEVICE_PART_COUNTS, GG_MAX_CLOUD_PARTS);
    OFF(n_parts); OFF(parts); OFF(dev_T_map_from_part); OFF(dev_part_counts); OFF(parts_per_slot);
    printf("\n");
    return 0;
}
"""


def test_step_parts_binding_matches_the_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(HEADER_PROBE)
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)], check=True)
    vals = list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    size, flag, max_parts, offsets = vals[0], vals[1], vals[2], vals[3:]
    S = capi.StepParts
    assert capi.C.sizeof(S) == size
    assert [getattr(S, f).offset for f in FIELDS] == offsets
    assert [name for name, _ in S._fields_] == list(FIELDS)
    assert capi.SCAN_DEVICE_PART_COUNTS == flag and capi.MAX_CLOUD_PARTS == max_parts
    assert flag & (capi.SCAN_DEVICE_POSE | capi.SCAN_DEVICE_COUNT) == 0
