"""The ctypes image of gg_device_resets (capi.DeviceResets) against the C header: size and every field offset, compiled
with the host C compiler.  No GPU needed."""
import os
import subprocess

from groundgrid_b200 import capi

FIELDS = ("xyz", "mask")

HEADER_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "groundgrid_b200.h"
int main(void) {
    printf("%zu %zu %zu\n", sizeof(gg_device_resets), offsetof(gg_device_resets, xyz), offsetof(gg_device_resets, mask));
    return 0;
}
"""


def test_device_resets_binding_matches_the_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(HEADER_PROBE)
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)], check=True)
    size, *offsets = map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split())
    R = capi.DeviceResets
    assert capi.C.sizeof(R) == size
    assert [getattr(R, f).offset for f in FIELDS] == offsets
    assert [name for name, _ in R._fields_] == list(FIELDS)
