"""The ctypes image of gg_step_desc (capi.StepDesc) against the C header: size and every field offset, compiled with the
host C compiler.  No GPU needed."""
import os
import subprocess

from groundgrid_b200 import capi

FIELDS = ("count", "scans", "dev_points", "msgs", "dev_T_map_from_frame", "dev_n_points", "poses", "dev_moved", "outs", "select",
          "dev_counts")

HEADER_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "groundgrid_b200.h"
#define OFF(f) printf(" %zu", offsetof(gg_step_desc, f))
int main(void) {
    printf("%zu %zu", sizeof(gg_step_desc), sizeof(gg_device_poses));
    OFF(count); OFF(scans); OFF(dev_points); OFF(msgs); OFF(dev_T_map_from_frame); OFF(dev_n_points); OFF(poses);
    OFF(dev_moved); OFF(outs); OFF(select); OFF(dev_counts);
    printf("\n");
    return 0;
}
"""


def test_step_desc_binding_matches_the_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(HEADER_PROBE)
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)], check=True)
    vals = list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    size, poses_size, offsets = vals[0], vals[1], vals[2:]
    S = capi.StepDesc
    assert capi.C.sizeof(S) == size
    assert capi.C.sizeof(capi.DevicePoses) == poses_size
    assert [getattr(S, f).offset for f in FIELDS] == offsets
    assert [name for name, _ in S._fields_] == list(FIELDS)
