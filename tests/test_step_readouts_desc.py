"""The ctypes image of gg_step_readouts (capi.StepReadouts) against the C header: size, every field offset and the field
order, compiled with the host C compiler.  No GPU needed."""
import os
import subprocess

from groundgrid_b200 import capi

FIELDS = ("n_layer_names", "layer_names", "layers", "n_image_names", "image_names", "images", "image_ranges", "terrain_images",
          "n_sample_names", "sample_names", "samples", "sample_mode", "point_info", "eval_counts")

HEADER_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "groundgrid_b200.h"
#define OFF(f) printf(" %zu", offsetof(gg_step_readouts, f))
int main(void) {
    printf("%zu", sizeof(gg_step_readouts));
    OFF(n_layer_names); OFF(layer_names); OFF(layers); OFF(n_image_names); OFF(image_names); OFF(images); OFF(image_ranges);
    OFF(terrain_images); OFF(n_sample_names); OFF(sample_names); OFF(samples); OFF(sample_mode); OFF(point_info);
    OFF(eval_counts);
    printf("\n");
    return 0;
}
"""


def test_step_readouts_binding_matches_the_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(HEADER_PROBE)
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)], check=True)
    vals = list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    size, offsets = vals[0], vals[1:]
    S = capi.StepReadouts
    assert capi.C.sizeof(S) == size
    assert [getattr(S, f).offset for f in FIELDS] == offsets
    assert [name for name, _ in S._fields_] == list(FIELDS)
