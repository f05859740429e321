"""The scan-mask flag and the two scan-mask calls of the Python bindings (capi.SCAN_DEVICE_MASK,
gg_set_scan_masks_from_device, gg_step_plan_create_with_scan_masks) against the C header, compiled with the host C
compiler.  No GPU needed."""
import ctypes as C
import os
import subprocess

from groundgrid_b200 import capi

HEADER_PROBE = r"""
#include <stdio.h>
#include "groundgrid_b200.h"
/* the prototypes the bindings assume: a mismatch does not compile (-Werror) */
static int (*set_fn)(gg_handle, int, const int*, const int32_t*, void*) = gg_set_scan_masks_from_device;
static int (*plan_fn)(gg_handle, const gg_step_desc*, const gg_step_parts*, const gg_device_resets*, const gg_device_configs*,
                      const gg_step_snapshots*, const gg_step_readouts*, const int32_t*, gg_step_plan*) = gg_step_plan_create_with_scan_masks;
int main(void) {
    (void)set_fn; (void)plan_fn;
    printf("%d %d %d %d\n", GG_SCAN_DEVICE_POSE, GG_SCAN_DEVICE_COUNT, GG_SCAN_DEVICE_PART_COUNTS, GG_SCAN_DEVICE_MASK);
    return 0;
}
"""


def probe(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(HEADER_PROBE)
    subprocess.run(["gcc", "-Werror", "-I", os.path.join(root, "include"), "-c", "-o", str(exe) + ".o", str(src)], check=True)
    # link without the library: the probe only takes the functions' addresses, so stub them in a second unit
    stub = tmp_path / "stub.c"
    stub.write_text("#include \"groundgrid_b200.h\"\n"
                    "int gg_set_scan_masks_from_device(gg_handle h, int c, const int* s, const int32_t* m, void* st) { return 0; }\n"
                    "int gg_step_plan_create_with_scan_masks(gg_handle h, const gg_step_desc* d, const gg_step_parts* p,\n"
                    "    const gg_device_resets* r, const gg_device_configs* c, const gg_step_snapshots* s, const gg_step_readouts* o,\n"
                    "    const int32_t* m, gg_step_plan* out) { return 0; }\n")
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(exe) + ".o", str(stub)], check=True)
    return list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))


def test_scan_flags_match_the_header(tmp_path):
    pose, count, parts, mask = probe(tmp_path)
    assert (capi.SCAN_DEVICE_POSE, capi.SCAN_DEVICE_COUNT, capi.SCAN_DEVICE_PART_COUNTS, capi.SCAN_DEVICE_MASK) == (pose, count, parts, mask)
    assert mask == 8
    # one bit each, so any combination can be flagged on one scan
    assert len({pose, count, parts, mask}) == 4 and all(f & (f - 1) == 0 for f in (pose, count, parts, mask))


def test_binding_argtypes():
    L = capi.load(build_if_missing=False)
    vp, i = C.c_void_p, C.c_int
    assert L.gg_set_scan_masks_from_device.restype is i
    assert L.gg_set_scan_masks_from_device.argtypes == [vp, i, vp, vp, vp]
    assert L.gg_step_plan_create_with_scan_masks.restype is i
    assert L.gg_step_plan_create_with_scan_masks.argtypes == [vp, C.POINTER(capi.StepDesc), C.POINTER(capi.StepParts), C.POINTER(capi.DeviceResets),
                                                              C.POINTER(capi.DeviceConfigs), C.POINTER(capi.StepSnapshots),
                                                              C.POINTER(capi.StepReadouts), vp, C.POINTER(vp)]


def test_null_handle_is_rejected_without_a_device():
    L = capi.load(build_if_missing=False)
    assert L.gg_set_scan_masks_from_device(None, 1, None, None, None) == -1
    p = C.c_void_p()
    assert L.gg_step_plan_create_with_scan_masks(None, None, None, None, None, None, None, None, C.byref(p)) == -1 and not p.value


def test_device_descs_flag_the_masks():
    """What the scan calls hand the C API: device_masks adds the flag to the others, never replaces them."""
    d = capi.GroundGridB200._device_descs([3, 5], [10, 20], "device", None, device_counts=True, device_masks=True)
    assert list(d["flags"]) == [capi.SCAN_DEVICE_COUNT | capi.SCAN_DEVICE_POSE | capi.SCAN_DEVICE_MASK] * 2
    d = capi.GroundGridB200._device_descs([3], [10], [[0.0, 0.0, 1.0]], 0.5, device_masks=True)
    assert list(d["flags"]) == [capi.SCAN_DEVICE_MASK]
    d = capi.GroundGridB200._device_descs([3], [10], [[0.0, 0.0, 1.0]], 0.5)
    assert list(d["flags"]) == [0]
