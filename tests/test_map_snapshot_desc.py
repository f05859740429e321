"""The ctypes images of the map snapshot header and of the snapshot call arguments (capi.MapSnapshot, MapRestore,
StepSnapshots) against the C header, the record-size formula, and the argument types of the new bindings, compiled with
the host C compiler.  No GPU needed."""
import ctypes as C
import os
import subprocess

from groundgrid_b200 import capi

SNAPSHOT_FIELDS = ("magic", "version", "cells_per_side", "resolution", "position", "reserved")
RESTORE_FIELDS = ("pool", "n_pool", "index", "status")
STEP_FIELDS = ("restore", "save", "save_mask")

HEADER_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "groundgrid_b200.h"
/* the prototypes the bindings assume: a mismatch does not compile (-Werror) */
static size_t (*bytes_fn)(gg_handle) = gg_map_snapshot_bytes;
static int (*save_fn)(gg_handle, int, const int*, void*, const int32_t*, void*) = gg_save_maps_to_device;
static int (*restore_fn)(gg_handle, int, const int*, const gg_map_restore*, void*) = gg_restore_maps_from_device;
static int (*plan_fn)(gg_handle, const gg_step_desc*, const gg_step_parts*, const gg_device_resets*, const gg_device_configs*,
                      const gg_step_snapshots*, const gg_step_readouts*, gg_step_plan*) = gg_step_plan_create_with_snapshots;
#define OFF(t, f) printf(" %zu", offsetof(t, f))
int main(void) {
    (void)bytes_fn; (void)save_fn; (void)restore_fn; (void)plan_fn;
    printf("%zu %u %d", sizeof(gg_map_snapshot), GG_SNAPSHOT_MAGIC, GG_SNAPSHOT_VERSION);
    OFF(gg_map_snapshot, magic); OFF(gg_map_snapshot, version); OFF(gg_map_snapshot, cells_per_side);
    OFF(gg_map_snapshot, resolution); OFF(gg_map_snapshot, position); OFF(gg_map_snapshot, reserved);
    printf(" %zu", sizeof(gg_map_restore));
    OFF(gg_map_restore, pool); OFF(gg_map_restore, n_pool); OFF(gg_map_restore, index); OFF(gg_map_restore, status);
    printf(" %zu", sizeof(gg_step_snapshots));
    OFF(gg_step_snapshots, restore); OFF(gg_step_snapshots, save); OFF(gg_step_snapshots, save_mask);
    printf("\n");
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
                    "size_t gg_map_snapshot_bytes(gg_handle h) { (void)h; return 0; }\n"
                    "int gg_save_maps_to_device(gg_handle h, int c, const int* s, void* d, const int32_t* m, void* st) { return 0; }\n"
                    "int gg_restore_maps_from_device(gg_handle h, int c, const int* s, const gg_map_restore* r, void* st) { return 0; }\n"
                    "int gg_step_plan_create_with_snapshots(gg_handle h, const gg_step_desc* d, const gg_step_parts* p, const gg_device_resets* r,\n"
                    "    const gg_device_configs* c, const gg_step_snapshots* s, const gg_step_readouts* o, gg_step_plan* out) { return 0; }\n")
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(exe) + ".o", str(stub)], check=True)
    return list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))


def test_snapshot_bindings_match_the_header(tmp_path):
    v = probe(tmp_path)
    size, magic, version = v[:3]
    assert size == 64 == C.sizeof(capi.MapSnapshot)
    assert magic == capi.SNAPSHOT_MAGIC and version == capi.SNAPSHOT_VERSION
    assert magic.to_bytes(4, "little") == b"GGMS"
    assert [getattr(capi.MapSnapshot, f).offset for f in SNAPSHOT_FIELDS] == v[3:9] == [0, 4, 8, 12, 16, 32]
    assert [name for name, _ in capi.MapSnapshot._fields_] == list(SNAPSHOT_FIELDS)
    assert C.sizeof(capi.MapRestore) == v[9]
    assert [getattr(capi.MapRestore, f).offset for f in RESTORE_FIELDS] == v[10:14]
    assert [name for name, _ in capi.MapRestore._fields_] == list(RESTORE_FIELDS)
    assert C.sizeof(capi.StepSnapshots) == v[14]
    assert [getattr(capi.StepSnapshots, f).offset for f in STEP_FIELDS] == v[15:18]
    assert [name for name, _ in capi.StepSnapshots._fields_] == list(STEP_FIELDS)


def test_record_size_formula():
    """64 + 8 * N2p with N2p = N * N rounded up to a multiple of 4: every record, and every plane in it, 16-byte aligned."""
    for n, want in ((1, 96), (2, 96), (3, 64 + 8 * 12), (55, 64 + 8 * 3028), (300, 720064), (364, 64 + 8 * 132496), (4096, 64 + 8 * 4096 * 4096)):
        assert capi.snapshot_bytes(n) == want, n
        assert want % 16 == 0 and (4 * ((n * n + 3) // 4 * 4)) % 16 == 0


def test_binding_argtypes():
    L = capi.load(build_if_missing=False)
    vp, i = C.c_void_p, C.c_int
    assert L.gg_map_snapshot_bytes.restype is C.c_size_t and L.gg_map_snapshot_bytes.argtypes == [vp]
    assert L.gg_save_maps_to_device.argtypes == [vp, i, vp, vp, vp, vp]
    assert L.gg_restore_maps_from_device.argtypes == [vp, i, vp, C.POINTER(capi.MapRestore), vp]
    assert L.gg_step_plan_create_with_snapshots.argtypes == [vp, C.POINTER(capi.StepDesc), C.POINTER(capi.StepParts), C.POINTER(capi.DeviceResets),
                                                             C.POINTER(capi.DeviceConfigs), C.POINTER(capi.StepSnapshots),
                                                             C.POINTER(capi.StepReadouts), C.POINTER(vp)]


def test_null_handle_is_rejected_without_a_device():
    L = capi.load(build_if_missing=False)
    assert L.gg_map_snapshot_bytes(None) == 0
    assert L.gg_save_maps_to_device(None, 1, None, None, None, None) == -1
    r = capi.MapRestore(None, -1, None, None)
    assert L.gg_restore_maps_from_device(None, 1, None, C.byref(r), None) == -1
    p = C.c_void_p()
    assert L.gg_step_plan_create_with_snapshots(None, None, None, None, None, None, None, C.byref(p)) == -1 and not p.value


def test_step_snapshots_marshalling():
    """What step_plan hands the C call: the restore inside the struct, the save pointers after it."""
    s = capi.StepSnapshots()
    s.restore = capi.MapRestore(0x1000, 7, 0x2000, 0x3000)
    s.save, s.save_mask = 0x4000, 0x5000
    raw = bytes(s)
    words = [int.from_bytes(raw[o:o + 8], "little") for o in range(0, len(raw), 8)]
    assert words[0] == 0x1000 and (words[1] & 0xFFFFFFFF) == 7 and words[2:] == [0x2000, 0x3000, 0x4000, 0x5000]
