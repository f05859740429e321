"""The ctypes images of gg_device_configs (capi.DeviceConfigs) and gg_config (capi.Config) against the C header, compiled
with the host C compiler; and config_tensor / config_field on CPU tensors against bytes(capi.Config).  No GPU needed."""
import math
import os
import subprocess

import numpy as np
import pytest

from groundgrid_b200 import capi

torch = pytest.importorskip("torch")

CONFIG_FIELDS = [name for name, _ in capi.Config._fields_]

HEADER_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "groundgrid_b200.h"
#define OFF(s, f) printf(" %zu", offsetof(s, f))
int main(void) {
    printf("%zu %zu", sizeof(gg_device_configs), sizeof(gg_config));
    OFF(gg_device_configs, cfg); OFF(gg_device_configs, mask);
%s
    printf("\n");
    return 0;
}
"""


def test_device_configs_binding_matches_the_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(HEADER_PROBE.replace("%s", "\n".join(f"    OFF(gg_config, {f});" for f in CONFIG_FIELDS)))
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)], check=True)
    vals = list(map(int, subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()))
    dc_size, cfg_size, dc_off, cfg_off = vals[0], vals[1], vals[2:4], vals[4:]
    D = capi.DeviceConfigs
    assert capi.C.sizeof(D) == dc_size
    assert [D.cfg.offset, D.mask.offset] == dc_off
    assert [name for name, _ in D._fields_] == ["cfg", "mask"]
    assert capi.C.sizeof(capi.Config) == cfg_size == 104
    assert [getattr(capi.Config, f).offset for f in CONFIG_FIELDS] == cfg_off


def _configs():
    a = capi.default_config()
    b = capi.default_config()
    b.outlier_tolerance = math.nan
    b.max_ring = -3
    b.point_count_cell_variance_threshold = 2**31 - 1
    b.patch_size_change_distance = -math.inf
    return [a, b, {"occupied_cells_decrease_factor": 0.5, "distance_factor": math.inf}, {}]


def test_config_tensor_round_trips_to_the_struct_bytes():
    cfgs = _configs()
    t = capi.config_tensor(cfgs, device="cpu")
    assert t.dtype == torch.uint8 and tuple(t.shape) == (4, capi.C.sizeof(capi.Config))
    want = []
    for c in cfgs:
        if isinstance(c, dict):
            d, c = c, capi.default_config()
            for k, v in d.items():
                setattr(c, k, v)
        want.append(bytes(c))
    assert [bytes(row.numpy().tobytes()) for row in t] == want
    assert capi.config_tensor([], device="cpu").shape == (0, 104)
    with pytest.raises(KeyError):
        capi.config_tensor([{"no_such_field": 1}], device="cpu")


def test_config_field_views_write_the_struct_fields():
    t = capi.config_tensor([capi.default_config()] * 3, device="cpu")
    for name, ctype in capi.Config._fields_:
        f = capi.config_field(t, name)
        assert f.shape == (3,)
        assert f.dtype == (torch.int32 if ctype is capi.C.c_int else torch.float64)
    capi.config_field(t, "outlier_tolerance").copy_(torch.tensor([0.05, math.nan, -math.inf], dtype=torch.float64))
    capi.config_field(t, "max_ring").copy_(torch.tensor([0, -1, 2**31 - 1], dtype=torch.int32))
    capi.config_field(t, "min_outlier_detection_ground_confidence").fill_(2.5)
    for k, (tol, ring) in enumerate([(0.05, 0), (math.nan, -1), (-math.inf, 2**31 - 1)]):
        c = capi.default_config()
        c.outlier_tolerance = tol
        c.max_ring = ring
        c.min_outlier_detection_ground_confidence = 2.5
        assert t[k].numpy().tobytes() == bytes(c)
    with pytest.raises(ValueError):
        capi.config_field(t[:, :100], "max_ring")
    with pytest.raises(ValueError):
        capi.config_field(t.to(torch.int16), "max_ring")


def test_host_constants_unchanged_by_the_shared_derivation():
    # the host derivation now lives in the header shared with the device; its constants are the reference's expressions
    c = capi.default_config()
    k = capi.host_config_constants(c)
    assert k["df_sq"] == c.distance_factor * c.distance_factor
    m10 = c.minimum_distance_factor * 10
    assert k["mdf10_sq"] == m10 * m10
    assert k["occ_factor2"] == c.occupied_cells_point_count_factor * float(np.float32(2.0))
    assert k["lab_fac"] == c.minimum_distance_factor * 5
    o = float(np.float32(0.001))
    assert k["decay_floor_ok"] == (1.0 if (c.occupied_cells_decrease_factor >= 1.0 and o - o / c.occupied_cells_decrease_factor < 0.000999) else 0.0)
