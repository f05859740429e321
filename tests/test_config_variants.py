"""Per-slot configuration, host side: the split of the derived constants (geometry / configuration) and the
bookkeeping of configuration variants (gg_host.cpp:ConfigRegistry).  No device needed."""
import numpy as np

from groundgrid_b200 import capi


def random_config(rng):
    c = capi.default_config()
    c.point_count_cell_variance_threshold = int(rng.integers(1, 40))
    c.max_ring = int(rng.choice([16, 32, 48, 64, 128, 1024]))
    c.distance_factor = float(rng.uniform(1e-5, 1e-3))
    c.minimum_distance_factor = float(rng.uniform(1e-5, 2e-3))
    c.miminum_point_height_threshold = float(rng.uniform(0.05, 0.6))
    c.minimum_point_height_obstacle_threshold = float(rng.uniform(0.01, 0.3))
    c.outlier_tolerance = float(rng.uniform(0.0, 0.4))
    c.ground_patch_detection_minimum_point_count_threshold = float(rng.uniform(0.05, 0.6))
    c.patch_size_change_distance = float(rng.uniform(2.0, 40.0))
    c.occupied_cells_decrease_factor = float(rng.choice([0.5, 1.0, 1.5, 5.0, 20.0]))
    c.occupied_cells_point_count_factor = float(rng.uniform(2.0, 60.0))
    c.min_outlier_detection_ground_confidence = float(rng.uniform(0.2, 3.0))
    return c


def expected_config_constants(c):
    """The expressions of the single derive_constants the split replaced, restated (fp64, no FMA)."""
    f64 = np.float64
    dec = f64(c.occupied_cells_decrease_factor)
    o = f64(np.float32(0.001))
    m10 = f64(c.minimum_distance_factor) * 10
    return {
        "max_ring": c.max_ring,
        "pc_var_thresh_f": float(np.float32(c.point_count_cell_variance_threshold)),
        "min_outlier_conf": c.min_outlier_detection_ground_confidence,
        "outlier_tol": c.outlier_tolerance,
        "gp_thresh": c.ground_patch_detection_minimum_point_count_threshold,
        "df_sq": c.distance_factor * c.distance_factor,
        "mdf_sq": c.minimum_distance_factor * c.minimum_distance_factor,
        "mdf10_sq": float(m10 * m10),
        "psc_sq": c.patch_size_change_distance * c.patch_size_change_distance,
        "occ_factor": c.occupied_cells_point_count_factor,
        "occ_factor2": c.occupied_cells_point_count_factor * 2.0,
        "dec_factor": c.occupied_cells_decrease_factor,
        "lab_fac": c.minimum_distance_factor * 5,
        "lab_thres": c.miminum_point_height_threshold,
        "lab_obs": c.minimum_point_height_obstacle_threshold,
        "decay_floor_ok": 1 if (dec >= 1.0 and (o - o / dec) < 0.000999) else 0,
    }


def test_config_constants_match_the_unsplit_derivation_field_by_field():
    rng = np.random.default_rng(11)
    cfgs = [capi.default_config()] + [random_config(rng) for _ in range(40)]
    for c in cfgs:
        got, want = capi.host_config_constants(c), expected_config_constants(c)
        assert list(got) == list(want)
        for name in want:
            assert np.float64(got[name]).tobytes() == np.float64(want[name]).tobytes(), (name, got[name], want[name])
    floors = {capi.host_config_constants(c)["decay_floor_ok"] for c in cfgs}
    assert floors == {0.0, 1.0}


def test_geometry_constants_do_not_depend_on_the_configuration():
    for dim, res, full in ((120.0, 0.33, False), (99.0, 0.33, True), (33.33, 0.33, False), (81.2, 0.4, True)):
        g = capi.host_geometry_constants(dim, res, full)
        r = np.float64(np.float32(res))
        n = int(np.round(np.float64(np.float32(dim)) / r))
        assert (g["N"], g["N2"], g["full_layers"]) == (n, n * n, 1.0 if full else 0.0)
        assert g["N"] == capi.host_cells_per_side(dim, res)
        assert (g["res_f"], g["res"], g["rres"]) == (r, r, 1.0 / r)
        assert g["len"] == n * r and g["half"] == 0.5 * (n * r) and g["res_sq"] == r * r


def cfg_with(**kw):
    c = capi.default_config()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_equal_configs_share_one_variant():
    a = cfg_with(max_ring=48)
    b = cfg_with(max_ring=48)
    ops, final = capi.host_config_registry(6, [(1, a), (3, b), (5, cfg_with(max_ring=48, thread_count=1))])
    # the first change builds a variant, equal ones (thread_count is not part of the constants) join it
    assert ops[:, 1].tolist() == [1, 0, 0]
    assert ops[0, 0] == ops[1, 0] == ops[2, 0] != 0
    assert final.tolist() == [0, ops[0, 0], 0, ops[0, 0], 0, ops[0, 0]]
    assert ops[:, 2].tolist() == [2, 2, 2] and ops[:, 3].tolist() == [2, 2, 2]
    # setting a slot to what it already runs changes nothing
    ops, _ = capi.host_config_registry(2, [(0, capi.default_config())])
    assert ops.tolist() == [[0, 0, 1, 1]]


def test_unused_variants_are_reused_and_refcounts_drop():
    a, b, c = cfg_with(max_ring=48), cfg_with(outlier_tolerance=0.3), cfg_with(patch_size_change_distance=7.5)
    d0 = capi.default_config()
    ops, final = capi.host_config_registry(3, [
        (0, a),   # 0 -> new variant 1 (built)
        (0, b),   # variant 1 loses its only slot: b reuses id 1 (built again)
        (1, b),   # joins
        (0, d0),  # back to the default variant
        (1, d0),  # variant 1 unused now
        (2, c),   # c takes the unused id 1
        (2, c),   # no-op
        (2, d0),
        (2, c),   # id 1 still holds c's data: no rebuild
    ])
    assert ops[:, 0].tolist() == [1, 1, 1, 0, 0, 1, 1, 0, 1]
    assert ops[:, 1].tolist() == [1, 1, 0, 0, 0, 1, 0, 0, 0]
    assert ops[:, 2].tolist() == [2, 2, 2, 2, 1, 2, 2, 1, 2]
    assert ops[:, 3].max() == 2            # never more than two device buffers
    assert final.tolist() == [0, 0, 1]


def test_live_variants_never_exceed_distinct_configurations():
    rng = np.random.default_rng(5)
    pool = [random_config(rng) for _ in range(4)]
    n_slots = 40
    slot_cfg = [-1] * n_slots   # -1: default
    ops = []
    for _ in range(400):
        s = int(rng.integers(0, n_slots))
        k = int(rng.integers(-1, len(pool)))
        ops.append((s, pool[k] if k >= 0 else capi.default_config()))
    out, final = capi.host_config_registry(n_slots, ops)
    for i, ((s, c), row) in enumerate(zip(ops, out)):
        slot_cfg[s] = next((j for j, p in enumerate(pool) if p is c), -1)
        distinct = len(set(slot_cfg))
        assert row[2] == distinct, (i, row, distinct)
        assert row[3] <= len(pool) + 1           # buffers: at most one per configuration ever in use at once
    # slots with the same configuration share a variant, different ones do not
    by_cfg = {}
    for s in range(n_slots):
        by_cfg.setdefault(slot_cfg[s], set()).add(int(final[s]))
    assert all(len(v) == 1 for v in by_cfg.values())
    assert len({next(iter(v)) for v in by_cfg.values()}) == len(by_cfg)


def test_handle_wide_config_collapses_every_slot_onto_one_variant():
    rng = np.random.default_rng(9)
    pool = [random_config(rng) for _ in range(3)]
    ops = [(s, pool[s % 3]) for s in range(8)] + [(None, pool[1])]
    out, final = capi.host_config_registry(8, ops)
    assert out[7, 2] == 3                      # slot 0..7 on three configurations (the default has no slot left)
    assert out[8].tolist() == [0, 1, 1, out[7, 3]]
    assert final.tolist() == [0] * 8
    # afterwards a slot change reuses a buffer instead of allocating one
    out2, _ = capi.host_config_registry(8, ops + [(4, pool[2])])
    assert out2[-1, 3] == out[7, 3] and out2[-1, 2] == 2


def test_a_variant_whose_build_failed_is_built_again_when_taken():
    a, b, d0 = cfg_with(max_ring=48), cfg_with(outlier_tolerance=0.3), capi.default_config()
    ops, final = capi.host_config_registry(3, [   # slot 2 keeps the default variant 0 in use
        (1, a),                    # variant 1 built
        (0, b),                    # variant 2 built
        (0, d0),                   # variant 2 unused, still holding b's data ...
        (("invalidate", 2), None), # ... until a failed rebuild of it leaves its data unknown
        (1, b),                    # b is not matched against the unknown data: built again (in the unused id 1)
        (0, b),                    # shares it
    ])
    assert ops[:, 1].tolist() == [1, 1, 0, 0, 1, 0]
    assert ops[4, 0] == ops[5, 0] == 1 and final.tolist() == [1, 1, 0]
    # without the failure b would have been found intact in variant 2
    ops, _ = capi.host_config_registry(3, [(1, a), (0, b), (0, d0), (1, b)])
    assert ops[3].tolist()[:2] == [2, 0]
