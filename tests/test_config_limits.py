"""Configurations at the limits of every GroundGridConfig field (tests/config_limits.py) on the oracle port, against the
reference's stored answers (tests/ref_scenarios.py:config_limits), and the coverage of the case list itself."""
import math

import pytest

import config_limits as cl
import ref_scenarios as rs
from groundgrid_b200 import capi


@pytest.mark.parametrize("n", list(rs.DENSE_GEOMETRY))
def test_config_limits_on_the_oracle(n):
    """Every case: three scans with a roll in between; labels, output order and cloud, all eleven layers, bit for bit."""
    rs.run("config_limits", rs.Oracle, n)


def test_every_field_at_its_ends_and_at_the_nonfinite_values():
    assert set(cl.RANGES) == set(cl.FIELDS), "a GroundGridConfig field without its cfg range"
    singles = [c for c in cl.CASES.values() if len(c) == 2]
    assert all(c["thread_count"] == 1 for c in cl.CASES.values())

    def has(field, pred):
        return any(field in c and pred(c[field]) for c in singles)

    for f in cl.DOUBLES:
        lo, hi = cl.RANGES[f]
        for v in (lo, hi, 0.0, -1.0, math.inf, -math.inf):
            assert has(f, lambda x, v=v: x == v), (f, v)
        assert has(f, math.isnan), f
        assert has(f, lambda x: x == 0.0 and math.copysign(1.0, x) < 0), f
    for f in cl.INTS:
        for v in cl.RANGES[f] + cl.INT_VALUES:
            assert has(f, lambda x, v=v: x == v), (f, v)
    assert has("max_ring", lambda x: x == 65535) and has("max_ring", lambda x: x == 65536)
    both = [c for c in cl.CASES.values() if len(c) == len(cl.FIELDS)]
    assert sorted(both, key=lambda c: c[cl.DECAY]) == [{f: cl.RANGES[f][e] if f != "thread_count" else 1 for f in cl.FIELDS}
                                                      for e in (0, 1)]


def test_decay_floor_shortcut_switches_between_the_two_cases():
    """derive_config's decay_floor_ok read back through gg_host_config_constants: on the factors around the switch and
    on every decrease factor of the cases, equal to the formula restated in config_limits.decay_floor_ok."""
    below, above = cl.decay_switch()
    assert above == math.nextafter(below, math.inf) and 999.9 < below < 1000.0

    def flag(factor):
        c = capi.default_config()
        c.occupied_cells_decrease_factor = factor
        return capi.host_config_constants(c)["decay_floor_ok"]

    assert flag(below) == 1.0 and flag(above) == 0.0
    assert {repr(below), repr(above)} <= {repr(f) for f in cl.decay_factors()}
    for f in cl.decay_factors():
        assert flag(f) == float(cl.decay_floor_ok(f)), f
