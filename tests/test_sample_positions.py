"""CPU checks of the terrain-lookup rules (gg_sample_layers_to_device) as tests/sample_ref.py restates them: the cell
of a position against the reference's own grid_map geometry, and hand-computed answers for nearest and linear."""
import numpy as np
import pytest

import sample_ref
from groundgrid_b200 import capi


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def f32(v):
    return np.float32(v)


@pytest.mark.parametrize("dim,res", [(99.0, 0.33), (33.33, 0.33), (120.0, 0.5)])
def test_geometry_matches_the_handle(dim, res):
    N = capi.host_cells_per_side(dim, res)
    k = capi.host_geometry_constants(dim, res)
    r, length, half = sample_ref.geometry(N, res)
    assert (r, length, half) == (k["res"], k["len"], k["half"])


def edge_positions(centres, res):
    """float32 positions on both sides of every cell edge of one axis (the edge = centre + res / 2, where the index
    changes), plus the centres themselves."""
    out = []
    for c in centres:
        for e in (c + 0.5 * res, c - 0.5 * res):
            v = f32(e)
            out += [np.nextafter(np.nextafter(v, f32(-np.inf)), f32(-np.inf)), np.nextafter(v, f32(-np.inf)), v,
                    np.nextafter(v, f32(np.inf)), np.nextafter(np.nextafter(v, f32(np.inf)), f32(np.inf))]
        out.append(f32(c))
    return np.array(out, np.float32)


@pytest.mark.parametrize("dim,res,pos", [(99.0, 0.33, (3.7, -12.2)), (33.0, 0.33, (-0.4, 101.3))])
def test_cells_match_the_reference_geometry(dim, res, pos):
    from oracle import ref as refmod

    if not refmod.available():
        pytest.skip("oracle/_ref is not built")
    r = refmod.Reference(dim, res)
    r.init_map(pos[0], pos[1], 0.0)
    px, py = r.position()
    N = r.n
    cx = np.array([r.cell_position(i, 0)[0] for i in range(N)])
    cy = np.array([r.cell_position(0, j)[1] for j in range(N)])
    xs, ys = edge_positions(cx, float(np.float32(res))), edge_positions(cy, float(np.float32(res)))
    far = np.array([px + 1e3, px - 1e3, px + 1e12, -1e30, np.nan, np.inf, -np.inf], np.float32)
    # every x edge at a middle row, every y edge at a middle column, the corners, and non-finite / far positions
    qx = np.concatenate([xs, np.full(len(ys), f32(cx[N // 2])), xs[:40], far, np.full(len(far), f32(px))])
    qy = np.concatenate([np.full(len(xs), f32(cy[N // 3])), ys, ys[-40:], np.full(len(far), f32(py)), far])
    i, j, inside = sample_ref.cells(N, res, px, py, qx, qy)
    _, cell = sample_ref.sample_layers([np.zeros((N, N), np.float32)], N, res, px, py, qx, qy, "nearest")
    for q in range(len(qx)):
        ri, rj, rin = r.grid_index(float(qx[q]), float(qy[q]))
        rin = rin and 0 <= ri < N and 0 <= rj < N
        assert inside[q] == rin, f"query {q} ({qx[q]!r}, {qy[q]!r}): inside {inside[q]} != reference {rin}"
        if rin:
            assert (i[q], j[q]) == (ri, rj), f"query {q} ({qx[q]!r}, {qy[q]!r}): cell ({i[q]}, {j[q]}) != reference ({ri}, {rj})"
            assert cell[q] == ri + rj * N
        else:
            assert cell[q] == -1
    assert inside.sum() > len(qx) // 2


# A 10 x 10 map of resolution 0.5 at (0, 0): half = 2.5, centre of cell (i, j) = (2.25 - 0.5 i, 2.25 - 0.5 j), every
# number below exact in binary.  plane[i, j] = 10 i + j, a linear function, so the bilinear value is known by hand.
N, RES = 10, 0.5


def centre(i):
    return 2.25 - 0.5 * i


def plane():
    i, j = np.meshgrid(np.arange(N), np.arange(N), indexing="ij")
    return (10 * i + j).astype(np.float32)


def sample(planes, x, y, mode):
    return sample_ref.sample_layers(planes, N, RES, 0.0, 0.0, np.asarray(x, np.float32), np.asarray(y, np.float32), mode)


def test_known_answers_at_cell_centres():
    p = plane()
    x = [centre(3), centre(0), centre(9)]
    y = [centre(4), centre(9), centre(0)]
    for mode in ("nearest", "linear"):
        v, c = sample([p], x, y, mode)
        assert v[0].tolist() == [34.0, 9.0, 90.0]
        assert c.tolist() == [3 + 4 * N, 0 + 9 * N, 9 + 0 * N]


@pytest.mark.parametrize("dx,dy", [(0.125, 0.0625), (0.125, -0.0625), (-0.125, 0.0625), (-0.125, -0.0625)])
def test_known_answers_on_each_quadrant_side(dx, dy):
    # x >= cx: the neighbour is i - 1 (i grows toward -x); tx = |dx| / res, ty = |dy| / res
    i, j = 4, 6
    v, c = sample([plane()], [centre(i) + dx], [centre(j) + dy], "linear")
    fi = i - abs(dx) / RES if dx >= 0 else i + abs(dx) / RES
    fj = j - abs(dy) / RES if dy >= 0 else j + abs(dy) / RES
    assert v[0, 0] == np.float32(10 * fi + fj)
    assert c[0] == i + j * N
    vn, _ = sample([plane()], [centre(i) + dx], [centre(j) + dy], "nearest")
    assert vn[0, 0] == 10 * i + j


@pytest.mark.parametrize("i,j,dx,dy", [(0, 5, 0.125, 0.0), (9, 5, -0.125, 0.0), (5, 0, 0.0, 0.125), (5, 9, 0.0, -0.125),
                                       (0, 0, 0.2, 0.2), (9, 9, -0.2, -0.2)])
def test_linear_falls_back_to_nearest_at_the_map_edges(i, j, dx, dy):
    # the neighbour i + si or j + sj would be outside [0, N): the nearest value, even where the fraction is not zero
    v, c = sample([plane()], [centre(i) + dx], [centre(j) + dy], "linear")
    assert v[0, 0] == 10 * i + j and c[0] == i + j * N


def test_linear_interpolates_next_to_the_map_edges():
    # at i = 0 with x < cx the neighbour is i = 1: inside, so the value interpolates
    v, _ = sample([plane()], [centre(0) - 0.125], [centre(5)], "linear")
    assert v[0, 0] == np.float32(10 * 0.25 + 5)


def test_non_finite_cells():
    p = plane()
    p[4, 6] = np.inf                      # the neighbour b of a query at the centre of (5, 6) with x >= cx
    pay = np.array([0x7FA00001], np.uint32).view(np.float32)[0]
    p[2, 2] = pay                         # a NaN with a payload
    p[7, 7] = np.float32(-0.0)
    x = [centre(5), centre(2), centre(7), centre(5)]
    y = [centre(6), centre(2), centre(7), centre(6) - 0.125]
    vn, _ = sample([p], x, y, "nearest")
    assert bits(vn[0]).tolist() == [bits(56.0)[()], 0x7FA00001, 0x80000000, bits(56.0)[()]]
    vl, _ = sample([p], x, y, "linear")
    b = bits(vl[0]).tolist()
    assert b[0] == 0x7FC00000             # weight 0 times inf is NaN, stored as the canonical quiet NaN
    assert b[1] == 0x7FC00000             # NaN cell: NaN
    assert b[2] == 0x80000000 or b[2] == 0  # -0 with zero-weight neighbours: the sum of -0 and +0 terms
    assert b[3] == 0x7FC00000


def test_outside_the_map():
    p = plane()
    x = [3.0, -2.5, np.nan, np.inf, -np.inf, 0.0, 1e30, centre(0) + 0.25]
    y = [0.0, 0.0, 0.0, 0.0, 0.0, np.nan, 0.0, 0.0]
    for mode in ("nearest", "linear"):
        v, c = sample([p, p], x, y, mode)
        assert c.tolist()[:7] == [-1] * 7
        assert (bits(v[:, :7]) == 0x7FC00000).all()
    # x = +2.5 (the +x edge of the map): t = -((x - px) - half) = 0 is inside, cell 0
    _, c = sample([p], [2.5], [0.0], "nearest")
    assert c[0] == 0 + 5 * N
    _, c = sample([p], [centre(0) + 0.25], [0.0], "nearest")
    assert c[0] == 0 + 5 * N
    _, c = sample([p], [np.nextafter(np.float32(2.5), np.float32(np.inf))], [0.0], "nearest")
    assert c[0] == -1
    _, c = sample([p], [-2.5], [0.0], "nearest")   # t = len: outside
    assert c[0] == -1
