"""CPU restatement (numpy float64, test infrastructure only) of gg_sample_layers_to_device: the checker of
tests/test_gpu_sample_layers.py and bench_sample_layers.py.  The rules are those of the header comment
(include/groundgrid_b200.h): the cell is grid_map's getIndexFromPosition / checkIfPositionWithinMap as the rasterizer
computes them, and GG_SAMPLE_LINEAR is the project's own bilinear definition.  numpy's float64 operations are correctly
rounded and never contracted, so each expression below is one rounding, in the header's order."""
import numpy as np

NAN_BITS = np.uint32(0x7FC00000)   # what the device stores outside the map and for a NaN linear value


def geometry(N, res):
    """(res, len, half) in fp64 from the handle's float resolution, as gg_create derives them."""
    r = float(np.float32(res))
    length = N * r
    return r, length, 0.5 * length


def cells(N, res, px, py, x, y):
    """(i, j, inside) of every query: x, y float32 arrays in the map frame, (px, py) the map position."""
    r, length, half = geometry(N, res)
    dx, dy = np.asarray(x, np.float32).astype(np.float64), np.asarray(y, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        qx, qy = ((dx - half) - px) / r, ((dy - half) - py) / r
        tx, ty = -((dx - px) - half), -((dy - py) - half)
        inside = (tx >= 0.0) & (ty >= 0.0) & (tx < length) & (ty < length)
    fin = np.isfinite(qx) & np.isfinite(qy) & (np.abs(qx) < 1e9) & (np.abs(qy) < 1e9)
    i = np.where(fin, -np.trunc(np.where(fin, qx, 0.0)), -1).astype(np.int64)
    j = np.where(fin, -np.trunc(np.where(fin, qy, 0.0)), -1).astype(np.int64)
    inside &= fin & (i >= 0) & (j >= 0) & (i < N) & (j < N)
    return i, j, inside


def sample_layers(planes, N, res, px, py, x, y, mode):
    """planes: [n_names] arrays N x N indexed [i, j] (like GroundGridB200.layer), x / y float32 [n], mode "nearest" or
    "linear".  Returns (values float32 [n_names, n], cells int32 [n]) with the device's bits."""
    planes = [np.asarray(p, np.float32) for p in planes]
    r, _, half = geometry(N, res)
    i, j, inside = cells(N, res, px, py, x, y)
    n = len(i)
    cell = np.where(inside, i + j * N, -1).astype(np.int32)
    vals = np.empty((len(planes), n), np.float32)
    vals.view(np.uint32)[:] = NAN_BITS
    ii, jj = i[inside], j[inside]
    lin = np.zeros(n, bool)
    if mode == "linear":
        dx = np.asarray(x, np.float32).astype(np.float64)
        dy = np.asarray(y, np.float32).astype(np.float64)
        off = half - 0.5 * r
        cx = (px + off) + r * (-i).astype(np.float64)
        cy = (py + off) + r * (-j).astype(np.float64)
        with np.errstate(invalid="ignore"):
            si = np.where(dx >= cx, -1, 1)
            sj = np.where(dy >= cy, -1, 1)
        lin = inside & (i + si >= 0) & (i + si < N) & (j + sj >= 0) & (j + sj < N)
        with np.errstate(invalid="ignore"):
            tx = np.abs(dx - cx) / r
            ty = np.abs(dy - cy) / r
        ux, uy = 1.0 - tx, 1.0 - ty
        wa, wb, wc, wd = ux * uy, tx * uy, ux * ty, tx * ty
    elif mode != "nearest":
        raise ValueError(mode)
    for l, p in enumerate(planes):
        vals[l, inside] = p[ii, jj]                       # nearest: the cell's bits
        if lin.any():
            m = lin
            with np.errstate(invalid="ignore", over="ignore"):   # signalling NaN cells and inf * 0 are expected here
                a = p[i[m], j[m]].astype(np.float64)
                b = p[i[m] + si[m], j[m]].astype(np.float64)
                c = p[i[m], j[m] + sj[m]].astype(np.float64)
                d = p[i[m] + si[m], j[m] + sj[m]].astype(np.float64)
                v = (((wa[m] * a + wb[m] * b) + wc[m] * c) + wd[m] * d).astype(np.float32)
            vb = v.view(np.uint32).copy()
            vb[np.isnan(v)] = NAN_BITS
            vals[l, m] = vb.view(np.float32)
    return vals, cell
