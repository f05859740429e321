"""CPU restatements (numpy, test infrastructure only) of the steps next to the hot path
(SURVEY.md section 8f) -- checkers for tests/test_gpu_next_rows.py.

  unpack_transform : pcl::fromROSMsg + per-point tf2::doTransform, src/GroundGridNodelet.cpp:119-120,148-184
  terrain_image    : publish_grid_map_layer "terrain" branch, src/GroundGridNodelet.cpp:247-270
  eval_counts      : callback_predicted_cloud tallies, scripts/eval_groundpoint_classifier.py:95-118
"""
import numpy as np

from . import POINT_DTYPE


def unpack_transform(raw, n, point_step, offsets, T=None):
    raw = np.frombuffer(np.ascontiguousarray(raw, np.uint8).tobytes(), np.uint8).reshape(n, point_step)
    out = np.zeros(n, POINT_DTYPE)

    def f32(off):
        return raw[:, off:off + 4].copy().view(np.float32).reshape(n)

    x, y, z = f32(offsets[0]), f32(offsets[1]), f32(offsets[2])
    if offsets[3] >= 0:
        out["intensity"] = f32(offsets[3])
    if offsets[4] >= 0:
        out["ring"] = raw[:, offsets[4]:offsets[4] + 2].copy().view(np.uint16).reshape(n)
    if T is not None:
        T = np.asarray(T, np.float64).reshape(3, 4)
        dx, dy, dz = x.astype(np.float64), y.astype(np.float64), z.astype(np.float64)
        x = (((T[0, 0] * dx + T[0, 1] * dy) + T[0, 2] * dz) + T[0, 3]).astype(np.float32)   # row.dot(v) left to right, + origin
        y = (((T[1, 0] * dx + T[1, 1] * dy) + T[1, 2] * dz) + T[1, 3]).astype(np.float32)
        z = (((T[2, 0] * dx + T[2, 1] * dy) + T[2, 2] * dz) + T[2, 3]).astype(np.float32)
    out["x"], out["y"], out["z"] = x, y, z
    return out


def terrain_image(ground, points_raw):
    n = ground.shape[0]
    img = np.zeros((n, n, 3), np.float32)
    img[:, :, 0] = ground
    img[:, :, 2] = points_raw
    s = np.zeros((n, n), np.float32)
    for di in (-1, 0, 1):
        for dj in (-1, 0, 1):
            # integers; near 2^24 their fp32 sum rounds and depends on the order, but not on which side of 27 it lies
            s[1:-1, 1:-1] += points_raw[1 + di:n - 1 + di, 1 + dj:n - 1 + dj]
    img[1:-1, 1:-1, 1] = (s[1:-1, 1:-1] >= 27).astype(np.float32)   # border cells: the reference reads out of bounds; defined as 0
    return img


def eval_counts(labels, rings, n_ids=1024):
    counts = np.zeros((n_ids, 2), np.uint64)
    present = labels != 0
    r = rings[present].astype(np.int64)
    ng = (labels[present] == 99).astype(np.int64)
    ok = r < n_ids
    np.add.at(counts, (r[ok], ng[ok]), 1)
    return counts


def layer_image_u8(layer):
    """grid_map::GridMapCvConverter::toImage<unsigned char, 1>(map, layer, CV_8UC1, img) as called by
    publish_grid_map_layer (src/GroundGridNodelet.cpp:238-245; grid_map_cv 1.6.x GridMapCvConverter.hpp): range = min / max
    over the finite cells, pixel = (uchar)(((v - lower) / (upper - lower)) * 255.f) in fp32, non-finite cells 0."""
    a = np.asarray(layer, np.float32)
    fin = np.isfinite(a)
    lower, upper = np.float32(a[fin].min()), np.float32(a[fin].max())
    with np.errstate(invalid="ignore", divide="ignore"):
        t = ((a - lower) / (upper - lower)) * np.float32(255.0)
    img = np.zeros(a.shape, np.uint8)
    ok = fin & np.isfinite(t)
    img[ok] = t[ok].astype(np.int32).astype(np.uint8)
    return img, float(lower), float(upper)
