"""ctypes binding of the CPU oracle (oracle/gg_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and the CPU arm of
bench.py (cpu_baseline / --impl reference).  Nothing under groundgrid_b200/ imports it.
Pinned by oracle/_ref (the unmodified reference sources on CPU stand-ins, oracle/ref.py) -- see the header of gg_oracle.cpp.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgg_oracle.so")

# include/velodyne_pointcloud/point_types.h:27-33 -- 32-byte PointXYZIR record.
POINT_DTYPE = np.dtype(
    {
        "names": ["x", "y", "z", "intensity", "ring"],
        "formats": ["<f4", "<f4", "<f4", "<f4", "<u2"],
        "offsets": [0, 4, 8, 16, 20],
        "itemsize": 32,
    }
)

LAYERS = (
    "points", "ground", "groundpatch", "minGroundHeight", "maxGroundHeight",
    "groundCandidates", "planeDist", "m2", "meanVariance", "pointsRaw", "variance",
)


class Config(C.Structure):
    """cfg/GroundGrid.cfg:8-21 -- same order and defaults."""

    _fields_ = [
        ("point_count_cell_variance_threshold", C.c_int),
        ("max_ring", C.c_int),
        ("groundpatch_detection_minimum_threshold", C.c_double),
        ("distance_factor", C.c_double),
        ("minimum_distance_factor", C.c_double),
        ("miminum_point_height_threshold", C.c_double),
        ("minimum_point_height_obstacle_threshold", C.c_double),
        ("outlier_tolerance", C.c_double),
        ("ground_patch_detection_minimum_point_count_threshold", C.c_double),
        ("patch_size_change_distance", C.c_double),
        ("occupied_cells_decrease_factor", C.c_double),
        ("occupied_cells_point_count_factor", C.c_double),
        ("min_outlier_detection_ground_confidence", C.c_double),
        ("thread_count", C.c_int),
    ]


def build(force=False):
    """Compile the oracle shared library (g++ only; no GPU needed)."""
    src = [os.path.join(_HERE, f) for f in ("gg_oracle.cpp", "eigen_redux.hpp", "gridmap_semantics.hpp", "Makefile")]
    if not force and os.path.exists(_LIB_PATH):
        if all(os.path.getmtime(_LIB_PATH) >= os.path.getmtime(s) for s in src):
            return _LIB_PATH
    subprocess.run(["make", "-C", _HERE, "-B", "libgg_oracle.so"], check=True, capture_output=True)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.ggo_create.restype = C.c_void_p
        L.ggo_create.argtypes = [C.c_double, C.c_float]
        L.ggo_destroy.argtypes = [C.c_void_p]
        L.ggo_cells_per_side.argtypes = [C.c_void_p]
        L.ggo_set_config.argtypes = [C.c_void_p, C.POINTER(Config)]
        L.ggo_get_config.argtypes = [C.c_void_p, C.POINTER(Config)]
        L.ggo_init_map.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double]
        L.ggo_update.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p]
        L.ggo_get_position.argtypes = [C.c_void_p, C.c_void_p]
        L.ggo_get_expected.argtypes = [C.c_void_p, C.c_void_p]
        L.ggo_get_layer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        L.ggo_set_layer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        L.ggo_filter_cloud.restype = C.c_long
        L.ggo_filter_cloud.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_double, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ggo_interpolate_cell.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ggo_spiral.argtypes = [C.c_void_p, C.c_double]
        L.ggo_detect_ground_patches.argtypes = [C.c_void_p]
        L.ggo_detect_ground_patch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.ggo_add_layer.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
        L.ggo_grid_index.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
        L.ggo_cell_position.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.ggo_block_sum3.restype = C.c_float
        L.ggo_block_sum3.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.ggo_block_sum5.restype = C.c_float
        L.ggo_block_sum5.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class Oracle:
    """One GroundGrid + GroundSegmentation pair on the CPU (thread_count semantics selectable)."""

    def __init__(self, dimension_m=120.0, resolution=0.33):
        self._l = lib()
        self._h = self._l.ggo_create(float(dimension_m), np.float32(resolution))
        self.n = self._l.ggo_cells_per_side(self._h)

    def close(self):
        if self._h:
            self._l.ggo_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_config(self, **kw):
        cfg = Config()
        self._l.ggo_get_config(self._h, C.byref(cfg))
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._l.ggo_set_config(self._h, C.byref(cfg))

    def init_map(self, x, y, z):
        self._l.ggo_init_map(self._h, x, y, z)

    def update(self, x, y, T_base_from_map):
        T = np.ascontiguousarray(T_base_from_map, dtype=np.float64).reshape(12)
        return self._l.ggo_update(self._h, x, y, _ptr(T))

    def position(self):
        xy = np.zeros(2, np.float64)
        self._l.ggo_get_position(self._h, _ptr(xy))
        return xy

    def expected_points(self):
        out = np.empty((self.n, self.n), np.float32, order="F")
        self._l.ggo_get_expected(self._h, _ptr(out))
        return out

    def layer(self, name):
        """Layer as an (n, n) array indexed [i, j] (column-major storage like Eigen::MatrixXf)."""
        out = np.empty((self.n, self.n), np.float32, order="F")
        if self._l.ggo_get_layer(self._h, name.encode(), _ptr(out)) != 0:
            raise KeyError(name)
        return out

    def set_layer(self, name, arr):
        a = np.asfortranarray(arr, dtype=np.float32)
        assert a.shape == (self.n, self.n)
        if self._l.ggo_set_layer(self._h, name.encode(), _ptr(a)) != 0:
            raise KeyError(name)

    def filter_cloud(self, points, origin, base_z, threads=1, stop_after=0, want_cloud=False, want_classes=False):
        """Returns (labels[u8 per input point: 0 absent / 49 ground / 99 non-ground],
        out_index[u32: input index of each output point in reference order], out_cloud or None); with want_classes
        also classes[u8 per input point]: 0 outside the map, 1 kept, 2 kept in a border cell, 3 ignored, 4 ignored in a
        border cell, 5 outlier (the classes of gg_get_point_classes)."""
        pts = np.ascontiguousarray(points, dtype=POINT_DTYPE)
        n = pts.shape[0]
        labels = np.zeros(n, np.uint8)
        out_index = np.zeros(n, np.uint32)
        out_cloud = np.zeros(n, POINT_DTYPE) if want_cloud else None
        classes = np.zeros(n, np.uint8) if want_classes else None
        org = np.ascontiguousarray(origin, dtype=np.float32)
        nout = self._l.ggo_filter_cloud(self._h, _ptr(pts), n, _ptr(org), float(base_z), int(threads), int(stop_after),
                                        _ptr(labels), _ptr(out_cloud), _ptr(out_index), _ptr(classes))
        if nout < 0:
            raise RuntimeError("oracle: map not initialised")
        out = (labels, out_index[:nout], (out_cloud[:nout] if want_cloud else None))
        return out + (classes,) if want_classes else out

    def interpolate_cell(self, x, y):
        self._l.ggo_interpolate_cell(self._h, x, y)

    def spiral(self, base_z):
        self._l.ggo_spiral(self._h, float(base_z))

    def detect_ground_patches(self):
        """detect_ground_patches over all four sections, with the variance recompute each starts with (:323)."""
        if self._l.ggo_detect_ground_patches(self._h) != 0:
            raise RuntimeError("oracle: detection needs a map with 'm2' and 'variance' layers")

    def detect_ground_patch(self, size, i, j):
        """detect_ground_patch<size>(map, i, j): one cell, the stored variance."""
        if self._l.ggo_detect_ground_patch(self._h, int(size), int(i), int(j)) != 0:
            raise RuntimeError("oracle: detection needs a map with a 'variance' layer")

    def add_layer(self, name, value=0.0):
        """grid_map::GridMap::add(name, value)."""
        if self._l.ggo_add_layer(self._h, name.encode(), float(value)) != 0:
            raise KeyError(name)

    def grid_index(self, x, y):
        idx = np.zeros(2, np.int32)
        inside = C.c_int(0)
        self._l.ggo_grid_index(self._h, x, y, _ptr(idx), C.byref(inside))
        return int(idx[0]), int(idx[1]), bool(inside.value)

    def cell_position(self, i, j):
        xy = np.zeros(2, np.float64)
        self._l.ggo_cell_position(self._h, i, j, _ptr(xy))
        return xy


def block_sum(mat, r0, c0, size):
    m = np.asfortranarray(mat, dtype=np.float32)
    f = lib().ggo_block_sum3 if size == 3 else lib().ggo_block_sum5
    return float(f(_ptr(m), m.shape[0], r0, c0))
