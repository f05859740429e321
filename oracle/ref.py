"""ctypes binding of oracle/_ref/libgg_ref.so -- the UNMODIFIED reference classes on CPU stand-ins.

TEST INFRASTRUCTURE ONLY (tests/, bench.py CPU legs).  See oracle/ref_harness.cpp and oracle/build_ref.py.
Every Reference() instance loads a PRIVATE COPY of the library: the reference keeps function-local statics
bound to the first map it sees, so one loaded copy can serve one map only.
"""
import atexit
import ctypes as C
import math
import os
import shutil
import tempfile

import numpy as np

from . import Config, POINT_DTYPE, LAYERS  # noqa: F401  (same config layout as the oracle port)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libgg_ref.so")

_tmpdir = None
_count = 0


def available():
    """True if the library exists (built here from a checkout of the reference, or copied here prebuilt)."""
    from . import build_ref

    if os.path.exists(LIB_PATH):
        return True
    if build_ref.have_sources():
        build_ref.build()
        return os.path.exists(LIB_PATH)
    return False


def _private_copy():
    global _tmpdir, _count
    from . import build_ref

    if build_ref.have_sources():
        build_ref.build()
    if _tmpdir is None:
        _tmpdir = tempfile.mkdtemp(prefix="gg_ref_")
        atexit.register(shutil.rmtree, _tmpdir, True)
    _count += 1
    dst = os.path.join(_tmpdir, f"libgg_ref_{os.getpid()}_{_count}.so")
    shutil.copyfile(LIB_PATH, dst)
    return dst


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


from groundgrid_b200.synth import base_from_map_qt, quat_from_yaw_pitch, tf2_matrix  # noqa: E402,F401  (pose helpers shared with bench.py)

IDENTITY_Q = np.array([0.0, 0.0, 0.0, 1.0])


class Reference:
    """One GroundGrid + GroundSegmentation pair of the reference itself.  Same calls as oracle.Oracle, except that
    transforms are (quaternion, translation) pairs like the ROS messages the reference consumes."""

    def __init__(self, dimension_m=120.0, resolution=0.33):
        L = C.CDLL(_private_copy())
        L.ggr_create.restype = C.c_void_p
        L.ggr_create.argtypes = [C.c_double, C.c_float]
        L.ggr_destroy.argtypes = [C.c_void_p]
        L.ggr_cells_per_side.argtypes = [C.c_void_p]
        L.ggr_set_config.argtypes = [C.c_void_p, C.POINTER(Config)]
        L.ggr_get_config.argtypes = [C.c_void_p, C.POINTER(Config)]
        L.ggr_update.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
        L.ggr_get_position.argtypes = [C.c_void_p, C.c_void_p]
        L.ggr_get_expected.argtypes = [C.c_void_p, C.c_void_p]
        L.ggr_get_layer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        L.ggr_set_layer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        L.ggr_filter_cloud.restype = C.c_long
        L.ggr_filter_cloud.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ggr_detect_ground_patches.argtypes = [C.c_void_p, C.c_int]
        # a library built elsewhere from an older harness may lack the one-cell entry point; only that call needs it
        self._has_detect_patch = hasattr(L, "ggr_detect_ground_patch")
        if self._has_detect_patch:
            L.ggr_detect_ground_patch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.ggr_interpolate_cell.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ggr_spiral.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ggr_add_layer.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
        L.ggr_grid_index.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
        L.ggr_cell_position.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        self._l = L
        self._h = L.ggr_create(float(dimension_m), np.float32(resolution))
        if not self._h:
            raise ValueError("reference: GroundSegmentation::init(size_t dimension) and the map disagree on the cell count "
                             f"for dimension {dimension_m} (non-integer dimension?)")
        self.n = L.ggr_cells_per_side(self._h)
        self.set_config(thread_count=1)  # parity is defined at thread_count = 1 (the shipped 8 races)
        self.last_filter_seconds = 0.0

    def close(self):
        # the handle is leaked on purpose: the library copy holds static references into its map
        self._h = None

    def set_config(self, **kw):
        cfg = Config()
        self._l.ggr_get_config(self._h, C.byref(cfg))
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._l.ggr_set_config(self._h, C.byref(cfg))

    def init_map(self, x, y, z):
        """First odometry message -> GroundGrid::update -> initGroundGrid."""
        rc = self._l.ggr_update(self._h, x, y, z, _ptr(IDENTITY_Q), _ptr(np.zeros(3)))
        if rc != 2:
            raise RuntimeError(f"reference: map creation returned {rc}")

    def update(self, x, y, q, t, z=0.0):
        q = np.ascontiguousarray(q, np.float64)
        t = np.ascontiguousarray(t, np.float64)
        rc = self._l.ggr_update(self._h, x, y, z, _ptr(q), _ptr(t))
        if rc < 0 or rc == 2:
            raise RuntimeError(f"reference: update returned {rc}")
        return rc

    def position(self):
        xy = np.zeros(2, np.float64)
        self._l.ggr_get_position(self._h, _ptr(xy))
        return xy

    def expected_points(self):
        out = np.empty((self.n, self.n), np.float32, order="F")
        self._l.ggr_get_expected(self._h, _ptr(out))
        return out

    def layer(self, name):
        out = np.empty((self.n, self.n), np.float32, order="F")
        if self._l.ggr_get_layer(self._h, name.encode(), _ptr(out)) != 0:
            raise KeyError(name)
        return out

    def set_layer(self, name, arr):
        a = np.asfortranarray(arr, dtype=np.float32)
        assert a.shape == (self.n, self.n)
        if self._l.ggr_set_layer(self._h, name.encode(), _ptr(a)) != 0:
            raise KeyError(name)

    def add_layer(self, name, value=0.0):
        self._l.ggr_add_layer(self._h, name.encode(), float(value))

    def filter_cloud(self, points, origin, base_z, want_cloud=False, q=None, t=None):
        """(labels, out_index, out_cloud | None); base_z is the translation z of mapToBase unless (q, t) is given."""
        pts = np.ascontiguousarray(points, dtype=POINT_DTYPE)
        n = pts.shape[0]
        labels = np.zeros(n, np.uint8)
        out_index = np.zeros(n, np.uint32)
        out_cloud = np.zeros(n, POINT_DTYPE) if want_cloud else None
        org = np.ascontiguousarray(origin, dtype=np.float32)
        q = IDENTITY_Q if q is None else np.ascontiguousarray(q, np.float64)
        t = np.array([0.0, 0.0, float(base_z)]) if t is None else np.ascontiguousarray(t, np.float64)
        sec = C.c_double(0.0)
        nout = self._l.ggr_filter_cloud(self._h, _ptr(pts), n, _ptr(org), _ptr(q), _ptr(t), _ptr(labels), _ptr(out_cloud),
                                        _ptr(out_index), C.byref(sec))
        if nout < 0:
            raise RuntimeError("reference: no map yet (scan before the first odometry message)")
        self.last_filter_seconds = sec.value
        return labels, out_index[:nout], (out_cloud[:nout] if want_cloud else None)

    def detect_ground_patches(self, section=None):
        """One section (0 .. 3) of GroundSegmentation::detect_ground_patches, or all four in order (section=None)."""
        for s in range(4) if section is None else (section,):
            self._l.ggr_detect_ground_patches(self._h, int(s))

    def detect_ground_patch(self, size, i, j):
        """GroundSegmentation::detect_ground_patch<size>(map, i, j)."""
        assert size in (3, 5)
        if not self._has_detect_patch:
            raise RuntimeError("reference: this oracle/_ref library predates ggr_detect_ground_patch; rebuild it with oracle/build_ref.py")
        self._l.ggr_detect_ground_patch(self._h, int(size), int(i), int(j))

    def interpolate_cell(self, x, y):
        self._l.ggr_interpolate_cell(self._h, x, y)

    def spiral(self, base_z):
        self._l.ggr_spiral(self._h, _ptr(IDENTITY_Q), _ptr(np.array([0.0, 0.0, float(base_z)])))

    def grid_index(self, x, y):
        idx = np.zeros(2, np.int32)
        inside = C.c_int(0)
        self._l.ggr_grid_index(self._h, x, y, _ptr(idx), C.byref(inside))
        return int(idx[0]), int(idx[1]), bool(inside.value)

    def cell_position(self, i, j):
        xy = np.zeros(2, np.float64)
        self._l.ggr_cell_position(self._h, i, j, _ptr(xy))
        return xy
