"""ctypes binding of the C-ABI (include/groundgrid_b200.h) -- the same calls the C++ host
classes make.  Python here is plumbing for tests / bench only; there is no Python compute
path and no CPU fallback: every compute call raises GroundGridError without an H100.
"""
import ctypes as C
import os
import weakref

import numpy as np

from . import build as _build
from .synth import POINT_DTYPE

GG_FLAG_FULL_LAYERS = 1
LABEL_ABSENT, LABEL_GROUND, LABEL_NONGROUND = 0, 49, 99
SELECT_GROUND, SELECT_NONGROUND = 1, 2
SELECT = {None: 0, "ground": SELECT_GROUND, "nonground": SELECT_NONGROUND, "all": SELECT_GROUND | SELECT_NONGROUND}


class GroundGridError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"groundgrid_b200 error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    """gg_config == groundgrid::GroundGridConfig (cfg/GroundGrid.cfg:8-21)."""

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


class ScanDesc(C.Structure):
    _fields_ = [
        ("slot", C.c_int),
        ("flags", C.c_int),
        ("n_points", C.c_size_t),
        ("origin", C.c_float * 3),
        ("_pad", C.c_float),
        ("base_z", C.c_double),
    ]


class CloudMsg(C.Structure):
    """gg_cloud_msg: one PointCloud2 payload in device memory (data), T_map_from_frame a host pointer or None."""

    _fields_ = [
        ("data", C.c_void_p),
        ("point_step", C.c_int),
        ("field_offsets", C.c_int * 5),
        ("T_map_from_frame", C.c_void_p),
    ]


# numpy image of an array of gg_cloud_msg (CloudMsg)
CLOUD_MSG_DTYPE = np.dtype({"names": ["data", "point_step", "field_offsets", "T_map_from_frame"],
                            "formats": [np.uint64, np.int32, (np.int32, 5), np.uint64], "offsets": [0, 8, 12, 32],
                            "itemsize": C.sizeof(CloudMsg)})

MAX_CLOUD_PARTS = 16   # GG_MAX_CLOUD_PARTS


class CloudPart(C.Structure):
    """gg_cloud_part: one sensor's payload of a merged scan and its point count."""

    _fields_ = [("msg", CloudMsg), ("n_points", C.c_size_t)]


# numpy image of an array of gg_cloud_part (CloudPart)
CLOUD_PART_DTYPE = np.dtype({"names": ["data", "point_step", "field_offsets", "T_map_from_frame", "n_points"],
                             "formats": [np.uint64, np.int32, (np.int32, 5), np.uint64, np.uint64],
                             "offsets": [0, 8, 12, 32, C.sizeof(CloudMsg)], "itemsize": C.sizeof(CloudPart)})


def _per_part(value, n_parts, item_ndim, name):
    """`value` for every part, or nested [scan][part] -> a flat list over the parts.  An item has item_ndim dimensions
    (None counts as an item: a part without T)."""
    def is_item(v):
        if v is None:
            return True
        try:
            a = np.asarray(v)          # nested lists holding None or ragged ones are no item
        except ValueError:
            return False
        return a.dtype != object and a.ndim == item_ndim

    if is_item(value):
        return [value] * int(sum(n_parts))
    if len(value) != len(n_parts) or any(len(v) != m for v, m in zip(value, n_parts)):
        raise ValueError(f"{name} must be one value or nested [scan][part] like the payloads")
    flat = [v for scan in value for v in scan]
    if not all(is_item(v) for v in flat):
        raise ValueError(f"{name} must be one value or nested [scan][part] like the payloads")
    return flat


def cloud_parts(nbytes, data_ptrs, point_step, field_offsets, T):
    """Flattens the nested arguments of merged scans into what gg_run_merged_cloud_msgs_to_device / gg_upload_cloud_msgs
    take.  nbytes / data_ptrs: nested [scan][part] payload sizes in bytes and addresses; point_step, field_offsets
    (5-tuple) and T (None or a 3x4 of lookupTransform("map", frame_id)) one value for every part or nested [scan][part].
    Returns (n_parts int32 [count], parts CLOUD_PART_DTYPE [total], T array): the T pointers of `parts` point into the T
    array, which must stay alive until the call."""
    n_parts = np.array([len(s) for s in nbytes], np.int32)
    if len(data_ptrs) != len(n_parts) or any(len(d) != m for d, m in zip(data_ptrs, n_parts)):
        raise ValueError("data_ptrs must be nested [scan][part] like nbytes")
    total = int(n_parts.sum())
    steps = _per_part(point_step, n_parts, 0, "point_step")
    offs = _per_part(field_offsets, n_parts, 1, "field_offsets")
    Ts = _per_part(T, n_parts, 2, "T")
    parts = np.zeros(max(1, total), CLOUD_PART_DTYPE)
    Tarr = np.zeros((max(1, total), 12), np.float64)
    for p, (nb, ptr, step, off, t) in enumerate(zip((b for s in nbytes for b in s), (d for s in data_ptrs for d in s), steps, offs, Ts)):
        step = int(step)
        if step <= 0 or int(nb) % step:
            raise ValueError(f"part {p}: {nb} bytes is not a multiple of point_step {step}")
        parts["data"][p] = int(ptr)
        parts["point_step"][p] = step
        parts["field_offsets"][p] = np.asarray(off, np.int32).reshape(5)
        parts["n_points"][p] = int(nb) // step
        if t is not None:
            Tarr[p] = np.asarray(t, np.float64).reshape(12)
            parts["T_map_from_frame"][p] = Tarr.ctypes.data + 96 * p
    return n_parts, parts[:total], Tarr

class Positions(C.Structure):
    """gg_positions: one set of query positions of a slot (device memory) and where its results go."""

    _fields_ = [
        ("data", C.c_void_p),
        ("n", C.c_size_t),
        ("point_step", C.c_int),
        ("off_x", C.c_int),
        ("off_y", C.c_int),
        ("dst", C.c_void_p),
        ("cell", C.c_void_p),
    ]


# numpy image of an array of gg_positions (Positions)
POSITIONS_DTYPE = np.dtype({"names": ["data", "n", "point_step", "off_x", "off_y", "dst", "cell"],
                            "formats": [np.uint64, np.uint64, np.int32, np.int32, np.int32, np.uint64, np.uint64],
                            "offsets": [Positions.data.offset, Positions.n.offset, Positions.point_step.offset, Positions.off_x.offset,
                                        Positions.off_y.offset, Positions.dst.offset, Positions.cell.offset],
                            "itemsize": C.sizeof(Positions)})
SAMPLE_MODES = {"nearest": 0, "linear": 1}   # GG_SAMPLE_NEAREST, GG_SAMPLE_LINEAR

# numpy image of an array of gg_point_info: device addresses of one slot's codes and heights (0 = none)
POINT_INFO_DTYPE = np.dtype({"names": ["codes", "height"], "formats": [np.uint64, np.uint64], "offsets": [0, 8], "itemsize": 16})
# per-point classes of gg_get_point_classes / gg_point_info_to_device (code >> 24)
PC_ABSENT, PC_KEPT, PC_KEPT_BORDER, PC_IGNORED, PC_IGNORED_BORDER, PC_OUTLIER = range(6)

# numpy image of an array of gg_scan_desc (ScanDesc)
SCAN_DESC_DTYPE = np.dtype({"names": ["slot", "flags", "n_points", "origin", "base_z"],
                            "formats": [np.int32, np.int32, np.uint64, (np.float32, 3), np.float64],
                            "offsets": [ScanDesc.slot.offset, ScanDesc.flags.offset, ScanDesc.n_points.offset, ScanDesc.origin.offset,
                                        ScanDesc.base_z.offset], "itemsize": C.sizeof(ScanDesc)})
SCAN_DEVICE_POSE = 1   # GG_SCAN_DEVICE_POSE: the scan's origin / base_z come from the slot's device scan pose
SCAN_DEVICE_COUNT = 2  # GG_SCAN_DEVICE_COUNT: n_points is the capacity; the scan runs on the slot's stored device count
SCAN_DEVICE_PART_COUNTS = 4  # GG_SCAN_DEVICE_PART_COUNTS: merged scans only; each part's n_points is its capacity and the part
                             # runs on the slot's stored part count
SCAN_DEVICE_MASK = 8   # GG_SCAN_DEVICE_MASK: the scan runs only if the slot's stored device scan mask is nonzero; else it is skipped


class DevicePoses(C.Structure):
    """gg_device_poses: device addresses of the per-slot pose arrays of gg_update_poses_from_device (None = not given)."""

    _fields_ = [
        ("xy", C.c_void_p),
        ("T_base_from_map", C.c_void_p),
        ("origin", C.c_void_p),
        ("base_z", C.c_void_p),
    ]


class DeviceResets(C.Structure):
    """gg_device_resets: device addresses of the odometry poses and the mask of gg_init_maps_from_device (None = NULL)."""

    _fields_ = [
        ("xyz", C.c_void_p),
        ("mask", C.c_void_p),
    ]


class DeviceConfigs(C.Structure):
    """gg_device_configs: device addresses of the configurations and the mask of gg_set_slot_configs_from_device (None =
    NULL)."""

    _fields_ = [
        ("cfg", C.c_void_p),
        ("mask", C.c_void_p),
    ]


SNAPSHOT_MAGIC = 0x534D4747   # GG_SNAPSHOT_MAGIC ("GGMS")
SNAPSHOT_VERSION = 1          # GG_SNAPSHOT_VERSION


class MapSnapshot(C.Structure):
    """gg_map_snapshot: the 64-byte header of a map snapshot record; "ground" follows at byte 64 and "groundpatch" at
    64 + 4 * N2p (N2p = N * N rounded up to a multiple of 4), both column-major."""

    _fields_ = [
        ("magic", C.c_uint32),
        ("version", C.c_uint32),
        ("cells_per_side", C.c_int32),
        ("resolution", C.c_float),
        ("position", C.c_double * 2),
        ("reserved", C.c_uint32 * 8),
    ]


def snapshot_bytes(n):
    """The size of one snapshot record of an n x n map: 64 + 8 * N2p, N2p = n * n rounded up to a multiple of 4."""
    return C.sizeof(MapSnapshot) + 8 * ((n * n + 3) // 4 * 4)


class MapRestore(C.Structure):
    """gg_map_restore: device addresses of the snapshot pool, the index and the status of gg_restore_maps_from_device
    (None = NULL)."""

    _fields_ = [
        ("pool", C.c_void_p),
        ("n_pool", C.c_int),
        ("index", C.c_void_p),
        ("status", C.c_void_p),
    ]


class StepSnapshots(C.Structure):
    """gg_step_snapshots: a step plan's restore (stage 3) and save (stage 9) stages (gg_step_plan_create_with_snapshots)."""

    _fields_ = [
        ("restore", MapRestore),
        ("save", C.c_void_p),
        ("save_mask", C.c_void_p),
    ]


class StepDesc(C.Structure):
    """gg_step_desc: the fixed batch and caller device buffers of a step plan (gg_step_plan_create)."""

    _fields_ = [
        ("count", C.c_int),
        ("scans", C.c_void_p),
        ("dev_points", C.c_void_p),
        ("msgs", C.c_void_p),
        ("dev_T_map_from_frame", C.c_void_p),
        ("dev_n_points", C.c_void_p),
        ("poses", DevicePoses),
        ("dev_moved", C.c_void_p),
        ("outs", C.c_void_p),
        ("select", C.c_uint),
        ("dev_counts", C.c_void_p),
    ]


class StepParts(C.Structure):
    """gg_step_parts: the parts of a step plan whose step is a merged scan (gg_step_plan_create_with_parts)."""

    _fields_ = [
        ("n_parts", C.c_void_p),
        ("parts", C.c_void_p),
        ("dev_T_map_from_part", C.c_void_p),
        ("dev_part_counts", C.c_void_p),
        ("parts_per_slot", C.c_int),
    ]


class StepReadouts(C.Structure):
    """gg_step_readouts: the read-out calls of a step plan's stage 8 (gg_step_plan_create_with_readouts); zero = not run."""

    _fields_ = [
        ("n_layer_names", C.c_int),
        ("layer_names", C.c_void_p),
        ("layers", C.c_void_p),
        ("n_image_names", C.c_int),
        ("image_names", C.c_void_p),
        ("images", C.c_void_p),
        ("image_ranges", C.c_void_p),
        ("terrain_images", C.c_void_p),
        ("n_sample_names", C.c_int),
        ("sample_names", C.c_void_p),
        ("samples", C.c_void_p),
        ("sample_mode", C.c_int),
        ("point_info", C.c_void_p),
        ("eval_counts", C.c_void_p),
    ]


class PlanReadouts:
    """The read-out tensors of a step plan (StepPlan.readouts), rewritten by every replay; None where not asked for.
    Each has the shape and layout of the standalone method's result:
      layers        : float32 [count, n_names, N, N] with column-major planes (get_layers_to_device)
      images, ranges: uint8 [count, n_names, N, N] and float32 [count, n_names, 2] (layer_images_to_device)
      terrain       : float32 [count, N, N, 3] (terrain_images_to_device)
      positions     : the CUDA position tensors the plan reads at every replay (write the next step's positions into them)
      samples, cells: per slot float32 [n_names, n] and int32 [n] (sample_layers_to_device)
      codes, height : per slot int32 / float32 [n], n the scan's capacity; the first last_scan_points entries are
                      written (point_info_to_device)
      tallies       : int64 [count, 1024, 2], to which every replay adds its tallies (eval_counts_to_device(out=))"""

    def __init__(self):
        self.layers = self.images = self.ranges = self.terrain = None
        self.positions = self.samples = self.cells = self.codes = self.height = self.tallies = None


class DeviceOutputs:
    """What GroundGridB200.run_scans_to_device returns: per-scan views into flat CUDA tensors.
      labels[k] : uint8 [n_k], the labels of every input point (None unless asked for)
      cloud[k]  : float32 [n_k, 8], the selected output points as 32-byte records, intensity 49 / 99 (None without select)
      index[k]  : int32 [n_k], input index of each selected point (None unless asked for)
      counts    : int32 [count] on the device, selected points of each scan (None without select)
    Only the first counts[k] entries of cloud[k] / index[k] are written.  They are complete in the order of `stream`.
    With device_counts=True every n_k is the scan's capacity: labels[k] then has capacity length and only its first u
    entries are written, u being the count the scan used (last_scan_points)."""

    def __init__(self, labels, cloud, index, counts, stream):
        self.labels, self.cloud, self.index, self.counts, self.stream = labels, cloud, index, counts, stream

    def trimmed(self):
        """(cloud, index) with every view cut to its count: one host synchronisation (counts.tolist()) per batch."""
        import torch

        with torch.cuda.stream(self.stream):
            n = self.counts.tolist()

        def cut(views):
            return None if views is None else [v[:k] for v, k in zip(views, n)]

        return cut(self.cloud), cut(self.index)


class StepPlan:
    """What GroundGridB200.step_plan returns: one step of a fixed batch recorded as a CUDA graph (gg_step_plan_create).
      launch(stream=None) : replays the step on `stream` (default: the current stream), without a host wait; inside a
                            torch.cuda.graph capture it adds the step to the captured graph
      outputs             : DeviceOutputs of the step (allocated at capacity), rewritten by every replay
      moved               : int32 [count] dev_moved of the roll, or None
      readouts            : PlanReadouts of the step's read-outs (all None for a plan without them)
      restore_status      : int32 [count] status of the step's restore, or None
      saved               : uint8 [count, snapshot_bytes] records of the step's save, or None
      kernels             : kernel launches per replay
      close()             : gg_step_plan_destroy (waits for the device); the slots accept every call again
    The plan keeps its input and output tensors alive; write the next step's inputs into them (e.g. with copy_) on the
    stream before launching."""

    def __init__(self, owner, p, outputs, moved, keep, readouts=None):
        self._owner, self._p, self.outputs, self.moved, self._keep = owner, p, outputs, moved, keep
        self.readouts = readouts if readouts is not None else PlanReadouts()
        self.restore_status = self.saved = None
        owner._plans.add(self)

    def launch(self, stream=None):
        import torch

        if not self._p:
            raise GroundGridError(-3, "the step plan is closed")
        st = torch.cuda.current_stream(torch.device("cuda", self._owner.device)) if stream is None else stream
        _check(self._owner._l.gg_step_plan_launch(self._p, st.cuda_stream or None))

    @property
    def kernels(self):
        return self._owner._l.gg_step_plan_kernels(self._p)

    def close(self):
        if getattr(self, "_p", None):
            p, self._p = self._p, None
            self._owner._plans.discard(self)
            # a plan collected in one cycle with its handle may find the handle closed already: gg_destroy destroyed it
            # (the handle's weak set of plans is emptied before either finaliser runs)
            if self._owner._h:
                _check(self._owner._l.gg_step_plan_destroy(p))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_lib = None


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """Loads libgroundgrid_b200.so (building it in-tree with nvcc if it is missing/stale)."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        try:
            _build.build_core()
        except Exception:
            if not os.path.exists(_build.LIB):
                raise
    L = C.CDLL(_build.LIB)
    vp, i, d, sz = C.c_void_p, C.c_int, C.c_double, C.c_size_t
    sig = {
        "gg_default_config": (None, [C.POINTER(Config)]),
        "gg_last_error": (C.c_char_p, []),
        "gg_create": (i, [d, C.c_float, i, i, sz, C.c_uint, vp, C.POINTER(vp)]),
        "gg_destroy": (i, [vp]),
        "gg_cells_per_side": (i, [vp]),
        "gg_num_slots": (i, [vp]),
        "gg_set_config": (i, [vp, C.POINTER(Config)]),
        "gg_get_config": (i, [vp, C.POINTER(Config)]),
        "gg_set_slot_config": (i, [vp, i, C.POINTER(Config)]),
        "gg_get_slot_config": (i, [vp, i, C.POINTER(Config)]),
        "gg_init_map": (i, [vp, i, d, d, d]),
        "gg_update_pose": (i, [vp, i, d, d, vp, C.POINTER(i)]),
        "gg_update_pose_batch": (i, [vp, i, vp, vp, vp, vp]),
        "gg_get_map_position": (i, [vp, i, vp]),
        "gg_set_map_position": (i, [vp, i, d, d]),
        "gg_filter_cloud": (i, [vp, i, vp, sz, vp, d, vp, vp, vp, C.POINTER(sz)]),
        "gg_filter_cloud_batch": (i, [vp, i, vp, vp, vp]),
        "gg_filter_cloud_batch_begin": (i, [vp, i, vp, vp, vp, C.POINTER(i)]),
        "gg_filter_cloud_batch_wait": (i, [vp, i]),
        "gg_upload_points": (i, [vp, i, vp, sz]),
        "gg_run_scans": (i, [vp, i, vp, i]),
        "gg_download_labels": (i, [vp, i, vp, sz]),
        "gg_synchronize": (i, [vp]),
        "gg_run_scans_device": (i, [vp, i, vp, vp, i]),
        "gg_run_scans_to_device": (i, [vp, i, vp, vp, vp, C.c_uint, vp, vp]),
        "gg_upload_cloud_msg": (i, [vp, i, vp, sz, i, vp, vp]),
        "gg_run_cloud_msgs_to_device": (i, [vp, i, vp, vp, vp, C.c_uint, vp, vp]),
        "gg_run_merged_cloud_msgs_to_device": (i, [vp, i, vp, vp, vp, vp, C.c_uint, vp, vp]),
        "gg_upload_cloud_msgs": (i, [vp, i, i, vp]),
        "gg_terrain_image": (i, [vp, i, vp]),
        "gg_layer_image_u8": (i, [vp, i, C.c_char_p, vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
        "gg_get_point_classes": (i, [vp, i, vp, sz]),
        "gg_detect_ground_patches": (i, [vp, i]),
        "gg_detect_ground_patch": (i, [vp, i, i, i, i]),
        "gg_spiral_ground_interpolation": (i, [vp, i, d]),
        "gg_interpolate_cell": (i, [vp, i, i, i]),
        "gg_eval_accumulate": (i, [vp, i]),
        "gg_eval_read": (i, [vp, vp, i]),
        "gg_eval_counts_to_device": (i, [vp, i, vp, vp, vp]),
        "gg_point_info_to_device": (i, [vp, i, vp, vp, vp]),
        "gg_update_poses_from_device": (i, [vp, i, vp, C.POINTER(DevicePoses), vp, vp]),
        "gg_last_scan_points": (i, [vp, i, C.POINTER(sz)]),
        "gg_set_point_counts_from_device": (i, [vp, i, vp, vp, vp]),
        "gg_set_part_counts_from_device": (i, [vp, i, vp, i, vp, vp]),
        "gg_step_plan_create": (i, [vp, C.POINTER(StepDesc), C.POINTER(vp)]),
        "gg_init_maps_from_device": (i, [vp, i, vp, C.POINTER(DeviceResets), vp]),
        "gg_step_plan_create_with_resets": (i, [vp, C.POINTER(StepDesc), C.POINTER(DeviceResets), C.POINTER(vp)]),
        "gg_step_plan_create_with_readouts": (i, [vp, C.POINTER(StepDesc), C.POINTER(DeviceResets), C.POINTER(StepReadouts), C.POINTER(vp)]),
        "gg_step_plan_create_with_parts": (i, [vp, C.POINTER(StepDesc), C.POINTER(StepParts), C.POINTER(DeviceResets), C.POINTER(StepReadouts),
                                               C.POINTER(vp)]),
        "gg_set_slot_configs_from_device": (i, [vp, i, vp, C.POINTER(DeviceConfigs), vp]),
        "gg_step_plan_create_with_configs": (i, [vp, C.POINTER(StepDesc), C.POINTER(StepParts), C.POINTER(DeviceResets), C.POINTER(DeviceConfigs),
                                                 C.POINTER(StepReadouts), C.POINTER(vp)]),
        "gg_map_snapshot_bytes": (sz, [vp]),
        "gg_save_maps_to_device": (i, [vp, i, vp, vp, vp, vp]),
        "gg_restore_maps_from_device": (i, [vp, i, vp, C.POINTER(MapRestore), vp]),
        "gg_step_plan_create_with_snapshots": (i, [vp, C.POINTER(StepDesc), C.POINTER(StepParts), C.POINTER(DeviceResets), C.POINTER(DeviceConfigs),
                                                   C.POINTER(StepSnapshots), C.POINTER(StepReadouts), C.POINTER(vp)]),
        "gg_set_scan_masks_from_device": (i, [vp, i, vp, vp, vp]),
        "gg_step_plan_create_with_scan_masks": (i, [vp, C.POINTER(StepDesc), C.POINTER(StepParts), C.POINTER(DeviceResets), C.POINTER(DeviceConfigs),
                                                    C.POINTER(StepSnapshots), C.POINTER(StepReadouts), vp, C.POINTER(vp)]),
        "gg_step_plan_launch": (i, [vp, vp]),
        "gg_step_plan_kernels": (i, [vp]),
        "gg_step_plan_destroy": (i, [vp]),
        "gg_profile_enable": (i, [vp, i]),
        "gg_profile_read": (i, [vp, vp, vp, i]),
        "gg_profile_kernel_count": (i, []),
        "gg_profile_kernel_name": (C.c_char_p, [i]),
        "gg_get_output": (i, [vp, i, vp, vp, C.POINTER(sz)]),
        "gg_get_layer": (i, [vp, i, C.c_char_p, vp]),
        "gg_set_layer": (i, [vp, i, C.c_char_p, vp]),
        "gg_layer_device_ptr": (i, [vp, i, C.c_char_p, C.POINTER(vp)]),
        "gg_get_layers_to_device": (i, [vp, i, vp, i, vp, vp, vp]),
        "gg_set_layers_from_device": (i, [vp, i, vp, i, vp, vp, vp]),
        "gg_sample_layers_to_device": (i, [vp, i, vp, vp, i, vp, i, vp]),
        "gg_layer_images_to_device": (i, [vp, i, vp, i, vp, vp, vp, vp]),
        "gg_terrain_images_to_device": (i, [vp, i, vp, vp, vp]),
        "gg_stream": (vp, [vp]),
        "gg_num_streams": (i, [vp]),
        "gg_host_pack_threads": (i, [vp]),
        "gg_last_batch_transfer": (i, [vp, C.POINTER(C.c_size_t)]),
        "gg_fork_streams": (i, [vp]),
        "gg_join_streams": (i, [vp]),
        "gg_kernel_launches": (C.c_uint64, [vp]),
        "gg_spiral_schedule_info": (i, [vp, C.POINTER(i), C.POINTER(i), C.POINTER(i)]),
        # host-only helpers (no device needed)
        "gg_host_cells_per_side": (i, [d, C.c_float]),
        "gg_host_expected_points": (i, [d, C.c_float, vp]),
        "gg_host_spiral_schedule": (i, [i, vp, i, vp, i, C.POINTER(i), C.POINTER(i)]),
        "gg_host_move_map": (i, [d, vp, d, d, vp]),
        "gg_host_resolve_move": (i, [d, vp, d, d, vp]),
        "gg_host_geometry_constants": (i, [d, C.c_float, C.c_uint, vp]),
        "gg_host_config_constants": (i, [C.POINTER(Config), vp]),
        "gg_host_config_registry": (i, [i, i, vp, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _check(rc):
    if rc != 0:
        raise GroundGridError(rc, load().gg_last_error().decode(errors="replace"))


# ---- host-only helpers --------------------------------------------------------------------
def host_cells_per_side(dimension_m, resolution):
    return load().gg_host_cells_per_side(float(dimension_m), np.float32(resolution))


def host_expected_points(dimension_m, resolution):
    n = host_cells_per_side(dimension_m, resolution)
    out = np.empty((n, n), np.float32, order="F")
    load().gg_host_expected_points(float(dimension_m), np.float32(resolution), _ptr(out))
    return out


def host_spiral_schedule(n):
    """(level_start[int32, levels+1], visits[(x, y) per visit, grouped by level])."""
    L = load()
    nl, nv = C.c_int(0), C.c_int(0)
    L.gg_host_spiral_schedule(n, None, 0, None, 0, C.byref(nl), C.byref(nv))
    ls = np.zeros(nl.value + 1, np.int32)
    vs = np.zeros(nv.value, np.uint32)
    L.gg_host_spiral_schedule(n, _ptr(ls), ls.size, _ptr(vs), vs.size, C.byref(nl), C.byref(nv))
    return ls, np.stack([vs & 0xFFFF, vs >> 16], axis=1).astype(np.int32)


def host_move_map(res, pos_xy, new_xy):
    pos = np.array(pos_xy, np.float64)
    shift = np.zeros(2, np.int32)
    moved = load().gg_host_move_map(float(res), _ptr(pos), float(new_xy[0]), float(new_xy[1]), _ptr(shift))
    return bool(moved), pos, (int(shift[0]), int(shift[1]))


def host_resolve_move(res, pos_xy, new_xy):
    """The cell-shift resolve of gg_update_poses_from_device run on the host: (1 moved / 0 not / -1 invalid, new position,
    shift).  An invalid pose (non-finite, or a shift outside int32) leaves the position and the zero shift untouched."""
    pos = np.array(pos_xy, np.float64)
    shift = np.zeros(2, np.int32)
    status = load().gg_host_resolve_move(float(res), _ptr(pos), float(new_xy[0]), float(new_xy[1]), _ptr(shift))
    return int(status), pos, (int(shift[0]), int(shift[1]))


GEOMETRY_CONSTANTS = ("N", "N2", "full_layers", "res_f", "res", "rres", "len", "half", "res_sq")
CONFIG_CONSTANTS = ("max_ring", "pc_var_thresh_f", "min_outlier_conf", "outlier_tol", "gp_thresh", "df_sq", "mdf_sq", "mdf10_sq",
                    "psc_sq", "occ_factor", "occ_factor2", "dec_factor", "lab_fac", "lab_thres", "lab_obs", "decay_floor_ok")


def default_config():
    cfg = Config()
    load().gg_default_config(C.byref(cfg))
    return cfg


def config_tensor(configs, device="cuda"):
    """uint8 tensor [n, sizeof(gg_config)] holding `configs` (a list of Config objects, or dicts of the fields that differ
    from the defaults) in the gg_config layout, on `device`: the input of set_configs_from_device and of a step plan's
    configs.  config_field gives typed views of its fields."""
    import torch

    rows = []
    for c in configs:
        if not isinstance(c, Config):
            d, c = c, default_config()
            for k, v in d.items():
                if not hasattr(c, k):
                    raise KeyError(k)
                setattr(c, k, v)
        rows.append(np.frombuffer(bytes(c), np.uint8))
    a = np.stack(rows) if rows else np.zeros((0, C.sizeof(Config)), np.uint8)
    return torch.from_numpy(a.copy()).to(device)


def config_field(t, name):
    """The `name` field of every row of a config_tensor as a strided view ([n], int32 or float64), so that the field can be
    written in place on the GPU: config_field(t, "outlier_tolerance").uniform_(0.05, 0.3)."""
    import torch

    if t.dtype != torch.uint8 or t.dim() != 2 or t.shape[1] != C.sizeof(Config) or not t.is_contiguous():
        raise ValueError("t must be a contiguous uint8 tensor [n, sizeof(gg_config)] (config_tensor)")
    ctype = dict(Config._fields_)[name]
    off = getattr(Config, name).offset
    if ctype is C.c_int:
        return t.view(torch.int32)[:, off // 4]
    return t.view(torch.float64)[:, off // 8]


def host_geometry_constants(dimension_m, resolution, full_layers=False):
    """{name: value} of the geometry constants the kernels get (gg::Const)."""
    out = np.zeros(len(GEOMETRY_CONSTANTS), np.float64)
    load().gg_host_geometry_constants(float(dimension_m), np.float32(resolution), GG_FLAG_FULL_LAYERS if full_layers else 0, _ptr(out))
    return dict(zip(GEOMETRY_CONSTANTS, out.tolist()))


def host_config_constants(cfg):
    """{name: value} of the constants derived from one configuration (gg::CfgConst)."""
    out = np.zeros(len(CONFIG_CONSTANTS), np.float64)
    load().gg_host_config_constants(C.byref(cfg), _ptr(out))
    return dict(zip(CONFIG_CONSTANTS, out.tolist()))


def host_config_registry(n_slots, ops):
    """Replays ops = [(slot or None for the whole handle, Config)] on the configuration-variant bookkeeping of a new
    handle; (("invalidate", v), None) marks variant v as holding unknown device data (a failed build).  Returns (per op: (variant id, built, live variants, variant ids) as int array [n_ops, 4], final variant
    of every slot)."""
    n = len(ops)
    slots = np.array([-1 if s is None else (-2 - s[1] if isinstance(s, tuple) else s) for s, _ in ops], np.int32)
    cfgs = (Config * max(1, n))(*[c if c is not None else default_config() for _, c in ops])
    out = np.zeros(4 * n + n_slots, np.int32)
    rc = load().gg_host_config_registry(int(n_slots), n, _ptr(slots), C.cast(cfgs, C.c_void_p), _ptr(out))
    if rc != 0:
        raise GroundGridError(rc, "gg_host_config_registry: bad argument")
    return out[:4 * n].reshape(n, 4), out[4 * n:]


# ---- device handle ------------------------------------------------------------------------
class GroundGridB200:
    """One handle = `n_slots` independent GroundGrid maps on one GPU (see the C header)."""

    def __init__(self, dimension_m=120.0, resolution=0.33, device=0, n_slots=1, max_points=131072,
                 full_layers=False, stream=None):
        self._l = load()
        h = C.c_void_p()
        flags = GG_FLAG_FULL_LAYERS if full_layers else 0
        _check(self._l.gg_create(float(dimension_m), np.float32(resolution), int(device), int(n_slots), int(max_points),
                                 flags, C.c_void_p(stream) if stream else None, C.byref(h)))
        self._h = h
        self.device = int(device)
        self.n = self._l.gg_cells_per_side(h)
        self.n_slots = n_slots
        self.max_points = max_points
        self._plans = weakref.WeakSet()   # live step plans (gg_destroy destroys them)

    def close(self):
        if getattr(self, "_h", None):
            for plan in list(getattr(self, "_plans", ())):   # gg_destroy destroys them
                plan._p = None
            self._l.gg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- config / state
    def set_config(self, slot=None, **kw):
        """Changes the given fields.  slot=None: the handle-wide configuration (every slot's, gg_set_config);
        an integer: that slot's own configuration only (gg_set_slot_config)."""
        cfg = self.get_config(slot)
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        if slot is None:
            _check(self._l.gg_set_config(self._h, C.byref(cfg)))
        else:
            _check(self._l.gg_set_slot_config(self._h, int(slot), C.byref(cfg)))

    def get_config(self, slot=None):
        """The handle-wide configuration (slot=None) or the one a slot runs with (on a device-configured slot: the stored
        configuration, after a wait for the slot's work)."""
        cfg = Config()
        if slot is None:
            _check(self._l.gg_get_config(self._h, C.byref(cfg)))
        else:
            _check(self._l.gg_get_slot_config(self._h, int(slot), C.byref(cfg)))
        return cfg

    def init_map(self, x, y, z, slot=0):
        _check(self._l.gg_init_map(self._h, slot, x, y, z))

    def update_pose(self, x, y, T_base_from_map, slot=0):
        T = np.ascontiguousarray(T_base_from_map, dtype=np.float64).reshape(12)
        moved = C.c_int(0)
        _check(self._l.gg_update_pose(self._h, slot, x, y, _ptr(T), C.byref(moved)))
        return bool(moved.value)

    def update_pose_batch(self, slots, xy, T):
        slots = np.ascontiguousarray(slots, np.int32)
        xy = np.ascontiguousarray(xy, np.float64).reshape(len(slots), 2)
        T = np.ascontiguousarray(T, np.float64).reshape(len(slots), 12)
        moved = np.zeros(len(slots), np.int32)
        _check(self._l.gg_update_pose_batch(self._h, len(slots), _ptr(slots), _ptr(xy), _ptr(T), _ptr(moved)))
        return moved.astype(bool)

    def update_poses_from_device_ptrs(self, slots, xy_ptr, T_ptr, origin_ptr, base_z_ptr, moved_ptr, stream_ptr):
        """gg_update_poses_from_device with raw device addresses (ints, or None for NULL); stream_ptr None = the legacy
        default stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        p = DevicePoses(xy_ptr, T_ptr, origin_ptr, base_z_ptr)
        _check(self._l.gg_update_poses_from_device(self._h, len(sl), _ptr(sl), C.byref(p), moved_ptr, stream_ptr))

    def update_poses_from_device(self, slots, xy=None, T=None, origins=None, base_z=None, moved=False, stream=None):
        """Rolls and / or scan poses of `slots` from CUDA tensors, resolved on the device (gg_update_poses_from_device).
          xy      : float64 [count, 2] odometry positions, with T float64 [count, 3, 4] (or [count, 12]) of
                    lookupTransform("base_link", "map"): rolls bit-identical to update_pose_batch
          origins : float32 [count, 3] cloudOrigin, with base_z float64 [count]: the scan pose that scans run with
                    origins="device" use
          moved   : also return an int32 [count] tensor: 1 the cells shifted, 0 not, -1 invalid pose (map untouched)
          stream  : torch.cuda.Stream the work is ordered on (default: the current stream); `moved` is allocated on it.
        Every tensor must be contiguous on this handle's device.  The call returns without waiting for the device; the
        pose tensors may be freed or refilled right after it when they belong to `stream` (others are marked in use on
        `stream`).  Afterwards the slots' map positions live on the device: position() and the other host calls that
        need them wait for the slots' work first."""
        torch, dev, current, stream = self._layer_stream(stream)
        count = len(slots)
        want = {"xy": (xy, torch.float64, (count, 2)), "T": (T, torch.float64, (count, 12)), "origins": (origins, torch.float32, (count, 3)),
                "base_z": (base_z, torch.float64, (count,))}
        ptrs = {}
        for name, (t, dtype, shape) in want.items():
            if t is None:
                ptrs[name] = None
                continue
            if t.dtype != dtype or t.device != dev or not t.is_contiguous() or t.numel() != int(np.prod(shape)) or t.shape[0] != count:
                raise ValueError(f"{name} must be a contiguous {dtype} tensor {shape} on {dev}")
            if stream != current:
                t.record_stream(stream)
            ptrs[name] = t.data_ptr() if count else None
        out = None
        if moved:
            with torch.cuda.stream(stream):
                out = torch.empty(count, dtype=torch.int32, device=dev)
        self.update_poses_from_device_ptrs(slots, ptrs["xy"], ptrs["T"], ptrs["origins"], ptrs["base_z"],
                                           out.data_ptr() if out is not None and count else None, stream.cuda_stream or None)
        return out

    def set_point_counts_from_device_ptrs(self, slots, counts_ptr, stream_ptr):
        """gg_set_point_counts_from_device with a raw device address (int32 [count]); stream_ptr None = the legacy default
        stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        _check(self._l.gg_set_point_counts_from_device(self._h, len(sl), _ptr(sl), counts_ptr, stream_ptr))

    def set_point_counts_from_device(self, slots, counts, stream=None):
        """The point counts of the slots' next scans from a CUDA tensor (gg_set_point_counts_from_device): scans run with
        device_counts=True use them.
          counts : int32 [count] (int64 is converted on `stream`, without a host wait), contiguous on this handle's device
          stream : torch.cuda.Stream the work is ordered on (default: the current stream).
        The call returns without waiting for the device; `counts` may be freed or overwritten right after it when it
        belongs to `stream` (another stream's tensor is marked in use on `stream`).  A count outside [0, capacity] runs the
        scan empty."""
        torch, dev, current, stream = self._layer_stream(stream)
        count = len(slots)
        if counts.device != dev or counts.numel() != count or counts.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"counts must be an int32 or int64 tensor of {count} entries on {dev}")
        if stream != current:
            counts.record_stream(stream)
        if counts.dtype != torch.int32 or not counts.is_contiguous():
            with torch.cuda.stream(stream):
                counts = counts.reshape(-1).to(torch.int32).contiguous()
        self.set_point_counts_from_device_ptrs(slots, counts.data_ptr() if count else None, stream.cuda_stream or None)

    def set_scan_masks_from_device_ptrs(self, slots, mask_ptr, stream_ptr):
        """gg_set_scan_masks_from_device with a raw device address (int32 [count]); stream_ptr None = the legacy default
        stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        _check(self._l.gg_set_scan_masks_from_device(self._h, len(sl), _ptr(sl), mask_ptr, stream_ptr))

    def set_scan_masks_from_device(self, slots, mask, stream=None):
        """Which of the slots' next scans run, from a CUDA tensor (gg_set_scan_masks_from_device): scans run with
        device_masks=True run where the slot's mask is nonzero and are skipped where it is 0 (the map, position and stored
        inputs stay untouched, no output is written but a zero count, and the slot's last scan becomes an empty one).
          mask   : int32 [count] (int64 or bool is converted on `stream`, without a host wait), on this handle's device
          stream : torch.cuda.Stream the work is ordered on (default: the current stream).
        The call returns without waiting for the device; `mask` may be freed or overwritten right after it when it belongs
        to `stream` (another stream's tensor is marked in use on `stream`)."""
        torch, dev, current, stream = self._layer_stream(stream)
        count = len(slots)
        if mask.device != dev or mask.numel() != count or mask.dtype not in (torch.int32, torch.int64, torch.bool):
            raise ValueError(f"mask must be an int32, int64 or bool tensor of {count} entries on {dev}")
        if stream != current:
            mask.record_stream(stream)
        if mask.dtype != torch.int32 or not mask.is_contiguous():
            with torch.cuda.stream(stream):
                mask = mask.reshape(-1).to(torch.int32).contiguous()
        self.set_scan_masks_from_device_ptrs(slots, mask.data_ptr() if count else None, stream.cuda_stream or None)

    def set_part_counts_from_device_ptrs(self, slots, parts_per_slot, counts_ptr, stream_ptr):
        """gg_set_part_counts_from_device with a raw device address (int32 [count, parts_per_slot]); stream_ptr None = the
        legacy default stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        _check(self._l.gg_set_part_counts_from_device(self._h, len(sl), _ptr(sl), int(parts_per_slot), counts_ptr, stream_ptr))

    def set_part_counts_from_device(self, slots, counts, stream=None):
        """The per-part point counts of the slots' next merged scans from a CUDA tensor (gg_set_part_counts_from_device):
        merged scans run with device_counts=True use them.
          counts : int32 [count, P] (int64 is converted on `stream`, without a host wait), on this handle's device; entry
                   [k, p] is the count of part p of slots[k], P (1 ... MAX_CLOUD_PARTS) the most parts such a scan may have
          stream : torch.cuda.Stream the work is ordered on (default: the current stream).
        The call returns without waiting for the device; `counts` may be freed or overwritten right after it when it
        belongs to `stream` (another stream's tensor is marked in use on `stream`).  A count outside [0, capacity] runs
        the part empty."""
        torch, dev, current, stream = self._layer_stream(stream)
        count = len(slots)
        if counts.device != dev or counts.dim() != 2 or counts.shape[0] != count or counts.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"counts must be an int32 or int64 tensor [{count}, parts] on {dev}")
        if stream != current:
            counts.record_stream(stream)
        if counts.dtype != torch.int32 or not counts.is_contiguous():
            with torch.cuda.stream(stream):
                counts = counts.to(torch.int32).contiguous()
        self.set_part_counts_from_device_ptrs(slots, counts.shape[1], counts.data_ptr() if count else None, stream.cuda_stream or None)

    def init_maps_from_device_ptrs(self, slots, xyz_ptr, mask_ptr, stream_ptr):
        """gg_init_maps_from_device with raw device addresses (ints, or None for NULL); stream_ptr None = the legacy
        default stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        r = DeviceResets(xyz_ptr, mask_ptr)
        _check(self._l.gg_init_maps_from_device(self._h, len(sl), _ptr(sl), C.byref(r), stream_ptr))

    def init_maps_from_device(self, slots, xyz, mask=None, stream=None):
        """init_map of the slots a device mask picks, at device poses (gg_init_maps_from_device).
          xyz    : float64 [count, 3] odometry x, y, z, as init_map takes them
          mask   : int32 [count], nonzero = start slots[k] over; None = every slot (which then needs no map beforehand)
          stream : torch.cuda.Stream the work is ordered on (default: the current stream).
        Every tensor must be contiguous on this handle's device.  The call returns without waiting for the device; the
        tensors may be freed or refilled right after it when they belong to `stream` (others are marked in use on
        `stream`).  Afterwards every slot of the call has a device-owned position, keeps its stored device scan pose and
        count, and refuses point_info_to_device until its next scan, reset or not (see the C header)."""
        if xyz is None:
            raise ValueError("xyz is required")
        torch, dev, current, stream = self._layer_stream(stream)
        count = len(slots)
        ptrs = []
        for name, t, dtype, shape in (("xyz", xyz, torch.float64, (count, 3)), ("mask", mask, torch.int32, (count,))):
            if t is None:
                ptrs.append(None)
                continue
            if t.dtype != dtype or t.device != dev or not t.is_contiguous() or t.numel() != int(np.prod(shape)) or (count and t.shape[0] != count):
                raise ValueError(f"{name} must be a contiguous {dtype} tensor {shape} on {dev}")
            if stream != current:
                t.record_stream(stream)
            ptrs.append(t.data_ptr() if count else None)
        self.init_maps_from_device_ptrs(slots, ptrs[0], ptrs[1], stream.cuda_stream or None)

    def set_configs_from_device_ptrs(self, slots, cfg_ptr, mask_ptr, stream_ptr):
        """gg_set_slot_configs_from_device with raw device addresses (ints, or None for NULL); stream_ptr None = the legacy
        default stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        c = DeviceConfigs(cfg_ptr, mask_ptr)
        _check(self._l.gg_set_slot_configs_from_device(self._h, len(sl), _ptr(sl), C.byref(c), stream_ptr))

    def set_configs_from_device(self, slots, cfgs, mask=None, stream=None):
        """set_config(slot=...) for the slots a device mask picks, with configurations in GPU memory
        (gg_set_slot_configs_from_device).
          cfgs   : uint8 [count, sizeof(gg_config)] (config_tensor), one configuration per slot
          mask   : int32 [count], nonzero = reconfigure slots[k]; None = every slot
          stream : torch.cuda.Stream the work is ordered on (default: the current stream).
        Every tensor must be contiguous on this handle's device.  The call returns without waiting for the device; the
        tensors may be freed or refilled right after it when they belong to `stream` (others are marked in use on
        `stream`).  Afterwards every slot of the call is device-configured, reconfigured or not: get_config(slot) waits
        for the slot's work and returns the stored configuration (see the C header)."""
        torch, dev, current, stream = self._layer_stream(stream)
        count = len(slots)
        ptrs = []
        for name, t, dtype, shape in (("cfgs", cfgs, torch.uint8, (count, C.sizeof(Config))), ("mask", mask, torch.int32, (count,))):
            if t is None:
                ptrs.append(None)
                continue
            if t.dtype != dtype or t.device != dev or not t.is_contiguous() or t.numel() != int(np.prod(shape)) or (count and t.shape[0] != count):
                raise ValueError(f"{name} must be a contiguous {dtype} tensor {shape} on {dev}")
            if stream != current:
                t.record_stream(stream)
            ptrs.append(t.data_ptr() if count else None)
        if cfgs is None and count:
            raise ValueError("cfgs is required")
        self.set_configs_from_device_ptrs(slots, ptrs[0], ptrs[1], stream.cuda_stream or None)

    @property
    def snapshot_bytes(self):
        """Bytes of one map snapshot record of this handle (gg_map_snapshot_bytes)."""
        return int(self._l.gg_map_snapshot_bytes(self._h))

    def save_maps_to_device_ptrs(self, slots, dst_ptr, mask_ptr, stream_ptr):
        """gg_save_maps_to_device with raw device addresses (ints, or None for NULL); stream_ptr None = the legacy default
        stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        _check(self._l.gg_save_maps_to_device(self._h, len(sl), _ptr(sl), dst_ptr, mask_ptr, stream_ptr))

    def save_maps_to_device(self, slots, mask=None, out=None, stream=None):
        """Snapshots of the maps of `slots` -- "ground", "groundpatch" and the map position -- as one uint8 CUDA tensor
        [count, snapshot_bytes] (gg_save_maps_to_device); record k starts with a MapSnapshot header.
          mask   : int32 [count] or None: a record whose entry is zero is left untouched (a new `out` starts zeroed then)
          out    : uint8 [count, snapshot_bytes] to fill instead of a new tensor (contiguous, 16-byte aligned)
          stream : torch.cuda.Stream the work is ordered on (default: the current stream).
        The call returns without waiting for the device; work enqueued on `stream` afterwards sees the records.  The
        slots' state does not change."""
        torch, dev, current, stream = self._layer_stream(stream)
        count, rb = len(slots), self.snapshot_bytes
        if out is None:
            with torch.cuda.stream(stream):
                out = (torch.zeros if mask is not None else torch.empty)((count, rb), dtype=torch.uint8, device=dev)
        elif out.dtype != torch.uint8 or out.device != dev or not out.is_contiguous() or tuple(out.shape) != (count, rb):
            raise ValueError(f"out must be a contiguous uint8 tensor {(count, rb)} on {dev}")
        elif stream != current:
            out.record_stream(stream)
        mask_ptr = None
        if mask is not None:
            if mask.dtype != torch.int32 or mask.device != dev or not mask.is_contiguous() or mask.numel() != count:
                raise ValueError(f"mask must be a contiguous int32 tensor ({count},) on {dev}")
            if stream != current:
                mask.record_stream(stream)
            mask_ptr = mask.data_ptr() if count else None
        self.save_maps_to_device_ptrs(slots, out.data_ptr() if count else None, mask_ptr, stream.cuda_stream or None)
        return out

    def restore_maps_from_device_ptrs(self, slots, pool_ptr, n_pool, index_ptr, status_ptr, stream_ptr):
        """gg_restore_maps_from_device with raw device addresses (ints, or None for NULL); stream_ptr None = the legacy
        default stream."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        r = MapRestore(pool_ptr, int(n_pool), index_ptr, status_ptr)
        _check(self._l.gg_restore_maps_from_device(self._h, len(sl), _ptr(sl), C.byref(r), stream_ptr))

    def restore_maps_from_device(self, slots, pool, index=None, status=False, stream=None):
        """Restores slots[k] from snapshot pool[index[k]] (gg_restore_maps_from_device): "ground", "groundpatch" and the
        map position as saved, every other layer as init_map starts it.
          pool   : uint8 CUDA tensor [n_pool, snapshot_bytes] (save_maps_to_device records, or their bytes from a file)
          index  : int32 [count] or None (= k): an index outside [0, n_pool) leaves the slot untouched
          status : True: also return an int32 [count] tensor, 1 restored, 0 index out of range, -1 record rejected
                   (another map size or resolution, or not a snapshot)
          stream : torch.cuda.Stream the work is ordered on (default: the current stream).
        Every slot needs a map already.  The call returns without waiting for the device; afterwards every slot of the
        call has a device-owned position and refuses point_info_to_device until its next scan, restored or not."""
        torch, dev, current, stream = self._layer_stream(stream)
        count, rb = len(slots), self.snapshot_bytes
        if pool.dtype != torch.uint8 or pool.device != dev or not pool.is_contiguous() or pool.dim() != 2 or pool.shape[1] != rb:
            raise ValueError(f"pool must be a contiguous uint8 tensor [n_pool, {rb}] on {dev}")
        if index is not None and (index.dtype != torch.int32 or index.device != dev or not index.is_contiguous() or index.numel() != count):
            raise ValueError(f"index must be a contiguous int32 tensor ({count},) on {dev}")
        ptrs = []
        for t in (pool, index):
            if t is None:
                ptrs.append(None)
                continue
            if stream != current:
                t.record_stream(stream)
            ptrs.append(t.data_ptr() if t.numel() else None)
        st = None
        if status:
            with torch.cuda.stream(stream):
                st = torch.empty(count, dtype=torch.int32, device=dev)
        self.restore_maps_from_device_ptrs(slots, ptrs[0], pool.shape[0], ptrs[1], st.data_ptr() if st is not None and count else None,
                                           stream.cuda_stream or None)
        return st

    def position(self, slot=0):
        xy = np.zeros(2, np.float64)
        _check(self._l.gg_get_map_position(self._h, slot, _ptr(xy)))
        return xy

    def set_position(self, x, y, slot=0):
        _check(self._l.gg_set_map_position(self._h, slot, x, y))

    def layer(self, name, slot=0):
        out = np.empty((self.n, self.n), np.float32, order="F")
        _check(self._l.gg_get_layer(self._h, slot, name.encode(), _ptr(out)))
        return out

    def set_layer(self, name, arr, slot=0):
        a = np.asfortranarray(arr, dtype=np.float32)
        assert a.shape == (self.n, self.n)
        _check(self._l.gg_set_layer(self._h, slot, name.encode(), _ptr(a)))

    def layer_device_ptr(self, name, slot=0):
        p = C.c_void_p()
        _check(self._l.gg_layer_device_ptr(self._h, slot, name.encode(), C.byref(p)))
        return p.value

    @staticmethod
    def _layer_batch_args(slots, names):
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        nm = None if names is None else (C.c_char_p * max(1, len(names)))(*[None if n is None else n.encode() for n in names])
        return sl, (0 if names is None else len(names)), nm

    def get_layers_to_device_ptrs(self, slots, names, dst_ptr, stream_ptr):
        """gg_get_layers_to_device with raw device addresses: dst_ptr float32 [count][n_names][N*N] (each plane
        column-major), stream_ptr an int or None (None = the legacy default stream)."""
        sl, n, nm = self._layer_batch_args(slots, names)
        _check(self._l.gg_get_layers_to_device(self._h, len(sl), _ptr(sl), n, nm, dst_ptr, stream_ptr))

    def set_layers_from_device_ptrs(self, slots, names, src_ptr, stream_ptr):
        """gg_set_layers_from_device with raw device addresses (the layout of get_layers_to_device_ptrs)."""
        sl, n, nm = self._layer_batch_args(slots, names)
        _check(self._l.gg_set_layers_from_device(self._h, len(sl), _ptr(sl), n, nm, src_ptr, stream_ptr))

    def _layer_stream(self, stream):
        import torch

        dev = torch.device("cuda", self.device)
        current = torch.cuda.current_stream(dev)
        return torch, dev, current, (current if stream is None else stream)

    def get_layers_to_device(self, slots, names=("ground", "groundpatch"), out=None, stream=None):
        """Layers `names` of `slots` as one float32 CUDA tensor [count, n_names, N, N] indexed [k, l, i, j] like layer()
        (gg_get_layers_to_device).  Each plane is column-major: the tensor is a transpose(-1, -2) view of a contiguous
        buffer.  It is allocated on `stream` (a torch.cuda.Stream; default: the current stream), or `out` (same shape
        and storage order) is filled.  The call returns without waiting for the device; work enqueued on `stream`
        afterwards sees the layers as of the slots' last enqueued scan or roll."""
        torch, dev, current, stream = self._layer_stream(stream)
        shape = (len(slots), len(names), self.n, self.n)
        if out is None:
            with torch.cuda.stream(stream):
                out = torch.empty(shape, dtype=torch.float32, device=dev).transpose(-1, -2)
        else:
            if tuple(out.shape) != shape or out.dtype != torch.float32 or out.device != dev or not out.transpose(-1, -2).is_contiguous():
                raise ValueError(f"out must be a float32 tensor {shape} on {dev} whose planes are column-major (a transpose(-1, -2) "
                                 "view of a contiguous tensor)")
            if stream != current:
                out.record_stream(stream)
        self.get_layers_to_device_ptrs(slots, names, out.data_ptr(), stream.cuda_stream or None)
        return out

    def set_layers_from_device(self, slots, names, src, stream=None):
        """Writes src [count, n_names, N, N] (indexed [k, l, i, j] like get_layers_to_device returns it) into layers
        `names` of `slots` (gg_set_layers_from_device), ordered on `stream` (default: the current stream).  A tensor
        that is not float32 on this device with column-major planes is first copied into that layout on `stream`.
        `src` may be freed right after the call (a tensor of another stream is marked in use on `stream`)."""
        torch, dev, current, stream = self._layer_stream(stream)
        shape = (len(slots), len(names), self.n, self.n)
        if tuple(src.shape) != shape:
            raise ValueError(f"src must have shape {shape}")
        buf = src.transpose(-1, -2)
        if buf.dtype != torch.float32 or buf.device != dev or not buf.is_contiguous():
            with torch.cuda.stream(stream):
                buf = buf.to(device=dev, dtype=torch.float32).contiguous()
        elif stream != current:
            buf.record_stream(stream)
        self.set_layers_from_device_ptrs(slots, names, buf.data_ptr(), stream.cuda_stream or None)

    def sample_layers_to_device_ptrs(self, slots, queries, names, mode, stream_ptr):
        """gg_sample_layers_to_device with raw device addresses: queries a POSITIONS_DTYPE array, one set per slot;
        mode "nearest" / "linear" (or GG_SAMPLE_*); stream_ptr an int or None (None = the legacy default stream)."""
        sl, n, nm = self._layer_batch_args(slots, names)
        q = None if queries is None else np.ascontiguousarray(queries, POSITIONS_DTYPE)
        m = SAMPLE_MODES[mode] if isinstance(mode, str) else int(mode)
        _check(self._l.gg_sample_layers_to_device(self._h, len(sl), _ptr(sl), _ptr(q), n, nm, m, stream_ptr))

    def sample_layers_to_device(self, slots, positions, names=("ground", "groundpatch"), mode="nearest", cells=False, out=None, stream=None):
        """Values of layers `names` of `slots` at map-frame positions (gg_sample_layers_to_device).
          positions : one CUDA tensor per slot: float32 [n, >= 2] with x, y in columns 0 and 1 and unit column stride
                      (e.g. [n, 2], or the float32 [n, 8] view of 32-byte point records); the row stride is the record step
          mode      : "nearest" (the cell's value) or "linear" (the header's bilinear definition)
          cells     : also return each query's cell i + j * N (-1 outside the map)
          out       : None, or one contiguous float32 [n_names, n] tensor per slot to fill
          stream    : torch.cuda.Stream the work is ordered on (default: the current stream); outputs are allocated on it.
        Returns a list of float32 [n_names, n] tensors (value of name l at query q at [l, q]; NaN outside the map), and
        with cells=True also a list of int32 [n] tensors.  The call returns without waiting for the device; the positions
        may be freed right after it when they were allocated on `stream` (others are marked in use on `stream`)."""
        torch, dev, current, stream = self._layer_stream(stream)
        if len(positions) != len(slots):
            raise ValueError("positions needs one tensor per slot")
        if mode not in SAMPLE_MODES:
            raise ValueError(f"mode must be one of {list(SAMPLE_MODES)}")
        L = len(names)
        q, ns = self._position_sets(torch, dev, positions)
        if out is not None:
            if len(out) != len(slots):
                raise ValueError("out needs one tensor per slot")
            out = [self._stream_out(torch, dev, current, stream, o, (L, n), torch.float32, f"out[{k}]") for k, (o, n) in enumerate(zip(out, ns))]
        out, cell = self._sample_outputs(torch, dev, stream, q, ns, L, out, cells)
        if stream != current:
            for p in positions:
                p.record_stream(stream)
        self.sample_layers_to_device_ptrs(slots, q[:len(slots)], names, mode, stream.cuda_stream or None)
        return (out, cell) if cells else out

    @staticmethod
    def _position_sets(torch, dev, positions):
        """(POSITIONS_DTYPE array with data, n, point_step and offsets of each set of positions, the sets' sizes)."""
        q = np.zeros(max(1, len(positions)), POSITIONS_DTYPE)
        ns = []
        for k, p in enumerate(positions):
            if p.dtype != torch.float32 or p.device != dev or p.dim() != 2 or p.shape[1] < 2 or (p.shape[0] > 1 and p.stride(1) != 1):
                raise ValueError(f"positions[{k}] must be a float32 tensor [n, >= 2] on {dev} with unit column stride")
            n = int(p.shape[0])
            step = 4 * (p.stride(0) if n > 1 else max(2, p.shape[1]))
            if n > 1 and p.stride(0) < 2:
                raise ValueError(f"positions[{k}]: a row stride of {p.stride(0)} elements is no record layout")
            ns.append(n)
            q["data"][k], q["n"][k], q["point_step"][k], q["off_x"][k], q["off_y"][k] = p.data_ptr() if n else 0, n, step, 0, 4
        return q, ns

    @staticmethod
    def _sample_outputs(torch, dev, stream, q, ns, L, out, cells):
        """The lookup results of sets of ns[k] positions: `out` (or float32 [L, n] tensors allocated on `stream`) and, with
        `cells`, int32 [n] tensors; their addresses are written into q.  Returns (out, cells or None)."""
        total = sum(ns)
        if out is None:
            with torch.cuda.stream(stream):
                flat = torch.empty(L * total, dtype=torch.float32, device=dev)
            out = [t.view(L, n) for t, n in zip(torch.split(flat, [L * n for n in ns]), ns)]
        cell = None
        if cells:
            with torch.cuda.stream(stream):
                cell = list(torch.split(torch.empty(total, dtype=torch.int32, device=dev), ns))
        for k, n in enumerate(ns):
            if n:
                q["dst"][k] = out[k].data_ptr()
                q["cell"][k] = cell[k].data_ptr() if cells else 0
        return out, cell

    def layer_images_to_device_ptrs(self, slots, names, dst_ptr, range_ptr, stream_ptr):
        """gg_layer_images_to_device with raw device addresses: dst_ptr uint8 [count][n_names][N][N] (row-major planes),
        range_ptr float32 [count][n_names][2] or None, stream_ptr an int or None (None = the legacy default stream)."""
        sl, n, nm = self._layer_batch_args(slots, names)
        _check(self._l.gg_layer_images_to_device(self._h, len(sl), _ptr(sl), n, nm, dst_ptr, range_ptr, stream_ptr))

    def terrain_images_to_device_ptrs(self, slots, dst_ptr, stream_ptr):
        """gg_terrain_images_to_device with raw device addresses: dst_ptr float32 [count][N][N][3]."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        _check(self._l.gg_terrain_images_to_device(self._h, len(sl), _ptr(sl), dst_ptr, stream_ptr))

    @staticmethod
    def _stream_out(torch, dev, current, stream, out, shape, dtype, what):
        """`out` checked (contiguous `dtype` `shape` on `dev`) and marked in use on `stream`, or a new tensor allocated on `stream`."""
        if out is None:
            with torch.cuda.stream(stream):
                return torch.empty(shape, dtype=dtype, device=dev)
        if tuple(out.shape) != shape or out.dtype != dtype or out.device != dev or not out.is_contiguous():
            raise ValueError(f"{what} must be a contiguous {dtype} tensor {shape} on {dev}")
        if stream != current:
            out.record_stream(stream)
        return out

    def layer_images_to_device(self, slots, names=("ground", "groundpatch"), out=None, ranges=None, stream=None):
        """The 8-bit images gg_layer_image_u8 gives for layers `names` of `slots` (gg_layer_images_to_device):
        (uint8 CUDA tensor [count, n_names, N, N] indexed [k, l, i, j] like the cv::Mat, C-contiguous;
        float32 [count, n_names, 2] = lower, upper).  Allocated on `stream` (a torch.cuda.Stream; default: the current
        stream), or `out` / `ranges` are filled.  The call returns without waiting for the device; work enqueued on
        `stream` afterwards sees the images of the slots' layers as of their last enqueued scan or roll."""
        torch, dev, current, stream = self._layer_stream(stream)
        shape = (len(slots), len(names), self.n, self.n)
        out = self._stream_out(torch, dev, current, stream, out, shape, torch.uint8, "out")
        ranges = self._stream_out(torch, dev, current, stream, ranges, shape[:2] + (2,), torch.float32, "ranges")
        self.layer_images_to_device_ptrs(slots, names, out.data_ptr(), ranges.data_ptr(), stream.cuda_stream or None)
        return out, ranges

    def terrain_images_to_device(self, slots, out=None, stream=None):
        """The terrain images gg_terrain_image gives for `slots` (gg_terrain_images_to_device): float32 CUDA tensor
        [count, N, N, 3], C-contiguous, allocated on `stream` (default: the current stream) or filled into `out`.
        Needs the full layers."""
        torch, dev, current, stream = self._layer_stream(stream)
        out = self._stream_out(torch, dev, current, stream, out, (len(slots), self.n, self.n, 3), torch.float32, "out")
        self.terrain_images_to_device_ptrs(slots, out.data_ptr(), stream.cuda_stream or None)
        return out

    @property
    def stream(self):
        return self._l.gg_stream(self._h)

    @property
    def n_streams(self):
        return self._l.gg_num_streams(self._h)

    @property
    def host_pack_threads(self):
        return self._l.gg_host_pack_threads(self._h)

    def last_batch_transfer(self):
        """(scans packed, scans raw, packed H2D bytes, raw H2D bytes, feed us, total us, packers' pack us,
        packers' slot-wait us, feeder idle us) of the last batch call."""
        info = (C.c_size_t * 9)()
        _check(self._l.gg_last_batch_transfer(self._h, info))
        return tuple(int(v) for v in info)

    def fork_streams(self):
        _check(self._l.gg_fork_streams(self._h))

    def join_streams(self):
        _check(self._l.gg_join_streams(self._h))

    @property
    def kernel_launches(self):
        return int(self._l.gg_kernel_launches(self._h))

    def spiral_schedule_info(self):
        a, b, c = C.c_int(0), C.c_int(0), C.c_int(0)
        _check(self._l.gg_spiral_schedule_info(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    # -- the reference-facing call: GroundSegmentation::filter_cloud with host buffers
    def filter_cloud(self, points, origin, base_z, slot=0, want_index=False, want_cloud=False):
        pts = np.ascontiguousarray(points, dtype=POINT_DTYPE)
        n = pts.shape[0]
        labels = np.zeros(n, np.uint8)
        org = np.ascontiguousarray(origin, dtype=np.float32)
        index = np.zeros(n, np.uint32) if want_index else None
        cloud = np.zeros(n, POINT_DTYPE) if want_cloud else None
        nout = C.c_size_t(0)
        _check(self._l.gg_filter_cloud(self._h, slot, _ptr(pts), n, _ptr(org), float(base_z), _ptr(labels), _ptr(index),
                                       _ptr(cloud), C.byref(nout) if (want_index or want_cloud) else None))
        if want_index or want_cloud:
            k = nout.value
            return labels, (index[:k] if want_index else None), (cloud[:k] if want_cloud else None)
        return labels

    # -- device-resident pieces
    def upload_points(self, points, slot=0):
        pts = np.ascontiguousarray(points, dtype=POINT_DTYPE)
        _check(self._l.gg_upload_points(self._h, slot, _ptr(pts), pts.shape[0]))
        return pts  # keep alive until synchronize()

    def upload_points_ptr(self, ptr, n, slot=0):
        _check(self._l.gg_upload_points(self._h, slot, C.c_void_p(ptr), n))

    @staticmethod
    def make_descs(slots, n_points, origins, base_z):
        """ScanDesc array; origins="device" flags every scan GG_SCAN_DEVICE_POSE (base_z is then ignored)."""
        arr = (ScanDesc * len(slots))()
        device = isinstance(origins, str) and origins == "device"
        for k, s in enumerate(slots):
            arr[k].slot = int(s)
            arr[k].n_points = int(n_points[k])
            if device:
                arr[k].flags = SCAN_DEVICE_POSE
                continue
            arr[k].origin[0], arr[k].origin[1], arr[k].origin[2] = [float(v) for v in origins[k]]
            arr[k].base_z = float(base_z[k])
        return arr

    def run_scans(self, descs, stop_after=0):
        _check(self._l.gg_run_scans(self._h, len(descs), descs, stop_after))

    def run_scans_device(self, descs, dev_ptrs, stop_after=0, device_counts=False, device_masks=False):
        """dev_ptrs: device addresses (ints) of the per-scan clouds (32-byte records).  device_counts: flag every scan
        GG_SCAN_DEVICE_COUNT (its n_points is then the capacity; set_point_counts_from_device stores the counts).
        device_masks: flag every scan GG_SCAN_DEVICE_MASK (it runs only where set_scan_masks_from_device stored a nonzero
        mask)."""
        flags = (SCAN_DEVICE_COUNT if device_counts else 0) | (SCAN_DEVICE_MASK if device_masks else 0)
        if flags and isinstance(descs, np.ndarray):
            descs["flags"] |= flags
        elif flags:
            for d in descs:
                d.flags |= flags
        pp = (C.c_void_p * len(descs))(*dev_ptrs)
        _check(self._l.gg_run_scans_device(self._h, len(descs), _ptr(descs) if isinstance(descs, np.ndarray) else descs, pp, stop_after))

    def run_scans_to_device_ptrs(self, descs, dev_ptrs, out_ptrs, select, counts_ptr, stream_ptr):
        """gg_run_scans_to_device with raw device addresses.  descs: ScanDesc array or SCAN_DESC_DTYPE array;
        out_ptrs: uint64 [count, 3] (labels, index, cloud; 0 = none) or None; select: GG_SELECT_* bits;
        counts_ptr / stream_ptr: ints or None (stream None = the legacy default stream)."""
        count = len(descs)
        d = _ptr(descs) if isinstance(descs, np.ndarray) else descs
        pp = np.ascontiguousarray(np.array(dev_ptrs, dtype=np.uint64).reshape(count))
        op = None if out_ptrs is None else np.ascontiguousarray(out_ptrs, dtype=np.uint64).reshape(count, 3)
        _check(self._l.gg_run_scans_to_device(self._h, count, d, _ptr(pp), _ptr(op), int(select), counts_ptr, stream_ptr))

    def run_scans_to_device(self, clouds, slots, origins, base_z, labels=True, select="nonground", index=False, stream=None,
                            device_counts=False, device_masks=False):
        """One scan per slot on caller-owned CUDA tensors, results left in new CUDA tensors (gg_run_scans_to_device).
          clouds : contiguous CUDA tensors of 32-byte point records (e.g. float32 [n, 8] or uint8 [n * 32]), 16-byte aligned
          origins: [count][3] sensor positions in the map frame; base_z: one value or one per scan.  origins="device"
                   (base_z unused): every scan takes the slot's latest device scan pose (update_poses_from_device)
          select : labels of the output cloud to return: "nonground" (the obstacle points), "ground", "all" (what get_output
                   returns) or None (no cloud)
          index  : also return the input index of each returned point
          stream : torch.cuda.Stream the work is ordered on (default: the current stream); the outputs are allocated on it.
          device_counts : each cloud's length is the scan's capacity, and the scan runs on the slot's stored device count
                   (set_point_counts_from_device, GG_SCAN_DEVICE_COUNT); the outputs are allocated at capacity.
          device_masks : every scan runs only where the slot's stored scan mask is nonzero (set_scan_masks_from_device,
                   GG_SCAN_DEVICE_MASK); a skipped scan leaves its map untouched, writes none of its outputs and counts 0.
        The call returns without waiting for the device.  Work enqueued on `stream` afterwards sees complete outputs, and
        the inputs may be freed right after the call when they were allocated on `stream` (other streams' inputs are
        marked in use on `stream`).  Returns DeviceOutputs."""
        torch, dev, stream, sel = self._device_call(select, index, stream)
        n = []
        for c in clouds:
            nbytes = c.numel() * c.element_size()
            if c.device != dev or not c.is_contiguous() or nbytes % 32:
                raise ValueError(f"clouds must be contiguous tensors of 32-byte records on {dev}")
            n.append(nbytes // 32)
        descs = self._device_descs(slots, n, origins, base_z, device_counts, device_masks)
        out, ptrs = self._device_outputs(torch, dev, stream, n, labels, sel, index, clouds)
        self.run_scans_to_device_ptrs(descs, [c.data_ptr() for c in clouds], ptrs, sel,
                                      out.counts.data_ptr() if out.counts is not None else None, stream.cuda_stream or None)
        return out

    def run_cloud_msgs_to_device_ptrs(self, descs, data_ptrs, point_step, field_offsets, T, out_ptrs, select, counts_ptr, stream_ptr):
        """gg_run_cloud_msgs_to_device with raw device addresses.  data_ptrs: one device address (int, 0 = NULL) per scan;
        point_step / field_offsets: one value / one 5-tuple, or one per scan; T: None, an array [count, 3, 4] or a list
        with None entries (None: the payload is in the map frame); the rest as in run_scans_to_device_ptrs."""
        count = len(descs)
        d = _ptr(descs) if isinstance(descs, np.ndarray) else descs
        msgs = np.zeros(max(1, count), CLOUD_MSG_DTYPE)
        msgs["data"][:count] = np.asarray(data_ptrs, np.uint64).reshape(count)
        msgs["point_step"][:count] = point_step
        msgs["field_offsets"][:count] = np.asarray(field_offsets, np.int32).reshape(-1, 5)
        if isinstance(T, np.ndarray):                  # read during the call only
            Tarr = np.ascontiguousarray(T, np.float64).reshape(count, 12)
            msgs["T_map_from_frame"][:count] = Tarr.ctypes.data + 96 * np.arange(count, dtype=np.uint64)
        elif T is not None:
            if len(T) != count:
                raise ValueError("T needs one entry per scan")
            Tarr = np.zeros((count, 12), np.float64)
            for k, t in enumerate(T):
                if t is not None:
                    Tarr[k] = np.asarray(t, np.float64).reshape(12)
                    msgs["T_map_from_frame"][k] = Tarr.ctypes.data + 96 * k
        op = None if out_ptrs is None else np.ascontiguousarray(out_ptrs, dtype=np.uint64).reshape(count, 3)
        _check(self._l.gg_run_cloud_msgs_to_device(self._h, count, d, _ptr(msgs), _ptr(op), int(select), counts_ptr, stream_ptr))

    def run_cloud_msgs_to_device(self, payloads, point_step, field_offsets, T, slots, origins, base_z, labels=True, select="nonground",
                                 index=False, stream=None, device_counts=False, device_masks=False):
        """One sensor_msgs/PointCloud2 payload per slot, in caller-owned CUDA memory, unpacked and transformed to the map frame
        on the device and then run like run_scans_to_device (gg_run_cloud_msgs_to_device).
          payloads      : contiguous CUDA tensors of any dtype whose byte size is a multiple of the scan's point_step
                          (e.g. float32 [n, 4] with step 16, or uint8 [n, 18])
          point_step    : bytes per point, one value or one per scan
          field_offsets : byte offsets of x, y, z, intensity, ring (-1 absent), one 5-tuple or one per scan
          T             : None (every payload in the map frame), an array [count, 3, 4] of lookupTransform("map", frame_id), or
                          a list with None entries
        origins, base_z, labels, select, index, stream, device_counts (each payload's length is then the capacity) and
        device_masks as in run_scans_to_device.  Each payload may be freed right after the call when it was allocated on `stream` (other
        streams' payloads are marked in use on `stream`).  Returns DeviceOutputs."""
        torch, dev, stream, sel = self._device_call(select, index, stream)
        count = len(payloads)
        steps = np.broadcast_to(np.asarray(point_step, np.int64), (count,))
        n = []
        for c, step in zip(payloads, steps):
            nbytes = c.numel() * c.element_size()
            if c.device != dev or not c.is_contiguous() or step <= 0 or nbytes % step:
                raise ValueError(f"payloads must be contiguous tensors on {dev} whose byte size is a multiple of point_step")
            n.append(int(nbytes // step))
        descs = self._device_descs(slots, n, origins, base_z, device_counts, device_masks)
        out, ptrs = self._device_outputs(torch, dev, stream, n, labels, sel, index, payloads)
        self.run_cloud_msgs_to_device_ptrs(descs, [c.data_ptr() for c in payloads], steps, field_offsets, T, ptrs, sel,
                                           out.counts.data_ptr() if out.counts is not None else None, stream.cuda_stream or None)
        return out

    def run_merged_cloud_msgs_to_device_ptrs(self, descs, n_parts, parts, out_ptrs, select, counts_ptr, stream_ptr):
        """gg_run_merged_cloud_msgs_to_device with raw device addresses.  n_parts: int32 [count]; parts: CLOUD_PART_DTYPE
        array (see cloud_parts); the rest as in run_scans_to_device_ptrs."""
        count = len(descs)
        d = _ptr(descs) if isinstance(descs, np.ndarray) else descs
        n_parts = np.ascontiguousarray(n_parts, np.int32)
        parts = np.ascontiguousarray(parts, CLOUD_PART_DTYPE)
        op = None if out_ptrs is None else np.ascontiguousarray(out_ptrs, dtype=np.uint64).reshape(count, 3)
        _check(self._l.gg_run_merged_cloud_msgs_to_device(self._h, count, d, _ptr(n_parts), _ptr(parts), _ptr(op), int(select), counts_ptr,
                                                          stream_ptr))

    def run_merged_cloud_msgs_to_device(self, payloads, point_step, field_offsets, T, slots, origins, base_z, labels=True,
                                        select="nonground", index=False, stream=None, device_counts=False, device_masks=False):
        """Scans made of several sensor_msgs/PointCloud2 payloads each (a multi-LiDAR rig), in caller-owned CUDA memory:
        every part is unpacked and transformed to the map frame on the device, the parts of a scan are concatenated in
        order in the slot's buffer, and the merged scans then run like run_scans_to_device
        (gg_run_merged_cloud_msgs_to_device).
          payloads      : payloads[k] is the list of contiguous CUDA tensors of scan k (at most MAX_CLOUD_PARTS), any
                          dtype whose byte size is a multiple of the part's point_step
          point_step    : bytes per point, one value for every part or nested [k][p]
          field_offsets : byte offsets of x, y, z, intensity, ring (-1 absent), one 5-tuple or nested [k][p]
          T             : lookupTransform("map", frame_id) as a 3x4, one for every part or nested [k][p]; None: the part
                          is already in the map frame
        origins (one cloudOrigin per merged scan), base_z, labels, select, index, stream and device_masks as in
        run_scans_to_device.
          device_counts : each payload's length is its part's capacity, and each part runs on the slot's stored part count
                          (set_part_counts_from_device, GG_SCAN_DEVICE_PART_COUNTS); the outputs are allocated at capacity
        Each payload may be freed right after the call when it was allocated on `stream` (other streams' payloads are
        marked in use on `stream`).  Returns DeviceOutputs."""
        torch, dev, stream, sel = self._device_call(select, index, stream)
        for scan in payloads:
            for c in scan:
                if c.device != dev or not c.is_contiguous():
                    raise ValueError(f"payloads must be contiguous tensors on {dev}")
        n_parts, parts, Tarr = cloud_parts([[c.numel() * c.element_size() for c in scan] for scan in payloads],
                                           [[c.data_ptr() for c in scan] for scan in payloads], point_step, field_offsets, T)
        first = np.cumsum(n_parts) - n_parts
        n = [int(parts["n_points"][b:b + m].sum()) for b, m in zip(first, n_parts)]
        descs = self._device_descs(slots, n, origins, base_z, device_masks=device_masks)
        if device_counts:
            descs["flags"] |= SCAN_DEVICE_PART_COUNTS
        out, ptrs = self._device_outputs(torch, dev, stream, n, labels, sel, index, [c for scan in payloads for c in scan])
        self.run_merged_cloud_msgs_to_device_ptrs(descs, n_parts, parts, ptrs, sel, out.counts.data_ptr() if out.counts is not None else None,
                                                  stream.cuda_stream or None)
        del Tarr                   # the transforms `parts` points to: read during the call only
        return out

    def step_plan(self, slots, clouds=None, payloads=None, point_step=32, field_offsets=(0, 4, 8, 16, 20), T=None, origins="device",
                  base_z=None, counts=None, xy=None, T_base_from_map=None, pose_origins=None, pose_base_z=None, moved=False, labels=True,
                  select="nonground", index=False, reset_xyz=None, reset_mask=None, layers=None, layer_images=None, terrain_images=False,
                  samples=None, sample_names=("ground", "groundpatch"), sample_mode="nearest", sample_cells=False, point_info=None,
                  tallies=None, parts=None, part_counts=None, configs=None, config_mask=None, restore_pool=None, restore_index=None,
                  restore_status=False, save=None, save_mask=None, scan_mask=None):
        """One step of a fixed batch recorded once as a CUDA graph and replayed from these tensors (gg_step_plan_create).
        Its step is the call sequence set_point_counts_from_device(counts) -> update_poses_from_device(xy, T_base_from_map,
        pose_origins, pose_base_z) -> run_scans_to_device(clouds) / run_cloud_msgs_to_device(payloads), each part only when
        its inputs are given, and every replay is bit-identical to it run on the tensors' contents at replay time.  With
        reset_xyz the step starts with init_maps_from_device(reset_xyz, reset_mask) (gg_step_plan_create_with_resets).
          clouds / payloads / parts : exactly one: contiguous CUDA tensors as in run_scans_to_device /
                              run_cloud_msgs_to_device, or nested [scan][part] as in run_merged_cloud_msgs_to_device (the
                              step's scan is then that call, gg_step_plan_create_with_parts); their lengths are the
                              scans' (or parts') capacities
          point_step, field_offsets : the payloads' layout (one value or one per scan; with parts one value or nested [k][p])
          T        : payloads only.  None (map frame); a CUDA float64 tensor [count, 12] (or [count, 3, 4]) or a list of
                     CUDA float64 [12] tensors / None: lookupTransform("map", frame_id) read at every replay; a numpy
                     [count, 3, 4] or a list of numpy 3x4 / None: fixed host transforms.  With parts: one value or nested
                     [k][p] of those entries, or a CUDA float64 tensor [count, P, 12] (or [count, P, 3, 4]) read at every
                     replay
          part_counts : parts only.  CUDA int32 [count, P] or None: the parts' point counts, read at every replay
                     (set_part_counts_from_device, GG_SCAN_DEVICE_PART_COUNTS)
          origins  : "device" (the slots' device scan poses, GG_SCAN_DEVICE_POSE) or host [count][3] with base_z
          counts   : CUDA int32 [count] or None: the scans' point counts, read at every replay (GG_SCAN_DEVICE_COUNT)
          xy, T_base_from_map, pose_origins, pose_base_z : CUDA tensors as in update_poses_from_device, or None
          moved    : also allocate dev_moved (plan.moved)
          labels, select, index : the outputs, as in run_scans_to_device
          reset_xyz, reset_mask : CUDA float64 [count, 3] and int32 [count] (or None: every slot) as in
                     init_maps_from_device, read at every replay; reset_mask without reset_xyz is an error
          configs, config_mask : CUDA uint8 [count, sizeof(gg_config)] (config_tensor) and int32 [count] (or None: every
                     slot) as in set_configs_from_device, read at every replay: the step then starts with that call
                     (gg_step_plan_create_with_configs), and the slots are device-configured from the plan's creation;
                     config_mask without configs is an error
          restore_pool, restore_index, restore_status : CUDA uint8 [n_pool, snapshot_bytes], int32 [count] (or None: k)
                     and True for plan.restore_status, as in restore_maps_from_device, read at every replay: the step then
                     restores after the resets and before the counts (gg_step_plan_create_with_snapshots)
          save, save_mask : True (a new tensor) or a CUDA uint8 [count, snapshot_bytes], and int32 [count] (or None: every
                     slot), as in save_maps_to_device: the step then ends with that call, into plan.saved
          scan_mask : CUDA int32 [count] or None: which scans run, read at every replay.  The step then stores it with
                     set_scan_masks_from_device just before the counts, and every scan is flagged device_masks
                     (gg_step_plan_create_with_scan_masks)
        Read-outs: with any of these the step has a stage of read-out calls after the scan (gg_step_plan_create_with_readouts),
        whose results land in plan.readouts (PlanReadouts) at every replay:
          layers       : layer names, as get_layers_to_device
          layer_images : layer names, as layer_images_to_device
          terrain_images : True: terrain_images_to_device (needs the full layers)
          samples      : one CUDA position tensor per slot, as sample_layers_to_device(positions); the plan looks up what
                         they hold at each replay, and their row counts are fixed capacities.  sample_names,
                         sample_mode and sample_cells are that call's names, mode and cells
          point_info   : ("codes", "height"), either or both: point_info_to_device into buffers of the scans' capacities
          tallies      : int64 CUDA tensor [count, 1024, 2] to which every replay adds its tallies (eval_counts_to_device(out=))
        Returns a StepPlan.  Until it is closed the slots are bound to it (see the C header)."""
        import torch

        torch_, dev, stream, sel = self._device_call(select, index, None)
        count = len(slots)
        if (clouds is not None) + (payloads is not None) + (parts is not None) != 1:
            raise ValueError("give exactly one of clouds, payloads and parts")
        if part_counts is not None and parts is None:
            raise ValueError("part_counts needs parts")
        keep = []

        def dptr(t, dtype, shape, name):
            if t is None:
                return None
            if t.dtype != dtype or t.device != dev or not t.is_contiguous() or t.numel() != int(np.prod(shape)):
                raise ValueError(f"{name} must be a contiguous {dtype} tensor {shape} on {dev}")
            keep.append(t)
            return t.data_ptr()

        d = StepDesc()
        d.count = count
        sp = None
        if parts is not None:
            n, sp = self._plan_parts(torch, dev, parts, point_step, field_offsets, T, part_counts, keep, dptr)
        elif clouds is not None:
            n = []
            for c in clouds:
                nbytes = c.numel() * c.element_size()
                if c.device != dev or not c.is_contiguous() or nbytes % 32:
                    raise ValueError(f"clouds must be contiguous tensors of 32-byte records on {dev}")
                n.append(nbytes // 32)
            pp = np.array([c.data_ptr() for c in clouds], np.uint64)
            keep += [clouds, pp]
            d.dev_points = pp.ctypes.data
        else:
            steps = np.broadcast_to(np.asarray(point_step, np.int64), (count,))
            n = []
            for c, step in zip(payloads, steps):
                nbytes = c.numel() * c.element_size()
                if c.device != dev or not c.is_contiguous() or step <= 0 or nbytes % step:
                    raise ValueError(f"payloads must be contiguous tensors on {dev} whose byte size is a multiple of point_step")
                n.append(int(nbytes // step))
            msgs = np.zeros(count, CLOUD_MSG_DTYPE)
            msgs["data"] = [c.data_ptr() for c in payloads]
            msgs["point_step"] = steps
            msgs["field_offsets"] = np.asarray(field_offsets, np.int32).reshape(-1, 5)
            keep += [payloads, msgs]
            d.msgs = msgs.ctypes.data
            if isinstance(T, torch.Tensor):
                T = list(T.reshape(count, 12))
            if T is not None:
                if len(T) != count:
                    raise ValueError("T needs one entry per scan")
                tp = np.zeros(count, np.uint64)
                Tarr = np.zeros((count, 12), np.float64)   # host transforms: read by gg_step_plan_create
                for k, t in enumerate(T):
                    if isinstance(t, torch.Tensor):
                        tp[k] = dptr(t, torch.float64, (12,), "T")
                    elif t is not None:
                        Tarr[k] = np.asarray(t, np.float64).reshape(12)
                        msgs["T_map_from_frame"][k] = Tarr.ctypes.data + 96 * k
                keep += [tp, Tarr]
                if tp.any():
                    d.dev_T_map_from_frame = tp.ctypes.data
        descs = self._device_descs(slots, n, origins, base_z, counts is not None, scan_mask is not None)
        if part_counts is not None:
            descs["flags"] |= SCAN_DEVICE_PART_COUNTS
        sl = np.ascontiguousarray(slots, np.int32)
        keep += [descs, sl]
        d.scans = descs.ctypes.data
        d.dev_n_points = dptr(counts, torch.int32, (count,), "counts")
        d.poses = DevicePoses(dptr(xy, torch.float64, (count, 2), "xy"), dptr(T_base_from_map, torch.float64, (count, 12), "T_base_from_map"),
                              dptr(pose_origins, torch.float32, (count, 3), "pose_origins"), dptr(pose_base_z, torch.float64, (count,), "pose_base_z"))
        mv = torch.empty(count, dtype=torch.int32, device=dev) if moved else None
        d.dev_moved = mv.data_ptr() if mv is not None else None
        out, ptrs = self._device_outputs(torch_, dev, stream, n, labels, sel, index, [])
        keep.append(ptrs)
        d.outs = ptrs.ctypes.data
        d.select = sel
        d.dev_counts = out.counts.data_ptr() if out.counts is not None else None
        ro, ro_c = self._plan_readouts(torch_, dev, stream, slots, n, keep, layers, layer_images, terrain_images, samples, sample_names,
                                       sample_mode, sample_cells, point_info, tallies)
        p = C.c_void_p()
        if reset_mask is not None and reset_xyz is None:
            raise ValueError("reset_mask needs reset_xyz")
        r = None if reset_xyz is None else DeviceResets(dptr(reset_xyz, torch.float64, (count, 3), "reset_xyz"),
                                                        dptr(reset_mask, torch.int32, (count,), "reset_mask"))
        if config_mask is not None and configs is None:
            raise ValueError("config_mask needs configs")
        if (restore_index is not None or restore_status) and restore_pool is None:
            raise ValueError("restore_index and restore_status need restore_pool")
        if save_mask is not None and save is None:
            raise ValueError("save_mask needs save")
        snap, rstatus, saved = None, None, None
        if restore_pool is not None or save is not None:
            snap = StepSnapshots()
            rb = self.snapshot_bytes
            if restore_pool is not None:
                if restore_pool.dim() != 2 or restore_pool.shape[1] != rb:
                    raise ValueError(f"restore_pool must be a CUDA uint8 tensor [n_pool, {rb}]")
                rstatus = torch.empty(count, dtype=torch.int32, device=dev) if restore_status else None
                snap.restore = MapRestore(dptr(restore_pool, torch.uint8, tuple(restore_pool.shape), "restore_pool"), restore_pool.shape[0],
                                          dptr(restore_index, torch.int32, (count,), "restore_index"),
                                          rstatus.data_ptr() if rstatus is not None else None)
            if save is not None:
                saved = torch.zeros((count, rb), dtype=torch.uint8, device=dev) if save is True else save
                snap.save = dptr(saved, torch.uint8, (count, rb), "save")
                snap.save_mask = dptr(save_mask, torch.int32, (count,), "save_mask")
        cc = None if configs is None else DeviceConfigs(dptr(configs, torch.uint8, (count, C.sizeof(Config)), "configs"),
                                                        dptr(config_mask, torch.int32, (count,), "config_mask"))
        _check(self._l.gg_step_plan_create_with_scan_masks(self._h, C.byref(d), None if sp is None else C.byref(sp),
                                                           None if r is None else C.byref(r), None if cc is None else C.byref(cc),
                                                           None if snap is None else C.byref(snap), None if ro_c is None else C.byref(ro_c),
                                                           dptr(scan_mask, torch.int32, (count,), "scan_mask"), C.byref(p)))
        plan = StepPlan(self, p, out, mv, keep, ro)
        plan.restore_status, plan.saved = rstatus, saved
        return plan

    @staticmethod
    def _plan_parts(torch, dev, parts, point_step, field_offsets, T, part_counts, keep, dptr):
        """step_plan's merged scans: (capacity of each scan, StepParts).  Host arrays and the tensors go to keep."""
        count = len(parts)
        m = [len(scan) for scan in parts]
        for scan in parts:
            for c in scan:
                if c.device != dev or not c.is_contiguous():
                    raise ValueError(f"parts must be contiguous tensors on {dev}")
        if isinstance(T, torch.Tensor):
            T3 = T.reshape(count, -1, 12)
            T = [[T3[k, q] for q in range(mk)] for k, mk in enumerate(m)]
        dev_T = np.zeros(max(1, sum(m)), np.uint64)
        if isinstance(T, (list, tuple)) and any(isinstance(t, torch.Tensor) for scan in T if isinstance(scan, (list, tuple)) for t in scan):
            if len(T) != count or any(len(scan) != mk for scan, mk in zip(T, m)):
                raise ValueError("T must be nested [scan][part] like the parts")
            host, at = [], 0
            for scan in T:
                row = []
                for t in scan:
                    if isinstance(t, torch.Tensor):
                        dev_T[at] = dptr(t, torch.float64, (12,), "T")
                        t = None
                    row.append(t)
                    at += 1
                host.append(row)
            T = host
        n_parts, arr, Tarr = cloud_parts([[c.numel() * c.element_size() for c in scan] for scan in parts],
                                         [[c.data_ptr() for c in scan] for scan in parts], point_step, field_offsets, T)
        first = np.cumsum(n_parts) - n_parts
        n = [int(arr["n_points"][b:b + mk].sum()) for b, mk in zip(first, n_parts)]
        arr = np.ascontiguousarray(arr)
        keep += [parts, n_parts, arr, Tarr, dev_T]   # host transforms: read by gg_step_plan_create_with_parts
        sp = StepParts(n_parts.ctypes.data, arr.ctypes.data, dev_T.ctypes.data if dev_T.any() else None, None, 0)
        if part_counts is not None:
            if part_counts.dim() != 2:
                raise ValueError("part_counts must be a CUDA int32 tensor [count, parts]")
            sp.dev_part_counts = dptr(part_counts, torch.int32, (count, part_counts.shape[1]), "part_counts")
            sp.parts_per_slot = part_counts.shape[1]
        return n, sp

    def _plan_readouts(self, torch, dev, stream, slots, n, keep, layers, layer_images, terrain_images, samples, sample_names, sample_mode,
                       sample_cells, point_info, tallies):
        """step_plan's read-outs: (PlanReadouts with tensors allocated on `stream`, their StepReadouts or None for none).
        n[k] is scan k's capacity."""
        ro, r = PlanReadouts(), StepReadouts()
        count, N = len(slots), self.n
        given = False
        with torch.cuda.stream(stream):
            if layers:
                _, r.n_layer_names, nm = self._layer_batch_args(slots, layers)
                ro.layers = torch.empty((count, len(layers), N, N), dtype=torch.float32, device=dev).transpose(-1, -2)
                r.layer_names, r.layers = C.cast(nm, C.c_void_p), ro.layers.data_ptr()
                keep.append(nm)
                given = True
            if layer_images:
                _, r.n_image_names, nm = self._layer_batch_args(slots, layer_images)
                ro.images = torch.empty((count, len(layer_images), N, N), dtype=torch.uint8, device=dev)
                ro.ranges = torch.empty((count, len(layer_images), 2), dtype=torch.float32, device=dev)
                r.image_names, r.images, r.image_ranges = C.cast(nm, C.c_void_p), ro.images.data_ptr(), ro.ranges.data_ptr()
                keep.append(nm)
                given = True
            if terrain_images:
                ro.terrain = torch.empty((count, N, N, 3), dtype=torch.float32, device=dev)
                r.terrain_images = ro.terrain.data_ptr()
                given = True
            if samples is not None:
                if len(samples) != count:
                    raise ValueError("samples needs one position tensor per slot")
                if sample_mode not in SAMPLE_MODES:
                    raise ValueError(f"sample_mode must be one of {list(SAMPLE_MODES)}")
                q, ns = self._position_sets(torch, dev, samples)
                ro.positions = list(samples)
                ro.samples, ro.cells = self._sample_outputs(torch, dev, stream, q, ns, len(sample_names), None, sample_cells)
                _, r.n_sample_names, nm = self._layer_batch_args(slots, sample_names)
                r.sample_names, r.samples, r.sample_mode = C.cast(nm, C.c_void_p), q.ctypes.data, SAMPLE_MODES[sample_mode]
                keep += [q, nm]
                given = True
            if point_info:
                fields = (point_info,) if isinstance(point_info, str) else tuple(point_info)
                if not set(fields) <= {"codes", "height"}:
                    raise ValueError('point_info takes "codes", "height" or both')
                o = np.zeros(max(1, count), POINT_INFO_DTYPE)
                for field, dtype in (("codes", torch.int32), ("height", torch.float32)):
                    if field in fields:
                        views = list(torch.split(torch.empty(int(sum(n)), dtype=dtype, device=dev), list(n)))
                        o[field][:count] = [t.data_ptr() if m else 0 for t, m in zip(views, n)]
                        setattr(ro, field, views)
                r.point_info = o.ctypes.data
                keep.append(o)
                given = True
        if tallies is not None:
            shape = (count, 1024, 2)
            if tuple(tallies.shape) != shape or tallies.dtype != torch.int64 or tallies.device != dev or not tallies.is_contiguous():
                raise ValueError(f"tallies must be a contiguous int64 tensor {shape} on {dev}")
            ro.tallies = tallies
            r.eval_counts = tallies.data_ptr()
            given = True
        return ro, (r if given else None)

    # shared by run_scans_to_device / run_cloud_msgs_to_device / run_merged_cloud_msgs_to_device
    def _device_call(self, select, index, stream):
        """(torch, device, stream, select bits); stream defaults to the current stream."""
        import torch

        if select not in SELECT:
            raise ValueError(f"select must be one of {list(SELECT)}")
        sel = SELECT[select]
        if index and not sel:
            raise ValueError("index needs a select")
        dev = torch.device("cuda", self.device)
        return torch, dev, (torch.cuda.current_stream(dev) if stream is None else stream), sel

    @staticmethod
    def _device_descs(slots, n, origins, base_z, device_counts=False, device_masks=False):
        count = len(n)
        descs = np.zeros(count, SCAN_DESC_DTYPE)
        descs["slot"] = np.asarray(slots, np.int32)
        descs["n_points"] = n
        if device_counts:   # n is the capacity; the slots' stored device counts (set_point_counts_from_device)
            descs["flags"] = SCAN_DEVICE_COUNT
        if device_masks:    # the slots' stored scan masks (set_scan_masks_from_device)
            descs["flags"] |= SCAN_DEVICE_MASK
        if isinstance(origins, str) and origins == "device":   # the slots' device scan poses (update_poses_from_device)
            descs["flags"] |= SCAN_DEVICE_POSE
            return descs
        descs["origin"] = np.asarray(origins, np.float32).reshape(count, 3)
        descs["base_z"] = np.broadcast_to(np.asarray(base_z, np.float64), (count,))
        return descs

    @staticmethod
    def _device_outputs(torch, dev, stream, n, labels, sel, index, inputs):
        """Flat output tensors allocated on `stream` for scans of n[k] points, as DeviceOutputs, and their per-scan addresses
        uint64 [count, 3] (labels, index, cloud).  Inputs of another stream than the current one are marked in use on
        `stream`."""
        count = len(n)
        offs = np.zeros(count, np.uint64)
        offs[1:] = np.cumsum(n[:-1], dtype=np.uint64)
        total = int(sum(n))
        with torch.cuda.stream(stream):
            lab = torch.empty(total, dtype=torch.uint8, device=dev) if labels else None
            cld = torch.empty((total, 8), dtype=torch.float32, device=dev) if sel else None
            idx = torch.empty(total, dtype=torch.int32, device=dev) if index else None
            counts = torch.empty(count, dtype=torch.int32, device=dev) if sel else None
        ptrs = np.zeros((count, 3), np.uint64)
        for col, t, size in ((0, lab, 1), (1, idx, 4), (2, cld, 32)):
            if t is not None and total:
                ptrs[:, col] = np.uint64(t.data_ptr()) + offs * np.uint64(size)
        if stream != torch.cuda.current_stream(dev):
            for c in inputs:
                c.record_stream(stream)

        def views(t):
            return None if t is None else list(torch.split(t, n))

        return DeviceOutputs(views(lab), views(cld), views(idx), counts, stream), ptrs

    # -- steps next to the path (SURVEY section 8f)
    def upload_cloud_msg(self, raw, n_points, point_step, field_offsets, T_map_from_frame=None, slot=0):
        """raw: uint8 array of the PointCloud2 payload; field_offsets: x, y, z, intensity, ring (-1 absent)."""
        raw = np.ascontiguousarray(raw, np.uint8)
        off = np.ascontiguousarray(field_offsets, np.int32)
        T = None if T_map_from_frame is None else np.ascontiguousarray(T_map_from_frame, np.float64).reshape(12)
        _check(self._l.gg_upload_cloud_msg(self._h, slot, _ptr(raw), int(n_points), int(point_step), _ptr(off), _ptr(T)))
        return raw

    def upload_cloud_msgs(self, parts, slot=0):
        """The payloads of one merged scan from host memory (gg_upload_cloud_msgs): parts = [(raw, point_step,
        field_offsets, T_map_from_frame or None), ...], raw a uint8 array of the part's PointCloud2 payload.  The records
        land in the slot's buffer back to back; follow with run_scans for the total point count.  Returns the payloads."""
        raws = [np.ascontiguousarray(p[0], np.uint8) for p in parts]
        n_parts, arr, Tarr = cloud_parts([[r.nbytes for r in raws]], [[r.ctypes.data for r in raws]], [[p[1] for p in parts]],
                                         [[p[2] for p in parts]], [[p[3] for p in parts]])
        _check(self._l.gg_upload_cloud_msgs(self._h, slot, int(n_parts[0]), _ptr(arr)))
        return raws

    def terrain_image(self, slot=0):
        img = np.zeros((self.n, self.n, 3), np.float32)
        _check(self._l.gg_terrain_image(self._h, slot, _ptr(img)))
        return img

    def layer_image_u8(self, name, slot=0):
        """(N x N uint8 image indexed [i, j], lower, upper): what toImage<unsigned char, 1> hands to cv::applyColorMap."""
        img = np.zeros((self.n, self.n), np.uint8)
        lo, hi = C.c_float(0), C.c_float(0)
        _check(self._l.gg_layer_image_u8(self._h, slot, name.encode(), _ptr(img), C.byref(lo), C.byref(hi)))
        return img, lo.value, hi.value

    # -- the reference's per-phase methods
    def point_classes(self, n, slot=0):
        codes = np.zeros(n, np.uint32)
        _check(self._l.gg_get_point_classes(self._h, slot, _ptr(codes), n))
        return codes

    def last_scan_points(self, slot=0):
        """Points of the slot's last scan (gg_last_scan_points): the length of its point_info_to_device outputs.  After a
        device_counts scan this waits for the slot's work (the count is on the device until then)."""
        n = C.c_size_t(0)
        _check(self._l.gg_last_scan_points(self._h, slot, C.byref(n)))
        return n.value

    def point_info_to_device_ptrs(self, slots, codes_ptrs, height_ptrs, stream_ptr):
        """gg_point_info_to_device with raw device addresses: codes_ptrs / height_ptrs one address per slot (int; 0 or None
        = none) or None for none at all; stream_ptr an int or None (None = the legacy default stream)."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        o = np.zeros(max(1, len(sl)), POINT_INFO_DTYPE)
        for field, ptrs in (("codes", codes_ptrs), ("height", height_ptrs)):
            if ptrs is not None:
                o[field][:len(sl)] = [0 if p is None else int(p) for p in ptrs]
        _check(self._l.gg_point_info_to_device(self._h, len(sl), _ptr(sl), _ptr(o), stream_ptr))

    def point_info_to_device(self, slots, codes=True, height=True, out=None, stream=None):
        """Per input point of each slot's last completed scan, its class code and height above the terrain
        (gg_point_info_to_device).  Returns (codes, height): each a list of one CUDA tensor per slot of the scan's
        n_points, or None when not asked for.
          codes  : int32 tensors, class << 24 | cell (the bits of gg_get_point_classes; the class is codes >> 24, PC_*)
          height : float32 tensors, z - ground[cell]; NaN for absent points
          out    : None, or a pair (codes list or None, height list or None) of contiguous tensors to fill
          stream : torch.cuda.Stream the work is ordered on (default: the current stream); outputs are allocated on it.
        The call returns without waiting for the device; work enqueued on `stream` afterwards sees the outputs.  The
        lengths come from last_scan_points, which waits after a device_counts scan; point_info_to_device_ptrs with
        buffers sized for the scan's capacity does not."""
        torch, dev, current, stream = self._layer_stream(stream)
        ns = [self.last_scan_points(int(s)) for s in slots]
        result = []
        for k, (want, dtype) in enumerate(((codes, torch.int32), (height, torch.float32))):
            given = None if out is None else out[k]
            if given is not None:
                if len(given) != len(slots):
                    raise ValueError("out needs one tensor per slot")
                result.append([self._stream_out(torch, dev, current, stream, t, (n,), dtype, f"out[{k}][{j}]")
                               for j, (t, n) in enumerate(zip(given, ns))])
            elif want:
                with torch.cuda.stream(stream):
                    result.append(list(torch.split(torch.empty(sum(ns), dtype=dtype, device=dev), ns)))
            else:
                result.append(None)
        ptrs = [None if r is None else [t.data_ptr() if n else 0 for t, n in zip(r, ns)] for r in result]
        self.point_info_to_device_ptrs(slots, ptrs[0], ptrs[1], stream.cuda_stream or None)
        return result[0], result[1]

    def detect_ground_patches(self, slot=0):
        _check(self._l.gg_detect_ground_patches(self._h, slot))

    def detect_ground_patch(self, size, i, j, slot=0):
        _check(self._l.gg_detect_ground_patch(self._h, slot, size, i, j))

    def spiral_ground_interpolation(self, base_z, slot=0):
        _check(self._l.gg_spiral_ground_interpolation(self._h, slot, float(base_z)))

    def interpolate_cell(self, x, y, slot=0):
        _check(self._l.gg_interpolate_cell(self._h, slot, x, y))

    def eval_accumulate(self, slot=0):
        _check(self._l.gg_eval_accumulate(self._h, slot))

    def eval_read(self, reset=False):
        counts = np.zeros((1024, 2), np.uint64)
        _check(self._l.gg_eval_read(self._h, _ptr(counts), 1 if reset else 0))
        return counts

    def eval_counts_to_device_ptrs(self, slots, dst_ptr, stream_ptr):
        """gg_eval_counts_to_device with raw device addresses: dst_ptr uint64 [count][1024][2] (8-byte aligned), to which
        the tallies are added; stream_ptr an int or None (None = the legacy default stream)."""
        sl = np.ascontiguousarray(slots, np.int32).reshape(-1)
        _check(self._l.gg_eval_counts_to_device(self._h, len(sl), _ptr(sl), dst_ptr, stream_ptr))

    def eval_counts_to_device(self, slots, out=None, stream=None):
        """The tallies eval_accumulate adds, for the last completed scan of each of `slots`, one tally per slot
        (gg_eval_counts_to_device): int64 CUDA tensor [count, 1024, 2] ([k, id, 0] ground, [k, id, 1] non-ground; the
        bits of the uint64 counts).  Without `out` a zeroed tensor is allocated on `stream` (a torch.cuda.Stream;
        default: the current stream); with `out` the tallies are added to it, so one tensor keeps running sums over a
        sequence.  The call returns without waiting for the device; work enqueued on `stream` afterwards sees them."""
        torch, dev, current, stream = self._layer_stream(stream)
        shape = (len(slots), 1024, 2)
        if out is None:
            with torch.cuda.stream(stream):
                out = torch.zeros(shape, dtype=torch.int64, device=dev)
        else:
            out = self._stream_out(torch, dev, current, stream, out, shape, torch.int64, "out")
        self.eval_counts_to_device_ptrs(slots, out.data_ptr(), stream.cuda_stream or None)
        return out

    def profile_enable(self, on=True):
        _check(self._l.gg_profile_enable(self._h, 1 if on else 0))

    def profile_read(self, reset=True):
        """{kernel name: (total ms, launches)} measured with CUDA events on the launching stream."""
        k = self._l.gg_profile_kernel_count()
        ms = np.zeros(k, np.float64)
        cnt = np.zeros(k, np.uint32)
        _check(self._l.gg_profile_read(self._h, _ptr(ms), _ptr(cnt), 1 if reset else 0))
        return {self._l.gg_profile_kernel_name(j).decode(): (float(ms[j]), int(cnt[j])) for j in range(k) if cnt[j]}

    def download_labels(self, n, slot=0, out=None):
        out = np.zeros(n, np.uint8) if out is None else out
        _check(self._l.gg_download_labels(self._h, slot, _ptr(out), n))
        return out

    def download_labels_ptr(self, ptr, n, slot=0):
        _check(self._l.gg_download_labels(self._h, slot, C.c_void_p(ptr), n))

    def filter_cloud_batch_ptrs(self, descs, point_ptrs, label_ptrs):
        """Host pointers (ints) per scan; see gg_filter_cloud_batch."""
        n = len(descs)
        pp = (C.c_void_p * n)(*point_ptrs)
        lp = (C.c_void_p * n)(*label_ptrs) if label_ptrs is not None else None
        _check(self._l.gg_filter_cloud_batch(self._h, n, descs, pp, lp))

    def filter_cloud_batch_begin(self, descs, point_ptrs, label_ptrs):
        """First half of filter_cloud_batch_ptrs: returns a ticket once everything is enqueued."""
        n = len(descs)
        pp = (C.c_void_p * n)(*point_ptrs)
        lp = (C.c_void_p * n)(*label_ptrs) if label_ptrs is not None else None
        ticket = C.c_int(-1)
        _check(self._l.gg_filter_cloud_batch_begin(self._h, n, descs, pp, lp, C.byref(ticket)))
        return ticket.value

    def filter_cloud_batch_wait(self, ticket):
        _check(self._l.gg_filter_cloud_batch_wait(self._h, ticket))

    def synchronize(self):
        _check(self._l.gg_synchronize(self._h))

    def get_output(self, slot=0, want_cloud=False):
        n = self.max_points
        index = np.zeros(n, np.uint32)
        cloud = np.zeros(n, POINT_DTYPE) if want_cloud else None
        nout = C.c_size_t(0)
        _check(self._l.gg_get_output(self._h, slot, _ptr(index), _ptr(cloud), C.byref(nout)))
        k = nout.value
        return index[:k], (cloud[:k] if want_cloud else None)

    def run_single(self, points, origin, base_z, slot=0, stop_after=0):
        """Upload + run (optionally only the first phases) + sync; returns labels if the run was complete."""
        keep = self.upload_points(points, slot)
        d = self.make_descs([slot], [keep.shape[0]], [origin], [base_z])
        self.run_scans(d, stop_after)
        labels = self.download_labels(keep.shape[0], slot) if stop_after == 0 else None
        self.synchronize()
        return labels
