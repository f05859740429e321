"""Host side of merged multi-sensor scans (gg_run_merged_cloud_msgs_to_device, gg_upload_cloud_msgs): the gg_cloud_part
record image, the flattening of nested per-part arguments, and the per-sensor clouds of synth.lidar_scan(split=True)."""
import ctypes as C

import numpy as np
import pytest

from groundgrid_b200 import capi, synth

L18 = (0, 4, 8, 12, 16)
L32 = (0, 4, 8, 16, 20)


def test_cloud_part_dtype_matches_the_ctypes_structure():
    dt = capi.CLOUD_PART_DTYPE
    assert dt.itemsize == C.sizeof(capi.CloudPart) == 48
    msg = capi.CloudPart.msg.offset
    assert msg == 0
    for name, field in (("data", "data"), ("point_step", "point_step"), ("field_offsets", "field_offsets"),
                        ("T_map_from_frame", "T_map_from_frame")):
        assert dt.fields[name][1] == msg + getattr(capi.CloudMsg, field).offset, name
    assert dt.fields["n_points"][1] == capi.CloudPart.n_points.offset
    # one record written through numpy reads back through ctypes
    a = np.zeros(2, dt)
    a["data"][1], a["point_step"][1], a["field_offsets"][1], a["T_map_from_frame"][1], a["n_points"][1] = 0x1234, 18, L18, 0x5678, 77
    s = capi.CloudPart.from_buffer(a, dt.itemsize)
    assert (s.msg.data, s.msg.point_step, tuple(s.msg.field_offsets), s.msg.T_map_from_frame, s.n_points) == (0x1234, 18, L18, 0x5678, 77)


def test_cloud_parts_nested_arguments():
    T1 = np.arange(12, dtype=np.float64).reshape(3, 4)
    T2 = -T1
    nbytes = [[18 * 5, 32 * 3], [], [18 * 0]]
    ptrs = [[100, 200], [], [0]]
    n_parts, parts, Tarr = capi.cloud_parts(nbytes, ptrs, [[18, 32], [], [18]], [[L18, L32], [], [L18]], [[T1, None], [], [T2]])
    assert n_parts.dtype == np.int32 and n_parts.tolist() == [2, 0, 1]
    assert parts.dtype == capi.CLOUD_PART_DTYPE and len(parts) == 3
    assert parts["data"].tolist() == [100, 200, 0]
    assert parts["point_step"].tolist() == [18, 32, 18]
    assert parts["n_points"].tolist() == [5, 3, 0]
    assert [tuple(o) for o in parts["field_offsets"]] == [L18, L32, L18]
    assert parts["T_map_from_frame"][1] == 0
    for p, want in ((0, T1), (2, T2)):
        addr = int(parts["T_map_from_frame"][p])
        got = np.ctypeslib.as_array((C.c_double * 12).from_address(addr))
        assert np.array_equal(got, want.reshape(12))
    assert Tarr.ctypes.data <= int(parts["T_map_from_frame"][0])


def test_cloud_parts_broadcast_arguments():
    nbytes = [[32 * 4, 32 * 2, 32], [32 * 7]]
    n_parts, parts, _ = capi.cloud_parts(nbytes, [[1, 2, 3], [4]], 32, L32, None)
    assert n_parts.tolist() == [3, 1]
    assert parts["n_points"].tolist() == [4, 2, 1, 7]
    assert (parts["point_step"] == 32).all() and (parts["T_map_from_frame"] == 0).all()
    assert all(tuple(o) == L32 for o in parts["field_offsets"])
    T = np.eye(3, 4)
    _, parts, _ = capi.cloud_parts(nbytes, [[1, 2, 3], [4]], 32, L32, T)
    assert len(set(parts["T_map_from_frame"].tolist())) == 4 and (parts["T_map_from_frame"] != 0).all()
    n_parts, parts, _ = capi.cloud_parts([], [], 18, L18, None)
    assert len(n_parts) == 0 and len(parts) == 0
    # one scan whose parts have no transform, or one each: nested, not one value
    for T in ([[None, None, None]], [[np.eye(3, 4), None, np.eye(3, 4)]], [[np.eye(3, 4)] * 3]):
        _, parts, _ = capi.cloud_parts(nbytes[:1], [[1, 2, 3]], 32, L32, T)
        assert [int(a) != 0 for a in parts["T_map_from_frame"]] == [t is not None for t in T[0]]


@pytest.mark.parametrize("kw", [
    dict(point_step=[[32, 32, 32]]),                      # one scan's worth for two scans
    dict(point_step=[[32, 32], [32]]),                    # too few parts in scan 0
    dict(field_offsets=[[L32, L32, L32], [L32, L32]]),    # too many parts in scan 1
    dict(T=[[None, None, None]]),
    dict(data_ptrs=[[1, 2, 3]]),
    dict(point_step=18),                                  # 32-byte multiples are not 18-byte multiples
])
def test_cloud_parts_rejects_mismatched_nesting(kw):
    args = dict(nbytes=[[32 * 4, 32 * 2, 32], [32 * 7]], data_ptrs=[[1, 2, 3], [4]], point_step=32, field_offsets=L32, T=None)
    args.update(kw)
    with pytest.raises(ValueError):
        capi.cloud_parts(**args)


def test_split_four_lidar_scan_concatenates_to_the_fused_cloud():
    scene = synth.make_scene(seed=21, stream_len=6.0)
    kw = dict(ego_xy=(3.0, -0.5), yaw=0.3, seed=99)
    fused, org = synth.scan_4lidar(scene, **kw)
    parts, org_s = synth.scan_4lidar(scene, split=True, **kw)
    assert len(parts) == len(synth.FOUR_LIDAR) and all(p.dtype == synth.POINT_DTYPE for p in parts)
    assert org_s.tobytes() == org.tobytes()
    assert b"".join(np.ascontiguousarray(p).tobytes() for p in parts) == fused.tobytes()
    _, _, ids = synth.scan_4lidar(scene, labels=True, **kw)
    _, _, ids_s = synth.scan_4lidar(scene, labels=True, split=True, **kw)
    assert [len(i) for i in ids_s] == [len(p) for p in parts] and np.array_equal(np.concatenate(ids_s), ids)
