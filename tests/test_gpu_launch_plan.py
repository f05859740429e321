"""The launch plan of every entry point that enqueues work: after each call, the number of kernels it launched
(gg_kernel_launches) and the launches per kernel (gg_profile_read) against a fixed table.  A handle of 6 slots on 3
stream groups (slots 0-1, 2-3, 4-5), so that each batched call is seen on one group and on several; a batched call
launches its kernels once per stream group with slots in the batch."""
import numpy as np
import pytest

from groundgrid_b200 import capi, synth

pytestmark = pytest.mark.gpu

PIPE = ("k_rasterize", "k_cell_tiles", "k_cell_place", "k_scatter", "k_cell_stats", "k_detect", "k_spiral", "k_label")
STOP = {0: PIPE, 1: PIPE[:5], 2: PIPE[:6], 3: PIPE[:7]}   # kernels of a scan run up to stop_after
OUT = ("k_out_count", "k_out_scan", "k_out_write")
ROLL = ("k_roll_gather", "k_roll_commit")
LAYERS = ("ground", "groundpatch", "points")
MSG = (32, (0, 4, 8, 16, 20))   # point_step and field offsets of a 32-byte PointXYZIR payload


def per_group(groups, *kernels):
    out = {}
    for k in kernels:
        out[k] = out.get(k, 0) + groups
    return out


def steps(g, torch, pts, org):
    """(name, call, {kernel: launches}); the calls run in this order on one handle."""
    n = len(pts)
    dev = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8).copy()).cuda()
    far = synth.base_from_map(3.0, 1.0)
    near = synth.base_from_map(0.0, 0.0)

    def roll(slots, xy):
        T = np.stack([(far if tuple(p) == (3.0, 1.0) else near).reshape(12) for p in xy])
        g.update_pose_batch(np.array(slots, np.int32), np.array(xy, np.float64), T)

    def run(slots, stop_after):
        for s in slots:
            g.upload_points(pts, slot=s)
        g.run_scans(g.make_descs(slots, [n] * len(slots), [org] * len(slots), [0.0] * len(slots)), stop_after)

    def to_device(slots, **kw):
        return g.run_scans_to_device([dev] * len(slots), slots, [org] * len(slots), 0.0, **kw)

    def msgs(slots):
        return g.run_cloud_msgs_to_device([dev] * len(slots), MSG[0], MSG[1], None, slots, [org] * len(slots), 0.0, select=None)

    def batch(slots):
        g.filter_cloud_batch_ptrs(g.make_descs(slots, [n] * len(slots), [org] * len(slots), [0.0] * len(slots)),
                                  [pts.ctypes.data] * len(slots), None)

    return [
        ("roll, 2 groups", lambda: roll([0, 1, 2], [(3.0, 1.0)] * 3), per_group(2, *ROLL)),
        ("roll without movement", lambda: roll([0, 1, 2, 3, 4, 5], [(3.0, 1.0)] * 3 + [(0.0, 0.0)] * 3), {}),
        ("roll, 1 of 2 groups moved", lambda: roll([3, 4], [(0.0, 0.0), (3.0, 1.0)]), per_group(1, *ROLL)),
        ("run_scans stop 1, 1 group", lambda: run([0, 1], 1), per_group(1, *STOP[1])),
        ("run_scans stop 2, 3 groups", lambda: run([0, 2, 4], 2), per_group(3, *STOP[2])),
        ("run_scans stop 3, 2 groups", lambda: run([1, 5], 3), per_group(2, *STOP[3])),
        ("run_scans stop 0, 3 groups", lambda: run([0, 1, 2, 3, 4, 5], 0), per_group(3, *STOP[0])),
        ("to_device labels, 2 groups", lambda: to_device([0, 1, 2], select=None), per_group(2, *PIPE, "k_out_write")),
        ("to_device index + cloud, 2 groups", lambda: to_device([3, 4, 5], labels=False, select="all", index=True),
         per_group(2, *PIPE, *OUT)),
        ("to_device labels + cloud, 1 group", lambda: to_device([4], select="nonground"), per_group(1, *PIPE, *OUT)),
        ("cloud msgs, 2 groups", lambda: msgs([0, 5]), per_group(2, "k_unpack_transform", *PIPE, "k_out_write")),
        ("cloud msgs, 1 group", lambda: msgs([2, 3]), per_group(1, "k_unpack_transform", *PIPE, "k_out_write")),
        ("upload_cloud_msg", lambda: g.upload_cloud_msg(np.ascontiguousarray(pts).view(np.uint8), n, *MSG, slot=1),
         per_group(1, "k_unpack_transform")),
        ("run_scans stop 0, 1 group", lambda: run([1], 0), per_group(1, *PIPE)),
        ("get_output", lambda: g.get_output(slot=0, want_cloud=True), per_group(1, *OUT)),
        ("layer export, 2 groups", lambda: g.get_layers_to_device([0, 1, 2, 3], LAYERS), per_group(2, "k_layer_copy")),
        ("layer export, 1 group", lambda: g.get_layers_to_device([5], LAYERS), per_group(1, "k_layer_copy")),
        ("layer import, 3 groups", lambda: g.set_layers_from_device([0, 3, 4], ("ground", "groundpatch"),
                                                                    g.get_layers_to_device([0, 3, 4], ("ground", "groundpatch"))),
         per_group(6, "k_layer_copy")),
        ("layer images, 3 groups", lambda: g.layer_images_to_device([0, 2, 4], LAYERS), per_group(3, "k_layer_range", "k_layer_image")),
        ("layer image, one slot", lambda: g.layer_image_u8("variance", slot=3), per_group(1, "k_layer_range", "k_layer_image")),
        ("terrain images, 3 groups", lambda: g.terrain_images_to_device([0, 1, 2, 3, 4, 5]), per_group(3, "k_terrain_image")),
        ("terrain image, one slot", lambda: g.terrain_image(slot=5), per_group(1, "k_terrain_image")),
        ("eval, 3 groups", lambda: g.eval_counts_to_device([5, 4, 3, 2, 1, 0]), per_group(3, "k_eval_counts")),
        ("eval, 1 group", lambda: g.eval_counts_to_device([3]), per_group(1, "k_eval_counts")),
        ("eval_accumulate", lambda: g.eval_accumulate(slot=2), per_group(1, "k_eval_counts")),
        ("detect_ground_patches", lambda: g.detect_ground_patches(slot=2), per_group(1, "k_detect")),
        ("spiral_ground_interpolation", lambda: g.spiral_ground_interpolation(0.0, slot=3), per_group(1, "k_spiral")),
        ("filter_cloud_batch, 3 groups", lambda: batch([0, 1, 2, 3, 4, 5]), per_group(3, *PIPE)),
        ("filter_cloud_batch, 1 group", lambda: batch([4, 5]), per_group(1, *PIPE)),
    ]


def test_launch_plan_of_every_entry_point(monkeypatch):
    import torch

    monkeypatch.setenv("GG_STREAMS", "3")
    g = capi.GroundGridB200(33.33, 0.33, n_slots=6, max_points=32768, full_layers=True)
    assert g.n_streams == 3
    scene = synth.make_scene(seed=7100, n_boxes=12)
    pts, org = synth.lidar_scan(scene, beams=32, az_steps=512, seed=7101)
    for s in range(6):
        g.init_map(0.0, 0.0, 0.0, slot=s)
    g.profile_enable(True)
    g.profile_read(reset=True)
    for name, call, want in steps(g, torch, pts, org):
        l0 = g.kernel_launches
        call()
        torch.cuda.synchronize()
        got = {k: c for k, (_, c) in g.profile_read(reset=True).items()}
        assert got == want, f"{name}: launches per kernel"
        assert g.kernel_launches - l0 == sum(want.values()), f"{name}: gg_kernel_launches"
    g.profile_enable(False)
    g.close()
