"""synth.lidar_scan(..., labels=True): the SemanticKITTI id of the surface each ray hit, with the cloud unchanged."""
import numpy as np
import pytest

from groundgrid_b200 import synth


@pytest.mark.parametrize("make", [synth.scan_64, synth.scan_128, synth.scan_4lidar], ids=["64beam", "128beam", "4lidar"])
def test_labels_leave_the_cloud_unchanged_and_name_the_surface(make):
    scene = synth.make_scene(seed=17, n_boxes=40, rmin=4.0, rmax=40.0)
    ego, yaw = (2.5, -1.0), 0.4
    pts, org = make(scene, ego_xy=ego, yaw=yaw, seed=17)
    pts_l, org_l, ids = make(scene, ego_xy=ego, yaw=yaw, seed=17, labels=True)
    assert pts_l.dtype == pts.dtype and pts_l.tobytes() == pts.tobytes()
    assert org_l.tobytes() == org.tobytes()
    assert ids.dtype == np.uint16 and ids.shape == (len(pts),)
    assert set(np.unique(ids)) == {synth.LABEL_CAR, synth.LABEL_ROAD, synth.LABEL_BUILDING}

    x = pts["x"].astype(np.float64)
    y = pts["y"].astype(np.float64)
    z = pts["z"].astype(np.float64)
    tol = 0.2   # 10 sigma of the range noise along the ray
    wall = ids == synth.LABEL_BUILDING
    cheb = np.maximum(np.abs(x - ego[0]), np.abs(y - ego[1]))
    assert np.all(np.abs(cheb[wall] - synth.WALL_HALF) < tol)
    assert np.all(cheb[~wall] < synth.WALL_HALF + tol)
    road = ids == synth.LABEL_ROAD
    assert np.all(np.abs(z[road]) < tol)
    car = ids == synth.LABEL_CAR
    b = scene.boxes
    inside = np.zeros(int(car.sum()), bool)
    for box in b:
        inside |= ((x[car] > box[0] - tol) & (x[car] < box[3] + tol) & (y[car] > box[1] - tol) & (y[car] < box[4] + tol)
                   & (z[car] > box[2] - tol) & (z[car] < box[5] + tol))
    assert inside.all()


def test_labels_in_the_base_frame_match_the_map_frame():
    scene = synth.make_scene(seed=3, stream_len=40.0)
    _, _, ids_map = synth.lidar_scan(scene, ego_xy=(10.0, 0.0), yaw=0.2, beams=32, az_steps=512, seed=3, labels=True)
    pts_b, _, ids_base = synth.lidar_scan(scene, ego_xy=(10.0, 0.0), yaw=0.2, beams=32, az_steps=512, seed=3, frame="base",
                                          labels=True)
    pts_b0, _ = synth.lidar_scan(scene, ego_xy=(10.0, 0.0), yaw=0.2, beams=32, az_steps=512, seed=3, frame="base")
    assert pts_b.tobytes() == pts_b0.tobytes()
    assert np.array_equal(ids_map, ids_base)
