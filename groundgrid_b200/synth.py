"""Seeded synthetic LiDAR scans shaped like the reference's input (SURVEY.md section 8d).

Not part of the compute path: this only fabricates PointXYZIR clouds (32-byte records,
include/velodyne_pointcloud/point_types.h:27-33 of the reference) for tests, smoke() and
bench.py.  Scene: ground plane (optionally undulating), axis-aligned boxes, an enclosure
wall so every beam returns; 64/128-beam spinning sensor, ring-major point order.
"""
import math

import numpy as np

# 32-byte PointXYZIR record: float x,y,z,(pad); float intensity; uint16 ring; (pad).
POINT_DTYPE = np.dtype(
    {
        "names": ["x", "y", "z", "intensity", "ring"],
        "formats": ["<f4", "<f4", "<f4", "<f4", "<u2"],
        "offsets": [0, 4, 8, 16, 20],
        "itemsize": 32,
    }
)

SENSOR_HEIGHT = 1.73  # launch/KITTIEvaluate.launch:13 static TF (sensor 1.73 m above base)
WALL_HALF = 45.0
WALL_HEIGHT = 20.0
BOX_SIZE = (4.5, 1.8, 1.5)


class Scene:
    def __init__(self, boxes, undulation=0.0):
        self.boxes = np.asarray(boxes, np.float64).reshape(-1, 6)  # xmin ymin zmin xmax ymax zmax
        self.undulation = float(undulation)

    def ground_height(self, x):
        if self.undulation == 0.0:
            return np.zeros_like(x)
        return self.undulation * np.sin(x / 15.0)


def make_scene(seed=1234, n_boxes=24, rmin=5.0, rmax=50.0, stream_len=0.0, undulation=0.0):
    """Boxes 4.5 x 1.8 x 1.5 m at seeded-uniform positions rmin..rmax from the ego start.
    With stream_len > 0 the boxes populate a corridor along +x (road |y| < 4 m kept free)."""
    rng = np.random.default_rng(seed)
    boxes = []
    if stream_len <= 0.0:
        for _ in range(n_boxes):
            r = rng.uniform(rmin, rmax)
            a = rng.uniform(0.0, 2.0 * math.pi)
            cx, cy = r * math.cos(a), r * math.sin(a)
            sx, sy = (BOX_SIZE[0], BOX_SIZE[1]) if rng.uniform() < 0.5 else (BOX_SIZE[1], BOX_SIZE[0])
            boxes.append([cx - sx / 2, cy - sy / 2, 0.0, cx + sx / 2, cy + sy / 2, BOX_SIZE[2]])
    else:
        count = int(round(n_boxes * (stream_len + 100.0) / 100.0))
        while len(boxes) < count:
            cx = rng.uniform(-50.0, stream_len + 50.0)
            cy = rng.uniform(-50.0, 50.0)
            sx, sy = (BOX_SIZE[0], BOX_SIZE[1]) if rng.uniform() < 0.5 else (BOX_SIZE[1], BOX_SIZE[0])
            if abs(cy) < 4.0 + sy / 2:
                continue
            boxes.append([cx - sx / 2, cy - sy / 2, 0.0, cx + sx / 2, cy + sy / 2, BOX_SIZE[2]])
    return Scene(boxes, undulation)


# SemanticKITTI ids of the surfaces (semantic-kitti.yaml): what lidar_scan(..., labels=True) reports per point
LABEL_ROAD, LABEL_CAR, LABEL_BUILDING = 40, 10, 50


def _cast(scene, origins, dirs, ego_xy):
    """Nearest hit distance along each ray (float64) and the SemanticKITTI id (uint16) of the surface hit: road for
    the ground, car for a box, building for the enclosure wall."""
    ox, oy, oz = origins[:, 0], origins[:, 1], origins[:, 2]
    dx, dy, dz = dirs[:, 0], dirs[:, 1], dirs[:, 2]
    big = 1.0e9
    with np.errstate(divide="ignore", invalid="ignore"):
        # ground (fixed-point iteration handles the gentle undulation)
        h = np.zeros_like(ox)
        t_g = np.full_like(ox, big)
        down = dz < -1e-9
        for _ in range(4 if scene.undulation != 0.0 else 1):
            t_g = np.where(down, (h - oz) / dz, big)
            h = scene.ground_height(ox + t_g * dx)
        t_g = np.where(down & (t_g > 0), t_g, big)
        # enclosure walls, ego-relative
        t_w = np.full_like(ox, big)
        for axis_o, axis_d, centre in ((ox, dx, ego_xy[0]), (oy, dy, ego_xy[1])):
            for sgn in (-1.0, 1.0):
                t = (centre + sgn * WALL_HALF - axis_o) / axis_d
                t = np.where((t > 0) & np.isfinite(t), t, big)
                t_w = np.minimum(t_w, t)
        t_best = np.minimum(t_g, t_w)
        ids = np.where(t_g <= t_w, LABEL_ROAD, LABEL_BUILDING).astype(np.uint16)
        # boxes: slab test
        for b in scene.boxes:
            inv = [1.0 / dx, 1.0 / dy, 1.0 / dz]
            t0 = (b[0] - ox) * inv[0]
            t1 = (b[3] - ox) * inv[0]
            tmin, tmax = np.minimum(t0, t1), np.maximum(t0, t1)
            t0 = (b[1] - oy) * inv[1]
            t1 = (b[4] - oy) * inv[1]
            tmin, tmax = np.maximum(tmin, np.minimum(t0, t1)), np.minimum(tmax, np.maximum(t0, t1))
            t0 = (b[2] - oz) * inv[2]
            t1 = (b[5] - oz) * inv[2]
            tmin, tmax = np.maximum(tmin, np.minimum(t0, t1)), np.minimum(tmax, np.maximum(t0, t1))
            hit = (tmax >= tmin) & (tmin > 0)
            closer = hit & (tmin < t_best)
            t_best = np.where(closer, tmin, t_best)
            ids[closer] = LABEL_CAR
    return t_best, ids


def lidar_scan(scene, ego_xy=(0.0, 0.0), yaw=0.0, beams=64, elev_deg=(2.0, -24.8), az_steps=2048,
               dropout=0.085, seed=1234, sensors=((0.0, 0.0, SENSOR_HEIGHT, 0.0),), range_noise=0.02,
               frame="map", labels=False, split=False):
    """One revolution of each sensor, concatenated sensor-major, ring-major then azimuth.

    sensors: (dx, dy, z, yaw_offset_deg) mounting poses in the ego frame.
    Returns (points[POINT_DTYPE], origin[3] float32) with points in the map frame
    (or in the ego/base frame when frame == "base").  With labels=True also a uint16 array of the
    SemanticKITTI id of the surface each point's ray hit (LABEL_ROAD, LABEL_CAR, LABEL_BUILDING); the
    points and origin are the same bytes as without it.  The evaluation flow puts the ids into "ring".
    With split=True the points (and ids) are lists with one array per sensor, as a multi-sensor rig delivers
    them; concatenated, they are the same bytes as without split.
    """
    rng = np.random.default_rng(seed)
    ego_xy = (float(ego_xy[0]), float(ego_xy[1]))
    elev = np.deg2rad(np.linspace(elev_deg[0], elev_deg[1], beams))[::-1]  # ring 0 = lowest beam
    az = np.arange(az_steps) * (2.0 * math.pi / az_steps)
    ce, se = np.cos(elev)[:, None], np.sin(elev)[:, None]
    clouds, ids = [], []
    for (sx, sy, sz, syaw) in sensors:
        a = az[None, :] + yaw + math.radians(syaw)
        d = np.stack([ce * np.cos(a), ce * np.sin(a), np.broadcast_to(se, (beams, az_steps))], axis=-1).reshape(-1, 3)
        cy_, sy_ = math.cos(yaw), math.sin(yaw)
        o = np.array([ego_xy[0] + cy_ * sx - sy_ * sy, ego_xy[1] + sy_ * sx + cy_ * sy, sz])
        origins = np.broadcast_to(o, d.shape)
        t, hit_id = _cast(scene, origins, d, ego_xy)
        t = t + rng.normal(0.0, range_noise, size=t.shape)
        p = origins + t[:, None] * d
        keep = rng.uniform(size=t.shape) >= dropout
        ring = np.repeat(np.arange(beams, dtype=np.uint16), az_steps)
        inten = rng.uniform(size=t.shape)
        pts = np.zeros(int(keep.sum()), POINT_DTYPE)
        if frame == "base":
            rx = p[:, 0] - ego_xy[0]
            ry = p[:, 1] - ego_xy[1]
            p = np.stack([cy_ * rx + sy_ * ry, -sy_ * rx + cy_ * ry, p[:, 2]], axis=-1)
        pts["x"] = p[keep, 0].astype(np.float32)
        pts["y"] = p[keep, 1].astype(np.float32)
        pts["z"] = p[keep, 2].astype(np.float32)
        pts["intensity"] = inten[keep].astype(np.float32)
        pts["ring"] = ring[keep]
        clouds.append(pts)
        ids.append(hit_id[keep])
    if split:
        cloud = clouds
    elif len(clouds) > 1:
        # np.concatenate drops the padding of the record dtype: fill a 32-byte-record array field by field instead
        cloud = np.zeros(sum(len(c) for c in clouds), POINT_DTYPE)
        at = 0
        for c in clouds:
            for f in ("x", "y", "z", "intensity", "ring"):
                cloud[f][at:at + len(c)] = c[f]
            at += len(c)
    else:
        cloud = clouds[0]
    origin = np.array([ego_xy[0], ego_xy[1], SENSOR_HEIGHT], np.float32)
    if labels:
        return cloud, origin, ids if split else np.concatenate(ids)
    return cloud, origin


FOUR_LIDAR = ((1.0, 0.5, SENSOR_HEIGHT, 0.0), (-1.0, 0.5, SENSOR_HEIGHT, 90.0),
              (-1.0, -0.5, SENSOR_HEIGHT, 180.0), (1.0, -0.5, SENSOR_HEIGHT, 270.0))


def scan_64(scene, ego_xy=(0.0, 0.0), yaw=0.0, seed=1234, **kw):
    """cfg1/2/5: 64 beams +2.0..-24.8 deg, 2048 azimuth steps, 8.5 % drop-out -> ~120 k returns."""
    return lidar_scan(scene, ego_xy, yaw, beams=64, elev_deg=(2.0, -24.8), seed=seed, **kw)


def scan_128(scene, ego_xy=(0.0, 0.0), yaw=0.0, seed=1234, **kw):
    """cfg3: 128 beams +15..-25 deg, 2048 azimuth steps -> ~240 k returns."""
    return lidar_scan(scene, ego_xy, yaw, beams=128, elev_deg=(15.0, -25.0), seed=seed, **kw)


def scan_4lidar(scene, ego_xy=(0.0, 0.0), yaw=0.0, seed=1234, **kw):
    """cfg4: four 64-beam sensors, clouds concatenated sensor-major -> ~480 k returns."""
    return lidar_scan(scene, ego_xy, yaw, beams=64, elev_deg=(2.0, -24.8), seed=seed, sensors=FOUR_LIDAR, **kw)


def base_from_map(ego_x, ego_y, yaw=0.0, base_z=0.0, pitch=0.0):
    """Row-major 3x4 [R|t] of lookupTransform("base_link", "map"): p_base = R p_map + t.
    A small pitch makes the seeded terrain of GroundGrid::update position dependent."""
    cy, sy = math.cos(yaw), math.sin(yaw)
    cp, sp = math.cos(pitch), math.sin(pitch)
    Rz = np.array([[cy, -sy, 0.0], [sy, cy, 0.0], [0.0, 0.0, 1.0]])
    Ry = np.array([[cp, 0.0, sp], [0.0, 1.0, 0.0], [-sp, 0.0, cp]])
    R_map_from_base = Rz @ Ry
    R = R_map_from_base.T
    t = -R @ np.array([ego_x, ego_y, base_z])
    return np.concatenate([R, t[:, None]], axis=1)


def quat_from_yaw_pitch(yaw=0.0, pitch=0.0):
    """Quaternion (x, y, z, w) of Rz(yaw) * Ry(pitch)."""
    cy, sy = math.cos(0.5 * yaw), math.sin(0.5 * yaw)
    cp, sp = math.cos(0.5 * pitch), math.sin(0.5 * pitch)
    return np.array([-sy * sp, cy * sp, sy * cp, cy * cp], np.float64)


def tf2_matrix(q, t):
    """Row-major 3x4 [R|t] of a geometry_msgs/Transform exactly as tf2::Matrix3x3::setRotation builds it (same fp64
    operation order), i.e. what tf2::doTransform applies.  Feeding (q, t) to the reference and this matrix to the C-ABI
    gives both the same numbers."""
    x, y, z, w = (float(v) for v in q)
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    return np.array([[1.0 - (yy + zz), xy - wz, xz + wy, float(t[0])],
                     [xy + wz, 1.0 - (xx + zz), yz - wx, float(t[1])],
                     [xz - wy, yz + wx, 1.0 - (xx + yy), float(t[2])]], np.float64)


def base_from_map_qt(ego_x, ego_y, yaw=0.0, base_z=0.0, pitch=0.0):
    """(q, t) of lookupTransform("base_link", "map") as the ROS message carries it, for a base frame at
    (ego_x, ego_y, base_z) with the given yaw / pitch in the map (the inverse of the base pose)."""
    q_pose = quat_from_yaw_pitch(yaw, pitch)
    q = np.array([-q_pose[0], -q_pose[1], -q_pose[2], q_pose[3]])
    R = tf2_matrix(q, (0.0, 0.0, 0.0))[:, :3]
    t = -(R @ np.array([ego_x, ego_y, base_z]))
    return q, t


def stream_pose(k, step=1.0, yaw_step_deg=0.5):
    """Pose of scan k of the 200-scan stream: +1.0 m/scan along x, 0.5 deg/scan yaw."""
    return (k * step, 0.0), math.radians(k * yaw_step_deg)
