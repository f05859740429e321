"""Cost of feeding sensor-frame PointCloud2 payloads from GPU memory, on the device-resident workload of bench.py's `value`.

    python bench_cloud_msgs.py [--streams 396] [--pool 8] [--steps 40] [--warmup 3] [--reps 3] [--u-steps 3]

Same scans as `value` (64-beam streams, rolls between steps, labels only), one step = one scan of every stream.  The
sensor-frame payloads are built once on the host from the generated map-frame clouds (inverse of a per-stream yaw + pitch
transform, rounded to float32) and kept in HBM: an 18-byte copy (x, y, z, intensity, ring: the KITTI player's layout) and a
32-byte PointXYZIR copy.  Every step is ordered on torch's current stream and timed with CUDA events recorded on it.
Variants, alternated --reps times in one run:
  B    gg_run_scans_to_device on the map-frame records already in HBM (today's device path; the floor)
  K18  gg_run_cloud_msgs_to_device on the 18-byte payloads
  K32  gg_run_cloud_msgs_to_device on the 32-byte payloads
  P    the caller in torch on the 32-byte payloads: fp64 elementwise transform in the reference's operation order, cast,
       packing into records, then gg_run_scans_to_device
  U    --u-steps steps of the host route: gg_upload_cloud_msg per slot from pinned host memory (18-byte payloads), then
       gg_run_scans and a synchronise (host clock; filling the pinned buffer is not timed)
After the timed steps of each variant, one more step is checked bit-exact on a seeded sample of --check streams against a
twin handle fed the same payload bytes from host memory through gg_upload_cloud_msg + gg_run_scans (its sampled slots
start from the handle's map position, "ground" and "groundpatch").  Whether P's labels equal the twin's is reported, not
assumed.  A serialised pass (one stream group, gg_profile) times the unpack kernel alone against the byte model
(point_step + 32) bytes per point at the H100 SXM data sheet's 3.35 TB/s.  Prints the card, its power limit, a table and
one JSON line; writes nothing.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generators and the pose sequence of bench.py)
from bench_slot_config import gpu_info  # noqa: E402

VARIANTS = {
    "B": "run_scans_to_device, map-frame records in HBM",
    "K18": "run_cloud_msgs_to_device, 18-byte payloads",
    "K32": "run_cloud_msgs_to_device, 32-byte payloads",
    "P": "torch fp64 transform + packing, run_scans_to_device",
    "U": "upload_cloud_msg x slots (pinned) + run_scans + sync",
}
LAYOUT = {18: (0, 4, 8, 12, 16), 32: (0, 4, 8, 16, 20)}
DATASHEET_TBS = 3.35


def map_from_sensor(origin, yaw, pitch):
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    R = np.array([[cy, -sy, 0.0], [sy, cy, 0.0], [0.0, 0.0, 1.0]]) @ np.array([[cp, 0.0, sp], [0.0, 1.0, 0.0], [-sp, 0.0, cp]])
    return np.concatenate([R, np.asarray(origin, np.float64).reshape(3, 1)], axis=1)


def payload(pts, T, step):
    """Sensor-frame PointCloud2 bytes [n, step] of map-frame points (inverse of T, float32)."""
    n = len(pts)
    p = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64) - T[:, 3]
    q = (p @ T[:, :3]).astype(np.float32)
    raw = np.zeros((n, step), np.uint8)
    off = LAYOUT[step]
    for c in range(3):
        raw[:, off[c]:off[c] + 4] = np.ascontiguousarray(q[:, c]).view(np.uint8).reshape(n, 4)
    raw[:, off[3]:off[3] + 4] = np.ascontiguousarray(pts["intensity"]).view(np.uint8).reshape(n, 4)
    raw[:, off[4]:off[4] + 2] = np.ascontiguousarray(pts["ring"]).view(np.uint8).reshape(n, 2)
    return raw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream (about 12 GB of HBM per 32-byte copy at 8)")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--u-steps", type=int, default=3)
    ap.add_argument("--prof-steps", type=int, default=3)
    ap.add_argument("--check", type=int, default=16, help="streams of the seeded sample checked after each variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_cloud_msgs.py needs a CUDA device")
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    origins = [np.array([streams[b][s][1] for b in range(B)], np.float32) for s in range(S)]
    Tsensor = [np.stack([map_from_sensor(streams[b][s][1], 0.013 * b + 0.2 * s, 0.02) for b in range(B)]) for s in range(S)]

    # per pose one flat device buffer per layout, streams back to back
    def upload(make, step):
        pools, views = [], []
        for s in range(S):
            n = npts[:, s]
            flat = torch.empty(int(n.sum()) * step, dtype=torch.uint8, device="cuda")
            o, vs = 0, []
            for b in range(B):
                raw = make(b, s).reshape(-1)
                flat[o:o + raw.size] = torch.from_numpy(raw)
                vs.append(flat[o:o + raw.size])
                o += raw.size
            pools.append(flat)
            views.append(vs)
        return pools, views

    t0 = time.time()
    rec_pool, clouds = upload(lambda b, s: np.ascontiguousarray(streams[b][s][0]).view(np.uint8), 32)
    k18_pool, k18 = upload(lambda b, s: payload(streams[b][s][0], Tsensor[s][b], 18), 18)
    k32_pool, k32 = upload(lambda b, s: payload(streams[b][s][0], Tsensor[s][b], 32), 32)
    del streams
    build_s = time.time() - t0
    pts_per_pose = npts.sum(axis=0)
    counts_dev = [torch.from_numpy(npts[:, s]).cuda() for s in range(S)]
    T_dev = [torch.from_numpy(Tsensor[s].reshape(B, 12)).cuda() for s in range(S)]

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    slots = np.arange(B, dtype=np.int32)
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    descs = [g.make_descs(list(range(B)), [int(npts[b, s]) for b in range(B)], list(origins[s]), [0.0] * B) for s in range(S)]
    pinned = torch.empty(int(npts.sum(axis=0).max()) * 18, dtype=torch.uint8).pin_memory()
    cur = torch.cuda.current_stream()
    tstep = [0]
    last = {}

    def torch_records(s):
        """P: what a caller writes in torch -- ((T00 x + T01 y) + T02 z) + T03 in fp64, one rounding per operation, cast to
        float32, packed into 32-byte records."""
        f = k32_pool[s].view(torch.float32).view(-1, 8)
        n = f.shape[0]
        scan = torch.repeat_interleave(torch.arange(B, device="cuda"), counts_dev[s], output_size=n)
        x, y, z = (f[:, c].double() for c in range(3))
        rec = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
        for r in range(3):
            T = T_dev[s][:, 4 * r:4 * r + 4][scan]
            rec[:, r] = (((T[:, 0] * x + T[:, 1] * y) + T[:, 2] * z) + T[:, 3]).float()
        rec[:, 4] = f[:, 4]
        rec.view(torch.int32)[:, 5] = f.view(torch.int32)[:, 5] & 0xFFFF
        return list(torch.split(rec, npts[:, s].tolist()))

    def launch(variant, h, s):
        if variant == "B":
            return h.run_scans_to_device(clouds[s], slots, origins[s], 0.0, labels=True, select=None)
        if variant in ("K18", "K32"):
            step = int(variant[1:])
            return h.run_cloud_msgs_to_device(k18[s] if step == 18 else k32[s], step, LAYOUT[step], Tsensor[s], slots, origins[s], 0.0,
                                              labels=True, select=None)
        if variant == "P":
            return h.run_scans_to_device(torch_records(s), slots, origins[s], 0.0, labels=True, select=None)
        raise ValueError(variant)

    def next_pose():
        s = bench.pingpong(tstep[0], S)
        if tstep[0]:
            g.update_pose_batch(slots, xy[s], Ts[s])
        tstep[0] += 1
        return s

    def step(variant):
        s = next_pose()
        last["out"], last["pose"] = launch(variant, g, s), s
        return int(pts_per_pose[s])

    def step_u(timed_out=None):
        """U: the pinned buffer is filled before the clock starts."""
        s = bench.pingpong(tstep[0], S)
        pinned[:k18_pool[s].numel()].copy_(k18_pool[s])
        torch.cuda.synchronize()
        t = time.perf_counter()
        s2 = next_pose()
        assert s2 == s
        base, off = pinned.data_ptr(), 0
        for b in range(B):
            n = int(npts[b, s])
            capi._check(g._l.gg_upload_cloud_msg(g._h, b, base + off, n, 18, capi._ptr(np.array(LAYOUT[18], np.int32)),
                                                 capi._ptr(np.ascontiguousarray(Tsensor[s][b]).reshape(12))))
            off += 18 * n
        g.run_scans(descs[s])
        g.synchronize()
        if timed_out is not None:
            timed_out.append((time.perf_counter() - t) * 1e3)
        last["out"], last["pose"] = None, s
        return int(pts_per_pose[s])

    def timed(variant):
        if variant == "U":
            step_u()
            per = []
            for _ in range(args.u_steps):
                step_u(per)
            return {"ms_per_step": float(np.mean(per)), "ms_step_median": float(np.median(per))}
        for _ in range(args.warmup):
            step(variant)
        g.synchronize()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        pts = 0
        ev[0].record(cur)
        for t in range(args.steps):
            pts += step(variant)
            ev[t + 1].record(cur)
        g.synchronize()
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[-1])
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.steps)]
        return {"ms_per_step": total / args.steps, "ms_step_median": float(np.median(per)), "mpoints_per_s": pts / (total * 1e-3) / 1e6}

    rng = np.random.default_rng(1234)
    sample = sorted(rng.choice(B, min(args.check, B), replace=False).tolist())
    twin = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=len(sample), max_points=bench.PCAP, full_layers=False)
    tslots = np.arange(len(sample), dtype=np.int32)
    checks = {v: [] for v in VARIANTS}

    def check(variant):
        """One more step of `variant`; its sampled scans against the twin fed the same bytes through gg_upload_cloud_msg."""
        torch.cuda.synchronize()
        g.synchronize()
        for i, b in enumerate(sample):
            pos = g.position(b)
            twin.init_map(float(pos[0]), float(pos[1]), 0.0, slot=i)
            twin.set_layer("ground", g.layer("ground", b), slot=i)
            twin.set_layer("groundpatch", g.layer("groundpatch", b), slot=i)
        if variant == "U":
            step_u()
        else:
            step(variant)
        s = last["pose"]
        torch.cuda.synchronize()
        g.synchronize()
        twin.update_pose_batch(tslots, xy[s][sample], Ts[s][sample])
        src = {"B": clouds, "K18": k18, "U": k18}.get(variant, k32)
        step_b = 32 if src is not k18 else 18
        keep = []
        for i, b in enumerate(sample):
            raw = src[s][b].cpu().numpy()
            keep.append(raw)
            twin.upload_cloud_msg(raw, int(npts[b, s]), step_b, LAYOUT[step_b], None if variant == "B" else Tsensor[s][b], slot=i)
        twin.run_scans(twin.make_descs(list(tslots), [int(npts[b, s]) for b in sample], [origins[s][b] for b in sample], [0.0] * len(sample)))
        same = True
        for i, b in enumerate(sample):
            want = twin.download_labels(int(npts[b, s]), slot=i)
            twin.synchronize()
            if variant == "U":
                got = g.download_labels(int(npts[b, s]), slot=b)
                g.synchronize()
            else:
                got = last["out"].labels[b].cpu().numpy()
            same = same and np.array_equal(got, want)
        if variant != "P":
            assert same, f"{variant}: labels differ from the twin"
        checks[variant].append(bool(same))

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            check(v)

    # serialised pass: one stream group, the unpack kernel's own time from gg_profile
    old = os.environ.get("GG_STREAMS")
    os.environ["GG_STREAMS"] = "1"
    g1 = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    if old is None:
        del os.environ["GG_STREAMS"]
    else:
        os.environ["GG_STREAMS"] = old
    for b in range(B):
        g1.init_map(0.0, 0.0, 0.0, slot=b)
    unpack = {}
    for variant in ("K18", "K32"):
        launch(variant, g1, 0)
        g1.synchronize()
        g1.profile_enable(True)
        g1.profile_read(reset=True)
        pts = 0
        for t in range(args.prof_steps):
            s = bench.pingpong(t + 1, S)
            g1.update_pose_batch(slots, xy[s], Ts[s])
            launch(variant, g1, s)
            pts += int(pts_per_pose[s])
        prof = g1.profile_read(reset=True)
        g1.profile_enable(False)
        ms, n_launch = prof["k_unpack_transform"]
        step_b = int(variant[1:])
        gbytes = (step_b + 32) * pts / 1e9
        unpack[variant] = {"ms_per_step": ms / args.prof_steps, "launches": n_launch, "model_gb_per_step": gbytes / args.prof_steps,
                           "tb_per_s": gbytes / (ms * 1e-3) / 1e3, "share_of_datasheet": gbytes / (ms * 1e-3) / 1e3 / DATASHEET_TBS,
                           "step_ms_serial": sum(v[0] for v in prof.values()) / args.prof_steps}
    g1.close()

    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, {args.steps} timed steps per run ({args.u_steps} for U), {args.reps} alternating runs; "
          f"{float(npts.mean()):.0f} points per scan; payloads built in {build_s:.0f} s")
    print(f"{'variant':<62} {'ms/step (runs)':<28} {'twin check':>10}")
    for v, desc in VARIANTS.items():
        ms = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<62} {' / '.join(f'{x:.2f}' for x in ms):<28} {'equal' if all(checks[v]) else 'DIFFERS':>10}")
    for v, u in unpack.items():
        print(f"k_unpack_transform {v} (serialised, one launch per step): {u['ms_per_step']:.3f} ms/step, byte model "
              f"{u['model_gb_per_step']:.2f} GB -> {u['tb_per_s']:.2f} TB/s = {100 * u['share_of_datasheet']:.0f} % of the data sheet's "
              f"{DATASHEET_TBS} TB/s (not a measured peak)")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "u_steps": args.u_steps, "reps": args.reps,
                      "points_per_scan_mean": float(npts.mean()), "sample": sample, "twin_equal": checks, "results": results,
                      "unpack": unpack}))
    twin.close()
    g.close()


if __name__ == "__main__":
    main()
