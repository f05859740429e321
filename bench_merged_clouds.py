"""Cost of feeding a multi-LiDAR rig's per-sensor PointCloud2 payloads from GPU memory, on the cfg4 workload of bench.py.

    python bench_merged_clouds.py [--streams 96] [--pool 2] [--steps 20] [--warmup 3] [--reps 3] [--u-steps 2]

cfg4 scans (BASELINE configs[3]: four 64-beam sensors of synth.FOUR_LIDAR, about 480 k points per scan, N = 364 at
120 m / 0.33 m), labels only, rolling between steps along the pose sequence of bench.py; one step = one scan of every
stream.  Each sensor's payload is built once on the host from its map-frame cloud: the inverse of T_map_from_sensor =
(ego pose) o (mount pose), rounded to float32.  It is kept in HBM as an 18-byte copy (x, y, z, intensity, ring: the KITTI
player's layout) and a 32-byte PointXYZIR copy; the part records of each pose are built once.  Every step is ordered on
torch's current stream and timed with CUDA events recorded on it.  Variants, alternated --reps times in one run:
  B    gg_run_scans_to_device on the fused map-frame records already in HBM (the floor)
  M18  gg_run_merged_cloud_msgs_to_device, four 18-byte payloads per scan
  M32  gg_run_merged_cloud_msgs_to_device, four 32-byte payloads per scan
  P    the caller in torch on the 32-byte payloads: per-part fp64 transform in tf2's operation order, cast, packing into
       records, concatenation, then gg_run_scans_to_device
  U    --u-steps steps of the host route: gg_upload_cloud_msgs per slot from pinned host memory (18-byte payloads), then
       gg_run_scans and a synchronise (host clock; filling the pinned buffer is not timed)
After the timed steps of each variant, one more step is checked bit-exact on a seeded sample of --check streams against a
twin handle fed the same payload bytes from host memory through gg_upload_cloud_msgs + gg_run_scans (its sampled slots
start from the handle's map position, "ground" and "groundpatch").  Whether P's labels equal the twin's is reported, not
assumed.  Also: one scan alone (one slot, M18 against B), and a serialised pass (one stream group, gg_profile) of the
unpack kernel against the byte model (point_step + 32) bytes per point at the H100 SXM data sheet's 3.35 TB/s.  Prints
the card, its power limit, a table and one JSON line; writes nothing.
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

import bench  # noqa: E402  (pose sequence and pingpong of bench.py)
from bench_slot_config import gpu_info  # noqa: E402

VARIANTS = {
    "B": "run_scans_to_device, fused map-frame records in HBM",
    "M18": "run_merged_cloud_msgs_to_device, 4 x 18-byte payloads",
    "M32": "run_merged_cloud_msgs_to_device, 4 x 32-byte payloads",
    "P": "torch fp64 per-part transform + packing + cat, run_scans_to_device",
    "U": "upload_cloud_msgs x slots (pinned) + run_scans + sync",
}
LAYOUT = {18: (0, 4, 8, 12, 16), 32: (0, 4, 8, 16, 20)}
DIM_M, RES, PCAP = 120.0, 0.33, 524288      # cfg4 of bench.py
DATASHEET_TBS = 3.35


def map_from_sensor(pose, mount):
    """Row-major 3x4 of T_map_from_sensor = (ego at (pose, 0), yaw 0) o (mount pose (dx, dy, z, yaw_deg))."""
    dx, dy, z, yaw = mount
    c, s = math.cos(math.radians(yaw)), math.sin(math.radians(yaw))
    return np.array([[c, -s, 0.0, float(pose) + dx], [s, c, 0.0, dy], [0.0, 0.0, 1.0, z]])


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


def _gen_task(args):
    """One stream's scan at one pose, per sensor (map frame), and its origin; the cfg4 seeds of bench.py."""
    from groundgrid_b200 import synth

    seed, pose, n_pose = args
    scene = synth.make_scene(seed=seed, stream_len=float(n_pose))
    return synth.scan_4lidar(scene, ego_xy=(float(pose), 0.0), yaw=0.0, seed=seed * 31 + pose, split=True)


def scan_bytes(parts, Ts):
    """(fused 32-byte records as bytes, 18-byte payloads, 32-byte payloads) of one scan's per-sensor clouds."""
    b = b"".join(np.ascontiguousarray(p).tobytes() for p in parts)
    return (np.frombuffer(b, np.uint8), [payload(p, T, 18) for p, T in zip(parts, Ts)], [payload(p, T, 32) for p, T in zip(parts, Ts)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=96)
    ap.add_argument("--pool", type=int, default=2, help="distinct ego poses per stream")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--u-steps", type=int, default=2)
    ap.add_argument("--single-steps", type=int, default=20)
    ap.add_argument("--prof-steps", type=int, default=3)
    ap.add_argument("--check", type=int, default=8, help="streams of the seeded sample checked after each variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    n_sensors = 4
    t0 = time.time()
    tasks = [(8000 + b, s, S) for b in range(B) for s in range(S)]
    procs = max(1, min(32, (os.cpu_count() or 2) - 1))
    if procs > 1:
        import multiprocessing as mp

        with mp.get_context("fork").Pool(procs) as pool:
            res = pool.map(_gen_task, tasks, chunksize=1)
    else:
        res = [_gen_task(t) for t in tasks]
    gen = [[res[b * S + s] for s in range(S)] for b in range(B)]
    del res

    import torch

    from groundgrid_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_merged_clouds.py needs a CUDA device")
    npart = np.array([[[len(p) for p in gen[b][s][0]] for s in range(S)] for b in range(B)], np.int64)   # [B][S][4]
    npts = npart.sum(axis=2)                                                                           # [B][S]
    assert npts.max() <= PCAP
    origins = [np.array([gen[b][s][1] for b in range(B)], np.float32) for s in range(S)]
    Tsensor = [[map_from_sensor(s, m) for m in synth.FOUR_LIDAR] for s in range(S)]   # the same mounts on every stream
    rng = np.random.default_rng(1234)
    sample = sorted(rng.choice(B, min(args.check, B), replace=False).tolist())

    # per pose one flat device buffer per layout: streams back to back, each stream's parts back to back; the host bytes
    # are kept for the sampled streams only (the twin's input)
    sizes = {0: 32 * npts, 18: 18 * npts, 32: 32 * npts}
    pools = {k: [torch.empty(int(v[:, s].sum()), dtype=torch.uint8, device="cuda") for s in range(S)] for k, v in sizes.items()}
    views = {k: [[] for _ in range(S)] for k in sizes}
    host = {k: {} for k in sizes}
    for s in range(S):
        at = {k: 0 for k in sizes}
        for b in range(B):
            fused_b, p18, p32 = scan_bytes(gen[b][s][0], Tsensor[s])
            gen[b][s] = None
            for k, raws in ((0, [fused_b]), (18, p18), (32, p32)):
                scan = []
                for raw in raws:
                    raw = raw.reshape(-1)
                    pools[k][s][at[k]:at[k] + raw.size] = torch.from_numpy(raw.copy())
                    scan.append(pools[k][s][at[k]:at[k] + raw.size])
                    at[k] += raw.size
                views[k][s].append(scan)
                if b in sample:
                    host[k][b, s] = raws
    del gen
    m18_pool, m32_pool = pools[18], pools[32]
    m18, m32 = views[18], views[32]
    build_s = time.time() - t0
    pts_per_pose = npts.sum(axis=0)
    clouds = [[v[0] for v in views[0][s]] for s in range(S)]
    dev = torch.device("cuda", 0)
    cur = torch.cuda.current_stream()

    g = capi.GroundGridB200(DIM_M, RES, n_slots=B, max_points=PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    slots = np.arange(B, dtype=np.int32)
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    descs = [g._device_descs(slots, npts[:, s], origins[s], 0.0) for s in range(S)]
    Tnest = [[Tsensor[s]] * B for s in range(S)]
    # the part records of each pose and layout, built once (the T arrays they point to are kept with them)
    recs = {step: [capi.cloud_parts([[v.numel() for v in scan] for scan in vw[s]], [[v.data_ptr() for v in scan] for scan in vw[s]],
                                    step, LAYOUT[step], Tnest[s]) for s in range(S)]
            for step, vw in ((18, m18), (32, m32))}
    pinned = torch.empty(max(p.numel() for p in m18_pool), dtype=torch.uint8).pin_memory()
    u_recs = []
    for s in range(S):
        offs = np.cumsum([0] + [v.numel() for b in range(B) for v in m18[s][b]])[:-1].reshape(B, n_sensors)
        u_recs.append(capi.cloud_parts([[v.numel() for v in m18[s][b]] for b in range(B)], (pinned.data_ptr() + offs).tolist(), 18, LAYOUT[18],
                                       Tnest[s]))
    part_counts = [torch.from_numpy(npart[:, s, :].reshape(-1)).cuda() for s in range(S)]
    T_dev = [torch.from_numpy(np.stack(Tsensor[s] * B).reshape(B * n_sensors, 12)).cuda() for s in range(S)]
    tstep = [0]
    last = {}

    def torch_records(s):
        """P: what a caller writes in torch -- ((T00 x + T01 y) + T02 z) + T03 in fp64 per part, one rounding per operation,
        cast to float32, packed into records; the parts of a scan are adjacent, so the packed buffer is their concatenation."""
        f = m32_pool[s].view(torch.float32).view(-1, 8)
        n = f.shape[0]
        part = torch.repeat_interleave(torch.arange(B * n_sensors, device="cuda"), part_counts[s], output_size=n)
        x, y, z = (f[:, c].double() for c in range(3))
        rec = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
        for r in range(3):
            T = T_dev[s][:, 4 * r:4 * r + 4][part]
            rec[:, r] = (((T[:, 0] * x + T[:, 1] * y) + T[:, 2] * z) + T[:, 3]).float()
        rec[:, 4] = f[:, 4]
        rec.view(torch.int32)[:, 5] = f.view(torch.int32)[:, 5] & 0xFFFF
        return list(torch.split(rec, npts[:, s].tolist()))

    def merged(h, step, s, sl=None):
        """gg_run_merged_cloud_msgs_to_device on the prebuilt part records, labels into new CUDA memory."""
        n_parts, parts, _ = recs[step][s]
        d = descs[s]
        if sl is not None:                          # one scan: slot sl alone
            first = int(n_parts[:sl].sum())
            n_parts, parts, d = n_parts[sl:sl + 1], parts[first:first + n_parts[sl]], h._device_descs([sl], [npts[sl, s]], origins[s][sl:sl + 1], 0.0)
        out, ptrs = h._device_outputs(torch, dev, cur, [int(x) for x in d["n_points"]], True, 0, False, [])
        h.run_merged_cloud_msgs_to_device_ptrs(d, n_parts, parts, ptrs, 0, None, cur.cuda_stream or None)
        return out

    def launch(variant, h, s):
        if variant == "B":
            return h.run_scans_to_device(clouds[s], slots, origins[s], 0.0, labels=True, select=None)
        if variant in ("M18", "M32"):
            return merged(h, int(variant[1:]), s)
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
        pinned[:m18_pool[s].numel()].copy_(m18_pool[s])
        torch.cuda.synchronize()
        t = time.perf_counter()
        s2 = next_pose()
        assert s2 == s
        n_parts, parts, _ = u_recs[s]
        for b in range(B):
            capi._check(g._l.gg_upload_cloud_msgs(g._h, b, n_sensors, capi._ptr(np.ascontiguousarray(parts[n_sensors * b:n_sensors * (b + 1)]))))
        capi._check(g._l.gg_run_scans(g._h, B, capi._ptr(descs[s]), 0))
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

    twin = capi.GroundGridB200(DIM_M, RES, n_slots=len(sample), max_points=PCAP, full_layers=False)
    tslots = np.arange(len(sample), dtype=np.int32)
    checks = {v: [] for v in VARIANTS}

    def check(variant):
        """One more step of `variant`; its sampled scans against the twin fed the same bytes through gg_upload_cloud_msgs."""
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
        keep = []
        for i, b in enumerate(sample):
            if variant == "B":
                parts = [(host[0][b, s][0], 32, LAYOUT[32], None)]
            else:
                step_b = 18 if variant in ("M18", "U") else 32
                parts = [(raw, step_b, LAYOUT[step_b], T) for raw, T in zip(host[step_b][b, s], Tsensor[s])]
            keep.append(twin.upload_cloud_msgs(parts, slot=i))
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

    # one scan alone: slot 0, strictly in sequence
    single = {}
    sl0 = np.array([0], np.int32)
    for variant in ("B", "M18"):
        def one(tt):
            s = bench.pingpong(tt, S)
            g.update_pose_batch(sl0, xy[s][:1], Ts[s][:1])
            if variant == "B":
                g.run_scans_to_device(clouds[s][:1], sl0, origins[s][:1], 0.0, labels=True, select=None)
            else:
                merged(g, 18, s, sl=0)

        for k in range(3):
            one(tstep[0] + k)
        g.synchronize()
        torch.cuda.synchronize()
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record(cur)
        for k in range(args.single_steps):
            one(tstep[0] + 3 + k)
        a1.record(cur)
        g.synchronize()
        torch.cuda.synchronize()
        single[variant] = a0.elapsed_time(a1) / args.single_steps
        tstep[0] += 3 + args.single_steps

    # serialised pass: one stream group, the unpack kernel's own time from gg_profile
    old = os.environ.get("GG_STREAMS")
    os.environ["GG_STREAMS"] = "1"
    g1 = capi.GroundGridB200(DIM_M, RES, n_slots=B, max_points=PCAP, full_layers=False)
    if old is None:
        del os.environ["GG_STREAMS"]
    else:
        os.environ["GG_STREAMS"] = old
    for b in range(B):
        g1.init_map(0.0, 0.0, 0.0, slot=b)
    unpack = {}
    for variant in ("M18", "M32"):
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
          f"{float(npts.mean()):.0f} points per scan in {n_sensors} parts; payloads built in {build_s:.0f} s")
    print(f"{'variant':<74} {'ms/step (runs)':<28} {'twin check':>10}")
    for v, desc in VARIANTS.items():
        ms = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<74} {' / '.join(f'{x:.2f}' for x in ms):<28} {'equal' if all(checks[v]) else 'DIFFERS':>10}")
    print(f"one scan alone (slot 0, in sequence): B {single['B']:.3f} ms, M18 {single['M18']:.3f} ms per scan")
    for v, u in unpack.items():
        print(f"k_unpack_transform {v} (serialised, {u['launches'] // args.prof_steps} launches per step): {u['ms_per_step']:.3f} ms/step, byte model "
              f"{u['model_gb_per_step']:.2f} GB -> {u['tb_per_s']:.2f} TB/s = {100 * u['share_of_datasheet']:.0f} % of the data sheet's "
              f"{DATASHEET_TBS} TB/s (not a measured peak)")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "u_steps": args.u_steps, "reps": args.reps,
                      "points_per_scan_mean": float(npts.mean()), "sample": sample, "twin_equal": checks, "results": results,
                      "single_scan_ms": single, "unpack": unpack}))
    twin.close()
    g.close()


if __name__ == "__main__":
    main()
