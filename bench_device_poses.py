"""Cost of the host pose round trip against poses resolved on the device (gg_update_poses_from_device), on the
device-resident workload of bench.py's `value`.

    python bench_device_poses.py [--streams 396] [--pool 8] [--steps 30] [--warmup 3] [--reps 3] [--latency-steps 60]

Same scans as `value` (64-beam streams, clouds resident in HBM, rolls between steps, labels only); one step = one roll
and one scan of every stream, ordered on the caller's stream (torch's current stream) and timed with CUDA events
recorded on it.  Variants, alternated --reps times in one run:
  B  host poses: gg_update_pose_batch + gg_run_scans_to_device with host origins
  D  the poses in device tensors: gg_update_poses_from_device + scans flagged GG_SCAN_DEVICE_POSE
  H  the poses produced on the device every step by a small torch op, then .cpu() and B's calls: the route a caller
     with GPU-produced poses has without D
After each variant a seeded sample of streams is checked bit-exact (labels of the last step, "ground" and
"groundpatch", the map position) against a twin handle that replays the same steps with host poses.  Then the
single-stream latency of B and D (one slot, median of --latency-steps steps, alternated), and a serialised pass (one
stream group, gg_profile) that gives the time of k_pose_resolve and k_stage_poses.  Prints the card, its power limit,
a table and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generators and the pose sequence of bench.py)
from bench_slot_config import gpu_info  # noqa: E402

VARIANTS = {
    "B": "host poses: update_pose_batch + scans",
    "D": "device poses: update_poses_from_device + flagged scans",
    "H": "device-produced poses -> .cpu() -> B",
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--latency-steps", type=int, default=60)
    ap.add_argument("--check", type=int, default=16, help="streams of the seeded sample checked after each variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_device_poses.py needs a CUDA device")
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    offs = np.zeros((B, S), np.int64)
    o = 0
    for b in range(B):
        for s in range(S):
            offs[b, s] = o
            o += int(npts[b, s]) * 8
    pool = torch.empty(o, dtype=torch.float32, device="cuda")
    for b in range(B):
        for s in range(S):
            raw = np.ascontiguousarray(streams[b][s][0]).view(np.float32).reshape(-1)
            pool[int(offs[b, s]):int(offs[b, s]) + raw.size] = torch.from_numpy(raw)
    recs = [[pool[int(offs[b, s]):int(offs[b, s]) + int(npts[b, s]) * 8].view(-1, 8) for b in range(B)] for s in range(S)]
    origins = [np.array([streams[b][s][1] for b in range(B)], np.float32) for s in range(S)]
    n_points = [int(npts[:, s].sum()) for s in range(S)]
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    base_z = np.zeros(B, np.float64)
    dxy = [torch.tensor(v, device="cuda") for v in xy]
    dT = [torch.tensor(v, device="cuda") for v in Ts]
    dorg = [torch.tensor(v, device="cuda") for v in origins]
    dbz = torch.tensor(base_z, device="cuda")

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    N = g.n
    slots = np.arange(B, dtype=np.int32)
    cur = torch.cuda.current_stream()
    tstep = [0]
    history = []   # the pose index of every step g ran
    last = {}

    def step(variant):
        s = bench.pingpong(tstep[0], S)
        first = tstep[0] == 0
        tstep[0] += 1
        history.append(s)
        if variant == "D":
            g.update_poses_from_device(slots, None if first else dxy[s], None if first else dT[s], dorg[s], dbz)
            last["out"] = g.run_scans_to_device(recs[s], slots, "device", None, labels=True, select=None)
            return
        if variant == "H":   # the poses exist on the device only: produced by a torch op, then copied to the host
            pxy, pT, porg = (t * 1.0 for t in (dxy[s], dT[s], dorg[s]))
            hxy, hT, horg = pxy.cpu().numpy(), pT.cpu().numpy(), porg.cpu().numpy()
        else:
            hxy, hT, horg = xy[s], Ts[s], origins[s]
        if not first:
            g.update_pose_batch(slots, hxy, hT)
        last["out"] = g.run_scans_to_device(recs[s], slots, horg, 0.0, labels=True, select=None)

    def timed(variant):
        for _ in range(args.warmup):
            step(variant)
        g.synchronize()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        ev[0].record(cur)
        for t in range(args.steps):
            step(variant)
            ev[t + 1].record(cur)
        g.synchronize()
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[-1])
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.steps)]
        return {"ms_per_step": total / args.steps, "ms_step_median": float(np.median(per)), "steps": args.steps}

    # the twin replays the steps of the sampled streams with host poses
    rng = np.random.default_rng(1234)
    sample = np.array(sorted(rng.choice(B, min(args.check, B), replace=False).tolist()), np.int32)
    m = len(sample)
    twin = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=m, max_points=bench.PCAP, full_layers=False)
    tslots = np.arange(m, dtype=np.int32)
    for j in range(m):
        twin.init_map(0.0, 0.0, 0.0, slot=j)
    replayed = [0]
    checked = {}

    def check(variant):
        torch.cuda.synchronize()
        g.synchronize()
        out = None
        for t in range(replayed[0], len(history)):
            s = history[t]
            if t:
                twin.update_pose_batch(tslots, xy[s][sample], Ts[s][sample])
            out = twin.run_scans_to_device([recs[s][b] for b in sample], tslots, origins[s][sample], 0.0, labels=True, select=None)
        replayed[0] = len(history)
        torch.cuda.synchronize()
        for j, b in enumerate(sample):
            assert torch.equal(last["out"].labels[b], out.labels[j]), f"{variant} stream {b}: labels differ from the host-driven twin"
            for name in ("ground", "groundpatch"):
                assert np.array_equal(g.layer(name, slot=int(b)).view(np.uint32), twin.layer(name, slot=j).view(np.uint32)), f"{variant} stream {b}: {name}"
            assert g.position(slot=int(b)).tolist() == twin.position(slot=j).tolist(), f"{variant} stream {b}: position"
        checked[variant] = checked.get(variant, 0) + m

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            check(v)

    # single-stream latency: one slot, one roll and one scan per step, B and D alternated
    g1 = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=1, max_points=bench.PCAP, full_layers=False)
    g1.init_map(0.0, 0.0, 0.0)
    one = np.zeros(1, np.int32)
    lat = {"B": [], "D": []}
    t1 = 0
    for rep in range(2 * args.reps):
        v = "BD"[rep % 2]
        per = []
        for t in range(args.latency_steps + args.warmup):
            s = bench.pingpong(t1, S)
            t1 += 1
            a, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(cur)
            if v == "D":
                g1.update_poses_from_device(one, dxy[s][:1], dT[s][:1], dorg[s][:1], dbz[:1])
                g1.run_scans_to_device(recs[s][:1], one, "device", None, labels=True, select=None)
            else:
                g1.update_pose_batch(one, xy[s][:1], Ts[s][:1])
                g1.run_scans_to_device(recs[s][:1], one, origins[s][:1], 0.0, labels=True, select=None)
            b_.record(cur)
            b_.synchronize()
            if t >= args.warmup:
                per.append(a.elapsed_time(b_))
        lat[v].append(float(np.median(per)))
    g1.close()

    # serialised pass: one stream group, rolls from device poses and flagged scans, timed per kernel
    os.environ["GG_STREAMS"] = "1"
    gs = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        gs.init_map(0.0, 0.0, 0.0, slot=b)
    gs.update_poses_from_device(slots, dxy[1], dT[1], dorg[1], dbz)
    gs.run_scans_to_device(recs[1], slots, "device", None, labels=True, select=None)
    torch.cuda.synchronize()
    gs.profile_enable(True)
    gs.profile_read(reset=True)
    rounds = 10
    for r in range(rounds):
        s = bench.pingpong(r + 2, S)
        gs.update_poses_from_device(slots, dxy[s], dT[s], dorg[s], dbz)
        gs.run_scans_to_device(recs[s], slots, "device", None, labels=True, select=None)
    prof = gs.profile_read(reset=True)
    gs.profile_enable(False)
    gs.close()
    kern = {k: prof[k] for k in ("k_pose_resolve", "k_stage_poses", "k_roll_gather", "k_roll_commit", "k_rasterize") if k in prof}

    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, N = {N}, {args.steps} timed steps per run, {args.reps} alternating runs, "
          f"{np.mean(n_points) / 1e6:.1f} M points per step")
    print(f"{'variant':<62} {'ms/step (runs)':<28}")
    for v, desc in VARIANTS.items():
        msv = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<62} {' / '.join(f'{x:.3f}' for x in msv):<28}")
    print(f"single-stream latency, median ms per step (runs): B {' / '.join(f'{x:.3f}' for x in lat['B'])}, "
          f"D {' / '.join(f'{x:.3f}' for x in lat['D'])}")
    print("serialised pass (one stream group, %d rounds): " % rounds +
          ", ".join(f"{k} {ms:.3f} ms / {n} launches" for k, (ms, n) in kern.items()))
    print(f"bit-exact checks: {checked}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "N": N, "steps": args.steps, "reps": args.reps,
                      "points_per_step": float(np.mean(n_points)), "single_stream_ms": lat, "serialised": kern,
                      "checked_streams": checked, "results": results}))
    g.close()
    twin.close()


if __name__ == "__main__":
    main()
