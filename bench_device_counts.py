"""Cost of the host point-count round trip against counts read on the device (gg_set_point_counts_from_device +
GG_SCAN_DEVICE_COUNT), on the device-resident workload of bench.py's `value`.

    python bench_device_counts.py [--streams 396] [--pool 8] [--steps 30] [--warmup 3] [--reps 3] [--gate 30]

Same scans as `value` (64-beam streams, clouds resident in HBM, rolls between steps, labels to device); one step = one
roll and one scan of every stream, ordered on the caller's stream (torch's current stream) and timed with CUDA events
recorded on it.  Variants, alternated --reps times in one run:
  B   host counts: gg_run_scans_to_device with each cloud's length
  D   the same counts from a device tensor, capacity = the count (the grids of B)
  D'  the same counts from a device tensor, capacity = max_points (oversized grids)
  G   every step a sync-free torch range gate (horizontal range < --gate m from the stream's origin: mask -> cumsum ->
      scatter) compacts each cloud and leaves its count on the device, then D's calls with capacity = the cloud's length
  H   G's gate, then .cpu() of the counts and B's calls on the compacted clouds: what such a caller does without D
After each variant a seeded sample of streams is checked bit-exact (labels of the last step, "ground", "groundpatch",
the map position) against a twin handle that replays the same steps with host counts.  Prints the card, its power
limit, a table and one JSON line; writes nothing.
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
    "B": "host counts",
    "D": "device counts, capacity = count",
    "D'": "device counts, capacity = max_points",
    "G": "torch range gate, counts stay on the device",
    "H": "torch range gate -> .cpu() of the counts -> B",
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gate", type=float, default=30.0, help="range of the gate of G and H, metres")
    ap.add_argument("--check", type=int, default=16, help="streams of the seeded sample checked after each variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_device_counts.py needs a CUDA device")
    P = bench.PCAP
    npts = np.array([[len(streams[b][s][0]) for b in range(B)] for s in range(S)], np.int64)   # [pose][stream]
    # per pose, the clouds of all streams back to back (the gate works on them at once), and max_points records of
    # slack at the end, so that every stream has a max_points view for D'
    offs = [np.concatenate([[0], np.cumsum(npts[s])[:-1]]) for s in range(S)]
    flat = []
    for s in range(S):
        t = torch.zeros((int(npts[s].sum()) + P + 1, 8), dtype=torch.float32, device="cuda")
        t[:int(npts[s].sum())] = torch.from_numpy(np.concatenate([np.ascontiguousarray(streams[b][s][0]).view(np.float32).reshape(-1, 8)
                                                                  for b in range(B)]))
        flat.append(t)
    recs = [[flat[s][int(offs[s][b]):int(offs[s][b] + npts[s][b])] for b in range(B)] for s in range(S)]
    wide = [[flat[s][int(offs[s][b]):int(offs[s][b]) + P] for b in range(B)] for s in range(S)]
    origins = [np.array([streams[b][s][1] for b in range(B)], np.float32) for s in range(S)]
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    dcount = [torch.tensor(npts[s].astype(np.int32), device="cuda") for s in range(S)]
    # the gate's per-point stream ids, stream starts and origins
    seg = [torch.repeat_interleave(torch.arange(B, device="cuda"), torch.tensor(npts[s], device="cuda")) for s in range(S)]
    dstart = [torch.tensor(offs[s], dtype=torch.int64, device="cuda") for s in range(S)]
    dorg = [torch.tensor(origins[s][:, :2], device="cuda") for s in range(S)]
    gated = torch.empty((max(int(npts[s].sum()) for s in range(S)) + 1, 8), dtype=torch.float32, device="cuda")

    def gate(s):
        """Points of pose s within --gate m (horizontal) of their stream's origin, compacted per stream in input order
        into `gated` (stream b from offs[s][b] on); returns the int32 counts, on the device, without a host wait."""
        n = int(npts[s].sum())
        src = flat[s][:n]
        d = src[:, :2] - dorg[s][seg[s]]
        keep = (d * d).sum(1) < args.gate * args.gate
        k64 = keep.to(torch.int64)
        before = torch.cumsum(k64, 0) - k64                    # kept points before each point
        rank = before - before[dstart[s]][seg[s]]              # ... within its stream
        dst = torch.where(keep, dstart[s][seg[s]] + rank, torch.full_like(rank, n))   # dropped points go to row n
        gated.index_copy_(0, dst, src)
        return torch.zeros(B, dtype=torch.int32, device="cuda").index_add_(0, seg[s], keep.to(torch.int32))

    def gated_views(s, lengths):
        return [gated[int(offs[s][b]):int(offs[s][b]) + int(lengths[b])] for b in range(B)]

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=P, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    N = g.n
    slots = np.arange(B, dtype=np.int32)
    cur = torch.cuda.current_stream()
    tstep = [0]
    history = []   # (pose, gated) of every step g ran
    last = {}

    def step(variant):
        s = bench.pingpong(tstep[0], S)
        if tstep[0]:
            g.update_pose_batch(slots, xy[s], Ts[s])
        tstep[0] += 1
        history.append((s, variant in ("G", "H")))
        if variant == "B":
            last["out"] = g.run_scans_to_device(recs[s], slots, origins[s], 0.0, labels=True, select=None)
        elif variant in ("D", "D'"):
            g.set_point_counts_from_device(slots, dcount[s])
            last["out"] = g.run_scans_to_device(recs[s] if variant == "D" else wide[s], slots, origins[s], 0.0, labels=True, select=None,
                                                device_counts=True)
        elif variant == "G":
            g.set_point_counts_from_device(slots, gate(s))
            last["out"] = g.run_scans_to_device(gated_views(s, npts[s]), slots, origins[s], 0.0, labels=True, select=None, device_counts=True)
        else:
            u = gate(s).cpu().numpy()
            last["out"] = g.run_scans_to_device(gated_views(s, u), slots, origins[s], 0.0, labels=True, select=None)

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

    # the twin replays the steps of the sampled streams with host counts on the same clouds
    rng = np.random.default_rng(1234)
    sample = np.array(sorted(rng.choice(B, min(args.check, B), replace=False).tolist()), np.int32)
    m = len(sample)
    twin = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=m, max_points=P, full_layers=False)
    tslots = np.arange(m, dtype=np.int32)
    for j in range(m):
        twin.init_map(0.0, 0.0, 0.0, slot=j)
    replayed = [0]
    checked = {}
    gate_kept = []

    def check(variant):
        torch.cuda.synchronize()
        g.synchronize()
        out, u = None, None
        for t in range(replayed[0], len(history)):
            s, gated_step = history[t]
            if t:
                twin.update_pose_batch(tslots, xy[s][sample], Ts[s][sample])
            if gated_step:
                u = gate(s).cpu().numpy()
                clouds = [v for j, v in enumerate(gated_views(s, u)) if j in set(sample.tolist())]
                u = u[sample]
            else:
                u = npts[s][sample]
                clouds = [recs[s][b] for b in sample]
            out = twin.run_scans_to_device(clouds, tslots, origins[s][sample], 0.0, labels=True, select=None)
            torch.cuda.synchronize()
        replayed[0] = len(history)
        if history[-1][1]:
            gate_kept.append(float(u.sum()) / float(npts[history[-1][0]][sample].sum()))
        for j, b in enumerate(sample):
            assert torch.equal(last["out"].labels[b][:int(u[j])], out.labels[j]), f"{variant} stream {b}: labels differ from the host-count twin"
            for name in ("ground", "groundpatch"):
                assert np.array_equal(g.layer(name, slot=int(b)).view(np.uint32), twin.layer(name, slot=j).view(np.uint32)), f"{variant} stream {b}: {name}"
            assert g.position(slot=int(b)).tolist() == twin.position(slot=j).tolist(), f"{variant} stream {b}: position"
            assert g.last_scan_points(slot=int(b)) == int(u[j]), f"{variant} stream {b}: last_scan_points"
        checked[variant] = checked.get(variant, 0) + m

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            check(v)

    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, N = {N}, {args.steps} timed steps per run, {args.reps} alternating runs, "
          f"{npts.sum(1).mean() / 1e6:.2f} M points per step before the gate, gate keeps {np.mean(gate_kept):.3f} of the sample's points")
    print(f"{'variant':<54} {'ms/step (runs)':<28}")
    for v, desc in VARIANTS.items():
        msv = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<54} {' / '.join(f'{x:.3f}' for x in msv):<28}")
    print(f"bit-exact checks (streams): {checked}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "N": N, "steps": args.steps, "reps": args.reps, "gate_m": args.gate,
                      "points_per_step": float(npts.sum(1).mean()), "gate_kept": float(np.mean(gate_kept)), "checked_streams": checked,
                      "results": results}))
    g.close()
    twin.close()


if __name__ == "__main__":
    main()
