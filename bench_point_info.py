"""Cost of per-point classes and heights (gg_point_info_to_device) on the device-resident workload of bench.py's `value`.

    python bench_point_info.py [--streams 396] [--pool 8] [--steps 30] [--warmup 3] [--reps 3] [--slow-steps 3]

Same scans as `value` (64-beam streams, clouds resident in HBM, rolls between steps); one step = one scan of every
stream through gg_run_scans_to_device (labels only), ordered on the caller's stream (torch's current stream) and timed
with CUDA events recorded on it.  Variants, alternated --reps times in one run:
  B  the scans alone
  P  B, then gg_point_info_to_device of every slot (codes and heights)
  S  B, then the heights as they can be composed without it: "ground" sampled nearest at every point of each stream's
     cloud (gg_sample_layers_to_device) and a torch subtraction (map-frame clouds that are still alive only)
  L  B, then gg_get_point_classes per slot (one host wait each), --slow-steps steps only
After P, S and L a seeded sample of streams is checked bit-exact against the per-slot route (gg_get_point_classes,
gg_get_layer and numpy float32 on the cloud's z); S's heights at the points inside the map.  Then a serialised pass: one
stream group, gg_profile, ten rounds of P's call after one scan: the kernel time and the bandwidth on the byte model (per
point 4 B code + the 8 B zw word + a 4 B ground gather + 4 B per output written).  Prints the card, its power limit, a
table and one JSON line; writes nothing.
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
    "B": "to_device: labels",
    "P": "B + point_info_to_device (codes + height)",
    "S": "B + sample ground nearest at the cloud + torch subtraction",
    "L": "B + gg_get_point_classes per slot (host route)",
}
HBM_TBPS = 3.35   # data sheet peak of the H100 SXM5 80 GB, not measured
QNAN = np.uint32(0x7FC00000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--slow-steps", type=int, default=3, help="timed steps of variant L")
    ap.add_argument("--check", type=int, default=16, help="streams of the seeded sample checked after each variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_point_info.py needs a CUDA device")
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

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    N = g.n
    slots = np.arange(B, dtype=np.int32)
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    cur = torch.cuda.current_stream()
    tstep = [0]
    last = {}

    def step(variant):
        s = bench.pingpong(tstep[0], S)
        if tstep[0]:
            g.update_pose_batch(slots, xy[s], Ts[s])
        tstep[0] += 1
        g.run_scans_to_device(recs[s], slots, origins[s], 0.0, labels=True, select=None)
        last["s"] = s
        if variant == "P":
            last["out"] = g.point_info_to_device(slots)
        elif variant == "S":
            vals, cells = g.sample_layers_to_device(slots, recs[s], ("ground",), cells=True)
            last["out"] = ([r[:, 2] - v[0] for r, v in zip(recs[s], vals)], cells)
        elif variant == "L":
            last["out"] = [g.point_classes(int(npts[b, s]), slot=b) for b in range(B)]

    def timed(variant):
        steps = args.slow_steps if variant == "L" else args.steps
        for _ in range(1 if variant == "L" else args.warmup):
            step(variant)
        g.synchronize()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
        ev[0].record(cur)
        for t in range(steps):
            step(variant)
            ev[t + 1].record(cur)
        g.synchronize()
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[-1])
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(steps)]
        return {"ms_per_step": total / steps, "ms_step_median": float(np.median(per)), "steps": steps}

    rng = np.random.default_rng(1234)
    sample = sorted(rng.choice(B, min(args.check, B), replace=False).tolist())
    checked = {}

    def per_slot(b, s):
        """(codes, height bits) through the per-slot route."""
        n = int(npts[b, s])
        codes = g.point_classes(n, slot=b)
        G = g.layer("ground", slot=b).reshape(-1, order="F")
        z = np.ascontiguousarray(streams[b][s][0]["z"], np.float32)
        cls, cell = codes >> 24, (codes & 0xFFFFFF).astype(np.int64)
        h = np.full(n, QNAN, np.uint32)
        h[cls != 0] = (z[cls != 0] - G[cell[cls != 0]]).astype(np.float32).view(np.uint32)
        return codes, h

    def check(variant):
        torch.cuda.synchronize()
        g.synchronize()
        s = last["s"]
        for b in sample:
            codes, h = per_slot(b, s)
            if variant == "P":
                got_c, got_h = last["out"][0][b].cpu().numpy().view(np.uint32), last["out"][1][b].cpu().numpy().view(np.uint32)
                assert np.array_equal(got_c, codes) and np.array_equal(got_h, h), f"P stream {b}: differs from the per-slot route"
            elif variant == "S":
                inside = last["out"][1][b].cpu().numpy() >= 0
                got = last["out"][0][b].cpu().numpy().view(np.uint32)
                assert np.array_equal(got[inside], h[inside]), f"S stream {b}: differs from the per-slot route"
            else:
                assert np.array_equal(last["out"][b], codes), f"L stream {b}"
        checked[variant] = checked.get(variant, 0) + len(sample)

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            if v != "B":
                check(v)

    # serialised pass: one stream group, one scan, then ten rounds of P's call, timed per kernel
    os.environ["GG_STREAMS"] = "1"
    gs = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        gs.init_map(0.0, 0.0, 0.0, slot=b)
    gs.run_scans_to_device(recs[0], slots, origins[0], 0.0, labels=True, select=None)
    gs.point_info_to_device(slots)
    torch.cuda.synchronize()
    gs.profile_enable(True)
    gs.profile_read(reset=True)
    rounds = 10
    for _ in range(rounds):
        gs.point_info_to_device(slots)
    prof = gs.profile_read(reset=True)
    gs.profile_enable(False)
    ms, launches = prof["k_point_info"]
    bytes_model = rounds * n_points[0] * (4 + 8 + 4 + 2 * 4)
    tbps = bytes_model / (ms * 1e-3) / 1e12
    gs.close()

    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, N = {N}, {args.steps} timed steps per run ({args.slow_steps} for L), {args.reps} alternating runs, "
          f"{np.mean(n_points) / 1e6:.1f} M points per step")
    print(f"{'variant':<62} {'ms/step (runs)':<28}")
    for v, desc in VARIANTS.items():
        msv = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<62} {' / '.join(f'{x:.3f}' for x in msv):<28}")
    print(f"serialised pass (one stream group, {rounds} rounds, {launches} launches): k_point_info {ms:.3f} ms, byte model "
          f"{bytes_model / 1e9:.3f} GB -> {tbps:.2f} TB/s = {100 * tbps / HBM_TBPS:.0f} % of the data sheet's {HBM_TBPS} TB/s "
          "(the card's HBM bandwidth was not measured)")
    print(f"bit-exact checks: {checked}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "N": N, "steps": args.steps, "slow_steps": args.slow_steps, "reps": args.reps,
                      "points_per_step": float(np.mean(n_points)), "serialised": {"ms": ms, "launches": launches, "bytes": bytes_model,
                                                                                  "tbps": tbps}, "checked_streams": checked,
                      "results": results}))
    g.close()


if __name__ == "__main__":
    main()
