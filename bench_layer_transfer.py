"""Cost of taking the terrain out of (and putting it back into) many slots at once, on the device-resident workload of
bench.py's `value`.

    python bench_layer_transfer.py [--streams 396] [--pool 8] [--steps 40] [--warmup 3] [--reps 3] [--slow-steps 3]

Same scans as `value` (64-beam streams, clouds resident in HBM, rolls between steps), one step = one scan of every
stream through gg_run_scans_to_device (labels only), ordered on the caller's stream (torch's current stream) and timed
with CUDA events recorded on it.  Variants, alternated --reps times in one run:
  B   the scans alone (labels into caller memory)
  G2  B + gg_get_layers_to_device of "ground" and "groundpatch" of every slot
  G5  B + the same for the five live layers ("ground", "groundpatch", "points", "variance", "minGroundHeight")
  M   B + a migration round: "ground" and "groundpatch" of every slot exported and imported into a second handle
  X   the export of G2 alone, no scans (the copy by itself)
  L   B + gg_get_layer of "ground" and "groundpatch" per slot (today's way out; --slow-steps steps only)
After the timed steps of G2, G5 and M a seeded sample of slots is checked bit-exact against gg_get_layer (for M: the
second handle's layers against the first's).  Prints the card, its power limit, a table and one JSON line; writes
nothing.
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

TERRAIN = ("ground", "groundpatch")
LIVE5 = ("ground", "groundpatch", "points", "variance", "minGroundHeight")
VARIANTS = {
    "B": "to_device: labels",
    "G2": "B + export ground, groundpatch",
    "G5": "B + export five live layers",
    "M": "B + export + import ground, groundpatch (2nd handle)",
    "X": "export ground, groundpatch alone",
    "L": "B + layer() x 2 x slots (today)",
}
HBM_TBPS = 3.35   # data sheet peak of the H100 SXM5 80 GB, not measured


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--slow-steps", type=int, default=3, help="timed steps of variant L")
    ap.add_argument("--check", type=int, default=16, help="slots of the seeded sample checked after G2, G5 and M")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_layer_transfer.py needs a CUDA device")
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    offs = np.zeros((B, S), np.int64)
    o = 0
    for b in range(B):
        for s in range(S):
            offs[b, s] = o
            o += int(npts[b, s]) * 32
    pool = torch.empty(o, dtype=torch.uint8, device="cuda")
    for b in range(B):
        for s in range(S):
            raw = np.ascontiguousarray(streams[b][s][0]).view(np.uint8).reshape(-1)
            pool[int(offs[b, s]):int(offs[b, s]) + raw.size] = torch.from_numpy(raw)
    clouds = [[pool[int(offs[b, s]):int(offs[b, s]) + int(npts[b, s]) * 32] for b in range(B)] for s in range(S)]
    origins = [np.array([streams[b][s][1] for b in range(B)], np.float32) for s in range(S)]

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    g2 = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
        g2.init_map(0.0, 0.0, 0.0, slot=b)
    N = g.n
    slots = np.arange(B, dtype=np.int32)
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    cur = torch.cuda.current_stream()
    tstep = [0]
    last = {}

    def step(variant):
        if variant != "X":
            s = bench.pingpong(tstep[0], S)
            if tstep[0]:
                g.update_pose_batch(slots, xy[s], Ts[s])
            tstep[0] += 1
            g.run_scans_to_device(clouds[s], slots, origins[s], 0.0, labels=True, select=None)
        if variant in ("G2", "X", "M"):
            last["exp"] = g.get_layers_to_device(slots, TERRAIN)
        elif variant == "G5":
            last["exp"] = g.get_layers_to_device(slots, LIVE5)
        elif variant == "L":
            for b in range(B):
                for name in TERRAIN:
                    g.layer(name, slot=b)
        if variant == "M":
            g2.set_layers_from_device(slots, TERRAIN, last["exp"])

    def timed(variant):
        steps = args.slow_steps if variant == "L" else args.steps
        for _ in range(1 if variant == "L" else args.warmup):
            step(variant)
        g.synchronize()
        g2.synchronize()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
        ev[0].record(cur)
        for t in range(steps):
            step(variant)
            ev[t + 1].record(cur)
        g.synchronize()
        g2.synchronize()
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[-1])
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(steps)]
        return {"ms_per_step": total / steps, "ms_step_median": float(np.median(per)), "steps": steps}

    rng = np.random.default_rng(1234)
    sample = sorted(rng.choice(B, min(args.check, B), replace=False).tolist())
    checked = {}

    def check(variant):
        exp = last["exp"]
        torch.cuda.synchronize()
        names = LIVE5 if variant == "G5" else TERRAIN
        got = exp.cpu().numpy()
        for b in sample:
            for l, name in enumerate(names):
                want = g.layer(name, slot=b)
                assert np.array_equal(np.ascontiguousarray(got[b, l]).view(np.uint32), want.view(np.uint32)), f"{variant} slot {b}: {name}"
                if variant == "M" and l < 2:
                    assert np.array_equal(g2.layer(name, slot=b).view(np.uint32), want.view(np.uint32)), f"M slot {b}: imported {name}"
        checked[variant] = checked.get(variant, 0) + len(sample)

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            if v in ("G2", "G5", "M"):
                check(v)
    card = gpu_info()
    gb2 = 2 * B * len(TERRAIN) * N * N * 4 / 1e9
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, N = {N}, {args.steps} timed steps per run ({args.slow_steps} for L), {args.reps} alternating runs")
    print(f"byte model of one export of ground + groundpatch of every slot: {gb2:.3f} GB read + written, "
          f"{gb2 / HBM_TBPS:.3f} ms at the data sheet's {HBM_TBPS} TB/s (not measured)")
    print(f"{'variant':<62} {'ms/step (runs)':<28}")
    for v, desc in VARIANTS.items():
        ms = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<62} {' / '.join(f'{x:.3f}' for x in ms):<28}")
    x = float(np.median([r["ms_per_step"] for r in results["X"]]))
    print(f"X median {x:.3f} ms -> {gb2 / x:.2f} TB/s effective (byte model over the measured step)")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "N": N, "steps": args.steps, "slow_steps": args.slow_steps,
                      "reps": args.reps, "byte_model_gb_two_layers": gb2, "checked_slots": checked, "results": results}))
    g.close()
    g2.close()


if __name__ == "__main__":
    main()
