"""Cost of terrain lookups at arbitrary positions (gg_sample_layers_to_device) on the device-resident workload of
bench.py's `value`.

    python bench_sample_layers.py [--streams 396] [--pool 8] [--steps 30] [--warmup 3] [--reps 3] [--slow-steps 3]

Same scans as `value` (64-beam streams, clouds resident in HBM, rolls between steps); one step = one scan of every
stream through gg_run_scans_to_device (labels only), ordered on the caller's stream (torch's current stream) and timed
with CUDA events recorded on it.  Variants, alternated --reps times in one run:
  B   the scans alone
  SN  B, then "ground" and "groundpatch" sampled nearest at every point of each stream's NEXT cloud (32-byte records)
  SL  the same, linear
  G   B, then a 64 x 64 float2 grid of positions per slot within +-20 m of the ego (small sets: the per-call overhead)
  Q   the torch route for SN: gg_get_layers_to_device of the two planes, the index arithmetic in torch float64
      (truncation toward zero, the inside test), then a gather
  L   the per-slot host route: gg_get_layer + numpy (tests/sample_ref.py), --slow-steps steps only
After each variant with outputs a seeded sample of streams is checked bit-exact against tests/sample_ref.py on
gg_get_layer planes and gg_get_map_position, and Q's values against SN's.  Then a serialised pass: one stream group,
gg_profile, ten rounds of SN's lookups without scans: the kernel time and the bandwidth on the byte model (per query
the 32-byte sector holding x, y and 4 bytes per name written; per slot and name 4 N^2 bytes read).  Prints the card,
its power limit, a table and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (workload generators and the pose sequence of bench.py)
import sample_ref  # noqa: E402  (the CPU restatement of the lookup rules)
from bench_slot_config import gpu_info  # noqa: E402

TERRAIN = ("ground", "groundpatch")
VARIANTS = {
    "B": "to_device: labels",
    "SN": "B + sample nearest at the next cloud",
    "SL": "B + sample linear at the next cloud",
    "G": "B + sample nearest on a 64 x 64 grid per slot",
    "Q": "B + export + torch index arithmetic + gather",
    "L": "B + layer() x 2 + numpy per slot (host route)",
}
HBM_TBPS = 3.35   # data sheet peak of the H100 SXM5 80 GB, not measured


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
        raise SystemExit("bench_sample_layers.py needs a CUDA device")
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
    # the torch route's inputs: per pose every stream's cloud back to back, and the slot of each point
    cat = [torch.cat(recs[s]) for s in range(S)]
    slot_of = [torch.repeat_interleave(torch.arange(B, device="cuda"), torch.from_numpy(npts[:, s]).cuda()) for s in range(S)]
    n_queries = [int(npts[:, s].sum()) for s in range(S)]

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    N = g.n
    res, length, half = sample_ref.geometry(N, bench.RES)
    slots = np.arange(B, dtype=np.int32)
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    lin = torch.linspace(-20.0, 20.0, 64, dtype=torch.float64, device="cuda")
    grid = [torch.stack(torch.meshgrid(lin + s, lin, indexing="ij"), -1).reshape(-1, 2).float().contiguous() for s in range(S)]
    cur = torch.cuda.current_stream()
    tstep = [0]
    last = {}

    def torch_route(s_next, s):
        exp = g.get_layers_to_device(slots, TERRAIN)                     # [B, 2, N, N], column-major planes
        flat = exp.transpose(-1, -2).reshape(B, 2, N * N)
        pos = torch.from_numpy(np.array([g.position(b) for b in range(B)])).cuda()   # host values: no device wait
        sl = slot_of[s_next]
        x, y = cat[s_next][:, 0].double(), cat[s_next][:, 1].double()
        px, py = pos[sl, 0], pos[sl, 1]
        r = torch.full_like(x, res)   # a tensor divisor: torch divides by a scalar as a multiply by its reciprocal
        i = -torch.trunc(((x - half) - px) / r)
        j = -torch.trunc(((y - half) - py) / r)
        tx, ty = -((x - px) - half), -((y - py) - half)
        inside = (tx >= 0) & (ty >= 0) & (tx < length) & (ty < length) & (i >= 0) & (j >= 0) & (i < N) & (j < N)
        cell = torch.where(inside, i + j * N, torch.zeros_like(i)).long()
        v = flat[sl, :, cell]                                               # [n, 2]
        return torch.where(inside[:, None], v, torch.full_like(v, float("nan")))

    def step(variant):
        s = bench.pingpong(tstep[0], S)
        s_next = bench.pingpong(tstep[0] + 1, S)
        if tstep[0]:
            g.update_pose_batch(slots, xy[s], Ts[s])
        tstep[0] += 1
        g.run_scans_to_device(recs[s], slots, origins[s], 0.0, labels=True, select=None)
        last["s_next"], last["s"] = s_next, s
        if variant in ("SN", "SL"):
            last["out"] = g.sample_layers_to_device(slots, recs[s_next], TERRAIN, mode="nearest" if variant == "SN" else "linear")
        elif variant == "G":
            last["out"] = g.sample_layers_to_device(slots, [grid[s]] * B, TERRAIN)
        elif variant == "Q":
            last["out"] = torch_route(s_next, s)
        elif variant == "L":
            for b in range(B):
                planes = [g.layer(name, slot=b) for name in TERRAIN]
                px, py = g.position(b)
                r = recs[s_next][b].cpu().numpy()
                sample_ref.sample_layers(planes, N, bench.RES, px, py, r[:, 0], r[:, 1], "nearest")

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

    def check(variant):
        torch.cuda.synchronize()
        g.synchronize()
        s_next = last["s_next"]
        if variant == "Q":
            # Q against SN: the same lookups through the kernel
            sn = g.sample_layers_to_device(slots, recs[s_next], TERRAIN)
            torch.cuda.synchronize()
            q = last["out"].cpu().numpy()
            starts = np.concatenate([[0], np.cumsum(npts[:, s_next])])
            for b in sample:
                want = sn[b].cpu().numpy().T
                assert np.array_equal(q[starts[b]:starts[b + 1]].view(np.uint32), want.view(np.uint32)), f"Q stream {b}: differs from SN"
        else:
            mode = "linear" if variant == "SL" else "nearest"
            for b in sample:
                planes = [g.layer(name, slot=b) for name in TERRAIN]
                px, py = g.position(b)
                r = (grid[last["s"]] if variant == "G" else recs[s_next][b]).cpu().numpy()
                want, _ = sample_ref.sample_layers(planes, N, bench.RES, px, py, r[:, 0], r[:, 1], mode)
                got = last["out"][b].cpu().numpy()
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{variant} stream {b}: differs from the restatement"
        checked[variant] = checked.get(variant, 0) + len(sample)

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            if v in ("SN", "SL", "G", "Q"):
                check(v)

    # serialised pass: one stream group, no scans, ten rounds of SN's lookups on the prior, timed per kernel
    os.environ["GG_STREAMS"] = "1"
    gs = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        gs.init_map(0.0, 0.0, 0.0, slot=b)
    gs.sample_layers_to_device(slots, recs[1], TERRAIN)
    torch.cuda.synchronize()
    gs.profile_enable(True)
    gs.profile_read(reset=True)
    rounds = 10
    for r in range(rounds):
        gs.sample_layers_to_device(slots, recs[r % S], TERRAIN)
    prof = gs.profile_read(reset=True)
    gs.profile_enable(False)
    ms, launches = prof["k_sample_layers"]
    q_total = sum(n_queries[r % S] for r in range(rounds))
    bytes_model = q_total * (32 + 4 * len(TERRAIN)) + rounds * B * len(TERRAIN) * 4 * N * N
    tbps = bytes_model / (ms * 1e-3) / 1e12
    gs.close()

    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, N = {N}, {args.steps} timed steps per run ({args.slow_steps} for L), {args.reps} alternating runs, "
          f"{np.mean(n_queries) / 1e6:.1f} M queries per SN / SL step")
    print(f"{'variant':<62} {'ms/step (runs)':<28}")
    for v, desc in VARIANTS.items():
        msv = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<62} {' / '.join(f'{x:.3f}' for x in msv):<28}")
    print(f"serialised pass (one stream group, {rounds} rounds, {launches} launches): k_sample_layers {ms:.3f} ms, byte model "
          f"{bytes_model / 1e9:.3f} GB -> {tbps:.2f} TB/s = {100 * tbps / HBM_TBPS:.0f} % of the data sheet's {HBM_TBPS} TB/s "
          "(the card's HBM bandwidth was not measured)")
    print(f"bit-exact checks: {checked}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "N": N, "steps": args.steps, "slow_steps": args.slow_steps, "reps": args.reps,
                      "queries_per_step": float(np.mean(n_queries)), "serialised": {"ms": ms, "launches": launches, "bytes": bytes_model,
                                                                                     "tbps": tbps}, "checked_streams": checked,
                      "results": results}))
    g.close()


if __name__ == "__main__":
    main()
