"""Cost of taking the results out of the handle, on the device-resident workload of bench.py's `value`.

    python bench_device_outputs.py [--streams 396] [--pool 8] [--steps 40] [--warmup 3] [--reps 3]

Same scans as `value` (64-beam streams, clouds resident in HBM, rolls between steps), one step = one scan of every
stream.  Every step is ordered on the caller's stream (torch's current stream) and timed with CUDA events recorded on
it.  Variants, alternated --reps times in one run:
  A  gg_run_scans_device; the caller's stream forks to / joins from the handle's streams around each step
     (results stay inside the handle)
  B  gg_run_scans_to_device, labels only
  C  gg_run_scans_to_device, labels + non-ground cloud (the obstacle points)
  D  gg_run_scans_to_device, labels + whole output cloud + index
  E  A, then gg_download_labels of every slot into pinned host memory and a host synchronise (today's way out)
plus A0, bench.py's own timing of `value` (one fork before and one join after all steps; steps are not ordered on
the caller's stream).  After the timed steps of B, C and D a seeded sample of scans is checked bit-exact against
gg_download_labels / gg_get_output.  Prints the card, its power limit, a table and one JSON line; writes nothing.
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
    "A0": "run_scans_device, fork/join once around all steps (bench.py value)",
    "A": "run_scans_device, fork/join per step",
    "B": "to_device: labels",
    "C": "to_device: labels + non-ground cloud",
    "D": "to_device: labels + whole cloud + index",
    "E": "run_scans_device + download_labels x slots + sync",
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=16, help="scans of the seeded sample checked after B, C and D")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_device_outputs.py needs a CUDA device")
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
    pts_per_pose = npts.sum(axis=0)

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    slots = np.arange(B, dtype=np.int32)
    descs = [g.make_descs(list(range(B)), [int(npts[b, s]) for b in range(B)], list(origins[s]), [0.0] * B) for s in range(S)]
    ptrs = [[c.data_ptr() for c in clouds[s]] for s in range(S)]
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    host_labels = torch.zeros((B, bench.PCAP), dtype=torch.uint8).pin_memory()
    lab_ptrs = [host_labels.data_ptr() + b * bench.PCAP for b in range(B)]
    cur = torch.cuda.current_stream()
    ext = torch.cuda.ExternalStream(g.stream)
    tstep = [0]
    last = {}

    def step(variant):
        s = bench.pingpong(tstep[0], S)
        if tstep[0]:
            g.update_pose_batch(slots, xy[s], Ts[s])
        tstep[0] += 1
        if variant in ("A", "E"):
            ext.wait_stream(cur)
            g.fork_streams()
            g.run_scans_device(descs[s], ptrs[s])
            if variant == "E":
                for b in range(B):
                    g.download_labels_ptr(lab_ptrs[b], int(npts[b, s]), slot=b)
            g.join_streams()
            cur.wait_stream(ext)
            if variant == "E":
                g.synchronize()
        elif variant == "A0":
            g.run_scans_device(descs[s], ptrs[s])
        else:
            sel, idx = {"B": (None, False), "C": ("nonground", False), "D": ("all", True)}[variant]
            last["out"] = g.run_scans_to_device(clouds[s], slots, origins[s], 0.0, labels=True, select=sel, index=idx)
        last["pose"] = s
        return int(pts_per_pose[s])

    def timed(variant):
        for _ in range(args.warmup):
            step(variant)
        g.synchronize()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        pts = 0
        if variant == "A0":
            ev[0].record(ext)
            g.fork_streams()
            for _ in range(args.steps):
                pts += step(variant)
            g.join_streams()
            ev[-1].record(ext)
        else:
            ev[0].record(cur)
            for t in range(args.steps):
                pts += step(variant)
                ev[t + 1].record(cur)
        g.synchronize()
        torch.cuda.synchronize()
        total = ev[0].elapsed_time(ev[-1])
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.steps)] if variant != "A0" else [total / args.steps]
        return {"ms_per_step": total / args.steps, "ms_step_median": float(np.median(per)), "mpoints_per_s": pts / (total * 1e-3) / 1e6}

    rng = np.random.default_rng(1234)
    sample = sorted(rng.choice(B, min(args.check, B), replace=False).tolist())
    checked = {}

    def check(variant):
        """The last step's outputs of the sampled scans against gg_download_labels / gg_get_output."""
        out, s = last["out"], last["pose"]
        torch.cuda.synchronize()
        g.synchronize()
        cloud, index = out.trimmed() if out.counts is not None else (None, None)
        for b in sample:
            lab = g.download_labels(int(npts[b, s]), slot=b)
            g.synchronize()
            assert np.array_equal(out.labels[b].cpu().numpy(), lab), f"{variant} slot {b}: labels"
            if cloud is None:
                continue
            want_i, want_c = g.get_output(slot=b, want_cloud=True)
            keep = np.ones(len(want_i), bool) if variant == "D" else lab[want_i] == capi.LABEL_NONGROUND
            got = cloud[b].cpu().numpy().view(np.uint8).reshape(-1, 32)
            want_raw = np.ascontiguousarray(want_c).view(np.uint8).reshape(-1, 32)   # masked as bytes: keeps the padding
            assert got.tobytes() == want_raw[keep].tobytes(), f"{variant} slot {b}: cloud"
            if index is not None:
                assert np.array_equal(index[b].cpu().numpy().view(np.uint32), want_i[keep]), f"{variant} slot {b}: index"
        checked[variant] = checked.get(variant, 0) + len(sample)

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            if v in ("B", "C", "D"):
                check(v)
    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, {args.steps} timed steps per run, {args.reps} alternating runs; {float(npts.mean()):.0f} points per scan")
    print(f"{'variant':<58} {'ms/step (runs)':<26} {'Mpoints/s (median)':>18}")
    for v, desc in VARIANTS.items():
        ms = [r["ms_per_step"] for r in results[v]]
        mp = float(np.median([r["mpoints_per_s"] for r in results[v]]))
        print(f"{v + '  ' + desc:<58} {' / '.join(f'{x:.2f}' for x in ms):<26} {mp:>18.0f}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "reps": args.reps,
                      "points_per_scan_mean": float(npts.mean()), "checked_scans": checked, "results": results}))
    g.close()


if __name__ == "__main__":
    main()
