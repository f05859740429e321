"""What skipping scans costs and saves: a step plan whose scans read a device scan mask (GG_SCAN_DEVICE_MASK), on the
device-resident workload of bench.py's `value`.

    python bench_scan_masks.py [--streams 396] [--pool 8] [--steps 30] [--warmup 3] [--reps 2] [--seed 7]

One step = the next cloud, point counts, poses and (where used) scan mask written into fixed CUDA tensors by torch
copies, then one roll and one scan of every stream with labels to the device, ordered on torch's current stream.  The
scanning slots of a step are drawn at random per step from --seed.  Variants, alternated --reps times:
  all       a step plan without masks: every slot scans (the reference point)
  mask100 / mask50 / mask10 / mask0
            the same plan with gg_step_plan_create_with_scan_masks, 100 / 50 / 10 / 0 % of the slots scanning
  count0_50 / count0_10
            the plan without masks, with a point count of 0 for the slots that do not scan (the workaround before
            masks; it computes something else: every count-0 scan still runs its spiral and decays its map)
  host50 / host10
            the call sequence issued from the host with the scanning subset known there: counts and poses of every slot,
            then gg_run_scans_to_device on the scanning slots only
Reported per variant: ms per step from CUDA events on the stream.  Prints the card and its power limit, a table and one
JSON line; writes nothing.
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

VARIANTS = {"all": ("plan", 1.0), "mask100": ("mask", 1.0), "mask50": ("mask", 0.5), "mask10": ("mask", 0.1), "mask0": ("mask", 0.0),
            "count0_50": ("count0", 0.5), "count0_10": ("count0", 0.1), "host50": ("host", 0.5), "host10": ("host", 0.1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    B, S = args.streams, args.pool

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_scan_masks.py needs a CUDA device")
    card = gpu_info()
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    cap = npts.max(1)
    first = np.concatenate([[0], np.cumsum(cap * 32)[:-1]]).astype(np.int64)
    total = int((cap * 32).sum())
    pool = []
    for s in range(S):
        buf = torch.zeros(total, dtype=torch.uint8, device="cuda")
        for b in range(B):
            raw = torch.from_numpy(np.ascontiguousarray(streams[b][s][0]).view(np.uint8).copy()).cuda()
            buf[int(first[b]):int(first[b]) + raw.numel()] = raw
        pool.append(buf)
    counts = [torch.tensor(npts[:, s].astype(np.int32), device="cuda") for s in range(S)]
    dxy = [torch.tensor(np.tile(np.array([float(s), 0.0]), (B, 1)), device="cuda") for s in range(S)]
    dT = [torch.tensor(np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)), device="cuda") for s in range(S)]
    dorg = [torch.tensor(np.array([streams[b][s][1] for b in range(B)], np.float32), device="cuda") for s in range(S)]
    bz = torch.zeros(B, dtype=torch.float64, device="cuda")

    frame = torch.zeros(total, dtype=torch.uint8, device="cuda")
    views = [frame[int(first[b]):int(first[b]) + int(cap[b]) * 32] for b in range(B)]
    f_counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    f_mask = torch.zeros(B, dtype=torch.int32, device="cuda")
    f_xy, f_T, f_org = dxy[0].clone(), dT[0].clone(), dorg[0].clone()

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    slots = np.arange(B, dtype=np.int32)
    cur = torch.cuda.current_stream()
    sp = cur.cuda_stream or None
    kw = dict(clouds=views, counts=f_counts, xy=f_xy, T_base_from_map=f_T, pose_origins=f_org, pose_base_z=bz, labels=True, select=None)
    plans = {"plan": g.step_plan(slots, **kw), "mask": None}
    c_descs = g._device_descs(slots, cap.tolist(), "device", None, True)
    _, c_ptrs = g._device_outputs(torch, torch.device("cuda", 0), cur, cap.tolist(), True, 0, False, [])
    rng = np.random.default_rng(args.seed)
    tstep = [0]

    def write(frac, zero_counts):
        s = bench.pingpong(tstep[0], S)
        tstep[0] += 1
        on = rng.random(B) < frac if 0.0 < frac < 1.0 else np.full(B, frac >= 1.0)
        frame.copy_(pool[s])
        f_counts.copy_(counts[s] * torch.from_numpy(on.astype(np.int32)).cuda() if zero_counts else counts[s])
        f_mask.copy_(torch.from_numpy(on.astype(np.int32)))
        f_xy.copy_(dxy[s])
        f_T.copy_(dT[s])
        f_org.copy_(dorg[s])
        return on

    def enqueue(kind, on):
        if kind in ("plan", "count0"):
            plans["plan"].launch(cur)
        elif kind == "mask":
            plans["mask"].launch(cur)
        else:
            g.set_point_counts_from_device_ptrs(slots, f_counts.data_ptr(), sp)
            g.update_poses_from_device_ptrs(slots, f_xy.data_ptr(), f_T.data_ptr(), f_org.data_ptr(), bz.data_ptr(), None, sp)
            k = np.flatnonzero(on)
            if len(k):
                g.run_scans_to_device_ptrs(c_descs[k], [views[i].data_ptr() for i in k], c_ptrs[k], 0, None, sp)

    def timed(kind, frac):
        zero = kind == "count0"
        for _ in range(args.warmup):
            enqueue(kind, write(frac, zero))
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        scanned = 0
        ev[0].record(cur)
        for t in range(args.steps):
            on = write(frac, zero)
            scanned += int(on.sum())
            enqueue(kind, on)
            ev[t + 1].record(cur)
        torch.cuda.synchronize()
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.steps)]
        return {"ms_per_step": ev[0].elapsed_time(ev[-1]) / args.steps, "ms_step_median": float(np.median(per)),
                "scanning": scanned / (args.steps * B)}

    results = {v: [] for v in VARIANTS}
    kernels = {"plan": plans["plan"].kernels}

    def bind(kind):
        """The plan the variant replays, recorded when needed; the other one is closed (a slot is bound to one plan)."""
        want = {"plan": "plan", "count0": "plan", "mask": "mask"}.get(kind)
        for k in ("plan", "mask"):
            if k != want and plans[k] is not None:
                plans[k].close()
                plans[k] = None
        if want and plans[want] is None:
            plans[want] = g.step_plan(slots, scan_mask=f_mask, **kw) if want == "mask" else g.step_plan(slots, **kw)
            kernels[want] = plans[want].kernels

    for _ in range(args.reps):
        for v, (kind, frac) in VARIANTS.items():
            bind(kind)
            results[v].append(timed(kind, frac))
    for p in plans.values():
        if p is not None:
            p.close()
    info = {"N": g.n, "points_per_step_all": float(npts.sum(0).mean()), "kernels_per_step": kernels}
    g.close()
    card_after = gpu_info()
    print(f"card, power limit, max SM clock: {card} (after the run: {card_after})")
    print(f"{B} streams x {S} poses, N = {info['N']}, {info['points_per_step_all'] / 1e6:.2f} M points per step with every slot scanning, "
          f"{args.steps} timed steps per run, {args.reps} alternating runs; kernels per replay {kernels}")
    print(f"  {'variant':<12} {'scanning':>9} {'ms/step (runs)':<30} {'median ms/step (runs)':<30}")
    for v in VARIANTS:
        ms = " / ".join(f"{x['ms_per_step']:.3f}" for x in results[v])
        md = " / ".join(f"{x['ms_step_median']:.3f}" for x in results[v])
        print(f"  {v:<12} {np.mean([x['scanning'] for x in results[v]]):>9.3f} {ms:<30} {md:<30}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "reps": args.reps, "seed": args.seed, **info, "results": results}))


if __name__ == "__main__":
    main()
