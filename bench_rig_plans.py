"""Cost of a multi-LiDAR rig whose per-sensor point counts live on the GPU, on the cfg4 workload of bench_merged_clouds.py.

    python bench_rig_plans.py [--streams 96] [--steps 20] [--warmup 3] [--reps 3] [--check 8]

cfg4 scans (four 64-beam sensors of synth.FOUR_LIDAR, about 480 k points per scan, N = 364 at 120 m / 0.33 m), four
18-byte payloads per scan, labels only.  Each payload tensor is a capacity buffer holding the sensor's whole sweep; every
step torch writes a seeded draw of each sensor's count (85-100 % of its points) into a CUDA int32 [streams, 4] tensor on
the caller's stream, and the rolls come from CUDA pose tensors (two positions, alternated).  Variants, alternated --reps
times in one run:
  H  the counts read back with .cpu(), then the host-count merged call (gg_update_poses_from_device first)
  D  gg_set_part_counts_from_device + the flagged merged call (GG_SCAN_DEVICE_PART_COUNTS)
  P  a step plan with parts (counts, poses, per-part transforms from CUDA tensors), gg_step_plan_launch
  G  P captured into a torch.cuda.graph and replayed
Reported per variant: ms per step from CUDA events on the caller's stream, host enqueue us per step (host clock around
the step's calls, count draw excluded), kernels per step.  After each variant one more step is checked bit-exact on a
seeded sample of --check streams against a twin running H (its sampled slots start from the handle's map position,
"ground" and "groundpatch").  Then one stream alone, and a serialised gg_profile pass of D (one stream group) for
k_stage_parts, k_store_part_counts and k_unpack_transform.  Prints the card, its power limit and SM clock, a table and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_merged_clouds import DIM_M, LAYOUT, PCAP, RES, _gen_task, map_from_sensor, payload  # noqa: E402
from bench_slot_config import gpu_info  # noqa: E402

import bench  # noqa: E402

VARIANTS = {"H": "counts .cpu() + host-count merged call", "D": "set_part_counts_from_device + flagged merged call",
            "P": "step plan with parts", "G": "P inside torch.cuda.graph"}
NS = 4


def run(torch, capi, synth, B, args, gen):
    caps = np.array([[len(p) for p in gen[b][0]] for b in range(B)], np.int64)     # [B][4]
    origins = np.array([gen[b][1] for b in range(B)], np.float32)
    Tsensor = [map_from_sensor(0, m) for m in synth.FOUR_LIDAR]
    bufs = [[torch.from_numpy(payload(gen[b][0][p], Tsensor[p], 18).reshape(-1).copy()).cuda() for p in range(NS)] for b in range(B)]
    dev = torch.device("cuda", 0)
    cur = torch.cuda.current_stream()
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(4321)
    sample = sorted(rng.choice(B, min(args.check, B), replace=False).tolist())
    counts = torch.zeros((B, NS), dtype=torch.int32, device="cuda")
    xy = torch.zeros((B, 2), dtype=torch.float64, device="cuda")
    Tb = torch.zeros((B, 12), dtype=torch.float64, device="cuda")
    org = torch.from_numpy(origins).cuda()
    bz = torch.zeros(B, dtype=torch.float64, device="cuda")
    T_dev = torch.from_numpy(np.stack([np.stack([t.reshape(12) for t in Tsensor])] * B)).cuda()   # [B, 4, 12]
    lo = torch.from_numpy((caps * 0.85).astype(np.int64)).cuda()
    span = torch.from_numpy(caps).cuda() - lo + 1
    gen_t = torch.Generator(device="cuda")
    gen_t.manual_seed(99)
    steps_done = [0]

    def draw():
        """The step's counts and pose, written by torch on the caller's stream."""
        k = steps_done[0]
        steps_done[0] += 1
        counts.copy_(lo + (torch.rand((B, NS), device="cuda", generator=gen_t) * span).floor().clamp_max(span - 1).long())
        s = bench.pingpong(k, 2)
        xy[:, 0] = float(s)
        xy[:, 1] = 0.0
        Tb.copy_(torch.from_numpy(np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1))))

    g = capi.GroundGridB200(DIM_M, RES, n_slots=B, max_points=PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    cap_n = [int(c) for c in caps.sum(axis=1)]
    nested_T = [Tsensor] * B
    recs_cap = capi.cloud_parts([[t.numel() for t in s] for s in bufs], [[t.data_ptr() for t in s] for s in bufs], 18, LAYOUT[18], nested_T)
    descs_cap = g._device_descs(slots, cap_n, "device", None)
    descs_flag = descs_cap.copy()
    descs_flag["flags"] |= capi.SCAN_DEVICE_PART_COUNTS

    def poses(h):
        h.update_poses_from_device(slots, xy, Tb, org, bz)

    def merged(h, descs, n_parts, parts):
        out, ptrs = h._device_outputs(torch, dev, cur, [int(x) for x in descs["n_points"]], True, 0, False, [])
        h.run_merged_cloud_msgs_to_device_ptrs(descs, n_parts, parts, ptrs, 0, None, cur.cuda_stream or None)
        return out

    def step_H(h=g):
        c = counts.cpu().numpy()
        poses(h)
        recs = capi.cloud_parts([[int(c[b, p]) * 18 for p in range(NS)] for b in range(B)], [[t.data_ptr() for t in s] for s in bufs], 18,
                                LAYOUT[18], nested_T)
        return merged(h, g._device_descs(slots, c.sum(axis=1), "device", None), recs[0], recs[1])

    def step_D(h=g):
        h.set_part_counts_from_device_ptrs(slots, NS, counts.data_ptr(), cur.cuda_stream or None)
        poses(h)
        return merged(h, descs_flag, recs_cap[0], recs_cap[1])

    plan = {}

    def step_P():
        plan["p"].launch()
        return plan["p"].outputs

    def step_G():
        plan["g"].replay()
        return plan["p"].outputs

    def make_plan():
        p = g.step_plan(list(slots), parts=bufs, point_step=18, field_offsets=LAYOUT[18],
                        T=[[T_dev[b, q] for q in range(NS)] for b in range(B)], origins="device", part_counts=counts, xy=xy,
                        T_base_from_map=Tb, pose_origins=org, pose_base_z=bz, labels=True, select=None)
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.graph(graph, stream=side):
            p.launch()
        cur.wait_stream(side)
        return p, graph

    fns = {"H": step_H, "D": step_D, "P": step_P, "G": step_G}
    twin = capi.GroundGridB200(DIM_M, RES, n_slots=B, max_points=PCAP, full_layers=False)

    def check(variant):
        """One more step on the handle and, for the sampled slots, on the twin through H from the same map state."""
        torch.cuda.synchronize()
        for b in sample:
            x, y = g.position(slot=b)
            twin.init_map(x, y, 0.0, slot=b)
            for name in ("ground", "groundpatch"):
                twin.set_layer(name, g.layer(name, slot=b), slot=b)
        draw()
        out = fns[variant]()
        torch.cuda.synchronize()
        c = counts.cpu().numpy()
        ts = np.array(sample, np.int32)
        twin.update_poses_from_device(ts, xy[ts].contiguous(), Tb[ts].contiguous(), org[ts].contiguous(), bz[ts].contiguous())
        recs = capi.cloud_parts([[int(c[b, p]) * 18 for p in range(NS)] for b in sample], [[t.data_ptr() for t in bufs[b]] for b in sample], 18,
                                LAYOUT[18], [Tsensor] * len(sample))
        d = twin._device_descs(ts, c[sample].sum(axis=1), "device", None)
        out_t = merged(twin, d, recs[0], recs[1])
        torch.cuda.synchronize()
        ok = all(torch.equal(out.labels[b][:int(c[b].sum())], out_t.labels[j]) for j, b in enumerate(sample))
        return bool(ok)

    def timed(variant):
        fn = fns[variant]
        for _ in range(args.warmup):
            draw()
            fn()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        host_us, kern = [], []
        ev[0].record(cur)
        for i in range(args.steps):
            draw()
            l0 = g.kernel_launches
            t = time.perf_counter()
            fn()
            host_us.append((time.perf_counter() - t) * 1e6)
            kern.append(g.kernel_launches - l0)
            ev[i + 1].record(cur)
        torch.cuda.synchronize()
        ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(args.steps)]
        return {"ms_per_step": float(np.mean(ms)), "ms_median": float(np.median(ms)), "host_us": float(np.median(host_us)),
                "kernels": int(np.median(kern)) if variant != "G" else None, "pts_per_step": int(caps.sum() * 0.925)}

    results = {v: [] for v in VARIANTS}
    checks = {v: [] for v in VARIANTS}
    for rep in range(args.reps):
        for v in VARIANTS:
            if v in ("P", "G") and not plan:
                draw()
                plan["p"], plan["g"] = make_plan()
            results[v].append(timed(v))
            checks[v].append(check(v))
    # the kernels one replay adds, for G too
    results["G_kernels"] = plan["p"].kernels
    plan["p"].close()
    g.close()
    prof = None
    if B > 1:   # serialised: one stream group, so no other group's kernels share the SMs with the timed ones
        os.environ["GG_STREAMS"] = "1"
        gp = capi.GroundGridB200(DIM_M, RES, n_slots=B, max_points=PCAP, full_layers=False)
        del os.environ["GG_STREAMS"]
        for b in range(B):
            gp.init_map(0.0, 0.0, 0.0, slot=b)
        for _ in range(2):
            draw()
            step_D(gp)
        gp.profile_enable(True)
        gp.profile_read()
        for _ in range(3):
            draw()
            step_D(gp)
        pr = gp.profile_read()
        gp.close()
        prof = {k: {"ms_total": pr[k][0], "launches": pr[k][1], "us_per_launch": 1e3 * pr[k][0] / max(pr[k][1], 1)}
                for k in ("k_stage_parts", "k_store_part_counts", "k_unpack_transform")}
    twin.close()
    return results, checks, prof


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=96)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=8)
    args = ap.parse_args()
    B = args.streams
    procs = max(1, min(32, (os.cpu_count() or 2) - 1))
    tasks = [(8000 + b, 0, 2) for b in range(B)]
    if procs > 1:
        import multiprocessing as mp

        with mp.get_context("fork").Pool(procs) as pool:
            gen = pool.map(_gen_task, tasks, chunksize=1)
    else:
        gen = [_gen_task(t) for t in tasks]
    import torch

    from groundgrid_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("bench_rig_plans.py needs a CUDA device")
    info = gpu_info()
    print(f"# {info}")
    out = {"gpu": info, "streams": B}
    for label, n in (("batch", B), ("single", 1)):
        res, chk, prof = run(torch, capi, synth, n, args, gen[:n])
        print(f"## {label}: {n} stream(s)")
        print("| variant | ms / step (runs) | host enqueue us (runs) | kernels / step | sample bit-exact |")
        print("|---|---|---|---|---|")
        for v, name in VARIANTS.items():
            r = res[v]
            kern = r[0]["kernels"] if r[0]["kernels"] is not None else res["G_kernels"]
            print(f"| {v} {name} | {' / '.join(f'{x['ms_per_step']:.2f}' for x in r)} | {' / '.join(f'{x['host_us']:.0f}' for x in r)} "
                  f"| {kern} | {all(chk[v])} |")
        if prof:
            for k, p in prof.items():
                print(f"{k}: {p['us_per_launch']:.1f} us per launch over {p['launches']} launches")
        out[label] = {"results": res, "checks": chk, "profile": prof}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
