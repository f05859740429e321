"""What replaying a recorded step saves: the call sequence against a step plan (gg_step_plan_launch) and against the plan
captured in a torch.cuda.graph, on the device-resident workload of bench.py's `value`.

    python bench_step_plans.py [--streams 396] [--pool 8] [--steps 30] [--warmup 3] [--reps 3] [--check 16]

One step = the next cloud, point counts and poses written into fixed CUDA tensors by torch copies (the same in every
variant), then one roll and one scan of every stream with labels to the device, ordered on torch's current stream.
Variants, alternated --reps times per workload:
  C  the call sequence: gg_set_point_counts_from_device + gg_update_poses_from_device + the scan call
  P  gg_step_plan_launch of a plan recorded once over the same tensors
  G  P's launch captured once in a torch.cuda.graph, replayed every step
Workloads: `value`'s streams x poses with 32-byte records (N = 300); one stream alone; the streams as 18-byte
sensor-frame payloads with their transforms in device memory (C passes the same transforms from host memory, as
gg_run_cloud_msgs_to_device takes them).  Reported per variant: ms per step from CUDA events on the stream, host time
per step spent in the enqueue calls alone (a host clock around them, excluding the input copies), and after each
variant a bit-exact check of a seeded sample of streams (labels of the last step, "ground", "groundpatch", the map
position) against a twin handle that ran the call sequence on the same inputs.  Prints the card and its power limit,
a table and one JSON line; writes nothing.
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

VARIANTS = {"C": "call sequence (device poses and counts)", "P": "gg_step_plan_launch", "G": "plan in a torch.cuda.graph"}
MSG18 = (18, (0, 4, 8, 12, 16))


def map_from_sensor(ego_x, yaw):
    c, s = math.cos(yaw), math.sin(yaw)
    return np.array([[c, -s, 0.0, ego_x], [s, c, 0.0, 0.0], [0.0, 0.0, 1.0, 1.7]])


def payloads18(torch, rec, T):
    """18-byte PointCloud2 bytes [n, 18] of map-frame records rec (float32 [n, 8]) in the sensor frame of T."""
    Td = torch.tensor(T, dtype=torch.float64, device=rec.device)
    p = rec[:, :3].double() - Td[:, 3]
    q = (p @ Td[:, :3]).float()
    ring = rec[:, 5].view(torch.int32).to(torch.int16).contiguous()
    return torch.cat([q.contiguous().view(torch.uint8).view(-1, 12), rec[:, 4:5].contiguous().view(torch.uint8).view(-1, 4),
                      ring.view(torch.uint8).view(-1, 2)], 1).contiguous()


def run_workload(torch, capi, streams, B, S, route, args):
    """(results per variant, checked streams, N, points per step) of one workload."""
    step_bytes = 32 if route == "records" else MSG18[0]
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    cap = npts.max(1)
    first = np.concatenate([[0], np.cumsum(cap * step_bytes)[:-1]]).astype(np.int64)
    total = int((cap * step_bytes).sum())
    Ts = [[map_from_sensor(float(s), 0.1 * b) for b in range(B)] for s in range(S)]
    pool = []
    for s in range(S):
        buf = torch.zeros(total, dtype=torch.uint8, device="cuda")
        for b in range(B):
            rec = torch.from_numpy(np.ascontiguousarray(streams[b][s][0]).view(np.float32).reshape(-1, 8).copy()).cuda()
            raw = rec.view(torch.uint8).reshape(-1) if route == "records" else payloads18(torch, rec, Ts[s][b]).reshape(-1)
            buf[int(first[b]):int(first[b]) + raw.numel()] = raw
        pool.append(buf)
    counts = [torch.tensor(npts[:, s].astype(np.int32), device="cuda") for s in range(S)]
    dxy = [torch.tensor(np.tile(np.array([float(s), 0.0]), (B, 1)), device="cuda") for s in range(S)]
    dT = [torch.tensor(np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)), device="cuda") for s in range(S)]
    dorg = [torch.tensor(np.array([streams[b][s][1] for b in range(B)], np.float32), device="cuda") for s in range(S)]
    dTm = [torch.tensor(np.stack([t.reshape(12) for t in Ts[s]]), device="cuda") for s in range(S)]
    bz = torch.zeros(B, dtype=torch.float64, device="cuda")

    # the fixed tensors every variant reads
    frame = torch.zeros(total, dtype=torch.uint8, device="cuda")
    views = [frame[int(first[b]):int(first[b]) + int(cap[b]) * step_bytes] for b in range(B)]
    f_counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    f_xy, f_T, f_org = dxy[0].clone(), dT[0].clone(), dorg[0].clone()
    f_Tm = dTm[0].clone()
    moved = torch.zeros(B, dtype=torch.int32, device="cuda")

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    slots = np.arange(B, dtype=np.int32)
    cur = torch.cuda.current_stream()
    sp = cur.cuda_stream or None
    descs = g._device_descs(slots, cap.tolist(), "device", None, True)
    c_out, c_ptrs = g._device_outputs(torch, torch.device("cuda", 0), cur, cap.tolist(), True, 0, False, [])
    kw = dict(counts=f_counts, xy=f_xy, T_base_from_map=f_T, pose_origins=f_org, pose_base_z=bz, moved=True, labels=True, select=None)
    if route == "records":
        plan = g.step_plan(slots, clouds=views, **kw)
    else:
        plan = g.step_plan(slots, payloads=views, point_step=MSG18[0], field_offsets=MSG18[1], T=list(f_Tm), **kw)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.launch()
    tstep = [0]
    history = []
    last = {}

    def write():
        s = bench.pingpong(tstep[0], S)
        tstep[0] += 1
        history.append(s)
        frame.copy_(pool[s])
        f_counts.copy_(counts[s])
        f_xy.copy_(dxy[s])
        f_T.copy_(dT[s])
        f_org.copy_(dorg[s])
        f_Tm.copy_(dTm[s])
        return s

    def enqueue(v, s):
        if v == "C":
            g.set_point_counts_from_device_ptrs(slots, f_counts.data_ptr(), sp)
            g.update_poses_from_device_ptrs(slots, f_xy.data_ptr(), f_T.data_ptr(), f_org.data_ptr(), bz.data_ptr(), moved.data_ptr(), sp)
            if route == "records":
                g.run_scans_to_device_ptrs(descs, [t.data_ptr() for t in views], c_ptrs, 0, None, sp)
            else:
                g.run_cloud_msgs_to_device_ptrs(descs, [t.data_ptr() for t in views], MSG18[0], MSG18[1], np.stack(Ts[s]), c_ptrs, 0, None, sp)
            last["labels"] = c_out.labels
        elif v == "P":
            plan.launch(cur)
            last["labels"] = plan.outputs.labels
        else:
            graph.replay()
            last["labels"] = plan.outputs.labels

    def timed(v):
        for _ in range(args.warmup):
            enqueue(v, write())
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        host = 0.0
        ev[0].record(cur)
        for t in range(args.steps):
            s = write()
            t0 = time.perf_counter()
            enqueue(v, s)
            host += time.perf_counter() - t0
            ev[t + 1].record(cur)
        torch.cuda.synchronize()
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.steps)]
        return {"ms_per_step": ev[0].elapsed_time(ev[-1]) / args.steps, "ms_step_median": float(np.median(per)),
                "host_enqueue_us_per_step": 1e6 * host / args.steps}

    # the twin runs the call sequence of the sampled streams on the pool's own tensors
    rng = np.random.default_rng(1234)
    sample = np.array(sorted(rng.choice(B, min(args.check, B), replace=False).tolist()), np.int32)
    m = len(sample)
    twin = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=m, max_points=bench.PCAP, full_layers=False)
    tslots = np.arange(m, dtype=np.int32)
    for j in range(m):
        twin.init_map(0.0, 0.0, 0.0, slot=j)
    idx = torch.tensor(sample.astype(np.int64), device="cuda")
    replayed = [0]
    checked = {}

    def check(v):
        torch.cuda.synchronize()
        out = None
        for t in range(replayed[0], len(history)):
            s = history[t]
            data = [pool[s][int(first[b]):int(first[b]) + int(cap[b]) * step_bytes] for b in sample]
            twin.set_point_counts_from_device(tslots, counts[s][idx])
            twin.update_poses_from_device(tslots, dxy[s][idx], dT[s][idx], dorg[s][idx], bz[idx])
            if route == "records":
                out = twin.run_scans_to_device(data, tslots, "device", None, labels=True, select=None, device_counts=True)
            else:
                out = twin.run_cloud_msgs_to_device(data, MSG18[0], MSG18[1], [Ts[s][b] for b in sample], tslots, "device", None, labels=True,
                                                    select=None, device_counts=True)
        replayed[0] = len(history)
        torch.cuda.synchronize()
        s = history[-1]
        for j, b in enumerate(sample):
            u = int(npts[b, s])
            assert torch.equal(last["labels"][b][:u], out.labels[j][:u]), f"{route} {v} stream {b}: labels differ from the call sequence"
            for name in ("ground", "groundpatch"):
                assert np.array_equal(g.layer(name, slot=int(b)).view(np.uint32), twin.layer(name, slot=j).view(np.uint32)), f"{route} {v} stream {b}: {name}"
            assert g.position(slot=int(b)).tolist() == twin.position(slot=j).tolist(), f"{route} {v} stream {b}: position"
        checked[v] = checked.get(v, 0) + m

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            check(v)
    info = {"kernels_per_step": plan.kernels, "N": g.n, "points_per_step": float(npts.sum(0).mean())}
    del graph
    plan.close()
    g.close()
    twin.close()
    return results, checked, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=16, help="streams of the seeded sample checked after each variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_step_plans.py needs a CUDA device")
    card = gpu_info()
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))
    workloads = {"value": (streams, B, "records"), "one_stream": (streams[:1], 1, "records"), "sensor18": (streams, B, "msgs18")}
    report = {}
    for name, (st, nb, route) in workloads.items():
        results, checked, info = run_workload(torch, capi, st, nb, S, route, args)
        report[name] = {"results": results, "checked_streams": checked, **info}
    card_after = gpu_info()
    print(f"card, power limit, max SM clock: {card} (after the run: {card_after})")
    print(f"{B} streams x {S} poses, {args.steps} timed steps per run, {args.reps} alternating runs")
    for name, r in report.items():
        print(f"{name}: N = {r['N']}, {r['points_per_step'] / 1e6:.2f} M points per step, {r['kernels_per_step']} kernels per replayed step")
        print(f"  {'variant':<46} {'ms/step (runs)':<28} {'host enqueue us/step (runs)':<30}")
        for v, desc in VARIANTS.items():
            ms = " / ".join(f"{x['ms_per_step']:.3f}" for x in r["results"][v])
            hu = " / ".join(f"{x['host_enqueue_us_per_step']:.0f}" for x in r["results"][v])
            print(f"  {v + '  ' + desc:<46} {ms:<28} {hu:<30}")
        print(f"  bit-exact checks: {r['checked_streams']}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "reps": args.reps, "workloads": report}))


if __name__ == "__main__":
    main()
