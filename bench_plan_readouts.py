"""What recording a step's read-outs into its plan saves: a plan followed by the standalone read-out calls against a plan
with read-outs (gg_step_plan_create_with_readouts), plain and captured in a torch.cuda.graph, on the device-resident
workload of bench.py's `value`.

    python bench_plan_readouts.py [--streams 396] [--pool 8] [--steps 30] [--warmup 3] [--reps 3] [--check 16]

One step = the next cloud, point counts and poses written into fixed CUDA tensors by torch copies (the same in every
variant), then one roll and one scan of every stream with labels to the device, ordered on torch's current stream.
The read-out set: "ground" and "groundpatch" of every slot, the height of every input point, a 64 x 64 grid of
nearest lookups per slot, and the running tallies.  Variants, alternated --reps times:
  P  gg_step_plan_launch of a plan without read-outs
  C  P, then the four standalone calls of the read-out set (gg_get_layers_to_device, gg_sample_layers_to_device,
     gg_point_info_to_device, gg_eval_counts_to_device) on the same stream
  R  gg_step_plan_launch of a plan with the read-out set
  G  R's launch captured once in a torch.cuda.graph, replayed every step
Reported per variant: ms per step from CUDA events on the stream, host time per step spent in the enqueue calls alone
(a host clock around them, excluding the input copies), and after each variant a bit-exact check of a seeded sample of
streams against a twin handle that ran the call sequence and the standalone read-outs on the same inputs: labels,
the read-outs of the last step and the tallies of every step.  Prints the card and its power limit, a table and one
JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generators and the pose sequence of bench.py)
from bench_slot_config import gpu_info  # noqa: E402

VARIANTS = {"P": "plan alone", "C": "plan, then the standalone read-outs", "R": "plan with read-outs",
            "G": "plan with read-outs in a torch.cuda.graph"}
NAMES = ("ground", "groundpatch")
GRID = 64


def run(torch, capi, streams, B, S, args):
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    cap = npts.max(1)
    first = np.concatenate([[0], np.cumsum(cap * 32)[:-1]]).astype(np.int64)
    total = int((cap * 32).sum())
    pool = []
    for s in range(S):
        buf = torch.zeros(total, dtype=torch.uint8, device="cuda")
        for b in range(B):
            rec = np.ascontiguousarray(streams[b][s][0]).view(np.uint8).reshape(-1)
            buf[int(first[b]):int(first[b]) + rec.size] = torch.from_numpy(rec.copy()).cuda()
        pool.append(buf)
    counts = [torch.tensor(npts[:, s].astype(np.int32), device="cuda") for s in range(S)]
    dxy = [torch.tensor(np.tile(np.array([float(s), 0.0]), (B, 1)), device="cuda") for s in range(S)]
    dT = [torch.tensor(np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)), device="cuda") for s in range(S)]
    dorg = [torch.tensor(np.array([streams[b][s][1] for b in range(B)], np.float32), device="cuda") for s in range(S)]
    bz = torch.zeros(B, dtype=torch.float64, device="cuda")
    # a 64 x 64 grid over the map around the poses, shared by every slot's lookups (inputs may share memory)
    ax = np.linspace(-45.0, 45.0 + S, GRID, dtype=np.float32)
    grid = torch.tensor(np.stack(np.meshgrid(ax, np.linspace(-45.0, 45.0, GRID, dtype=np.float32), indexing="ij"), -1).reshape(-1, 2),
                        device="cuda")

    frame = torch.zeros(total, dtype=torch.uint8, device="cuda")
    views = [frame[int(first[b]):int(first[b]) + int(cap[b]) * 32] for b in range(B)]
    f_counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    f_xy, f_T, f_org = dxy[0].clone(), dT[0].clone(), dorg[0].clone()

    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    slots = np.arange(B, dtype=np.int32)
    cur = torch.cuda.current_stream()
    sp = cur.cuda_stream or None
    kw = dict(counts=f_counts, xy=f_xy, T_base_from_map=f_T, pose_origins=f_org, pose_base_z=bz, moved=True, labels=True, select=None)

    # C's destinations of the standalone read-outs
    c_layers = torch.empty((B, len(NAMES), g.n, g.n), dtype=torch.float32, device="cuda").transpose(-1, -2)
    c_q, ns = g._position_sets(torch, torch.device("cuda", 0), [grid] * B)
    c_samples, _ = g._sample_outputs(torch, torch.device("cuda", 0), cur, c_q, ns, len(NAMES), None, False)
    c_height = list(torch.split(torch.empty(int(cap.sum()), dtype=torch.float32, device="cuda"), cap.tolist()))
    c_tallies = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")

    tstep = [0]
    history = []

    def write():
        s = bench.pingpong(tstep[0], S)
        tstep[0] += 1
        history.append(s)
        frame.copy_(pool[s])
        f_counts.copy_(counts[s])
        f_xy.copy_(dxy[s])
        f_T.copy_(dT[s])
        f_org.copy_(dorg[s])

    def setup(v):
        """(plan, graph or None, what the check reads: labels, layers, samples, heights, tallies) of variant v."""
        if v in ("P", "C"):
            plan = g.step_plan(slots, clouds=views, **kw)
            c_tallies.zero_()
            out = (plan.outputs.labels, c_layers, c_samples, c_height, c_tallies) if v == "C" else (plan.outputs.labels,)
            return plan, None, out
        plan = g.step_plan(slots, clouds=views, layers=NAMES, samples=[grid] * B, sample_names=NAMES, point_info=("height",),
                           tallies=torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda"), **kw)
        graph = None
        if v == "G":
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                plan.launch()
        ro = plan.readouts
        return plan, graph, (plan.outputs.labels, ro.layers, ro.samples, ro.height, ro.tallies)

    def enqueue(v, plan, graph):
        if v == "G":
            graph.replay()
            return
        plan.launch(cur)
        if v == "C":
            g.get_layers_to_device_ptrs(slots, NAMES, c_layers.data_ptr(), sp)
            g.sample_layers_to_device_ptrs(slots, c_q[:B], NAMES, "nearest", sp)
            g.point_info_to_device_ptrs(slots, None, [t.data_ptr() for t in c_height], sp)
            g.eval_counts_to_device_ptrs(slots, c_tallies.data_ptr(), sp)

    def timed(v, plan, graph):
        for _ in range(args.warmup):
            write()
            enqueue(v, plan, graph)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        host = 0.0
        k0 = g.kernel_launches
        ev[0].record(cur)
        for t in range(args.steps):
            write()
            t0 = time.perf_counter()
            enqueue(v, plan, graph)
            host += time.perf_counter() - t0
            ev[t + 1].record(cur)
        torch.cuda.synchronize()
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.steps)]
        return {"ms_per_step": ev[0].elapsed_time(ev[-1]) / args.steps, "ms_step_median": float(np.median(per)),
                "host_enqueue_us_per_step": 1e6 * host / args.steps, "kernels_per_step": plan.kernels if v == "G" else (g.kernel_launches - k0) / args.steps}   # a torch graph replay is not counted by the handle

    # the twin runs the call sequence and the standalone read-outs of the sampled streams on the pool's own tensors
    rng = np.random.default_rng(1234)
    sample = np.array(sorted(rng.choice(B, min(args.check, B), replace=False).tolist()), np.int32)
    m = len(sample)
    twin = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=m, max_points=bench.PCAP, full_layers=False)
    tslots = np.arange(m, dtype=np.int32)
    for j in range(m):
        twin.init_map(0.0, 0.0, 0.0, slot=j)
    idx = torch.tensor(sample.astype(np.int64), device="cuda")
    t_tallies = torch.zeros((m, 1024, 2), dtype=torch.int64, device="cuda")
    t_height = [torch.empty(int(cap[b]), dtype=torch.float32, device="cuda") for b in sample]
    replayed = [0]
    checked = {}

    def check(v, got):
        torch.cuda.synchronize()
        t_tallies.zero_()
        out = None
        for t in range(replayed[0], len(history)):
            s = history[t]
            data = [pool[s][int(first[b]):int(first[b]) + int(cap[b]) * 32] for b in sample]
            twin.set_point_counts_from_device(tslots, counts[s][idx])
            twin.update_poses_from_device(tslots, dxy[s][idx], dT[s][idx], dorg[s][idx], bz[idx])
            out = twin.run_scans_to_device(data, tslots, "device", None, labels=True, select=None, device_counts=True)
            twin.eval_counts_to_device(tslots, out=t_tallies)
        replayed[0] = len(history)
        layers = twin.get_layers_to_device(tslots, NAMES)
        samples = twin.sample_layers_to_device(tslots, [grid] * m, NAMES)
        twin.point_info_to_device_ptrs(tslots, None, [t.data_ptr() for t in t_height], torch.cuda.current_stream().cuda_stream or None)
        torch.cuda.synchronize()
        s = history[-1]
        for j, b in enumerate(sample):
            u = int(npts[b, s])
            assert torch.equal(got[0][b][:u], out.labels[j][:u]), f"{v} stream {b}: labels differ from the call sequence"
            if len(got) == 1:
                continue
            assert torch.equal(got[1][b].view(torch.int32), layers[j].view(torch.int32)), f"{v} stream {b}: layers"
            assert torch.equal(got[2][b].view(torch.int32), samples[j].view(torch.int32)), f"{v} stream {b}: lookups"
            assert torch.equal(got[3][b][:u].view(torch.int32), t_height[j][:u].view(torch.int32)), f"{v} stream {b}: heights"
            assert torch.equal(got[4][b], t_tallies[j]), f"{v} stream {b}: tallies"
        checked[v] = checked.get(v, 0) + m

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            plan, graph, got = setup(v)
            results[v].append(timed(v, plan, graph))
            check(v, got)
            del graph
            plan.close()
    info = {"kernels_per_step": {v: r[-1]["kernels_per_step"] for v, r in results.items()}, "N": g.n, "points_per_step": float(npts.sum(0).mean())}
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
        raise SystemExit("bench_plan_readouts.py needs a CUDA device")
    card = gpu_info()
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))
    results, checked, info = run(torch, capi, streams, B, S, args)
    card_after = gpu_info()
    print(f"card, power limit, max SM clock: {card} (after the run: {card_after})")
    print(f"{B} streams x {S} poses, N = {info['N']}, {info['points_per_step'] / 1e6:.2f} M points per step, {args.steps} timed steps per run, "
          f"{args.reps} alternating runs")
    print(f"  {'variant':<50} {'kernels':<8} {'ms/step (runs)':<28} {'host enqueue us/step (runs)':<30}")
    for v, desc in VARIANTS.items():
        ms = " / ".join(f"{x['ms_per_step']:.3f}" for x in results[v])
        hu = " / ".join(f"{x['host_enqueue_us_per_step']:.0f}" for x in results[v])
        print(f"  {v + '  ' + desc:<50} {info['kernels_per_step'][v]:<8.0f} {ms:<28} {hu:<30}")
    print(f"  bit-exact checks: {checked}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "reps": args.reps, **info, "results": results, "checked_streams": checked}))


if __name__ == "__main__":
    main()
