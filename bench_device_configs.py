"""Configurations chosen on the GPU inside a step: the host gg_set_slot_config a caller needs today against
gg_set_slot_configs_from_device, a step plan with configurations and that plan in a torch.cuda.graph, on bench.py's
`value` workload.

    python bench_device_configs.py [--streams 396] [--pool 8] [--steps 32] [--warmup 3] [--reps 3] [--check 16] [--p 0.03125]

One step = the next cloud, point counts, poses, configurations and configuration mask written into fixed CUDA tensors by
torch copies (the same in every variant), then the configurations, one roll and one scan of every stream with labels to
the device, ordered on torch's current stream.  The configurations are a seeded domain-randomisation draw: every field
uniform between the smallest and the largest value the four test configurations (tests/test_gpu_slot_config.py:CFGS)
give it; the mask picks each stream with probability --p per step, and one step of every timed run reconfigures every
stream.  Variants, alternated --reps times per workload:
  H  what a caller must do today: read the mask and configurations back to the host, gg_set_slot_config of each changed
     stream, then the call sequence (gg_set_point_counts_from_device + gg_update_poses_from_device + gg_run_scans_to_device)
  D  gg_set_slot_configs_from_device, then the same call sequence
  P  gg_step_plan_launch of a plan with configurations (gg_step_plan_create_with_configs) recorded once over the same tensors
  G  P's launch captured once in a torch.cuda.graph, replayed every step
H and D run on one handle, P and G on another (gg_set_slot_config is refused on slots bound to a plan).  Reported per
variant: ms per step from CUDA events on the stream, host time per step spent in the enqueue calls (a host clock around
them, excluding the input copies), and after each variant a bit-exact check of a seeded sample of streams (labels of the
last step, "ground", "groundpatch", the map position) against a twin handle that ran host gg_set_slot_config + the call
sequence on the same inputs.  Then k_store_configs and k_rebuild_detect_tables alone (gg_profile) reconfiguring every
stream: bytes written, GB/s and the share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), on a handle with one
stream group so that one launch covers every stream.  Prints the card and its power limit, a table and one JSON line;
writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generators and the pose sequence of bench.py)
from bench_slot_config import gpu_info  # noqa: E402

VARIANTS = {"H": "host gg_set_slot_config + call sequence", "D": "gg_set_slot_configs_from_device + call sequence",
            "P": "plan with configurations", "G": "plan with configurations in a torch.cuda.graph"}
DATASHEET_BPS = 3.35e12   # H100 SXM HBM3, NVIDIA data sheet (not a measured peak)
# the ranges of the draw: per field the smallest and largest value of the four test configurations
CFGS = [
    dict(),
    dict(max_ring=48, occupied_cells_decrease_factor=1.5, patch_size_change_distance=8.0, miminum_point_height_threshold=0.2,
         minimum_point_height_obstacle_threshold=0.05, outlier_tolerance=0.25, min_outlier_detection_ground_confidence=0.6,
         point_count_cell_variance_threshold=4),
    dict(max_ring=40, occupied_cells_decrease_factor=2000.0, patch_size_change_distance=30.0, distance_factor=0.0003,
         minimum_distance_factor=0.001, ground_patch_detection_minimum_point_count_threshold=0.15,
         occupied_cells_point_count_factor=8.0, outlier_tolerance=0.05),
    dict(occupied_cells_decrease_factor=1.5, patch_size_change_distance=12.0, outlier_tolerance=0.02,
         min_outlier_detection_ground_confidence=2.0, miminum_point_height_threshold=0.45,
         minimum_point_height_obstacle_threshold=0.2, point_count_cell_variance_threshold=20,
         ground_patch_detection_minimum_point_count_threshold=0.4, occupied_cells_point_count_factor=35.0),
]


def draw_configs(capi, rng, n):
    """n configurations as uint8 rows of gg_config: every field uniform over its range in CFGS."""
    base = []
    for kw in CFGS:
        c = capi.default_config()
        for k, v in kw.items():
            setattr(c, k, v)
        base.append(c)
    out = np.zeros((n, C.sizeof(capi.Config)), np.uint8)
    for j in range(n):
        c = capi.default_config()
        for name, t in capi.Config._fields_:
            lo, hi = min(getattr(b, name) for b in base), max(getattr(b, name) for b in base)
            setattr(c, name, int(rng.integers(lo, hi + 1)) if t is C.c_int else float(rng.uniform(lo, hi)))
        out[j] = np.frombuffer(bytes(c), np.uint8)
    return out


def run_workload(torch, capi, streams, B, S, args):
    """(results per variant, checked streams, info) of one workload."""
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    cap = npts.max(1)
    first = np.concatenate([[0], np.cumsum(cap * 32)[:-1]]).astype(np.int64)
    total = int((cap * 32).sum())
    pool = []
    for s in range(S):
        buf = torch.zeros(total, dtype=torch.uint8, device="cuda")
        for b in range(B):
            rec = torch.from_numpy(np.ascontiguousarray(streams[b][s][0]).view(np.uint8).copy()).cuda()
            buf[int(first[b]):int(first[b]) + rec.numel()] = rec
        pool.append(buf)
    counts = [torch.tensor(npts[:, s].astype(np.int32), device="cuda") for s in range(S)]
    hxy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    dxy = [torch.tensor(x, device="cuda") for x in hxy]
    dT = [torch.tensor(np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)), device="cuda") for s in range(S)]
    dorg = [torch.tensor(np.array([streams[b][s][1] for b in range(B)], np.float32), device="cuda") for s in range(S)]
    # draws: seeded configurations and Bernoulli masks, entry 0 = every stream
    rng = np.random.default_rng(4321)
    hcfg = [draw_configs(capi, rng, B) for _ in range(8)]
    dcfg = [torch.from_numpy(x).cuda() for x in hcfg]
    hmask = [np.ones(B, np.int32)] + [(rng.random(B) < args.p).astype(np.int32) for _ in range(31)]
    dmask = [torch.tensor(m, device="cuda") for m in hmask]
    bz = torch.zeros(B, dtype=torch.float64, device="cuda")

    # the fixed tensors every variant reads
    frame = torch.zeros(total, dtype=torch.uint8, device="cuda")
    views = [frame[int(first[b]):int(first[b]) + int(cap[b]) * 32] for b in range(B)]
    f_counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    f_xy, f_T, f_org, f_cfg, f_mask = dxy[0].clone(), dT[0].clone(), dorg[0].clone(), dcfg[0].clone(), dmask[1].clone()
    moved = torch.zeros(B, dtype=torch.int32, device="cuda")

    handles = {}
    for key in ("call", "plan"):
        h = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
        for b in range(B):
            h.init_map(0.0, 0.0, 0.0, slot=b)
        handles[key] = h
    g, gp = handles["call"], handles["plan"]
    slots = np.arange(B, dtype=np.int32)
    cur = torch.cuda.current_stream()
    sp = cur.cuda_stream or None
    descs = g._device_descs(slots, cap.tolist(), "device", None, True)
    c_out, c_ptrs = g._device_outputs(torch, torch.device("cuda", 0), cur, cap.tolist(), True, 0, False, [])
    kw = dict(counts=f_counts, xy=f_xy, T_base_from_map=f_T, pose_origins=f_org, pose_base_z=bz, moved=True, labels=True, select=None)
    plan = gp.step_plan(slots, clouds=views, configs=f_cfg, config_mask=f_mask, **kw)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.launch()
    tstep = [0]
    history = {"call": [], "plan": []}
    last = {}

    def write(key, all_cfg):
        s = bench.pingpong(tstep[0], S)
        m = 0 if all_cfg else 1 + tstep[0] % (len(hmask) - 1)
        c = tstep[0] % len(hcfg)
        tstep[0] += 1
        history[key].append((s, m, c))
        frame.copy_(pool[s])
        f_counts.copy_(counts[s])
        f_xy.copy_(dxy[s])
        f_T.copy_(dT[s])
        f_org.copy_(dorg[s])
        f_cfg.copy_(dcfg[c])
        f_mask.copy_(dmask[m])
        return s

    def sequence():
        g.set_point_counts_from_device_ptrs(slots, f_counts.data_ptr(), sp)
        g.update_poses_from_device_ptrs(slots, f_xy.data_ptr(), f_T.data_ptr(), f_org.data_ptr(), bz.data_ptr(), moved.data_ptr(), sp)
        g.run_scans_to_device_ptrs(descs, [t.data_ptr() for t in views], c_ptrs, 0, None, sp)
        last["labels"] = c_out.labels

    def enqueue(v):
        if v == "H":
            mask, cfg = f_mask.cpu().numpy(), f_cfg.cpu().numpy()   # a host wait for everything before on the stream
            for b in np.flatnonzero(mask):
                capi._check(g._l.gg_set_slot_config(g._h, int(b), C.byref(capi.Config.from_buffer_copy(cfg[b].tobytes()))))
            sequence()
        elif v == "D":
            g.set_configs_from_device_ptrs(slots, f_cfg.data_ptr(), f_mask.data_ptr(), sp)
            sequence()
        elif v == "P":
            plan.launch(cur)
            last["labels"] = plan.outputs.labels
        else:
            graph.replay()
            last["labels"] = plan.outputs.labels

    def timed(v):
        key = "call" if v in "HD" else "plan"
        for _ in range(args.warmup):
            write(key, False)
            enqueue(v)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
        host = 0.0
        ev[0].record(cur)
        for t in range(args.steps):
            write(key, t == args.steps // 2)
            t0 = time.perf_counter()
            enqueue(v)
            host += time.perf_counter() - t0
            ev[t + 1].record(cur)
        torch.cuda.synchronize()
        per = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.steps)]
        return {"ms_per_step": ev[0].elapsed_time(ev[-1]) / args.steps, "ms_step_median": float(np.median(per)),
                "host_enqueue_us_per_step": 1e6 * host / args.steps}

    # one twin per handle runs host gg_set_slot_config + the call sequence of the sampled streams on the pool's tensors
    rng = np.random.default_rng(1234)
    sample = np.array(sorted(rng.choice(B, min(args.check, B), replace=False).tolist()), np.int32)
    m = len(sample)
    twins = {}
    for key in ("call", "plan"):
        twins[key] = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=m, max_points=bench.PCAP, full_layers=False)
        for j in range(m):
            twins[key].init_map(0.0, 0.0, 0.0, slot=j)
    tslots = np.arange(m, dtype=np.int32)
    idx = torch.tensor(sample.astype(np.int64), device="cuda")
    replayed = {"call": 0, "plan": 0}
    checked = {}

    def check(v):
        key = "call" if v in "HD" else "plan"
        h, twin = handles[key], twins[key]
        torch.cuda.synchronize()
        out = None
        for s, mi, ci in history[key][replayed[key]:]:
            for j, b in enumerate(sample):
                if hmask[mi][b]:
                    capi._check(twin._l.gg_set_slot_config(twin._h, j, C.byref(capi.Config.from_buffer_copy(hcfg[ci][b].tobytes()))))
            data = [pool[s][int(first[b]):int(first[b]) + int(cap[b]) * 32] for b in sample]
            twin.set_point_counts_from_device(tslots, counts[s][idx])
            twin.update_poses_from_device(tslots, dxy[s][idx], dT[s][idx], dorg[s][idx], bz[idx])
            out = twin.run_scans_to_device(data, tslots, "device", None, labels=True, select=None, device_counts=True)
        replayed[key] = len(history[key])
        torch.cuda.synchronize()
        s = history[key][-1][0]
        for j, b in enumerate(sample):
            u = int(npts[b, s])
            assert torch.equal(last["labels"][b][:u], out.labels[j][:u]), f"{v} stream {b}: labels differ from the host configurations"
            for name in ("ground", "groundpatch"):
                assert np.array_equal(h.layer(name, slot=int(b)).view(np.uint32), twin.layer(name, slot=j).view(np.uint32)), f"{v} stream {b}: {name}"
            assert h.position(slot=int(b)).view(np.uint64).tolist() == twin.position(slot=j).view(np.uint64).tolist(), f"{v} stream {b}: position"
            assert bytes(h.get_config(slot=int(b))) == bytes(twin.get_config(slot=j)), f"{v} stream {b}: configuration"
        checked[v] = checked.get(v, 0) + m

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            check(v)
    changes = sum(int(hmask[mi].sum()) for key in history for _, mi, _ in history[key])
    steps = sum(len(x) for x in history.values())
    info = {"kernels_per_step": plan.kernels, "N": g.n, "points_per_step": float(npts.sum(0).mean()), "changes_per_step": changes / steps}
    del graph
    plan.close()
    for h in list(handles.values()) + list(twins.values()):
        h.close()
    return results, checked, info


def kernels_alone(torch, capi, B, reps):
    """k_store_configs and k_rebuild_detect_tables reconfiguring all B streams, timed with gg_profile: ms per launch,
    bytes written, GB/s, share of the data sheet; and the rebuild with every stream masked off.  The handle has one stream
    group, so one launch covers every stream."""
    saved = os.environ.get("GG_STREAMS")
    os.environ["GG_STREAMS"] = "1"
    try:
        g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=4096, full_layers=False)
    finally:
        if saved is None:
            del os.environ["GG_STREAMS"]
        else:
            os.environ["GG_STREAMS"] = saved
    assert g.n_streams == 1
    slots = np.arange(B, dtype=np.int32)
    cfg = torch.from_numpy(draw_configs(capi, np.random.default_rng(7), B)).cuda()
    mask = torch.ones(B, dtype=torch.int32, device="cuda")
    sp = torch.cuda.current_stream().cuda_stream or None
    for _ in range(3):
        g.set_configs_from_device_ptrs(slots, cfg.data_ptr(), mask.data_ptr(), sp)
    torch.cuda.synchronize()
    out = {}
    for case in ("all", "none"):
        if case == "none":
            mask.zero_()
        g.profile_enable(True)
        for _ in range(reps):
            g.set_configs_from_device_ptrs(slots, cfg.data_ptr(), mask.data_ptr(), sp)
        torch.cuda.synchronize()
        prof = g.profile_read()
        g.profile_enable(False)
        out[case] = {k: prof[k][0] / prof[k][1] for k in ("k_store_configs", "k_rebuild_detect_tables")}
    N = g.n
    g.close()
    tab_bytes = B * N * N * 16
    rec_bytes = B * (C.sizeof(capi.Config) + 120)
    res = {}
    for k, nbytes in (("k_rebuild_detect_tables", tab_bytes), ("k_store_configs", rec_bytes)):
        per = out["all"][k]
        res[k] = {"ms": per, "bytes": nbytes, "GBps": nbytes / (per * 1e-3) / 1e9, "share_of_datasheet": nbytes / (per * 1e-3) / DATASHEET_BPS,
                  "ms_none_masked": out["none"][k]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--check", type=int, default=16, help="streams of the seeded sample checked after each variant")
    ap.add_argument("--p", type=float, default=1.0 / 32, help="probability per stream and step of a new configuration")
    ap.add_argument("--kernel-reps", type=int, default=50)
    args = ap.parse_args()
    B, S = args.streams, args.pool

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_device_configs.py needs a CUDA device")
    card = gpu_info()
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))
    results, checked, info = run_workload(torch, capi, streams, B, S, args)
    kernel = kernels_alone(torch, capi, B, args.kernel_reps)
    card_after = gpu_info()
    print(f"card, power limit, max SM clock: {card} (after the run: {card_after})")
    print(f"{B} streams x {S} poses, {args.steps} timed steps per run, {args.reps} alternating runs, p = {args.p}")
    print(f"value: N = {info['N']}, {info['points_per_step'] / 1e6:.2f} M points per step, {info['changes_per_step']:.2f} reconfigured "
          f"streams per step, {info['kernels_per_step']} kernels per replayed step")
    print(f"  {'variant':<58} {'ms/step (runs)':<28} {'host enqueue us/step (runs)':<30}")
    for v, desc in VARIANTS.items():
        ms = " / ".join(f"{x['ms_per_step']:.3f}" for x in results[v])
        hu = " / ".join(f"{x['host_enqueue_us_per_step']:.0f}" for x in results[v])
        print(f"  {v + '  ' + desc:<58} {ms:<28} {hu:<30}")
    print(f"  bit-exact checks: {checked}")
    for k, r in kernel.items():
        print(f"{k}, {B} streams all reconfigured: {r['ms']:.3f} ms, {r['bytes'] / 1e6:.2f} MB written, {r['GBps']:.0f} GB/s = "
              f"{100 * r['share_of_datasheet']:.1f} % of the data-sheet 3.35 TB/s; none reconfigured: {r['ms_none_masked'] * 1e3:.1f} us")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "reps": args.reps, "p": args.p, "value": {"results": results,
                      "checked_streams": checked, **info}, "kernels": kernel}))


if __name__ == "__main__":
    main()
