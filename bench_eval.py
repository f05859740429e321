"""Cost of the evaluator's tallies (scripts/eval_groundpoint_classifier.py:95-118) for every stream of bench.py's `value`
workload, and a configuration sweep scored from them.

    python bench_eval.py [--streams 396] [--pool 8] [--steps 40] [--warmup 3] [--reps 3] [--slow-steps 3]

Same scans as `value` (64-beam streams, N = 300, rolls between steps, labels only), but each cloud is generated with
synth.lidar_scan(..., labels=True) and carries the SemanticKITTI id of the surface its ray hit in `ring`, as the KITTI
player sends it.  The ids are 10, 40 and 50, all below the default max_ring (1024), so the scans are those of `value`.
One step = one scan of every stream, ordered on torch's current stream and timed with CUDA events recorded on it.
Variants, alternated --reps times in one run:
  B  gg_run_scans_to_device on the 32-byte records in HBM, labels only
  E  B + gg_eval_counts_to_device of every slot, added into one running int64 [streams, 1024, 2] tensor
  K  gg_run_cloud_msgs_to_device on 18-byte sensor-frame payloads (x, y, z, intensity, label: the KITTI player's layout)
     + the tallies of E
  L  B + the per-slot route: gg_eval_accumulate + gg_eval_read(reset=1) per slot (--slow-steps steps only)
After each variant the tallies of a seeded sample of --check slots (one batched call) are checked bit-exact against the
per-slot route.  A serialised pass (one stream group, gg_profile) times k_eval_counts alone against its byte model:
per point the label byte and the 32-byte sector that holds the ring (33 B).  The sweep runs --sweep-steps steps of four
configurations x (streams / 4) streams on one handle and scores each configuration from its slots' summed tallies.
Its configurations differ from bench_slot_config.py's: those lower max_ring, and with the label in `ring` a max_ring
below 50 would keep every wall point out of the map.  Prints the card, its power limit, a table and one JSON line;
writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the pose sequence and geometry of bench.py)
from bench_cloud_msgs import map_from_sensor, payload  # noqa: E402
from bench_slot_config import gpu_info  # noqa: E402

VARIANTS = {
    "B": "run_scans_to_device, labels only",
    "E": "B + eval_counts_to_device of every slot",
    "K": "run_cloud_msgs_to_device, 18-byte payloads + E's tallies",
    "L": "B + eval_accumulate + eval_read(reset) per slot",
}
KITTI18 = (0, 4, 8, 12, 16)
BYTES_PER_POINT = 33   # the label byte + the 32-byte record (sector) that holds the ring
DATASHEET_TBS = 3.35   # H100 SXM5 80 GB data sheet, not measured
# four configurations of the sweep, max_ring left at its default
SWEEP = [
    {},
    dict(miminum_point_height_threshold=0.2, minimum_point_height_obstacle_threshold=0.05),
    dict(outlier_tolerance=0.05, patch_size_change_distance=30.0, distance_factor=0.0003),
    dict(occupied_cells_decrease_factor=1.5, min_outlier_detection_ground_confidence=0.6, point_count_cell_variance_threshold=20),
]


def _gen_labelled(args):
    """bench.py's scan of (stream, pose), generated with labels; the ids go into `ring`."""
    from groundgrid_b200 import synth

    seed, pose, n_pose = args
    scene = synth.make_scene(seed=seed, stream_len=float(n_pose))
    pts, org, ids = synth.scan_64(scene, ego_xy=(float(pose), 0.0), yaw=0.0, seed=seed * 31 + pose, labels=True)
    pts["ring"] = ids
    return pts[:bench.PCAP], org


def generate(first_seed, n_streams, n_pose, procs):
    tasks = [(first_seed + b, s, n_pose) for b in range(n_streams) for s in range(n_pose)]
    if procs > 1:
        import multiprocessing as mp

        with mp.get_context("fork").Pool(procs) as pool:
            res = pool.map(_gen_labelled, tasks, chunksize=1)
    else:
        res = [_gen_labelled(t) for t in tasks]
    return [[res[b * n_pose + s] for s in range(n_pose)] for b in range(n_streams)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--slow-steps", type=int, default=3, help="timed steps of variant L")
    ap.add_argument("--prof-steps", type=int, default=10, help="profiled tally rounds of the serialised pass")
    ap.add_argument("--sweep-steps", type=int, default=14, help="steps of the configuration sweep (one pose cycle at --pool 8)")
    ap.add_argument("--check", type=int, default=16, help="slots of the seeded sample checked after every variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = generate(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi, evalmetrics

    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    origins = [np.array([streams[b][s][1] for b in range(B)], np.float32) for s in range(S)]
    Tsensor = [np.stack([map_from_sensor(streams[b][s][1], 0.013 * b + 0.2 * s, 0.02) for b in range(B)]) for s in range(S)]

    def upload(make, step):
        views = []
        for s in range(S):
            flat = torch.empty(int(npts[:, s].sum()) * step, dtype=torch.uint8, device="cuda")
            o, vs = 0, []
            for b in range(B):
                raw = make(b, s).reshape(-1)
                flat[o:o + raw.size] = torch.from_numpy(raw)
                vs.append(flat[o:o + raw.size])
                o += raw.size
            views.append(vs)
        return views

    clouds = upload(lambda b, s: np.ascontiguousarray(streams[b][s][0]).view(np.uint8), 32)
    k18 = upload(lambda b, s: payload(streams[b][s][0], Tsensor[s][b], 18), 18)
    del streams
    pts_per_pose = npts.sum(axis=0)

    def make_handle(cfgs=None):
        h = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
        for b in range(B):
            if cfgs:
                h.set_config(slot=b, **cfgs[b * len(cfgs) // B])
            h.init_map(0.0, 0.0, 0.0, slot=b)
        return h

    g = make_handle()
    slots = np.arange(B, dtype=np.int32)
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    cur = torch.cuda.current_stream()
    acc = torch.zeros((B, 1024, 2), dtype=torch.int64, device="cuda")
    tstep = [0]

    def scan(h, variant):
        s = bench.pingpong(tstep[0], S)
        if tstep[0]:
            h.update_pose_batch(slots, xy[s], Ts[s])
        tstep[0] += 1
        if variant == "K":
            h.run_cloud_msgs_to_device(k18[s], 18, KITTI18, Tsensor[s], slots, origins[s], 0.0, labels=True, select=None)
        else:
            h.run_scans_to_device(clouds[s], slots, origins[s], 0.0, labels=True, select=None)
        return s

    def step(variant):
        s = scan(g, variant)
        if variant in ("E", "K"):
            g.eval_counts_to_device(slots, out=acc)
        elif variant == "L":
            for b in range(B):
                g.eval_accumulate(b)
                g.eval_read(reset=True)
        return int(pts_per_pose[s])

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
    sample = np.array(sorted(rng.choice(B, min(args.check, B), replace=False).tolist()), np.int32)
    checked = {}

    def check(variant):
        got = g.eval_counts_to_device(sample)
        torch.cuda.synchronize()
        got = got.cpu().numpy().view(np.uint64)
        for k, b in enumerate(sample):
            g.eval_accumulate(int(b))
            want = g.eval_read(reset=True)
            assert np.array_equal(got[k], want), f"{variant}: slot {b} differs from the per-slot route"
            assert want.sum() > 0
        checked[variant] = checked.get(variant, 0) + len(sample)

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            check(v)
    g.close()

    # serialised pass: one stream group, the kernel's own time from gg_profile
    old = os.environ.get("GG_STREAMS")
    os.environ["GG_STREAMS"] = "1"
    g1 = make_handle()
    if old is None:
        del os.environ["GG_STREAMS"]
    else:
        os.environ["GG_STREAMS"] = old
    tstep[0] = 0
    s = scan(g1, "B")
    one = torch.zeros_like(acc)
    g1.eval_counts_to_device(slots, out=one)
    g1.synchronize()
    torch.cuda.synchronize()
    g1.profile_enable(True)
    g1.profile_read(reset=True)
    for _ in range(args.prof_steps):
        g1.eval_counts_to_device(slots, out=one)
    prof = g1.profile_read(reset=True)
    g1.profile_enable(False)
    g1.close()
    ms, n_launch = prof["k_eval_counts"]
    per = ms / args.prof_steps
    gbytes = BYTES_PER_POINT * int(pts_per_pose[s]) / 1e9
    kernel = {"ms_per_round": per, "launches": n_launch, "points": int(pts_per_pose[s]), "model_gb": gbytes, "tb_per_s": gbytes / per,
              "share_of_datasheet": gbytes / per / DATASHEET_TBS}

    # the sweep: four configurations, B / 4 streams each, scored from their slots' summed tallies
    gs = make_handle(SWEEP)
    tstep[0] = 0
    run = torch.zeros_like(acc)
    for _ in range(args.sweep_steps):
        scan(gs, "B")
        gs.eval_counts_to_device(slots, out=run)
    torch.cuda.synchronize()
    per_cfg = run.view(len(SWEEP), B // len(SWEEP), 1024, 2).sum(dim=1).cpu().numpy()
    gs.close()
    sweep = []
    for c, kw in enumerate(SWEEP):
        m = evalmetrics.metrics(per_cfg[c])
        sweep.append({"config": kw, **{k: m[k] for k in ("precision", "recall", "f1", "iou_ground", "tp", "fp", "fn", "tn")}})

    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, N = {int(bench.DIM_M / bench.RES + 0.5)}, {float(npts.mean()):.0f} points per scan, "
          f"{args.steps} timed steps per run ({args.slow_steps} for L), {args.reps} alternating runs")
    print(f"{'variant':<62} {'ms/step (runs)':<28}")
    for v, desc in VARIANTS.items():
        ms_ = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<62} {' / '.join(f'{x:.3f}' for x in ms_):<28}")
    print(f"k_eval_counts (serialised, {B} slots, {kernel['points'] / 1e6:.1f} M points): {per:.3f} ms, byte model "
          f"{gbytes:.3f} GB -> {kernel['tb_per_s']:.2f} TB/s = {100 * kernel['share_of_datasheet']:.0f} % of the data sheet's "
          f"{DATASHEET_TBS} TB/s (not a measured peak)")
    print(f"sweep: {len(SWEEP)} configurations x {B // len(SWEEP)} streams, {args.sweep_steps} steps")
    for r in sweep:
        print(f"  {json.dumps(r['config']):<120} precision {r['precision']:.5f} recall {r['recall']:.5f} F1 {r['f1']:.5f} "
              f"IoU {r['iou_ground']:.5f}")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "steps": args.steps, "slow_steps": args.slow_steps, "reps": args.reps,
                      "points_per_scan_mean": float(npts.mean()), "checked_slots": checked, "results": results, "kernel": kernel,
                      "sweep": sweep}))


if __name__ == "__main__":
    main()
