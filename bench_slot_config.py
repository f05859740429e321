"""Cost of per-slot configurations (gg_set_slot_config) on the device-resident workload of bench.py.

    python bench_slot_config.py [--streams 396] [--steps 50] [--warmup 3] [--pool 4]

Same scans (bench.py's 64-beam streams, rolls between steps, clouds resident in HBM) in three setups:
  mixed     one handle, four configurations assigned slot by slot (slot b runs configuration b % 4)
  split     the same scans over four handles, one uniform configuration each
  uniform   one handle, one configuration (what bench.py measures)
plus the mixed handle with one slot reconfigured before every step, alternating between two configurations other
slots also use (no device work besides waiting for that slot's stream group) and between two no other slot uses (the
slot's variant is freed and its detect table rebuilt every step).  Both runs count the configuration changes and the
tables built (kernel launches of gg_set_slot_config) and check them against the number of steps.
A step is timed by the host clock from a device synchronize to the next, over all handles of the setup.  Prints one
JSON line; nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generators and the pose sequence of bench.py)

CFGS = [
    dict(),
    dict(max_ring=48, occupied_cells_decrease_factor=1.5, patch_size_change_distance=8.0, miminum_point_height_threshold=0.2,
         outlier_tolerance=0.25),
    dict(max_ring=40, occupied_cells_decrease_factor=2000.0, patch_size_change_distance=30.0, distance_factor=0.0003,
         minimum_distance_factor=0.001),
    dict(outlier_tolerance=0.02, min_outlier_detection_ground_confidence=2.0, miminum_point_height_threshold=0.45,
         point_count_cell_variance_threshold=20, occupied_cells_point_count_factor=35.0),
]


def full(kw):
    """Every field of a configuration (defaults where `kw` has none): set_config(**kw) changes only the fields it is
    given, so switching a slot between configurations needs all of them."""
    from groundgrid_b200 import capi

    c = capi.default_config()
    for k, v in kw.items():
        setattr(c, k, v)
    return {name: getattr(c, name) for name, _ in capi.Config._fields_}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=20)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pool", type=int, default=4, help="distinct ego poses / clouds per stream")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(1000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    npts = np.array([[len(streams[b][s][0]) for s in range(S)] for b in range(B)], np.int64)
    offs = np.zeros((B, S), np.int64)
    host = np.zeros(int(npts.sum()) * 32, np.uint8)
    o = 0
    for b in range(B):
        for s in range(S):
            raw = np.ascontiguousarray(streams[b][s][0]).view(np.uint8).reshape(-1)
            host[o:o + raw.size] = raw
            offs[b, s] = o
            o += raw.size
    dev = torch.from_numpy(host).cuda()
    pts_per_pose = npts.sum(axis=0)

    def make(slots, cfg_of_slot=None, uniform=None):
        g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=len(slots), max_points=bench.PCAP, full_layers=False)
        if uniform is not None:
            g.set_config(**full(uniform))
        for k, b in enumerate(slots):
            if cfg_of_slot is not None:
                g.set_config(slot=k, **full(cfg_of_slot(b)))
            g.init_map(0.0, 0.0, 0.0, slot=k)
        descs = [g.make_descs(list(range(len(slots))), [int(npts[b, s]) for b in slots], [streams[b][s][1] for b in slots], [0.0] * len(slots))
                 for s in range(S)]
        ptrs = [[dev.data_ptr() + int(offs[b, s]) for b in slots] for s in range(S)]
        xy = [np.tile(np.array([float(s), 0.0]), (len(slots), 1)) for s in range(S)]
        Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (len(slots), 1)) for s in range(S)]
        return g, descs, ptrs, xy, Ts, np.arange(len(slots), dtype=np.int32)

    def timed(handles, before_step=None):
        t = [0]

        def step():
            s = bench.pingpong(t[0], S)
            if before_step:
                before_step(t[0])
            for g, descs, ptrs, xy, Ts, sl in handles:
                if t[0]:
                    g.update_pose_batch(sl, xy[s], Ts[s])
                g.run_scans_device(descs[s], ptrs[s])
            t[0] += 1
            return s

        for _ in range(args.warmup):
            step()
        for h in handles:
            h[0].synchronize()
        torch.cuda.synchronize()
        pts = 0
        t0 = time.perf_counter()
        for _ in range(args.steps):
            pts += int(pts_per_pose[step()])
        for h in handles:
            h[0].synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        return {"ms_per_step": ms / args.steps, "mpoints_per_s": pts / (ms * 1e-3) / 1e6}

    out = {"gpu": gpu_info(), "streams": B, "steps": args.steps, "points_per_scan_mean": float(npts.mean()),
           "timing": "host clock between device synchronizes"}
    every = list(range(B))
    h = make(every, cfg_of_slot=lambda b: CFGS[b % 4])
    out["mixed_4_configs_one_handle"] = timed([h])

    def reconfigure(cfgs, record):
        """Before step t slot 0 gets cfgs[t % 2]; counts the configuration changes and the detect tables built."""
        def before(t):
            old = bytes(h[0].get_config(slot=0))
            n0 = h[0].kernel_launches
            h[0].set_config(slot=0, **full(cfgs[t % 2]))
            record["changes"] += bytes(h[0].get_config(slot=0)) != old
            record["tables_built"] += h[0].kernel_launches - n0
        return before

    steps_total = args.warmup + args.steps
    # slot 0 alternates between configurations 1 and 0, both in use by other slots: no device data is built
    rec = {"changes": 0, "tables_built": 0}
    r = timed([h], reconfigure([CFGS[1], CFGS[0]], rec))
    assert rec["changes"] == steps_total and rec["tables_built"] == 0, rec
    out["mixed_reconfigure_one_slot_shared"] = dict(r, **rec)
    # slot 0 alternates between two configurations no other slot uses: every step frees its variant and rebuilds it
    fresh = [dict(CFGS[2], outlier_tolerance=0.33), dict(CFGS[2], outlier_tolerance=0.34)]
    rec = {"changes": 0, "tables_built": 0}
    r = timed([h], reconfigure(fresh, rec))
    assert rec["changes"] == steps_total and rec["tables_built"] == steps_total, rec
    out["mixed_reconfigure_one_slot_new"] = dict(r, **rec)
    h[0].close()
    hs = [make([b for b in every if b % 4 == c], uniform=CFGS[c]) for c in range(4)]
    out["split_4_uniform_handles"] = timed(hs)
    for x in hs:
        x[0].close()
    h = make(every)
    out["uniform_one_handle"] = timed([h])
    h[0].close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
