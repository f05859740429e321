"""Map snapshots on the GPU: gg_save_maps_to_device and gg_restore_maps_from_device against the host recipe a caller
needs without them, and a step plan with and without a restore stage.

    python bench_map_snapshots.py [--streams 396] [--reps 50] [--plan-steps 32]

On bench.py's geometry (99 m at 0.33 m: N = 300, 720 kB of planes per slot) with --streams slots:
  save        gg_save_maps_to_device of every slot
  restore     gg_restore_maps_from_device of every slot (index NULL)
  restore10   the same call with about 10 % of the indices inside the pool (the others leave their slot untouched)
  host        the recipe without snapshots: gg_get_layers_to_device ("ground", "groundpatch") + gg_get_map_position and
              gg_init_map per slot (each waits on the host) + gg_set_layers_from_device
The call times are CUDA events around --reps calls on torch's current stream (handle with one stream group, so one
launch covers every slot); the host recipe is a host clock around whole recipes ending in a synchronise.  The kernels
alone come from gg_profile.  Each is set against the byte lower bound computed from shapes (not measured): a save reads
and writes 8 N^2 bytes per slot, a restore reads 8 N^2 and writes n_layers * 4 N^2, at the H100 SXM data-sheet HBM3
bandwidth of 3.35 TB/s.  Then a step plan over bench.py's `value` clouds (counts, device poses, scan, labels to the
device) with and without a restore stage of 10 % valid indices, replayed --plan-steps times: ms per step from CUDA events.
A bit-exact check restores every slot from a pool saved in reverse slot order and saves again.  Prints the card and its
power limit (read in the same run), a table and one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generator and geometry of bench.py)
from bench_slot_config import gpu_info  # noqa: E402

DATASHEET_BPS = 3.35e12   # H100 SXM HBM3, NVIDIA data sheet (not a measured peak)


def one_group_handle(capi, B, max_points):
    saved = os.environ.get("GG_STREAMS")
    os.environ["GG_STREAMS"] = "1"
    try:
        return capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=max_points, full_layers=False)
    finally:
        if saved is None:
            del os.environ["GG_STREAMS"]
        else:
            os.environ["GG_STREAMS"] = saved


def event_ms(torch, fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def calls(torch, capi, B, reps):
    g = one_group_handle(capi, B, 4096)
    assert g.n_streams == 1
    N = g.n
    slots = np.arange(B, dtype=np.int32)
    rng = np.random.default_rng(11)
    for s in range(B):
        g.init_map(float(s), -0.5 * s, 0.01 * s, slot=s)
    planes = torch.tensor(rng.uniform(-2.0, 2.0, (B, 2, N, N)).astype(np.float32), device="cuda")
    g.set_layers_from_device(slots, ["ground", "groundpatch"], planes)
    rb = g.snapshot_bytes
    pool = torch.empty((B, rb), dtype=torch.uint8, device="cuda")
    sp = torch.cuda.current_stream().cuda_stream or None
    g.save_maps_to_device(slots, out=pool)
    # bit-exact check: restore slot k from record B-1-k, save again
    rev = torch.tensor(np.arange(B - 1, -1, -1, dtype=np.int32), device="cuda")
    status = g.restore_maps_from_device(slots, pool, rev, status=True)
    again = g.save_maps_to_device(slots)
    torch.cuda.synchronize()
    exact = bool((status == 1).all()) and torch.equal(again, pool.flip(0))
    idx10 = torch.tensor(np.where(rng.random(B) < 0.1, np.arange(B), -1).astype(np.int32), device="cuda")
    valid10 = int((idx10 >= 0).sum())
    out = {}
    out["save"] = event_ms(torch, lambda: g.save_maps_to_device_ptrs(slots, pool.data_ptr(), None, sp), reps)
    out["restore"] = event_ms(torch, lambda: g.restore_maps_from_device_ptrs(slots, pool.data_ptr(), B, None, None, sp), reps)
    out["restore10"] = event_ms(torch, lambda: g.restore_maps_from_device_ptrs(slots, pool.data_ptr(), B, idx10.data_ptr(), None, sp), reps)
    # kernels alone
    kern = {}
    for key, fn, name in (("save", lambda: g.save_maps_to_device_ptrs(slots, pool.data_ptr(), None, sp), "k_save_maps"),
                          ("restore", lambda: g.restore_maps_from_device_ptrs(slots, pool.data_ptr(), B, None, None, sp), "k_reset_maps_restore"),
                          ("restore10", lambda: g.restore_maps_from_device_ptrs(slots, pool.data_ptr(), B, idx10.data_ptr(), None, sp),
                           "k_reset_maps_restore")):
        torch.cuda.synchronize()
        g.profile_enable(True)
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        ms, n = g.profile_read()[name]
        g.profile_enable(False)
        kern[key] = ms / n
    # the host recipe
    buf = torch.empty((B, 2, N, N), dtype=torch.float32, device="cuda").transpose(-1, -2)
    hrep = max(2, reps // 10)

    def recipe():
        g.get_layers_to_device(slots, ["ground", "groundpatch"], out=buf)
        for s in range(B):
            x, y = g.position(slot=s)
            g.init_map(x, y, 0.0, slot=s)
        g.set_layers_from_device(slots, ["ground", "groundpatch"], buf)
        torch.cuda.synchronize()

    recipe()
    t0 = time.perf_counter()
    for _ in range(hrep):
        recipe()
    out["host"] = (time.perf_counter() - t0) * 1e3 / hrep
    n_layers = 6
    bound = {"save": B * 2 * 8 * N * N / DATASHEET_BPS * 1e3, "restore": B * (8 + 4 * n_layers) * N * N / DATASHEET_BPS * 1e3,
             "restore10": valid10 * (8 + 4 * n_layers) * N * N / DATASHEET_BPS * 1e3}
    bound["host"] = bound["restore"]
    g.close()
    return {"N": N, "record_bytes": rb, "ms": out, "kernel_ms": kern, "bound_ms": bound, "valid10": valid10, "bit_exact": exact}


def plans(torch, capi, B, steps):
    streams = bench.generate_streams(2000, B, 1, max(1, min(32, (os.cpu_count() or 2) - 1)))
    npts = np.array([len(streams[b][0][0]) for b in range(B)], np.int64)
    g = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=False)
    for b in range(B):
        g.init_map(0.0, 0.0, 0.0, slot=b)
    slots = np.arange(B, dtype=np.int32)
    clouds = [torch.from_numpy(np.ascontiguousarray(streams[b][0][0]).view(np.uint8).copy()).cuda() for b in range(B)]
    counts = torch.tensor(npts.astype(np.int32), device="cuda")
    xy = torch.zeros((B, 2), dtype=torch.float64, device="cuda")
    T = torch.tensor(np.tile(bench.pose_T(0)[2].reshape(1, 12), (B, 1)), device="cuda")
    org = torch.tensor(np.array([streams[b][0][1] for b in range(B)], np.float32), device="cuda")
    bz = torch.zeros(B, dtype=torch.float64, device="cuda")
    kw = dict(counts=counts, xy=xy, T_base_from_map=T, pose_origins=org, pose_base_z=bz, labels=True, select=None)
    pool = g.save_maps_to_device(slots)
    rng = np.random.default_rng(12)
    idx = torch.tensor(np.where(rng.random(B) < 0.1, np.arange(B), -1).astype(np.int32), device="cuda")
    out = {}
    for key, extra in (("plain", {}), ("restore10", dict(restore_pool=pool, restore_index=idx))):
        plan = g.step_plan(slots, clouds=clouds, **kw, **extra)
        out[key] = {"ms_per_step": event_ms(torch, plan.launch, steps), "kernels": plan.kernels}
        plan.close()
    g.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--plan-steps", type=int, default=32)
    args = ap.parse_args()
    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_map_snapshots.py needs a CUDA device")
    card = gpu_info()
    c = calls(torch, capi, args.streams, args.reps)
    p = plans(torch, capi, args.streams, args.plan_steps)
    card_after = gpu_info()
    B = args.streams
    print(f"card, power limit, max SM clock: {card} (after the run: {card_after})")
    print(f"{B} slots at N = {c['N']}, record {c['record_bytes']} bytes; bit-exact reverse restore + save: {c['bit_exact']}")
    print(f"  {'call':<12} {'ms per call':>12} {'kernel ms':>10} {'byte bound ms':>14} {'bound / call':>13}")
    for k in ("save", "restore", "restore10", "host"):
        km = c["kernel_ms"].get(k)
        print(f"  {k:<12} {c['ms'][k]:>12.3f} {('%.3f' % km) if km else '-':>10} {c['bound_ms'][k]:>14.3f} {c['bound_ms'][k] / c['ms'][k]:>12.0%}")
    print(f"  restore10: {c['valid10']} of {B} indices valid")
    for k, r in p.items():
        print(f"plan {k:<10}: {r['ms_per_step']:.3f} ms per step, {r['kernels']} kernels")
    print(json.dumps({"gpu": card, "streams": B, "reps": args.reps, "calls": c, "plans": p}))


if __name__ == "__main__":
    main()
