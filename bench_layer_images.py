"""Cost of the images publish_grid_map_layer makes every scan (the 8-bit layer images and the terrain image), for many
slots at once, on the device-resident workload of bench.py's `value`.

    python bench_layer_images.py [--streams 396] [--pool 8] [--steps 20] [--warmup 3] [--reps 3] [--slow-steps 3]

Same scans as `value` (64-beam streams, clouds resident in HBM, rolls between steps), one step = one scan of every
stream through gg_run_scans_to_device (labels only), ordered on the caller's stream (torch's current stream) and timed
with CUDA events recorded on it.  The handle has GG_FLAG_FULL_LAYERS, because the terrain image reads "pointsRaw": that
is NOT the configuration of `value` (which runs without the full layers), so B here is not bench.py's number.
Variants, alternated --reps times in one run:
  B   the scans alone (labels into caller memory)
  I2  B + gg_layer_images_to_device of "ground" and "groundpatch" of every slot
  IA  B + the images of all eleven layers of the map + gg_terrain_images_to_device (what :216-228 publishes)
  Q   B + the same as IA written in torch on top of gg_get_layers_to_device (bit-exact restatement)
  L   B + the per-slot gg_layer_image_u8 / gg_terrain_image of IA (--slow-steps steps only)
After each variant a seeded sample of slots is checked bit-exact against the per-slot calls.  A serialised pass (one
stream group, gg_profile) then times the image kernels of IA alone against their byte model: 9 N^2 bytes per layer
image (4 N^2 read by the range pass, 4 N^2 read + N^2 written by the image pass), 20 N^2 per terrain image (8 N^2 read,
12 N^2 written).  Prints the card, its power limit, a table and one JSON line; writes nothing.
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

TERRAIN = ("ground", "groundpatch")
# the eleven layers of the reference's map (GroundSegmentation.cpp:15-27), each published as an image (:219-228)
ELEVEN = ("points", "ground", "groundpatch", "minGroundHeight", "maxGroundHeight", "variance", "groundCandidates", "planeDist",
          "m2", "meanVariance", "pointsRaw")
VARIANTS = {
    "B": "to_device: labels",
    "I2": "B + images of ground, groundpatch",
    "IA": "B + images of eleven layers + terrain",
    "Q": "B + IA in torch on get_layers_to_device",
    "L": "B + IA per slot (gg_layer_image_u8 / gg_terrain_image)",
}
HBM_TBPS = 3.35   # data sheet peak of the H100 SXM5 80 GB, not measured
KEY_POS_INF, KEY_NEG_INF = 0x7F800000, 0x807FFFFF - (1 << 32)   # ordered keys of +inf / -inf


def torch_layer_images(torch, planes):
    """toImage<unsigned char, 1> of planes [k, l, i, j] (any strides) with the ordered min / max (-0 below +0):
    (uint8 [k, l, N, N] row-major, float32 [k, l, 2])."""
    fin = torch.isfinite(planes)
    b = planes.contiguous().view(torch.int32)
    key = b ^ ((b >> 31) & 0x7FFFFFFF)
    big = torch.iinfo(torch.int32).max
    lo_k = torch.where(fin, key, big).amin(dim=(-2, -1))
    hi_k = torch.where(fin, key, -big - 1).amax(dim=(-2, -1))
    lo_k = torch.where(lo_k == big, torch.full_like(lo_k, KEY_POS_INF), lo_k)   # no finite cell: the range (+inf, -inf)
    hi_k = torch.where(hi_k == -big - 1, torch.full_like(hi_k, KEY_NEG_INF), hi_k)
    unkey = lambda k: (k ^ ((k >> 31) & 0x7FFFFFFF)).view(torch.float32)   # noqa: E731
    lo, hi = unkey(lo_k), unkey(hi_k)
    x = planes.contiguous()
    t = ((x - lo[..., None, None]) / (hi - lo)[..., None, None]) * 255.0
    img = torch.where(fin & (t == t), t.to(torch.int32).to(torch.uint8), torch.zeros((), dtype=torch.uint8, device=planes.device))
    return img, torch.stack((lo, hi), dim=-1)


def torch_terrain_images(torch, ground, raw):
    """[k, i, j] planes -> float32 [k, N, N, 3]; the 3x3 sum in the order of the kernels' tree9, border cells 0."""
    n = raw.shape[-1]
    e = [raw[:, q % 3:n - 2 + q % 3, q // 3:n - 2 + q // 3] for q in range(9)]   # cell (i - 1 + q % 3, j - 1 + q / 3)
    s = ((e[0] + e[1]) + (e[2] + e[3])) + ((e[4] + e[5]) + (e[6] + (e[7] + e[8])))
    vis = torch.zeros_like(raw)
    vis[:, 1:-1, 1:-1] = (s >= 27.0).to(torch.float32)
    return torch.stack((ground, vis, raw), dim=-1).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=396)
    ap.add_argument("--pool", type=int, default=8, help="distinct ego poses / clouds per stream")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--slow-steps", type=int, default=3, help="timed steps of variant L")
    ap.add_argument("--prof-steps", type=int, default=10, help="profiled image rounds of the serialised pass")
    ap.add_argument("--check", type=int, default=16, help="slots of the seeded sample checked after every variant")
    args = ap.parse_args()
    B, S = args.streams, args.pool
    streams = bench.generate_streams(2000, B, S, max(1, min(32, (os.cpu_count() or 2) - 1)))

    import torch

    from groundgrid_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("bench_layer_images.py needs a CUDA device")
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

    def make_handle():
        h = capi.GroundGridB200(bench.DIM_M, bench.RES, n_slots=B, max_points=bench.PCAP, full_layers=True)
        for b in range(B):
            h.init_map(0.0, 0.0, 0.0, slot=b)
        return h

    g = make_handle()
    N = g.n
    slots = np.arange(B, dtype=np.int32)
    xy = [np.tile(np.array([float(s), 0.0]), (B, 1)) for s in range(S)]
    Ts = [np.tile(bench.pose_T(s)[2].reshape(1, 12), (B, 1)) for s in range(S)]
    cur = torch.cuda.current_stream()
    tstep = [0]
    last = {}

    def scan(h):
        s = bench.pingpong(tstep[0], S)
        if tstep[0]:
            h.update_pose_batch(slots, xy[s], Ts[s])
        tstep[0] += 1
        h.run_scans_to_device(clouds[s], slots, origins[s], 0.0, labels=True, select=None)

    def step(variant):
        scan(g)
        if variant == "I2":
            last["img"] = g.layer_images_to_device(slots, TERRAIN)
        elif variant == "IA":
            last["img"] = g.layer_images_to_device(slots, ELEVEN)
            last["ter"] = g.terrain_images_to_device(slots)
        elif variant == "Q":
            planes = g.get_layers_to_device(slots, ELEVEN)
            last["img"] = torch_layer_images(torch, planes)
            last["ter"] = torch_terrain_images(torch, planes[:, 1], planes[:, 10])
        elif variant == "L":
            for b in range(B):
                for name in ELEVEN:
                    g.layer_image_u8(name, slot=b)
                g.terrain_image(slot=b)

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
        """The images of the last step of `variant` (or, for B and L, a fresh batched call) against the per-slot calls."""
        if variant in ("B", "L"):
            last["img"] = g.layer_images_to_device(slots, ELEVEN)
            last["ter"] = g.terrain_images_to_device(slots)
        torch.cuda.synchronize()
        img, rg = (t.cpu().numpy() for t in last["img"])
        names = TERRAIN if variant == "I2" else ELEVEN
        for b in sample:
            for l, name in enumerate(names):
                want, lo, hi = g.layer_image_u8(name, slot=b)
                assert np.array_equal(img[b, l], want), f"{variant} slot {b}: image of {name}"
                assert np.array_equal(rg[b, l].view(np.uint32), np.array([lo, hi], np.float32).view(np.uint32)), f"{variant} slot {b}: range of {name}"
            if variant != "I2":
                ter = last["ter"][b].cpu().numpy()
                assert np.array_equal(ter.view(np.uint32), g.terrain_image(slot=b).view(np.uint32)), f"{variant} slot {b}: terrain"
        checked[variant] = checked.get(variant, 0) + len(sample)
        last.clear()

    results = {v: [] for v in VARIANTS}
    for _ in range(args.reps):
        for v in VARIANTS:
            results[v].append(timed(v))
            check(v)
    g.close()

    # serialised pass: one stream group, the image kernels' own time from gg_profile
    old = os.environ.get("GG_STREAMS")
    os.environ["GG_STREAMS"] = "1"
    g1 = make_handle()
    if old is None:
        del os.environ["GG_STREAMS"]
    else:
        os.environ["GG_STREAMS"] = old
    for _ in range(2):
        scan(g1)
    g1.layer_images_to_device(slots, ELEVEN)
    g1.terrain_images_to_device(slots)
    g1.synchronize()
    torch.cuda.synchronize()
    g1.profile_enable(True)
    g1.profile_read(reset=True)
    for _ in range(args.prof_steps):
        g1.layer_images_to_device(slots, ELEVEN)
        g1.terrain_images_to_device(slots)
    prof = g1.profile_read(reset=True)
    g1.profile_enable(False)
    g1.close()
    plane = N * N
    model = {"k_layer_range": 4 * plane * B * len(ELEVEN), "k_layer_image": 5 * plane * B * len(ELEVEN), "k_terrain_image": 20 * plane * B}
    kernels = {}
    for name, nbytes in model.items():
        ms, n_launch = prof[name]
        per = ms / args.prof_steps
        kernels[name] = {"ms_per_round": per, "launches": n_launch, "model_gb": nbytes / 1e9, "tb_per_s": nbytes / 1e9 / per,
                         "share_of_datasheet": nbytes / 1e9 / per / HBM_TBPS}

    card = gpu_info()
    print(f"card, power limit, max SM clock: {card}")
    print(f"{B} streams x {S} poses, N = {N}, full layers (not the configuration of `value`), {args.steps} timed steps per run "
          f"({args.slow_steps} for L), {args.reps} alternating runs")
    print(f"{'variant':<62} {'ms/step (runs)':<28}")
    for v, desc in VARIANTS.items():
        ms = [r["ms_per_step"] for r in results[v]]
        print(f"{v + '  ' + desc:<62} {' / '.join(f'{x:.3f}' for x in ms):<28}")
    for name, k in kernels.items():
        print(f"{name} (serialised, IA's images of {B} slots): {k['ms_per_round']:.3f} ms, byte model {k['model_gb']:.3f} GB -> "
              f"{k['tb_per_s']:.2f} TB/s = {100 * k['share_of_datasheet']:.0f} % of the data sheet's {HBM_TBPS} TB/s (not a measured peak)")
    print(json.dumps({"gpu": card, "streams": B, "pool": S, "N": N, "full_layers": True, "steps": args.steps, "slow_steps": args.slow_steps,
                      "reps": args.reps, "checked_slots": checked, "results": results, "kernels": kernels}))


if __name__ == "__main__":
    main()
