"""Per-path maps (pqp_plan_create_maps, the mapped plan calls, set_occupancy_slots*; include/pqp_plan.h) on one GPU.

Prints one JSON line with the GPU's name and power limit read in the same run, and:
  - B = 1024 plan_points_device calls (TENSION2, from reference points) over M in {1, 64, 1024} distinct demo-sized
    maps, path b on map b % M: each map is the demo image with its own random 1.8 m blocks, all M built by one
    set_occupancy_slots_device call. ms per call (CUDA events, median of --steps calls), stage ms, status histogram;
  - on the same inputs and handle, alternated call by call with the mapped call, the unmapped plan_points_device on
    slot 0: what the slot lookup costs the shared-map path;
  - today's alternative at M = 64: 64 single-map planners, each planning its 16 paths, one after another on one
    stream;
  - set_occupancy_slots_device of 1024 demo images against 1024 set_occupancy_device calls.
Writes nothing to the source tree.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_plan import gpu_info  # noqa: E402


def _timed(fn):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def _blocked(demo, rng, count, res):
    """`count` copies of the demo image, each with 12 random 1.8 m (9-cell) obstacle blocks."""
    rows, cols = demo.shape
    out = np.repeat(demo[None], count, axis=0)
    side = int(round(1.8 / res))
    for k in range(count):
        for i, j in zip(rng.integers(0, rows - side, 12), rng.integers(0, cols - side, 12)):
            out[k, i:i + side, j:j + side] = 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    import torch
    from PIL import Image

    from path_optimizer_2_b200 import plan, sharedmap
    dev = torch.device("cuda:0")
    res = sharedmap.RES
    demo = np.asarray(Image.open(os.path.join(ROOT, "tests", "golden", "gridmap.png")).convert("L")).astype(np.uint8)
    dmap = sharedmap.DistanceMap()
    R, P, L, N, B = 64, 64, 64, 255, args.batch
    ref_x, ref_y, start, target = sharedmap.make_plan_points(B, dmap=dmap)
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_in = [t(px), t(py), t(m), t(start), t(target)]
    rng = np.random.default_rng(3)
    result = {"metric": "ms_per_mapped_plan_points_device", "gpu": gpu_info(), "batch": B, "steps": args.steps,
              "warmup": args.warmup, "method": "TENSION2", "maps": {}}
    zero = np.zeros(demo.shape, np.float32)
    for M in (1, 64, 1024):
        imgs = t(_blocked(demo, rng, M, res))
        pl = plan.Planner.from_maps([zero] * M, res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B)
        pl.set_occupancy_slots_device(imgs, res, obstacle_max=127)
        idx = t((np.arange(B) % M).astype(np.int32))
        mapped = lambda: pl.plan_points_device(*d_in, map_index=idx)  # noqa: E731
        shared = lambda: pl.plan_points_device(*d_in)  # noqa: E731
        for _ in range(args.warmup):
            mapped()
            shared()
        torch.cuda.synchronize()
        ms_m, ms_s, stages = [], [], []
        for _ in range(args.steps):  # alternated call by call
            ms_m.append(_timed(mapped))
            stages.append(pl.last_stage_ms)
            ms_s.append(_timed(shared))
        out = mapped()
        torch.cuda.synchronize()
        st = out["status"].cpu().numpy()
        entry = {"ms_mapped": float(np.median(ms_m)), "ms_unmapped_slot0": float(np.median(ms_s)),
                 "ms_mapped_min_max": [float(min(ms_m)), float(max(ms_m))],
                 "ms_unmapped_min_max": [float(min(ms_s)), float(max(ms_s))],
                 "stage_ms_mapped": {k: float(np.median([s[k] for s in stages])) for k in plan.STAGES},
                 "status": {plan.STATUS_NAMES[int(v)]: int((st == v).sum()) for v in np.unique(st)},
                 "layer_bytes": int(M * demo.size * 4)}
        result["maps"][str(M)] = entry
        pl.close()
        del imgs
        torch.cuda.empty_cache()

    # today's alternative at M = 64: one single-map planner per map, each on its B / 64 paths, back to back
    M = 64
    imgs = _blocked(demo, np.random.default_rng(4), M, res)
    singles = []
    per = B // M
    for k in range(M):
        p1 = plan.Planner(zero, res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=per)
        p1.set_occupancy(imgs[k], res, obstacle_max=127)
        rows = np.arange(k, B, M)
        singles.append((p1, [a[rows].contiguous() for a in d_in]))

    def one_by_one():
        for p1, a in singles:
            p1.plan_points_device(*a)

    for _ in range(args.warmup):
        one_by_one()
    torch.cuda.synchronize()
    ms_alt = [_timed(one_by_one) for _ in range(max(args.steps // 4, 5))]
    for p1, _ in singles:
        p1.close()
    result["alternative_64_single_map_planners"] = {"ms": float(np.median(ms_alt)), "paths_per_planner": per}

    # building 1024 layers: one batched call against one call per image
    count = 1024
    d_imgs = t(_blocked(demo, np.random.default_rng(5), count, res))
    pl = plan.Planner.from_maps([zero] * count, res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=1)
    one = plan.Planner(zero, res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=1)
    batched = lambda: pl.set_occupancy_slots_device(d_imgs, res, obstacle_max=127)  # noqa: E731

    def each():
        for k in range(count):
            one.set_occupancy_device(d_imgs[k], res, obstacle_max=127)

    for _ in range(2):
        batched()
        each()
    torch.cuda.synchronize()
    ms_b, ms_e = [], []
    for _ in range(5):
        ms_b.append(_timed(batched))
        ms_e.append(_timed(each))
    result["set_occupancy_1024_demo_images"] = {"ms_set_occupancy_slots_device": float(np.median(ms_b)),
                                                "ms_1024_set_occupancy_device": float(np.median(ms_e)),
                                                "launches_batched": plan.occupancy_slots_launches(count),
                                                "launches_one_by_one": count * plan.OCCUPANCY_LAUNCHES}
    pl.close()
    one.close()
    result["value"] = result["maps"]["1024"]["ms_mapped"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
