"""Map replacement cost (pqp_plan_set_occupancy*, include/pqp_plan.h) on one GPU.

Prints one JSON line with the GPU's name and power limit read in the same run, and:
  - ms per set_occupancy_device (CUDA events around --repeats calls after warm-up) on the demo map (gridmap.png,
    701 x 710) and on a 4096 x 4096 random grid with 1 % obstacles, with the algorithmic bytes (1 B in and 4 B out per
    cell, plus the column pass's int32 g written and read back through the layer: 8 B) and the share of the 3.35 TB/s
    HBM bound they give;
  - ms per host set_occupancy, end to end (image upload, both kernels, synchronisation);
  - cv2.distanceTransform (DIST_L2, DIST_MASK_PRECISE) of the same images on this machine's CPU, or "not measured"
    without OpenCV;
  - one receding-horizon tick of 1024 paths: set_occupancy_device + plan_points_device against plan_points_device
    alone (TENSION2, from reference points);
  - pqp_plan_destroy + pqp_plan_create on the same map: what following a map change costs without set_occupancy.
Writes nothing to the source tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_plan import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_CELL = 1 + 4 + 4 + 4  # image in, g out, g in, layer out


def _events_ms(fn, repeats, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(repeats):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / repeats


def _wall_ms(fn, repeats, warmup):
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    for _ in range(repeats):
        fn()
    return (time.perf_counter() - t0) * 1e3 / repeats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    import torch
    from PIL import Image

    from path_optimizer_2_b200 import plan, sharedmap
    dev = torch.device("cuda:0")
    png = os.path.join(ROOT, "tests", "golden", "gridmap.png")
    demo = np.asarray(Image.open(png).convert("L")).astype(np.uint8)
    big = np.where(np.random.default_rng(0).random((4096, 4096)) < 0.01, 0, 255).astype(np.uint8)
    try:
        import cv2
    except ImportError:
        cv2 = None

    dmap = sharedmap.DistanceMap()
    R, P, L, N, B = 64, 64, 64, 255, args.batch
    result = {"metric": "ms_per_set_occupancy_device", "gpu": gpu_info(), "repeats": args.repeats,
              "warmup": args.warmup, "maps": {}}
    for name, img in (("demo_701x710", demo), ("random_4096x4096_1pct", big)):
        pl = plan.Planner(np.zeros(img.shape, np.float32), sharedmap.RES, r_max=R, p_max=P, layers_max=L, n_max=N,
                          batch_max=1)
        d_img = torch.from_numpy(img).to(dev)
        ms_dev = _events_ms(lambda: pl.set_occupancy_device(d_img, sharedmap.RES), args.repeats, args.warmup)
        ms_host = _wall_ms(lambda: pl.set_occupancy(img, sharedmap.RES), max(args.repeats // 4, 20), 3)
        cells = img.size
        entry = {"ms_device": ms_dev, "ms_host_end_to_end": ms_host, "cells": cells,
                 "algorithmic_bytes": BYTES_PER_CELL * cells,
                 "share_of_hbm_bound": BYTES_PER_CELL * cells / (ms_dev * 1e-3) / HBM_BYTES_PER_S}
        if cv2 is not None:
            free = (img > 0).astype(np.uint8)
            entry["cv2_ms_cpu"] = _wall_ms(lambda: cv2.distanceTransform(free, cv2.DIST_L2, cv2.DIST_MASK_PRECISE),
                                           10 if cells > 1e7 else 50, 2)
            entry["cv2_threads"] = cv2.getNumThreads()
        else:
            entry["cv2_ms_cpu"] = "not measured"
        result["maps"][name] = entry
        pl.close()

    # one tick of B paths on the demo map
    ref_x, ref_y, start, target = sharedmap.make_plan_points(B, dmap=dmap)
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_in = [t(px), t(py), t(m), t(start), t(target)]
    d_img = t(demo)
    pl = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B)
    steps = max(args.repeats // 10, 20)

    def tick():
        pl.set_occupancy_device(d_img, sharedmap.RES, obstacle_max=127)
        pl.plan_points_device(*d_in)

    ms_plan = _events_ms(lambda: pl.plan_points_device(*d_in), steps, 3)
    ms_tick = _events_ms(tick, steps, 3)
    pl.close()

    def recreate():
        p = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B)
        p.close()

    ms_recreate = _wall_ms(recreate, 10, 2)
    result.update(value=result["maps"]["demo_701x710"]["ms_device"], tick_batch=B,
                  tick_ms_set_occupancy_device_plus_plan_points_device=ms_tick,
                  tick_ms_plan_points_device_alone=ms_plan, ms_plan_destroy_plus_create_same_map=ms_recreate)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
