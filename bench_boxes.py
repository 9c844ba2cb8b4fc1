"""Obstacle boxes stamped into the map slots on the GPU (set_occupancy_boxes*, include/pqp_bounds.h) on one GPU.

The bench_maps scene expressed as boxes: 1024 slots, the demo image shared by every slot, 12 boxes of 1.8 m per slot
at random places, first axis-aligned, then at random headings. Prints one JSON line with the GPU's name and power limit
read in the same run, and per heading mode (CUDA events, medians over --steps, after --warmup):
  - set_occupancy_boxes_device (image, boxes and counts already on the device) against set_occupancy_slots_device of
    the equivalent pre-stamped images (also already on the device), alternated call by call on one handle;
  - the host forms of both, host clock around the synchronous call: the box call with its ~0.5 MB of boxes, the
    image call including the numpy stamping of 1024 image copies and their 510 MB upload;
  - one tick: the device box update followed by plan_points_device of 1024 paths, path b on slot b (TENSION2).
Also how many of every 16th slot have layers equal between the box call and the stamped images (numpy's cos /
sin against the device's may decide a cell lying on a box edge at a random heading). Writes nothing to the source tree.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_maps import _timed  # noqa: E402
from bench_plan import gpu_info  # noqa: E402

SIDE = 1.8
PER_SLOT = 12


def _boxes(rng, shape, res, count, headings):
    """[count, PER_SLOT, 5]: boxes of SIDE m with centres uniform over the map."""
    rows, cols = shape
    b = np.zeros((count, PER_SLOT, 5))
    b[..., 0] = rng.uniform(-0.5 * rows * res, 0.5 * rows * res, (count, PER_SLOT))
    b[..., 1] = rng.uniform(-0.5 * cols * res, 0.5 * cols * res, (count, PER_SLOT))
    b[..., 2] = rng.uniform(-math.pi, math.pi, (count, PER_SLOT)) if headings else 0.0
    b[..., 3:] = SIDE
    return b


def stamp_images(demo, res, boxes):
    """What a caller of set_occupancy_slots writes today: `count` copies of the image, each box stamped by the header's
    predicate over the cells of its bounding box (map centred at the origin)."""
    rows, cols = demo.shape
    out = np.repeat(demo[None], len(boxes), axis=0)
    half_lx, half_ly = 0.5 * rows * res, 0.5 * cols * res
    for s, slot in enumerate(boxes):
        for x, y, h, length, width in slot:
            c, sn = math.cos(h), math.sin(h)
            r = 0.5 * length * abs(c) + 0.5 * width * abs(sn) + res, 0.5 * length * abs(sn) + 0.5 * width * abs(c) + res
            i0, i1 = max(int((half_lx - x - r[0]) / res), 0), min(int((half_lx - x + r[0]) / res) + 1, rows)
            j0, j1 = max(int((half_ly - y - r[1]) / res), 0), min(int((half_ly - y + r[1]) / res) + 1, cols)
            if i0 >= i1 or j0 >= j1:
                continue
            px = (half_lx - (np.arange(i0, i1) + 0.5) * res)[:, None]
            py = (half_ly - (np.arange(j0, j1) + 0.5) * res)[None, :]
            dx, dy = px - x, py - y
            inside = (np.abs(dx * c + dy * sn) <= 0.5 * length) & (np.abs(dy * c - dx * sn) <= 0.5 * width)
            out[s, i0:i1, j0:j1][inside] = 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--count", type=int, default=1024)
    args = ap.parse_args()
    import torch
    from PIL import Image

    from path_optimizer_2_b200 import plan, sharedmap
    dev = torch.device("cuda:0")
    res = sharedmap.RES
    demo = np.asarray(Image.open(os.path.join(ROOT, "tests", "golden", "gridmap.png")).convert("L")).astype(np.uint8)
    count = args.count
    R, P, L, N = 64, 64, 64, 255
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    result = {"metric": "ms_set_occupancy_boxes_device", "gpu": gpu_info(), "slots": count,
              "map": list(demo.shape), "boxes_per_slot": PER_SLOT, "box_side_m": SIDE, "steps": args.steps,
              "warmup": args.warmup, "modes": {}}
    zero = np.zeros(demo.shape, np.float32)
    pl = plan.Planner.from_maps([zero] * count, res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=count)
    ref_x, ref_y, start, target = sharedmap.make_plan_points(count, dmap=sharedmap.DistanceMap())
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((count, R)), np.zeros((count, R))
    for b in range(count):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    d_in = [t(px), t(py), t(m), t(start), t(target)]
    idx = t(np.arange(count, dtype=np.int32))
    d_demo = t(demo)
    k = np.full(count, PER_SLOT, np.int32)
    d_k = t(k)
    for mode, headings in (("axis_aligned", False), ("random_headings", True)):
        boxes = _boxes(np.random.default_rng(7 if headings else 3), demo.shape, res, count, headings)
        d_boxes = t(boxes)
        t0 = time.perf_counter()
        imgs = stamp_images(demo, res, boxes)
        ms_numpy_stamp = 1e3 * (time.perf_counter() - t0)
        d_imgs = t(imgs)
        by_boxes = lambda: pl.set_occupancy_boxes_device(d_demo, res, d_boxes, d_k, obstacle_max=127)  # noqa: E731
        by_images = lambda: pl.set_occupancy_slots_device(d_imgs, res, obstacle_max=127)  # noqa: E731
        # the two paths give the same layers (up to cells on a box edge at a random heading)
        check = list(range(0, count, 16))
        by_images()
        want = [pl.get_map(s)[0] for s in check]
        by_boxes()
        equal = sum(int(np.array_equal(pl.get_map(s)[0], w)) for s, w in zip(check, want))
        for _ in range(args.warmup):
            by_boxes()
            by_images()
        torch.cuda.synchronize()
        ms_b, ms_i = [], []
        for _ in range(args.steps):  # alternated call by call
            ms_b.append(_timed(by_boxes))
            ms_i.append(_timed(by_images))
        # host forms: boxes (0.5 MB) against numpy stamping + 510 MB of images
        host_b, host_i = [], []
        for it in range(args.warmup + max(args.steps // 2, 3)):
            t0 = time.perf_counter()
            pl.set_occupancy_boxes(demo, res, boxes, k, obstacle_max=127)
            tb = time.perf_counter()
            pl.set_occupancy_slots(stamp_images(demo, res, boxes), res, obstacle_max=127)
            ti = time.perf_counter()
            if it >= args.warmup:
                host_b.append(1e3 * (tb - t0))
                host_i.append(1e3 * (ti - tb))
        # one tick: the box update, then the plan of every path on its own slot
        tick = lambda: (by_boxes(), pl.plan_points_device(*d_in, map_index=idx))  # noqa: E731
        for _ in range(args.warmup):
            tick()
        torch.cuda.synchronize()
        ms_t = [_timed(tick) for _ in range(args.steps)]
        st = pl.plan_points_device(*d_in, map_index=idx)["status"].cpu().numpy()
        result["modes"][mode] = {
            "ms_set_occupancy_boxes_device": float(np.median(ms_b)),
            "ms_set_occupancy_slots_device_prestamped": float(np.median(ms_i)),
            "ms_boxes_min_max": [float(min(ms_b)), float(max(ms_b))],
            "ms_slots_min_max": [float(min(ms_i)), float(max(ms_i))],
            "ms_set_occupancy_boxes_host": float(np.median(host_b)),
            "ms_numpy_stamp_plus_set_occupancy_slots_host": float(np.median(host_i)),
            "ms_numpy_stamp_once": ms_numpy_stamp,
            "ms_tick_boxes_plus_plan_points_mapped_device": float(np.median(ms_t)),
            "launches_per_update": plan.occupancy_slots_launches(count),
            "bytes_boxes": int(boxes.nbytes + k.nbytes), "bytes_images": int(imgs.nbytes),
            "slots_checked": len(check), "slots_equal_to_stamped_images": equal,
            "status": {plan.STATUS_NAMES[int(v)]: int((st == v).sum()) for v in np.unique(st)},
        }
        del d_imgs, imgs, want
        torch.cuda.empty_cache()
    pl.close()
    result["value"] = result["modes"]["axis_aligned"]["ms_set_occupancy_boxes_device"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
