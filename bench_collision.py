"""Footprint collision check of final paths (pqp_plan_collision_check_device; include/pqp_bounds.h) on one GPU.

Workload: bench_plan.py --input points, B = 1024 plans (TENSION2) from reference points on gridmap.png. Prints one
JSON line with the GPU's name and power limit read in the same run, and:
  - ms per check_collision_device call on the plan's final paths (CUDA events around each call, median of --steps
    calls after --warmup), each check alternated with the plan_points_device call whose output it reads, and the
    plan call's ms from the same loop;
  - the same on a 1024-slot handle with distinct maps (bench_maps.py's workload: the demo image with its own random
    1.8 m blocks per slot), path b planned and checked on slot b;
  - how many PLAN_OK paths the check flags on each;
  - the Python oracle's (numpy) time for the same check of the 1024 shared-map paths on one core;
  - the bytes the check gathers per state: 7 bilinear lookups of 4 float32 cells.
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

from bench_maps import _blocked, _timed  # noqa: E402
from bench_plan import gpu_info  # noqa: E402


def _measure(pl, d_in, steps, warmup, map_index=None):
    import torch
    from path_optimizer_2_b200 import plan
    stream = torch.cuda.current_stream().cuda_stream
    out = {}

    def run_plan():
        out.update(pl.plan_points_device(*d_in, map_index=map_index))

    def run_check():
        out["check"] = pl.check_collision_device(out["path"], out["n"], map_index=map_index, stream=stream)

    for _ in range(warmup):
        run_plan()
        run_check()
    torch.cuda.synchronize()
    ms_plan, ms_check = [], []
    for _ in range(steps):  # alternated call by call
        ms_plan.append(_timed(run_plan))
        ms_check.append(_timed(run_check))
    status = out["status"].cpu().numpy()
    n = out["n"].cpu().numpy()
    hit = out["check"]["first_hit"].cpu().numpy()
    ok = status == plan.OK
    return {"ms_check": float(np.median(ms_check)), "ms_check_min_max": [float(min(ms_check)), float(max(ms_check))],
            "ms_plan": float(np.median(ms_plan)), "plan_ok": int(ok.sum()),
            "plan_ok_flagged": int(np.sum(ok & (hit < n))), "states_checked": int(n.sum())}, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=1024)
    args = ap.parse_args()
    import torch
    from PIL import Image

    from oracle import collision_oracle
    from path_optimizer_2_b200 import plan, sharedmap
    dev = torch.device("cuda:0")
    dmap = sharedmap.DistanceMap()
    res = dmap.res
    R, P, L, N, B = 64, 64, 64, 255, args.batch
    ref_x, ref_y, start, target = sharedmap.make_plan_points(B, dmap=dmap)
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_in = [t(px), t(py), t(m), t(start), t(target)]
    result = {"metric": "ms_per_collision_check_device", "gpu": gpu_info(), "batch": B, "steps": args.steps,
              "warmup": args.warmup, "method": "TENSION2", "input": "points",
              "gathered_bytes_per_state": 7 * 4 * 4}

    pl = plan.Planner(dmap.dist, res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B)
    shared, out = _measure(pl, d_in, args.steps, args.warmup)
    path, n = out["path"].cpu().numpy(), out["n"].cpu().numpy()
    gpu_hit = out["check"]["first_hit"].cpu().numpy()
    pl.close()
    t0 = time.perf_counter()
    oracle_hit = collision_oracle.check(dmap.dist, res, path, n)[0]
    shared["ms_python_oracle_one_core"] = (time.perf_counter() - t0) * 1e3
    shared["first_hit_equals_oracle"] = bool(np.array_equal(oracle_hit, gpu_hit))
    result["shared_map"] = shared

    demo = np.asarray(Image.open(os.path.join(ROOT, "tests", "golden", "gridmap.png")).convert("L")).astype(np.uint8)
    imgs = t(_blocked(demo, np.random.default_rng(3), B, res))
    zero = np.zeros(demo.shape, np.float32)
    pl = plan.Planner.from_maps([zero] * B, res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B)
    pl.set_occupancy_slots_device(imgs, res, obstacle_max=127)
    idx = t(np.arange(B, dtype=np.int32))
    result["slots_1024"], _ = _measure(pl, d_in, args.steps, args.warmup, map_index=idx)
    pl.close()
    result["value"] = result["shared_map"]["ms_check"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
