"""The demo's tick through the C++ PathOptimizer drop-in (include/pqp_path_optimizer.hpp) on one GPU, B = 1.

The demo constructs a PathOptimizer per tick with that tick's map, solves, reads getReferencePath() and destroys it
(demo.cpp:196-206). tests/cpp/path_optimizer_test (built by __graft_entry__.build()) times exactly that on the demo
map (gridmap.png, 701 x 710, a 2 MB distance layer) with a pool hit on every construction after the first, and the
first construction itself, which creates the plan handle. Between its runs this script times Planner.plan_points
(the same library call with B = 1, no trace, no map copy) and Planner.set_map (the 2 MB copy the drop-in's
construction makes), so the three alternate in blocks. It also reports a plan handle's device footprint with the
drop-in's capacities, from cudaMemGetInfo around its creation.

Prints the GPU's name and power limit and one JSON line with medians over --rounds x --ticks ticks, each round after
--warmup warm-up ticks. Writes nothing to the source tree (inputs go to a temporary directory).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_plan import gpu_info  # noqa: E402

BIN = os.path.join(ROOT, "tests", "cpp", "path_optimizer_test")
CAPS = dict(r_max=256, p_max=256, layers_max=160, n_max=511)  # PathOptimizerOptions' defaults


def _wall_ms(fn, n, warmup):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--ticks", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not os.path.exists(BIN):
        raise SystemExit("%s is missing: run __graft_entry__.build() first" % BIN)
    import torch
    from PIL import Image

    from oracle import edt_oracle
    from path_optimizer_2_b200 import plan, sharedmap
    from tests.test_path_optimizer_dropin import write_script

    gpu = gpu_info()
    print("GPU: %s, power limit %s" % (gpu["name"], gpu["power_limit"]))
    torch.cuda.init()
    torch.cuda.synchronize()
    img = np.asarray(Image.open(os.path.join(ROOT, "tests", "golden", "gridmap.png")).convert("L")).astype(np.uint8)
    dist = edt_oracle.transform(img, sharedmap.RES, 127)[1]
    params = plan.default_params()
    free0 = torch.cuda.mem_get_info(0)[0]
    pl = plan.Planner(dist, sharedmap.RES, batch_max=1, params=params, **CAPS)
    footprint = free0 - torch.cuda.mem_get_info(0)[0]

    # the first path of the demo's point sets that plans to the end
    ref_x, ref_y, start, target = sharedmap.make_plan_points(8, dmap=sharedmap.DistanceMap(dist=dist))
    b = next(i for i in range(8) if pl.plan_points([ref_x[i]], [ref_y[i]], start[[i]], target[[i]]).status[0] == plan.OK)
    inputs = ([ref_x[b]], [ref_y[b]], start[[b]], target[[b]])

    dropin, host, set_map, first_construct, first_tick, pool = [], [], [], [], [], []
    with tempfile.TemporaryDirectory() as d:
        script = write_script(d, params, [("dist", dist)], [(0, ref_x[b], ref_y[b], start[b], target[b])])
        for _ in range(args.rounds):
            out = subprocess.run([BIN, script, "bench", str(args.warmup), str(args.ticks)], capture_output=True,
                                 text=True, check=True).stdout.split("\n")
            head = out[0].split()
            if head[0] != "bench" or int(head[2]) != plan.OK:
                raise SystemExit("drop-in tick failed: %s" % out[0])
            kv = {head[i]: float(head[i + 1]) for i in range(1, len(head) - 1, 2)}
            first_construct.append(kv["first_construct_ms"])
            first_tick.append(kv["first_tick_ms"])
            pool.append((int(kv["creates"]), int(kv["hits"])))
            dropin += [float(v) for v in out[1].split()[1:]]
            host += _wall_ms(lambda: pl.plan_points(*inputs), args.ticks, args.warmup)
            set_map += _wall_ms(lambda: pl.set_map(dist, sharedmap.RES), args.ticks, args.warmup)
    pl.close()
    med = lambda v: float(np.median(v))  # noqa: E731
    result = {"metric": "ms_per_demo_tick_b1", "value": med(dropin), "gpu": gpu, "ticks": len(dropin),
              "warmup_per_round": args.warmup, "rounds": args.rounds, "capacities": CAPS,
              "dropin_tick_ms_median": med(dropin), "dropin_tick_ms_p90": float(np.percentile(dropin, 90)),
              "planner_plan_points_ms_median": med(host), "planner_set_map_ms_median": med(set_map),
              "host_call_plus_map_copy_ms": med(host) + med(set_map),
              "first_construct_ms": first_construct, "first_tick_ms": first_tick,
              "pool_creates_hits_per_round": pool, "plan_handle_device_bytes": int(footprint),
              "plan_handle_device_mib": footprint / 2**20}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
