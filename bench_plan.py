"""Whole-plan throughput (include/pqp_plan.h): PathOptimizer::solve for a batch of paths on one H100.

Workload: BASELINE configs[1]'s shape - reference lines through gridmap.png from sharedmap.make_lines, sampled about
every 1 m with 3 cm of noise as the bSpline() samples, the start up to 1 m beside the line near s = 0.5, the target
1 m before its end. Prints one JSON line: plans/s at B = 1024 (device call, CUDA events around the timed loop), ms per
plan at B = 1 (host call), the per-stage device times of the last call, kernel launches per plan, the status histogram,
the CPU Python oracle chain's plans/s on a sample (the Python restatement, not the reference), and the GPU's name and
power limit read in the same run. --smoothing-method selects the reference smoother (TENSION2, the default, or
TENSION). --input points starts each plan from "clicked" reference points instead (sharedmap.make_plan_points, 3-14 m
apart, through pqp_plan_points_device: bSpline() on the GPU); the JSON line then also carries "input" and the B-spline
degree histogram. Writes nothing to the source tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": q[0], "power_limit": q[1]}
    except Exception as e:  # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unavailable (%r)" % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-sample", type=int, default=8)
    ap.add_argument("--smoothing-method", choices=("TENSION2", "TENSION"), default="TENSION2",
                    help="the reference's --smoothing_method: TensionSmoother2 (default) or TensionSmoother")
    ap.add_argument("--input", choices=("samples", "points"), default="samples",
                    help="bSpline() samples (pqp_plan, default) or reference points (pqp_plan_points)")
    args = ap.parse_args()
    import torch

    from oracle import bspline_oracle, cartesian_oracle, plan_oracle
    from path_optimizer_2_b200 import plan, sharedmap
    dmap = sharedmap.DistanceMap()
    B = args.batch
    points = args.input == "points"
    make = sharedmap.make_plan_points if points else sharedmap.make_plan_inputs
    raw_x, raw_y, start, target = make(B, dmap=dmap)
    R, P, L, N = 64, 64, 64, 255  # the points' polygons are under 50 m: at most about 50 samples
    params = plan.default_params(args.smoothing_method)
    pl = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B, params=params)
    dev = torch.device("cuda:0")
    r = np.array([len(v) for v in raw_x], dtype=np.int32)
    rx, ry = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        rx[b, :r[b]], ry[b, :r[b]] = raw_x[b], raw_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_in = [t(rx), t(ry), t(r), t(start), t(target)]
    run = pl.plan_points_device if points else pl.plan_device
    for _ in range(args.warmup):
        out = run(*d_in)
    torch.cuda.synchronize()
    c0 = pl.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = run(*d_in)
    e1.record()
    torch.cuda.synchronize()
    ms_batch = e0.elapsed_time(e1) / args.steps
    launches = (pl.launch_count - c0) / args.steps
    stages = pl.last_stage_ms
    status = out["status"].cpu().numpy()
    hist = {plan.STATUS_NAMES[c]: int(np.sum(status == c)) for c in sorted(set(status.tolist()))}

    one = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=1, params=params)
    run_one = one.plan_points if points else one.plan
    for _ in range(args.warmup):
        run_one(raw_x[:1], raw_y[:1], start[:1], target[:1])
    t0 = time.perf_counter()
    n1 = max(args.steps, 10)
    for i in range(n1):
        run_one(raw_x[i:i + 1], raw_y[i:i + 1], start[i:i + 1], target[i:i + 1])
    ms_one = (time.perf_counter() - t0) * 1e3 / n1
    stages_one = one.last_stage_ms
    one.close()

    k = min(args.oracle_sample, B)
    oracle_plan = cartesian_oracle.plan if args.smoothing_method == "TENSION" else plan_oracle.plan
    t0 = time.perf_counter()
    for b in range(k):
        if points:
            bspline_oracle.plan(dmap.dist, dmap.res, raw_x[b], raw_y[b], start[b], target[b], r_max=R,
                                smoothing_method=args.smoothing_method, params=pl.params.solver, p_max=P, layers_max=L,
                                n_max=N)
        else:
            oracle_plan(dmap.dist, dmap.res, raw_x[b], raw_y[b], start[b], target[b], params=pl.params.solver,
                        p_max=P, layers_max=L, n_max=N)
    oracle_s = time.perf_counter() - t0
    pl.close()
    result = {
        "metric": "plans_per_s", "what": "PathOptimizer::solve batched, bSpline samples -> final path, gridmap.png, "
                                         "configs[1] shape (device call)",
        "batch": B, "value": B / (ms_batch * 1e-3), "ms_per_batch": ms_batch,
        "ms_per_plan_b1_host_call": ms_one, "stage_ms_last_batch": stages, "stage_ms_b1": stages_one,
        "kernel_launches_per_plan_call": launches, "status_histogram": hist,
        "python_oracle_chain_plans_per_s": k / oracle_s, "python_oracle_sample": k,
        "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "smoothing_method": args.smoothing_method}
    if points:
        result["what"] = result["what"].replace("bSpline samples", "reference points -> bSpline on the GPU")
        degree = [bspline_oracle.degree_for(bspline_oracle.polygon_length(x, y), len(x)) for x, y in zip(raw_x, raw_y)]
        result.update(input="points", bspline_degree_histogram={d: degree.count(d) for d in sorted(set(degree))})
    print(json.dumps(result))


if __name__ == "__main__":
    main()
