"""Whole-plan throughput (include/pqp_plan.h): PathOptimizer::solve for a batch of paths on one H100.

Workload: BASELINE configs[1]'s shape - reference lines through gridmap.png from sharedmap.make_lines, sampled about
every 1 m with 3 cm of noise as the bSpline() samples, the start up to 1 m beside the line near s = 0.5, the target
1 m before its end. Prints one JSON line: plans/s at B = 1024 (device call, CUDA events around the timed loop), ms per
plan at B = 1 (host call), the per-stage device times of the last call, kernel launches per plan, the status histogram,
the CPU Python oracle chain's plans/s on a sample (the Python restatement, not the reference), and the GPU's name and
power limit read in the same run. Writes nothing to the source tree.
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
    args = ap.parse_args()
    import torch

    from oracle import plan_oracle
    from path_optimizer_2_b200 import plan, sharedmap
    dmap = sharedmap.DistanceMap()
    B = args.batch
    raw_x, raw_y, start, target = sharedmap.make_plan_inputs(B, dmap=dmap)
    R, P, L, N = 64, 64, 64, 255
    pl = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B)
    dev = torch.device("cuda:0")
    r = np.array([len(v) for v in raw_x], dtype=np.int32)
    rx, ry = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        rx[b, :r[b]], ry[b, :r[b]] = raw_x[b], raw_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_in = [t(rx), t(ry), t(r), t(start), t(target)]
    for _ in range(args.warmup):
        out = pl.plan_device(*d_in)
    torch.cuda.synchronize()
    c0 = pl.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = pl.plan_device(*d_in)
    e1.record()
    torch.cuda.synchronize()
    ms_batch = e0.elapsed_time(e1) / args.steps
    launches = (pl.launch_count - c0) / args.steps
    stages = pl.last_stage_ms
    status = out["status"].cpu().numpy()
    hist = {plan.STATUS_NAMES[c]: int(np.sum(status == c)) for c in sorted(set(status.tolist()))}

    one = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=1)
    for _ in range(args.warmup):
        one.plan(raw_x[:1], raw_y[:1], start[:1], target[:1])
    t0 = time.perf_counter()
    n1 = max(args.steps, 10)
    for i in range(n1):
        one.plan(raw_x[i:i + 1], raw_y[i:i + 1], start[i:i + 1], target[i:i + 1])
    ms_one = (time.perf_counter() - t0) * 1e3 / n1
    stages_one = one.last_stage_ms
    one.close()

    k = min(args.oracle_sample, B)
    t0 = time.perf_counter()
    for b in range(k):
        plan_oracle.plan(dmap.dist, dmap.res, raw_x[b], raw_y[b], start[b], target[b], params=pl.params.solver,
                         p_max=P, layers_max=L, n_max=N)
    oracle_s = time.perf_counter() - t0
    pl.close()
    print(json.dumps({
        "metric": "plans_per_s", "what": "PathOptimizer::solve batched, bSpline samples -> final path, gridmap.png, "
                                         "configs[1] shape (device call)",
        "batch": B, "value": B / (ms_batch * 1e-3), "ms_per_batch": ms_batch,
        "ms_per_plan_b1_host_call": ms_one, "stage_ms_last_batch": stages, "stage_ms_b1": stages_one,
        "kernel_launches_per_plan_call": launches, "status_histogram": hist,
        "python_oracle_chain_plans_per_s": k / oracle_s, "python_oracle_sample": k,
        "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup}))


if __name__ == "__main__":
    main()
