"""The whole plan over several GPUs of one box (plan_multi.MultiPlanner, include/pqp_plan_multi.h).

Prints the GPU's name, power limit and the visible device count read in the same run, a scaling table and one JSON
line:
  - B = --batch plans from reference points (sharedmap.make_plan_points) on the demo map, TENSION2, at G = 1, 2, 4, 8
    devices as far as the box has them (the others are reported as not measured): plans/s of the device form
    (CUDA events on the home stream, median of --steps calls), of the host form (host clock around the synchronous
    C call, median of --host-steps calls), the efficiency rate_G / (G * rate_1) of both, and each device's shard time
    (pqp_plan_last_stage_ms of its handle after the last device-form call);
  - the outputs of every G against G = 1, bit for bit (status, n, path, cost, iters);
  - the per-path-maps workload of bench_maps.py at the largest G: --maps demo-sized slots built by one
    set_occupancy_slots_device call, path b on slot b % maps;
  - MultiPlanner(devices=[0]) against a Planner on the same inputs, device form, alternated call by call: what the
    multi-device layer costs on one GPU.
Writes nothing to the source tree.
"""
import argparse
import ctypes as C
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

R, P, L, N = 64, 64, 64, 255


def _same(a, b):
    return all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in ("status", "n", "path", "cost", "iters"))


def _host(out):
    return {k: v.cpu().numpy() for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--host-steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--maps", type=int, default=1024)
    args = ap.parse_args()
    import torch
    from PIL import Image

    from path_optimizer_2_b200 import plan, plan_multi, sharedmap
    visible = torch.cuda.device_count()
    if visible < 1:
        raise SystemExit("no CUDA device")
    B = args.batch
    dmap = sharedmap.DistanceMap()
    ref_x, ref_y, start, target = sharedmap.make_plan_points(B, dmap=dmap)
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    start, target = np.ascontiguousarray(start), np.ascontiguousarray(target)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda(0)  # noqa: E731
    d_in = [t(px), t(py), t(m), t(start), t(target)]
    host_in = plan.PlanPointsIn(B, R, px.ctypes.data, py.ctypes.data, m.ctypes.data, start.ctypes.data,
                                target.ctypes.data)
    params = plan.default_params("TENSION2")
    kw = dict(r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B, params=params)
    result = {"metric": "plans_per_s_multi_gpu_plan_points", "gpu": gpu_info(), "visible_devices": visible, "batch": B,
              "steps": args.steps, "host_steps": args.host_steps, "warmup": args.warmup, "method": "TENSION2",
              "scaling": {}}
    base = None
    largest = max(g for g in (1, 2, 4, 8) if g <= visible)
    for G in (1, 2, 4, 8):
        if G > visible:
            result["scaling"][str(G)] = "not measured (%d device%s visible)" % (visible, "s" if visible > 1 else "")
            continue
        mp = plan_multi.MultiPlanner([dmap.dist], dmap.res, devices=list(range(G)), **kw)
        call = lambda: mp.plan_points_device(*d_in)  # noqa: E731
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        ms = [_timed(call) for _ in range(args.steps)]
        shard_ms = [mp.last_stage_ms(i)["total"] for i in range(G)]
        out = _host(call())
        # the host form: the C call alone (host buffers, synchronous)
        res = plan.PlanResult(B, N)
        pout = plan.PlanOut(res.status.ctypes.data, res.n.ctypes.data, res.path.ctypes.data, res.cost.ctypes.data,
                            res.iters.ctypes.data, None)
        host_ms = []
        for i in range(1 + args.host_steps):
            t0 = time.perf_counter()
            mp._check(mp.L.pqp_plan_multi_points(mp.h, C.byref(host_in), None, C.byref(pout)))
            if i:  # the first call warms the host path
                host_ms.append((time.perf_counter() - t0) * 1e3)
        hres = {k: getattr(res, k) for k in ("status", "n", "path", "cost", "iters")}
        if base is None:
            base = out
        entry = {"ms_device": float(np.median(ms)), "ms_device_min_max": [float(min(ms)), float(max(ms))],
                 "plans_per_s_device": B / (float(np.median(ms)) / 1e3),
                 "ms_host": float(np.median(host_ms)), "plans_per_s_host": B / (float(np.median(host_ms)) / 1e3),
                 "shard_total_ms": shard_ms, "shards": [list(mp.shard(i)) for i in range(G)],
                 "bit_identical_to_g1": bool(_same(out, base) and _same(hres, base)),
                 "status": {plan.STATUS_NAMES[int(v)]: int((out["status"] == v).sum()) for v in np.unique(out["status"])}}
        one = result["scaling"].get("1")
        for form in ("device", "host"):
            entry["efficiency_" + form] = entry["plans_per_s_" + form] / (G * (one or entry)["plans_per_s_" + form])
        result["scaling"][str(G)] = entry
        mp.close()
        torch.cuda.empty_cache()

    # per-path maps at the largest G: path b on slot b % maps, the slots built on the home device and peer-copied
    demo = np.asarray(Image.open(os.path.join(ROOT, "tests", "golden", "gridmap.png")).convert("L")).astype(np.uint8)
    M = args.maps
    zero = np.zeros(demo.shape, np.float32)
    imgs = t(_blocked(demo, np.random.default_rng(3), M, dmap.res))
    idx = t((np.arange(B) % M).astype(np.int32))
    mp = plan_multi.MultiPlanner([zero] * M, dmap.res, devices=list(range(largest)), **kw)
    build_ms = _timed(lambda: mp.set_occupancy_slots_device(imgs, dmap.res, obstacle_max=127))
    call = lambda: mp.plan_points_device(*d_in, map_index=idx)  # noqa: E731
    for _ in range(args.warmup):
        call()
    torch.cuda.synchronize()
    ms = [_timed(call) for _ in range(args.steps)]
    st = call()["status"].cpu().numpy()
    result["per_path_maps"] = {"devices": largest, "maps": M, "ms_device": float(np.median(ms)),
                               "plans_per_s_device": B / (float(np.median(ms)) / 1e3),
                               "ms_set_occupancy_slots_device": build_ms,
                               "shard_total_ms": [mp.last_stage_ms(i)["total"] for i in range(largest)],
                               "status": {plan.STATUS_NAMES[int(v)]: int((st == v).sum()) for v in np.unique(st)}}
    mp.close()
    del imgs
    torch.cuda.empty_cache()

    # the multi-device layer on one GPU: MultiPlanner([0]) against a Planner, alternated call by call
    mp = plan_multi.MultiPlanner([dmap.dist], dmap.res, devices=[0], **kw)
    pl = plan.Planner(dmap.dist, dmap.res, **kw)
    calls = (lambda: mp.plan_points_device(*d_in), lambda: pl.plan_points_device(*d_in))
    for _ in range(args.warmup):
        for c in calls:
            c()
    torch.cuda.synchronize()
    ms_m, ms_p = [], []
    for _ in range(args.steps):
        ms_m.append(_timed(calls[0]))
        ms_p.append(_timed(calls[1]))
    result["one_gpu_multi_vs_planner"] = {
        "ms_multi_0": float(np.median(ms_m)), "ms_planner": float(np.median(ms_p)),
        "ms_multi_0_min_max": [float(min(ms_m)), float(max(ms_m))],
        "ms_planner_min_max": [float(min(ms_p)), float(max(ms_p))],
        "bit_identical": bool(_same(_host(calls[0]()), _host(calls[1]())))}
    mp.close()
    pl.close()

    print("%s, power limit %s, %d visible device(s); B = %d plans from points, TENSION2" % (
        result["gpu"]["name"], result["gpu"]["power_limit"], visible, B))
    print("%3s %12s %12s %8s %8s %8s  %s" % ("G", "dev plans/s", "host plans/s", "eff dev", "eff host", "same", "shard ms"))
    for G, e in result["scaling"].items():
        if isinstance(e, str):
            print("%3s %s" % (G, e))
        else:
            print("%3s %12.0f %12.0f %8.3f %8.3f %8s  %s" % (G, e["plans_per_s_device"], e["plans_per_s_host"],
                                                              e["efficiency_device"], e["efficiency_host"],
                                                              e["bit_identical_to_g1"],
                                                              " ".join("%.2f" % v for v in e["shard_total_ms"])))
    result["value"] = result["scaling"][str(largest)]["plans_per_s_device"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()
