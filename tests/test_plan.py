"""The whole plan (include/pqp_plan.h): PathOptimizer::solve for a batch, from bSpline() samples to final path.

CPU: the C ABI declaration, the glue's per-path source (pqp_plan_core.cuh compiled with g++) against
oracle/plan_oracle.py, and the oracle chain on a closed-form case. GPU: conditional stage parity through the trace
(each stage against its oracle fed with the GPU's previous stage), the independent oracle chain, every status code,
and device / host / batch invariance.
"""
import math
import os
import re

import numpy as np
import pytest

from oracle import bounds_oracle as bo
from oracle import dp_oracle, plan_oracle as po, smoother_oracle
from path_optimizer_2_b200 import abi, plan, sharedmap
from tests.emu import plan_emu as pe

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_MAX, P_MAX, L_MAX, N_MAX = 64, 64, 64, 255


# ------------------------------------------------------------------------------------------------- CPU
def test_header_symbols_match_binding():
    src = open(os.path.join(ROOT, "include", "pqp_plan.h")).read()
    declared = sorted(set(re.findall(r"\b(pqp_plan\w*)\s*\(", src)))
    assert declared == sorted(plan.EXPORTED_SYMBOLS)
    from path_optimizer_2_b200 import solver
    if os.path.exists(solver.LIB_PATH):
        out = os.popen("nm -D --defined-only %s" % solver.LIB_PATH).read()
        for s in plan.EXPORTED_SYMBOLS:
            assert re.search(r"\bT %s$" % s, out, re.M), s


def test_spline_fit_bitwise_random_and_circle():
    rng = np.random.default_rng(3)
    for k in (3, 4, 17, 120):
        sx = np.cumsum(rng.uniform(0.05, 2.0, k))
        y = rng.normal(0, 3, k)
        got, want = pe.fit(sx, y), bo.natural_spline(sx, y)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
    r = 12.0
    t = np.linspace(0, 1.5, 60)
    x, y = r * np.cos(t), r * np.sin(t)
    s, ok = pe.chord(x, y)
    assert ok and np.array_equal(s, po.chord_length(x, y))
    rows = pe.spline_rows(s, x, y)
    assert np.array_equal(rows, po.spline_rows(s, x, y))
    _, _, _, k, _ = pe.segment(rows, int(s[-1]))
    assert np.all(np.abs(k[2:-2] - 1.0 / r) < 1e-4)


def test_segmentation_matches_oracle():
    rng = np.random.default_rng(5)
    t = np.linspace(0, 30, 31)
    x, y = t + rng.normal(0, 0.05, 31), 0.02 * t * t + rng.normal(0, 0.05, 31)
    s, ok = pe.chord(x, y)
    assert ok
    p = pe.segment_count(s[-1])
    assert p == po.segment_count(s[-1]) == int(math.ceil(s[-1])) + 1  # the last sample overshoots the end
    assert (p - 1) >= s[-1] and (p - 2) < s[-1]
    assert pe.segment_count(s[-1], cap=p - 1) == p  # cap + 1: over capacity
    rows = po.spline_rows(s, x, y)
    got, want = pe.segment(rows, p), po.segment(rows, p)
    for g, w in zip(got, want):
        assert np.allclose(g, w, rtol=0, atol=1e-12)


def test_epilogues_match_oracle():
    rng = np.random.default_rng(7)
    tx = np.linspace(0, 40, 41)
    ty = np.sin(tx / 7.0) + rng.normal(0, 0.01, 41)
    ts, _ = pe.chord(tx, ty)
    rows, length = po.tension_epilogue(tx, ty, ts)
    assert np.array_equal(rows, pe.spline_rows(ts, tx, ty)) and length == ts[-1] + 3.0
    layer_s = np.arange(0.5, 40, 1.5)
    off = rng.uniform(-1, 1, len(layer_s))
    for g, w in zip(pe.post_points(rows, layer_s, off), po.post_epilogue(rows, layer_s, off)):
        assert np.allclose(g, w, rtol=0, atol=1e-12)


def _straight(length=40.0):
    s = np.arange(0.0, length + 1, 1.0)
    return po.spline_rows(s, s.copy(), np.zeros_like(s))


def test_process_reference_projection_and_gates():
    rows = _straight()
    # target on the line: exact projection
    st, l0, psi0, max_s = pe.process(rows, 40.0, [0.0, 0.0, 0.0, 0.0], [23.25, 0.0, 0.0])
    assert st == po.OK and max_s == 23.25
    assert (st, l0, psi0, max_s) == po.process_reference(rows, 40.0, [0.0, 0.0, 0.0, 0.0], [23.25, 0.0, 0.0])
    # target beyond the end: the length is kept
    st, _, _, max_s = pe.process(rows, 40.0, [0, 0, 0, 0], [45.0, 1.0, 0.0])
    assert st == po.OK and max_s == 40.0
    # init offset sign: the vehicle's lateral offset from the line, positive to the left
    _, l0, _, _ = pe.process(rows, 40.0, [0.0, 1.5, 0.0, 0.0], [20, 0, 0])
    assert l0 == 1.5
    _, l0, _, _ = pe.process(rows, 40.0, [0.0, -1.5, 0.0, 0.0], [20, 0, 0])
    assert l0 == -1.5
    # 75 degree gate, both sides, both signs
    for deg, want in ((74.9, po.OK), (75.1, po.INIT_HEADING), (-74.9, po.OK), (-75.1, po.INIT_HEADING)):
        h = math.radians(deg)
        got = pe.process(rows, 40.0, [0.0, 0.0, h, 0.0], [20, 0, 0])
        assert got[0] == want and got[0] == po.process_reference(rows, 40.0, [0.0, 0.0, h, 0.0], [20, 0, 0])[0]
        assert abs(got[2] - h) < 1e-12
    assert pe.process(rows, 0.0, [0, 0, 0, 0], [20, 0, 0])[0] == po.EMPTY_REFERENCE


def test_end_heading_rows_signed_and_blocked():
    for deg, rows_on in ((69.9, True), (70.1, False), (-69.9, True), (-80.0, True)):
        lo, hi = pe.end_heading(True, False, math.radians(deg), 0.0)
        assert (lo, hi) == po.end_heading_rows(True, False, math.radians(deg), 0.0)
        assert (abs(lo) < 1e29) == rows_on
        if rows_on:
            assert abs(lo - (math.radians(deg) - 0.087)) < 1e-15 and abs(hi - (math.radians(deg) + 0.087)) < 1e-15
    assert pe.end_heading(True, True, 0.1, 0.0) == (-1e30, 1e30)  # blocked path: no rows
    assert pe.end_heading(False, False, 0.1, 0.0) == (-1e30, 1e30)


def test_precise_size_rough_constraints():
    s = np.arange(0.0, 50.0, 0.3)
    assert pe.precise(s, False) == len(s)
    assert pe.precise(s, True, 30.0) == po.precise_size(s, len(s), True, 30.0) == int(np.sum(s < 30.0))
    assert pe.precise(s[:10], True, 30.0) == 10


def test_placeholder_line_is_valid_dp_input():
    from tests.emu import dp_emu
    s, x, y = pe.placeholder()
    rows = pe.spline_rows(s, x, y)
    assert np.array_equal(rows, po.spline_rows(s, x, y))
    dmap = sharedmap.DistanceMap()
    spline = np.zeros((3, 9, 8))
    spline[:, :, :3] = rows
    starts = np.array([[0.5, 0.0, 0.0], [0.5, 30.0, 1.0], [1e4, -1e4, 3.0]])
    r = dp_emu.search(dmap.dist, dmap.res, spline, np.full(3, 3, np.int32), np.full(3, 2.0), starts, layers_max=8)
    assert r.status[1] == 0 and r.status[2] == 0  # far vehicles: rejected at once
    assert r.status[0] in (0, 1) and 1 <= r.n_layers[0] <= 8 and r.n_out[0] <= r.n_layers[0]


def test_oracle_chain_straight_corridor():
    dist = np.full((400, 400), 20.0, dtype=np.float32)  # 80 m x 80 m, free
    xs = np.arange(-20.0, 20.5, 1.0)
    o = po.plan(dist, 0.2, xs, np.zeros_like(xs), [-20.0, 0.0, 0.0, 0.0], [18.0, 0.0, 0.0], params=abi.default_params(),
                p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX)
    assert o["status"] == po.OK
    assert o["l0"] == 0.0 and o["psi0"] == 0.0
    assert np.max(np.abs(o["path"][5])) < 1e-3


# ------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def world():
    dmap = sharedmap.DistanceMap()
    raw_x, raw_y, start, target = sharedmap.make_plan_inputs(64, dmap=dmap)
    return dmap, raw_x, raw_y, start, target


@pytest.fixture(scope="module")
def planner(world):
    pl = plan.Planner(world[0].dist, world[0].res, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=64)
    yield pl
    pl.close()


@pytest.fixture(scope="module")
def run64(world, planner):
    _, raw_x, raw_y, start, target = world
    return planner.plan(raw_x, raw_y, start, target, trace=True)


def _close(a, b, tol):
    return np.allclose(a, b, rtol=0, atol=tol)


@pytest.mark.gpu
def test_conditional_stage_parity(world, planner, run64):
    from tests import parity
    dmap, raw_x, raw_y, start, target = world
    T, params = run64.trace, planner.params.solver
    assert np.mean(run64.status == plan.OK) > 0.8, run64.status_names()
    for b in range(64):
        st = int(run64.status[b])
        s_raw = po.chord_length(raw_x[b], raw_y[b])
        r = len(raw_x[b])
        assert np.array_equal(T["raw_spline"][b, :, :r], po.spline_rows(s_raw, raw_x[b], raw_y[b])), b  # bitwise
        p = int(T["seg_p"][b])
        assert p == po.segment_count(s_raw[-1])
        seg = po.segment(T["raw_spline"][b, :, :r], p)
        for name, w in zip(("seg_x", "seg_y", "seg_angle", "seg_k", "seg_s"), seg):
            assert _close(T[name][b, :p], w, 1e-12), (b, name)
        if b < 8:  # the FP64 QP restatements are slow: a sample
            ok, tx, ty, _, g = smoother_oracle.osqp_smooth(*(T[n][b, :p] for n in ("seg_x", "seg_y", "seg_angle", "seg_k", "seg_s")))
            assert T["tension_status"][b] == g.status and T["tension_iters"][b] == g.iters
            assert _close(T["tension_x"][b, :p], tx, 1e-6) and _close(T["tension_y"][b, :p], ty, 1e-6)
        if st == plan.TENSION_FAILED:
            continue
        tx, ty, ts = T["tension_x"][b, :p], T["tension_y"][b, :p], T["tension_s"][b, :p]
        assert _close(ts, po.chord_length(tx, ty), 1e-12)
        rows, length = po.tension_epilogue(tx, ty, ts)
        assert np.array_equal(T["tension_spline"][b, :, :p], rows) and T["tension_length"][b] == length
        d = dp_oracle.graph_search_dp(dmap.dist, dmap.res, rows, length, start[b, :3])
        if not d["ok"]:
            assert st == plan.DP_VEHICLE_FAR
            continue
        n_out = int(T["dp_n_out"][b])
        assert n_out == d["n_out"] and np.array_equal(T["dp_chosen"][b, :n_out], d["chosen"]), b
        if st == plan.POST_TOO_SHORT:
            continue
        ls, lo, up = T["dp_layer_s"][b, :n_out], T["dp_lower"][b, :n_out], T["dp_upper"][b, :n_out]
        if b < 8:
            okp, off, gp = smoother_oracle.post_smooth(ls, lo, up, T["dp_vehicle_l"][b])
            assert T["post_status"][b] == gp.status and T["post_iters"][b] == gp.iters
            assert _close(T["post_offsets"][b, :n_out], off, 1e-6)
        if st == plan.POST_FAILED:
            continue
        ps, px, py = po.post_epilogue(T["tension_spline"][b, :, :p], ls, T["post_offsets"][b, :n_out])
        ref = T["ref_spline"][b, :, :n_out]
        assert _close(ref[0], ps, 1e-12) and _close(ref[4], px, 1e-12) and _close(ref[8], py, 1e-12)
        assert np.array_equal(ref, po.spline_rows(ref[0], ref[4], ref[8]))  # the fit itself: bitwise
        pst, l0, psi0, max_s = po.process_reference(ref, ref[0, -1], start[b], target[b])
        assert abs(T["inst"][b, abi.I_L0] - l0) <= 1e-12 and abs(T["inst"][b, abi.I_PSI0] - psi0) <= 1e-12
        if st in (plan.EMPTY_REFERENCE, plan.INIT_HEADING):
            assert pst == st
            continue
        assert abs(T["max_s"][b] - max_s) <= 1e-12
        s, x, y, h, k = bo.build_states(ref, T["max_s"][b], 0.15, 0.3, True)
        total = int(T["total"][b])
        assert total == len(s)
        if st == plan.TOO_MANY_KNOTS:
            continue
        for i, w in enumerate((s, x, y, h)):
            assert _close(T["states"][b, i, :total], w, 1e-9), (b, i)
        bnd, nv = bo.update_bounds(dmap.dist, dmap.res, ref, *T["states"][b, :, :total])
        assert nv == T["n_valid"][b]
        dd = np.abs(bnd[:, :nv] - T["bounds"][b, :, :nv])
        assert (dd > 1e-9).mean() < 5e-3 and dd.max() < 0.31  # as test_bounds.py / smoke()
        if st == plan.BLOCKED_AT_START:
            continue
        knots, inst, pp = po.instance_block(T["states"][b, :, :total], T["curvature"][b, :total], T["bounds"][b, :, :total],
                                            nv, start[b], target[b], T["inst"][b, 0], T["inst"][b, 1])
        assert pp == T["p"][b] and np.array_equal(inst, T["inst"][b])
        assert np.array_equal(knots, T["knots"][b, :, :nv])
        if b >= 8:
            continue
        hb = abi.HostBatch(T["knots"][b:b + 1], T["inst"][b:b + 1], np.array([nv], dtype=np.int32), np.array([pp], dtype=np.int32))
        res1 = abi.HostResult(1, N_MAX, full=True)
        res1.sol[0], res1.status[0], res1.iters[0] = T["sol1"][b], T["status1"][b], T["iters1"][b]
        res1.x_full[0], res1.y_full[0], res1.z_full[0] = T["x_full1"][b], T["y_full1"][b], T["z_full1"][b]
        res1.cost[0] = 0.5 * float(np.dot(parity.oracle_reference(params, hb, 0).problem()[0] * T["x_full1"][b, :6 * nv - 1],
                                          T["x_full1"][b, :6 * nv - 1]))
        parity.check_instance(params, hb, res1, 0, oracle_solver=parity.oracle_reference(params, hb, 0), label="plan 1st")
        if st == plan.PRE_SOLVE_FAILED:
            continue
        sol1 = T["sol1"][b]
        res2 = abi.HostResult(1, N_MAX, full=True)
        res2.status[0], res2.iters[0], res2.cost[0] = abi.PQP_SOLVED, run64.iters[b, 1], run64.cost[b]
        res2.x_full[0], res2.y_full[0], res2.z_full[0] = T["x_full2"][b], T["y_full2"][b], T["z_full2"][b]
        if st == plan.OK:
            n = int(run64.n[b])
            path = run64.path[b]
            res2.sol[0, 0, :n], res2.sol[0, 1, :n], res2.sol[0, 2, :n] = path[5, :n], path[6, :n], path[3, :n]
            res2.sol[0, 3, :n - 1] = path[4, :n - 1]
            parity.check_instance(params, hb, res2, 0, label="plan 2nd",
                                  oracle_solver=parity.oracle_reference(params, hb, 0, warm_from=(sol1[0], sol1[1], sol1[2])))
            from oracle import oracle
            xyh = oracle.frenet_to_cartesian(T["states"][b, 1:4, :n], path[5, :n], path[6, :n])
            assert _close(path[:3, :n], xyh, 1e-12)


@pytest.mark.gpu
def test_independent_oracle_chain(world, planner, run64):
    dmap, raw_x, raw_y, start, target = world
    differ = 0
    for b in range(64):
        o = po.plan(dmap.dist, dmap.res, raw_x[b], raw_y[b], start[b], target[b], params=planner.params.solver,
                    p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX)
        assert o["status"] == run64.status[b], (b, o["status"], run64.status_names()[b])
        if o["status"] != po.OK:
            continue
        n_out = int(run64.trace["dp_n_out"][b])
        if n_out != o["dp"]["n_out"] or not np.array_equal(run64.trace["dp_chosen"][b, :n_out], o["dp"]["chosen"]):
            differ += 1
            continue
        n = int(run64.n[b])
        if n == o["n"]:
            assert np.max(np.abs(run64.path[b, 5, :n] - o["path"][5])) < 1e-2, b  # the x* envelope of SURVEY §8c
    print("independent chain: %d of 64 paths chose a different DP corridor" % differ)


def _case_inputs(world, idx):
    _, raw_x, raw_y, start, target = world
    return [raw_x[i].copy() for i in idx], [raw_y[i].copy() for i in idx], start[idx].copy(), target[idx].copy()


@pytest.mark.gpu
def test_every_status_code_is_reached(world, planner, run64):
    dmap = world[0]
    idx = list(range(8))
    rx, ry, st, tg = _case_inputs(world, idx)
    rx[0], ry[0] = rx[0][:2], ry[0][:2]                      # too few samples
    h = st[1, 2]
    st[1, 0] -= 15.0 * math.sin(h)                          # vehicle 15 m off the line
    st[1, 1] += 15.0 * math.cos(h)
    st[2, 2] -= math.radians(80.0)                          # start heading rotated 80 degrees (clockwise)
    rx[4], ry[4] = rx[4][::-1].copy(), ry[4][::-1].copy()
    rx[4][1] = rx[4][0]                                      # repeated sample: non-increasing s
    ry[4][1] = ry[4][0]
    res = planner.plan(rx, ry, st, tg, trace=True)
    assert [res.status[b] for b in (0, 1, 2, 4)] == [plan.SPLINE_DEGENERATE, plan.DP_VEHICLE_FAR, plan.INIT_HEADING,
                                                     plan.SPLINE_DEGENERATE], res.status_names()
    for b in (3, 5, 6, 7):  # failed paths do not disturb their neighbours
        assert res.status[b] == run64.status[b] and np.array_equal(res.path[b], run64.path[b])
    # a reference longer than n_max allows: a planner with few knots
    small = plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=40, batch_max=2)
    rx2, ry2, st2, tg2 = _case_inputs(world, [0, 1])
    r2 = small.plan(rx2, ry2, st2, tg2)
    assert list(r2.status) == [plan.TOO_MANY_KNOTS] * 2
    # a raw list longer than p_max allows (about 45 samples resampled to about 46 points, p_max = 32)
    short = plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=32, layers_max=L_MAX, n_max=N_MAX, batch_max=2)
    assert list(short.plan(rx2, ry2, st2, tg2).status) == [plan.TOO_MANY_POINTS] * 2
    short.close()
    # too few DP layers: a planner whose layer capacity is below the path's
    few = plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=P_MAX, layers_max=8, n_max=N_MAX, batch_max=2)
    assert list(few.plan(rx2, ry2, st2, tg2).status) == [plan.TOO_MANY_POINTS] * 2
    small.close()
    few.close()
    # a pinch on the reference where the front circle of the first state reaches it (3.9 m ahead): a dot of a few
    # cells, small enough to pass between the DP's nodes, so the reference still runs through it
    b = int(np.nonzero(run64.status == plan.OK)[0][0])
    T = run64.trace
    i = int(np.argmin(np.abs(T["states"][b, 0, :T["total"][b]] - 3.9)))
    dist = dmap.dist.copy()
    ci = int((dmap.lx / 2 - T["states"][b, 1, i]) / dmap.res)
    cj = int((dmap.ly / 2 - T["states"][b, 2, i]) / dmap.res)
    dist[ci - 1:ci + 2, cj - 1:cj + 2] = 0.0
    pinch = plan.Planner(dist, dmap.res, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=1)
    rx3, ry3, st3, tg3 = _case_inputs(world, [b])
    r3 = pinch.plan(rx3, ry3, st3, tg3, trace=True)
    pinch.close()
    o3 = po.plan(dist, dmap.res, rx3[0], ry3[0], st3[0], tg3[0], params=planner.params.solver, p_max=P_MAX,
                 layers_max=L_MAX, n_max=N_MAX)
    assert r3.status[0] == o3["status"] == plan.BLOCKED_AT_START, (r3.status_names(), o3["status"])
    seen = set(int(v) for v in np.concatenate([res.status, r2.status, r3.status, run64.status]))
    print("status codes reached:", [plan.STATUS_NAMES[c] for c in sorted(seen)])


@pytest.mark.gpu
def test_device_call_and_batch_invariance(world, planner, run64):
    import torch
    _, raw_x, raw_y, start, target = world
    dev = torch.device("cuda:0")
    B = 64
    r = np.array([len(v) for v in raw_x], dtype=np.int32)
    rx, ry = np.zeros((B, R_MAX)), np.zeros((B, R_MAX))
    for b in range(B):
        rx[b, :r[b]], ry[b, :r[b]] = raw_x[b], raw_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    out = planner.plan_device(t(rx), t(ry), t(r), t(start), t(target), trace=True)
    torch.cuda.synchronize()
    for k in ("status", "n", "path", "cost", "iters"):
        assert np.array_equal(out[k].cpu().numpy(), getattr(run64, k)), k
    for k in ("knots", "sol1", "states", "ref_spline"):
        assert np.array_equal(out["trace"][k].cpu().numpy(), run64.trace[k]), k
    for b in (0, 17, 63):  # B = 1 equals its row of the batch, bitwise
        one = planner.plan([raw_x[b]], [raw_y[b]], start[b:b + 1], target[b:b + 1])
        assert one.status[0] == run64.status[b] and one.n[0] == run64.n[b]
        assert np.array_equal(one.path[0], run64.path[b]) and one.cost[0] == run64.cost[b]
    ms = planner.last_stage_ms
    assert ms["total"] > 0 and ms["total"] >= ms["smoothing"]
    assert planner.launch_count > 0


@pytest.mark.gpu
def test_ragged_batch():
    dmap = sharedmap.DistanceMap()
    raw_x, raw_y, start, target = [], [], [], []
    for i, n in enumerate((40, 120, 60, 200, 80, 300)):  # lines of 20 .. 98 m
        rx, ry, st, tg = sharedmap.make_plan_inputs(1, n=n, first=100 + i, dmap=dmap)
        raw_x += rx
        raw_y += ry
        start.append(st[0])
        target.append(tg[0])
    start, target = np.array(start), np.array(target)
    pl = plan.Planner(dmap.dist, dmap.res, r_max=128, p_max=128, layers_max=96, n_max=511, batch_max=6)
    res = pl.plan(raw_x, raw_y, start, target)
    for b in range(6):
        o = po.plan(dmap.dist, dmap.res, raw_x[b], raw_y[b], start[b], target[b], params=pl.params.solver, p_max=128,
                    layers_max=96, n_max=511)
        assert res.status[b] == o["status"], (b, res.status_names()[b], o["status"])
        if o["status"] == po.OK:
            assert res.n[b] == o["n"]
    assert np.mean(res.status == plan.OK) >= 0.5, res.status_names()
    pl.close()
