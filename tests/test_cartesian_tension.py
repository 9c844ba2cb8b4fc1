"""The reference's TENSION smoothing method (TensionSmoother::osqpSmooth, tension_smoother.cpp:49-177): the Cartesian
tension QP over x, y and a lateral shift d per point, bounded by the map's obstacle distance.

CPU: the oracle's structure and closed forms (oracle/cartesian_oracle.assemble), the kernel source
(pqp_smoother_core.cuh through tests/emu/cartesian_driver.cpp) against the oracle, the ctypes mirrors of the parameter
structs against the C layout, and the oracle chain with TENSION. GPU: the standalone C ABI, the shared-memory limit of
its wider band, and the whole plan with smoothing_method = TENSION (stage parity through the trace, the independent
oracle chain, invariance, and that the option takes effect).

Parity bar as for TENSION2 (tests/test_smoother.py): identical status, iteration count and rho updates; the primal
vector within 1e-6 of the oracle's and passing the primal part of OSQP's termination test on the oracle-assembled QP.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import bounds_oracle as bo
from oracle import cartesian_oracle as co
from oracle import osqp_generic, plan_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_MAX, P_MAX, L_MAX, N_MAX = 64, 64, 64, 255


def wiggly(seed, p):
    """Points 1 m apart along a wiggly line with headings and clearances; a tenth of the clearances are 0."""
    rng = np.random.default_rng(seed)
    kap = 0.15 * np.sin(2 * np.pi * rng.uniform(0.5, 2.0) * np.arange(p) / max(p - 1, 1) + rng.uniform(0, 6))
    a = rng.uniform(-1, 1) + np.concatenate(([0.0], np.cumsum(kap[:-1])))
    x = rng.uniform(-5, 5) + np.concatenate(([0.0], np.cumsum(np.cos(a[:-1])))) + rng.normal(0, 0.3, p)
    y = rng.uniform(-5, 5) + np.concatenate(([0.0], np.cumsum(np.sin(a[:-1])))) + rng.normal(0, 0.3, p)
    cl = rng.uniform(0.0, 3.0, p)
    cl[rng.uniform(size=p) < 0.1] = 0.0
    return x, y, a, cl


def _check(res, x, y, a, cl):
    """The bar of this module for one QP; returns the oracle's solver."""
    p = len(x)
    ok, rx, ry, rs, g = co.osqp_smooth(x, y, a, cl)
    xs, _, _ = g.solution()
    assert res["status"] == g.status and res["iters"] == g.iters, (res["status"], res["iters"], g.status, g.iters)
    if "rho_updates" in res:
        assert res["rho_updates"] == g.rho_updates
    assert np.max(np.abs(res["x_full"][:3 * p] - xs)) < 1e-6
    assert np.allclose(res["x"][:p], rx, rtol=0, atol=1e-6) and np.allclose(res["y"][:p], ry, rtol=0, atol=1e-6)
    assert np.allclose(res["s"][:p], po.chord_length(res["x"][:p], res["y"][:p]), rtol=0, atol=1e-12)
    H, q, A, lo, up = co.assemble(x, y, a, cl)
    Ax = A @ res["x_full"][:3 * p]
    viol = np.maximum(lo - Ax, 0) + np.maximum(Ax - up, 0)
    scale = max(np.max(np.abs(Ax)), np.max(np.abs(np.clip(lo, -1e30, 1e30))))
    assert np.max(viol) < 1e-3 + 1e-3 * scale  # primal part of the termination test
    return g


# ------------------------------------------------------------------------------------------------- CPU
def test_oracle_structure_and_bounds():
    p = 9
    x, y, a, cl = wiggly(1, p)
    cl[3], cl[4], cl[5] = 0.7, 5.0, 0.0
    H, q, A, lo, up = co.assemble(x, y, a, cl)
    assert H.shape == (3 * p, 3 * p) and A.shape == (3 * p, 3 * p) and np.all(q == 0)
    assert A.nnz == 5 * p
    assert np.array_equal(lo[:p], x) and np.array_equal(up[:p], x) and np.array_equal(lo[p:2 * p], y)
    d_lo, d_up = lo[2 * p:], up[2 * p:]
    assert d_lo[0] == d_up[0] == 0.0 and d_lo[-1] == -0.5 and d_up[-1] == 0.5
    assert (d_lo[3], d_up[3]) == (-0.7, 0.7) and (d_lo[4], d_up[4]) == (-2.0, 2.0) and (d_lo[5], d_up[5]) == (0.0, 0.0)
    inner = np.minimum(cl[1:-1], 2.0)
    assert np.array_equal(d_up[1:-1], inner) and np.array_equal(d_lo[1:-1], -inner)
    # A's rows: x_i - cos(theta_i) d_i, y_i - sin(theta_i) d_i, d_i
    Ad = A.toarray()
    th = a + np.pi / 2
    for i in range(p):
        assert Ad[i, i] == 1 and Ad[i, 2 * p + i] == -np.cos(th[i]) and Ad[p + i, 2 * p + i] == -np.sin(th[i])
    # P: no cost on d (default deviation weight 0), x and y blocks equal, band of 3 points
    Hd = H.toarray()
    assert np.all(Hd[2 * p:, :] == 0) and np.array_equal(Hd[:p, :p], Hd[p:2 * p, p:2 * p])
    assert np.all(np.triu(Hd[:p, :p], 4) == 0) and Hd[0, 3] == -50.0  # w_dk * (-1) * 1


def test_p3_has_no_third_difference():
    x, y, a, cl = wiggly(2, 3)
    H, _, _, _, _ = co.assemble(x, y, a, cl)
    dds = np.outer([1, -2, 1], [1, -2, 1]) * co.W_CURVATURE
    Hd = H.toarray()
    assert np.array_equal(Hd[:3, :3], dds) and np.array_equal(Hd[3:6, 3:6], dds)
    H4, _, _, _, _ = co.assemble(*wiggly(2, 4))
    assert H4.toarray()[0, 3] == -co.W_CURVATURE_RATE  # p = 4 has one


def test_straight_line_in_free_space_stays_put():
    """A straight line costs nothing, so it stays put: d = 0 from OSQP's cold start at 0 when the line runs through
    the origin. The cost is also blind to rotating the line about its pinned first point (d linear in i); from an
    offset line the solver ends somewhere on that family, and the result is still a straight line."""
    from tests.emu import cartesian_emu as ce
    p = 30
    t = np.arange(p, dtype=np.float64)
    for x0, y0, h in ((0.0, 0.0, 0.0), (0.0, 0.0, 0.4), (3.0, -2.0, 0.4)):
        x, y, a = x0 + t * np.cos(h), y0 + t * np.sin(h), np.full(p, h)
        ok, rx, ry, rs, g = co.osqp_smooth(x, y, a, np.full(p, 10.0))
        assert ok
        d = g.solution()[0][2 * p:]
        if x0 == y0 == 0.0:
            assert np.max(np.abs(d)) < 1e-3 and np.max(np.abs(rx - x)) < 1e-3 and np.max(np.abs(ry - y)) < 1e-3
        u = np.array([rx[-1] - rx[0], ry[-1] - ry[0]]) / np.hypot(rx[-1] - rx[0], ry[-1] - ry[0])
        assert np.max(np.abs(-(rx - rx[0]) * u[1] + (ry - ry[0]) * u[0])) < 1e-3  # still straight
        assert abs(d[0]) < 1e-3 and np.max(np.abs(np.diff(d, 2))) < 1e-3 and np.max(np.abs(d)) <= 0.5 + 1e-3
        _check(ce.cartesian(x, y, a, np.full(p, 10.0)), x, y, a, np.full(p, 10.0))


def test_zero_clearance_pins_the_shift():
    p = 40
    x, y, a, _ = wiggly(3, p)
    free = np.full(p, 3.0)
    _, _, _, _, g0 = co.osqp_smooth(x, y, a, free)
    d0 = g0.solution()[0][2 * p:]
    pinned = [i for i in np.argsort(-np.abs(d0[1:-1]))[:5] + 1]
    assert np.min(np.abs(d0[pinned])) > 0.05  # these points move when they may
    cl = free.copy()
    cl[pinned] = 0.0
    ok, rx, ry, _, g = co.osqp_smooth(x, y, a, cl)
    xs = g.solution()[0]
    tol = 1e-3 + 1e-3 * np.max(np.abs(xs))  # OSQP's relative tolerance on the rows
    assert ok and np.max(np.abs(xs[2 * p + np.array(pinned)])) < tol
    assert np.max(np.abs(rx[pinned] - x[pinned])) < tol and np.max(np.abs(ry[pinned] - y[pinned])) < tol


def _active_case():
    x, y, a, cl = wiggly(4, 50)
    return x, y, a, np.where(cl > 0, 0.08, 0.0)  # a tight corridor: the bounds hold the points back


@pytest.mark.parametrize("case", ["p3", "p4", "wiggly12", "wiggly60", "wiggly120", "active", "off_map"])
def test_kernel_source_on_cpu(case):
    from tests.emu import cartesian_emu as ce
    if case == "active":
        x, y, a, cl = _active_case()
    elif case == "off_map":
        x, y, a, cl = wiggly(9, 25)
        cl[:] = 0.0  # every point off the map: all interior shifts pinned
    else:
        p = {"p3": 3, "p4": 4, "wiggly12": 12, "wiggly60": 60, "wiggly120": 120}[case]
        x, y, a, cl = wiggly(10 + p, p)
    res = ce.cartesian(x, y, a, cl)
    g = _check(res, x, y, a, cl)
    assert g.status == osqp_generic.SOLVED
    if case == "active":
        p = len(x)
        d = res["x_full"][2 * p + 1:3 * p - 1]
        bound = np.minimum(cl[1:-1], 2.0)
        assert np.sum(np.abs(np.abs(d) - bound) < 2e-3 * (1 + np.max(np.abs(res["x_full"])))) >= 3  # bounds active


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "pqp_plan.h"
#define F(T, m) printf("%s %zu\n", #m, offsetof(T, m))
int main(void) {
    printf("smoother_size %zu\nplan_size %zu\n", sizeof(pqp_smoother_params), sizeof(pqp_plan_params));
    F(pqp_smoother_params, reserved);
    F(pqp_smoother_params, cartesian_curvature_weight);
    F(pqp_smoother_params, cartesian_curvature_rate_weight);
    F(pqp_smoother_params, cartesian_deviation_weight);
    F(pqp_plan_params, smoother);
    F(pqp_plan_params, output_spacing);
    F(pqp_plan_params, constraint_end_heading);
    F(pqp_plan_params, smoothing_method);
    printf("smooth_tension2 %d\nsmooth_tension %d\n", PQP_PLAN_SMOOTH_TENSION2, PQP_PLAN_SMOOTH_TENSION);
    printf("trace_clearance %zu\ntrace_size %zu\n", offsetof(pqp_plan_trace, tension_clearance), sizeof(pqp_plan_trace));
    return 0;
}
"""


def test_param_layout_matches_ctypes():
    from path_optimizer_2_b200 import plan, smoother
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(src, "w") as f:
            f.write(_LAYOUT_C)
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    got = {k: int(v) for k, v in got.items()}
    S, P, T = smoother.SmootherParams, plan.PlanParams, plan.PlanTrace
    want = {"smoother_size": ctypes.sizeof(S), "plan_size": ctypes.sizeof(P), "reserved": S.reserved.offset,
            "cartesian_curvature_weight": S.cartesian_curvature_weight.offset,
            "cartesian_curvature_rate_weight": S.cartesian_curvature_rate_weight.offset,
            "cartesian_deviation_weight": S.cartesian_deviation_weight.offset, "smoother": P.smoother.offset,
            "output_spacing": P.output_spacing.offset, "constraint_end_heading": P.constraint_end_heading.offset,
            "smoothing_method": P.smoothing_method.offset, "smooth_tension2": plan.SMOOTH_TENSION2,
            "smooth_tension": plan.SMOOTH_TENSION, "trace_clearance": T.tension_clearance.offset,
            "trace_size": ctypes.sizeof(T)}
    assert got == want


def test_oracle_chain_straight_corridor_tension():
    from path_optimizer_2_b200 import abi
    dist = np.full((400, 400), 20.0, dtype=np.float32)  # 80 m x 80 m, free
    xs = np.arange(-20.0, 20.5, 1.0)
    o = co.plan(dist, 0.2, xs, np.zeros_like(xs), [-20.0, 0.0, 0.0, 0.0], [18.0, 0.0, 0.0], params=abi.default_params(),
                p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX)
    assert o["status"] == po.OK
    assert np.all(o["tension_clearance"] == 20.0)
    assert np.max(np.abs(o["tension_y"])) < 1e-3 and np.max(np.abs(o["path"][5])) < 1e-3


# ------------------------------------------------------------------------------------------------- GPU
def _map_cases(dmap, count):
    """Resampled reference lines through the map (what the plan hands the smoother), of varied length, with the map's
    obstacle distance at each point; one cut to p = 3."""
    from path_optimizer_2_b200 import sharedmap
    cases = []
    for b in range(count):
        rx, ry, _, _ = sharedmap.make_plan_inputs(1, n=30 + 7 * b, first=300 + b, dmap=dmap)
        s = po.chord_length(rx[0], ry[0])
        rows = po.spline_rows(s, rx[0], ry[0])
        x, y, a, _, _ = po.segment(rows, po.segment_count(s[-1]))
        if b == 0:
            x, y, a = x[:3], y[:3], a[:3]
        cl = bo.map_distance(dmap.dist, dmap.res, x, y)
        if b % 2:
            cl = 0.02 * cl  # a tight corridor: the shift bounds become active
        if b % 4 == 2:
            cl[::5] = 0.0   # points on obstacles
        cases.append((x, y, a, cl))
    return cases


@pytest.mark.gpu
def test_gpu_standalone_matches_oracle_and_device_call():
    import torch
    from path_optimizer_2_b200 import sharedmap, smoother
    dmap = sharedmap.DistanceMap()
    cases = _map_cases(dmap, 24)
    p_max = max(len(c[0]) for c in cases)
    sm = smoother.Smoother(p_max=p_max, batch_max=32)
    r = sm.cartesian_tension(*[[c[i] for c in cases] for i in range(4)], full=True)
    zeros = active = 0
    for b, (x, y, a, cl) in enumerate(cases):
        p = len(x)
        xf = r["x_full"][b]
        _check(dict(status=r["status"][b], iters=r["iters"][b], x=r["x"][b], y=r["y"][b], s=r["s"][b], x_full=xf), x, y, a, cl)
        zeros += int(np.sum(cl[1:-1] == 0))
        active += int(np.sum(np.abs(np.abs(xf[2 * p + 1:3 * p - 1]) - np.minimum(cl[1:-1], 2.0)) < 1e-2))
    print("cartesian kernel: %.3f ms for %d QPs (p = 3 .. %d), %d zero clearances, %d shifts at their bound"
          % (sm.last_kernel_ms, len(cases), p_max, zeros, active))
    assert zeros > 0 and active > zeros
    dev = torch.device("cuda:0")
    t = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(dev)  # noqa: E731
    pad = lambda i: smoother._pad([c[i] for c in cases], p_max)  # noqa: E731
    out = sm.cartesian_tension_device(t(r["p"]), t(pad(0)), t(pad(1)), t(pad(2)), t(pad(3)), full=True)
    torch.cuda.synchronize()
    for k in ("x", "y", "s", "status", "iters", "x_full"):
        assert np.array_equal(out[k].cpu().numpy(), r[k]), k
    sm.close()


@pytest.mark.gpu
def test_gpu_cartesian_limit_leaves_the_handle_usable():
    from path_optimizer_2_b200 import plan, sharedmap, smoother, solver
    from tests.test_smoother import _check_tension, raw_reference
    sm = smoother.Smoother(p_max=900, batch_max=2)  # TENSION2's band fits at 900, the Cartesian one ends at 877
    x, y, a, cl = wiggly(5, 20)
    with pytest.raises(solver.PqpError) as e:
        sm.cartesian_tension([x], [y], [a], [cl])
    assert e.value.code == -1 and "shared-memory" in str(e.value), str(e.value)
    cases = [raw_reference(7, 30), raw_reference(8, 45)]
    r = sm.tension(*[[c[i] for c in cases] for i in range(5)], full=True)
    for b, c in enumerate(cases):
        p = len(c[0])
        _check_tension(dict(status=r["status"][b], iters=r["iters"][b], x=r["x"][b, :p], y=r["y"][b, :p], s=r["s"][b, :p],
                            x_full=r["x_full"][b, :4 * p - 1]), *c)
    sm.close()
    ok = smoother.Smoother(p_max=877, batch_max=1)  # the last p_max that fits
    r = ok.cartesian_tension([x], [y], [a], [cl], full=True)
    _check(dict(status=r["status"][0], iters=r["iters"][0], x=r["x"][0], y=r["y"][0], s=r["s"][0], x_full=r["x_full"][0]),
           x, y, a, cl)
    ok.close()
    dmap = sharedmap.DistanceMap()
    with pytest.raises(solver.PqpError) as e:  # the plan checks the limit at create
        plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=900, layers_max=L_MAX, n_max=N_MAX, batch_max=1,
                     params=plan.default_params("TENSION"))
    assert e.value.code == -1 and "TENSION" in str(e.value)
    with pytest.raises(solver.PqpError) as e:  # as the reference's flag validator: only the two methods
        plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=1,
                     params=plan.default_params(2))
    assert e.value.code == -1 and "smoothing_method" in str(e.value)


@pytest.fixture(scope="module")
def world():
    from path_optimizer_2_b200 import sharedmap
    dmap = sharedmap.DistanceMap()
    raw_x, raw_y, start, target = sharedmap.make_plan_inputs(64, dmap=dmap)
    return dmap, raw_x, raw_y, start, target


@pytest.fixture(scope="module")
def planners(world):
    from path_optimizer_2_b200 import plan
    dmap = world[0]
    mk = lambda params: plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX,  # noqa: E731
                                     n_max=N_MAX, batch_max=64, params=params)
    pls = {"TENSION": mk(plan.default_params("TENSION")), "TENSION2": mk(plan.default_params())}
    yield pls
    for pl in pls.values():
        pl.close()


@pytest.fixture(scope="module")
def runs(world, planners):
    _, raw_x, raw_y, start, target = world
    out = {}
    for name, pl in planners.items():
        c0 = pl.launch_count
        out[name] = pl.plan(raw_x, raw_y, start, target, trace=True)
        out[name + "_launches"] = pl.launch_count - c0
    return out


@pytest.mark.gpu
def test_gpu_plan_tension_stage_parity(world, planners, runs):
    from path_optimizer_2_b200 import plan
    dmap = world[0]
    run = runs["TENSION"]
    T = run.trace
    assert np.mean(run.status == plan.OK) >= 0.8, run.status_names()
    for b in range(64):
        p = int(T["seg_p"][b])
        if p == 0:
            continue
        sx, sy, sa = T["seg_x"][b, :p], T["seg_y"][b, :p], T["seg_angle"][b, :p]
        cl = T["tension_clearance"][b, :p]
        assert np.allclose(cl, bo.map_distance(dmap.dist, dmap.res, sx, sy), rtol=0, atol=1e-12), b
        if b < 8:
            ok, tx, ty, _, g = co.osqp_smooth(sx, sy, sa, cl)
            assert T["tension_status"][b] == g.status and T["tension_iters"][b] == g.iters, b
            assert np.allclose(T["tension_x"][b, :p], tx, rtol=0, atol=1e-6)
            assert np.allclose(T["tension_y"][b, :p], ty, rtol=0, atol=1e-6)
        if run.status[b] == plan.TENSION_FAILED:
            continue
        tx, ty, ts = T["tension_x"][b, :p], T["tension_y"][b, :p], T["tension_s"][b, :p]
        assert np.allclose(ts, po.chord_length(tx, ty), rtol=0, atol=1e-12)
        if run.status[b] == plan.SPLINE_DEGENERATE:
            continue
        rows, length = po.tension_epilogue(tx, ty, ts)
        assert np.array_equal(T["tension_spline"][b, :, :p], rows) and T["tension_length"][b] == length, b


@pytest.mark.gpu
def test_gpu_plan_tension_independent_oracle_chain(world, planners, runs):
    dmap, raw_x, raw_y, start, target = world
    run = runs["TENSION"]
    differ = compared = 0
    for b in range(64):
        o = co.plan(dmap.dist, dmap.res, raw_x[b], raw_y[b], start[b], target[b], params=planners["TENSION"].params.solver,
                    p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX)
        assert o["status"] == run.status[b], (b, o["status"], run.status_names()[b])
        if o["status"] != po.OK:
            continue
        n_out = int(run.trace["dp_n_out"][b])
        if n_out != o["dp"]["n_out"] or not np.array_equal(run.trace["dp_chosen"][b, :n_out], o["dp"]["chosen"]):
            differ += 1
            continue
        n = int(run.n[b])
        if n == o["n"]:
            compared += 1
            assert np.max(np.abs(run.path[b, 5, :n] - o["path"][5])) < 1e-2, b
    print("independent TENSION chain: %d of 64 paths chose a different DP corridor, %d final paths compared"
          % (differ, compared))


@pytest.mark.gpu
def test_gpu_plan_tension_invariance_and_selection(world, planners, runs):
    import torch
    from path_optimizer_2_b200 import plan
    dmap, raw_x, raw_y, start, target = world
    pl, run = planners["TENSION"], runs["TENSION"]
    # one more launch per call than TENSION2 (the clearance kernel)
    assert runs["TENSION_launches"] == runs["TENSION2_launches"] + 1, (runs["TENSION_launches"], runs["TENSION2_launches"])
    # device call = host call, bitwise
    B = 64
    r = np.array([len(v) for v in raw_x], dtype=np.int32)
    rx, ry = np.zeros((B, R_MAX)), np.zeros((B, R_MAX))
    for b in range(B):
        rx[b, :r[b]], ry[b, :r[b]] = raw_x[b], raw_y[b]
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    out = pl.plan_device(t(rx), t(ry), t(r), t(start), t(target), trace=True)
    torch.cuda.synchronize()
    for k in ("status", "n", "path", "cost", "iters"):
        assert np.array_equal(out[k].cpu().numpy(), getattr(run, k)), k
    for k in ("tension_clearance", "tension_x", "tension_y", "tension_spline", "ref_spline"):
        assert np.array_equal(out["trace"][k].cpu().numpy(), run.trace[k]), k
    # B = 1 equals its row of the batch, bitwise
    for b in (0, 17, 63):
        one = pl.plan([raw_x[b]], [raw_y[b]], start[b:b + 1], target[b:b + 1], trace=True)
        assert one.status[0] == run.status[b] and one.n[0] == run.n[b]
        assert np.array_equal(one.path[0], run.path[b]) and one.cost[0] == run.cost[b]
        p = int(run.trace["seg_p"][b])  # entries past p are unspecified
        assert one.trace["seg_p"][0] == p
        for k in ("tension_clearance", "tension_x", "tension_y"):
            assert np.array_equal(one.trace[k][0, :p], run.trace[k][b, :p]), k
    ms = pl.last_stage_ms
    assert ms["total"] > 0 and ms["total"] >= ms["smoothing"]
    # the option takes effect: the two methods smooth differently
    t2 = runs["TENSION2"].trace
    both = (run.trace["tension_status"] == 0) & (t2["tension_status"] == 0)
    assert both.sum() >= 32
    diff = [np.max(np.abs(run.trace["tension_x"][b] - t2["tension_x"][b])) for b in np.nonzero(both)[0]]
    assert np.median(diff) > 1e-3, diff
    # an explicit 0 is the default
    p0 = plan.default_params()
    p0.smoothing_method = plan.SMOOTH_TENSION2
    explicit = plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=64,
                            params=p0)
    e = explicit.plan(raw_x, raw_y, start, target)
    explicit.close()
    d = runs["TENSION2"]
    for k in ("status", "n", "path", "cost", "iters"):
        assert np.array_equal(getattr(e, k), getattr(d, k)), k
