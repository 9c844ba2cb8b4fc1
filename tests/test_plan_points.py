"""The whole plan from the reference points (pqp_plan_points): bSpline() on the GPU, then the pqp_plan chain.

CPU: oracle/bspline_oracle.py against scipy's B-spline, its end samples, degree thresholds and sample counts against
a literal transcription of the reference's loop; the kernel's source (pqp_plan_core.cuh under g++) against the oracle
bit for bit; the oracle chain from points on a free corridor; the C layouts of the new structs. GPU: the traced
samples against the oracle, pqp_plan_points against pqp_plan fed with those samples, the independent oracle chain,
every new failure with its neighbours unchanged, device / host / batch invariance, launch counts and stage times, under
both smoothing methods.
"""
import ctypes
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import bspline_oracle as bso
from oracle import plan_oracle as po
from path_optimizer_2_b200 import abi, plan, sharedmap
from tests.emu import bspline_emu as be

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_MAX, P_MAX, L_MAX, N_MAX = 64, 64, 64, 255


# ------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_scipy_bspline():
    from scipy.interpolate import BSpline
    rng = np.random.default_rng(1)
    worst = 0.0
    for degree in (3, 4, 5):
        for m in list(range(degree + 1, 16)) + [23, 31, 40]:
            px, py = np.cumsum(rng.normal(0, 8, m)), np.cumsum(rng.normal(0, 8, m))
            knots = np.array([bso.knot(i, degree, m) for i in range(m + degree + 1)])
            t = np.concatenate(([0.0], np.sort(rng.uniform(0, 1, 40)), knots[degree + 1:m], [1.0]))
            got = np.array([bso.de_boor(px, py, degree, v) for v in t])
            want = np.stack([BSpline(knots, px, degree)(t), BSpline(knots, py, degree)(t)], axis=1)
            worst = max(worst, float(np.max(np.abs(got - want))))
    assert worst < 1e-10, worst


def test_end_samples_are_the_end_points():
    rng = np.random.default_rng(2)
    for m in (4, 5, 6, 9, 17, 40):
        px, py = rng.uniform(-300, 300, m), rng.uniform(-300, 300, m)
        o = bso.b_spline(px, py, 100000)
        assert o["status"] == po.OK, o["status"]
        assert o["x"][0] == px[0] and o["y"][0] == py[0] and o["x"][-1] == px[-1] and o["y"][-1] == py[-1]
        e = be.b_spline(px, py, 100000)
        assert e["x"][0] == px[0] and e["y"][0] == py[0] and e["x"][-1] == px[-1] and e["y"][-1] == py[-1]


def test_collinear_points_give_samples_on_the_line():
    for spacing in (3.0, 7.0, 12.0):
        s = spacing * np.arange(8)
        o = bso.b_spline(s, np.zeros(8), 1000)
        assert o["status"] == po.OK and np.all(o["y"] == 0.0) and np.all(np.diff(o["x"]) > 0)
        c, h = math.cos(0.7), math.sin(0.7)
        o = bso.b_spline(3.0 + c * s, -2.0 + h * s, 1000)
        assert np.max(np.abs(-(o["x"] - 3.0) * h + (o["y"] + 2.0) * c)) < 1e-12  # distance from the line


def test_degree_thresholds():
    # strict comparisons: an average of exactly 10 gives 4, exactly 5 gives 5
    for spacing, m, want in ((11, 4, 3), (10, 5, 4), (6, 6, 4), (5, 6, 5), (1, 8, 5)):
        x = float(spacing) * np.arange(m)
        assert bso.polygon_length(x, np.zeros(m)) / (m - 1) == spacing
        assert bso.b_spline(x, np.zeros(m), 1000)["degree"] == want, (spacing, m)
        assert be.b_spline(x, np.zeros(m), 1000)["degree"] == want, (spacing, m)
    # degree >= m: tinyspline refuses the spline
    assert bso.b_spline(3.0 * np.arange(4), np.zeros(4), 1000)["status"] == bso.BSPLINE_DEGREE
    assert be.b_spline(3.0 * np.arange(4), np.zeros(4), 1000)["status"] == bso.BSPLINE_DEGREE
    assert be.b_spline(np.arange(3.0), np.zeros(3), 1000)["status"] == bso.POINT_COUNT


def _reference_count(length, guard):
    """The reference's loop as written (x_list_.size() after bSpline()), in float64; None when it runs past `guard`."""
    with np.errstate(divide="ignore", invalid="ignore"):
        delta_t = np.float64(1.0) / np.float64(length)
    tmp_t, n = np.float64(0.0), 0
    while tmp_t < 1:
        n += 1
        if n > guard:
            return None
        tmp_t += delta_t
    return n + 1


def test_sample_count_matches_the_reference_loop():
    rng = np.random.default_rng(4)
    lengths = list(rng.uniform(1.0, 300.0, 300)) + [1.0, 1.5, 2.0, 3.0, 10.0, 49.0, 100.0, 0.1 + 0.2, 1 / 3 * 30]
    for length in lengths:
        want = _reference_count(length, 10 ** 6)
        t = bso.abscissae(length, 10 ** 6)
        assert len(t) == want, length
        assert all(t[j + 1] > t[j] for j in range(len(t) - 1))
    # over capacity: cap + 1, from both
    assert bso.abscissae(300.0, 50) is None and _reference_count(300.0, 50) is None
    x = np.array([0.0, 100.0, 200.0, 300.0])
    e = be.b_spline(x, np.zeros(4), 50)
    assert e["status"] == po.TOO_MANY_POINTS and e["r"] == 51
    # zero length, below 1 m, NaN: two samples (t = 0 and t = 1); infinite: over capacity, and nothing hangs
    for length, want in ((0.0, 2), (0.5, 2), (float("nan"), 2)):
        assert len(bso.abscissae(length, 1000)) == want == _reference_count(length, 1000)
    assert bso.abscissae(float("inf"), 1000) is None and _reference_count(float("inf"), 1000) is None
    pts = {"zero": (np.ones(8), np.ones(8)), "short": (np.linspace(0, 0.5, 8), np.zeros(8)),
           "nan": (np.array([0, 1, 2, np.nan, 4, 5, 6, 7.0]), np.zeros(8)),
           "inf": (np.array([0, 1, 2, 3, 4, 5, 6, 1e308]), np.array([0, 0, 0, 0, 0, 0, 0, -1e308]))}
    for name, (x, y) in pts.items():
        e, o = be.b_spline(x, y, 1000), bso.b_spline(x, y, 1000)
        assert (e["status"], e["r"], e["degree"]) == (o["status"], o["r"], o["degree"]), name
        assert e["r"] == (1001 if name == "inf" else 2), name


def test_kernel_source_matches_oracle_bitwise():
    rng = np.random.default_rng(5)
    seen = set()
    for case in range(300):
        m = int(rng.integers(0, 41)) if case % 3 else int(rng.integers(3, 7))  # 4 or 5 short points: degree >= m
        spacing = float(rng.uniform(0.05, 16.0))
        h = np.cumsum(rng.normal(0, 0.3, m))
        px = np.cumsum(spacing * np.cos(h)) + rng.normal(0, 1.0)
        py = np.cumsum(spacing * np.sin(h)) + rng.normal(0, 1.0)
        cap = int(rng.choice([64, 256, 2000]))
        e = be.b_spline(px, py, cap)
        o = bso.b_spline(px, py, cap) if m >= 4 else dict(status=bso.POINT_COUNT, r=0, degree=0, x=[], y=[])
        assert (e["status"], e["r"], e["degree"]) == (o["status"], o["r"], o["degree"]), case
        assert np.array_equal(e["x"], o["x"]) and np.array_equal(e["y"], o["y"]), case
        seen.add((e["status"], e["degree"]))
    assert {(po.OK, 3), (po.OK, 4), (po.OK, 5), (bso.BSPLINE_DEGREE, 5), (po.TOO_MANY_POINTS, 3)} <= seen, seen
    # a row longer than m is never read beyond m; m above the row stride is rejected
    x = 4.0 * np.arange(10)
    assert be.b_spline(x, np.zeros(10), 100, m_max=9)["status"] == bso.POINT_COUNT


def test_oracle_chain_from_points_straight_corridor():
    dist = np.full((400, 400), 20.0, dtype=np.float32)  # 80 m x 80 m, free
    xs = np.arange(-20.0, 20.5, 4.0)
    o = bso.plan(dist, 0.2, xs, np.zeros_like(xs), [-20.0, 0.0, 0.0, 0.0], [18.0, 0.0, 0.0], r_max=R_MAX,
                 params=abi.default_params(), p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX)
    assert o["status"] == po.OK and o["bspline"]["degree"] == 5
    assert o["l0"] == 0.0 and o["psi0"] == 0.0
    assert np.max(np.abs(o["path"][5])) < 1e-3


def test_make_plan_points_workload():
    ref_x, ref_y, start, target = sharedmap.make_plan_points(64)
    _, _, s0, t0 = sharedmap.make_plan_inputs(64)
    assert np.array_equal(start, s0) and np.array_equal(target, t0)
    degrees = {bso.b_spline(x, y, R_MAX)["degree"] for x, y in zip(ref_x, ref_y)}
    assert degrees == {3, 4, 5}, degrees


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "pqp_plan.h"
int main(void) {
    printf("size %zu\nbatch %zu\nm_max %zu\nref_x %zu\nref_y %zu\nm %zu\nstart %zu\ntarget %zu\n",
           sizeof(pqp_plan_points_in), offsetof(pqp_plan_points_in, batch), offsetof(pqp_plan_points_in, m_max),
           offsetof(pqp_plan_points_in, ref_x), offsetof(pqp_plan_points_in, ref_y), offsetof(pqp_plan_points_in, m),
           offsetof(pqp_plan_points_in, start), offsetof(pqp_plan_points_in, target));
    printf("trace_size %zu\nraw_r %zu\nbspline_degree %zu\n", sizeof(pqp_plan_trace), offsetof(pqp_plan_trace, raw_r),
           offsetof(pqp_plan_trace, bspline_degree));
    printf("point_count %d\nbspline_degree_code %d\ntoo_many_points %d\n", PQP_PLAN_POINT_COUNT,
           PQP_PLAN_BSPLINE_DEGREE, PQP_PLAN_TOO_MANY_POINTS);
    return 0;
}
"""


def test_points_layout_matches_ctypes():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(src, "w") as f:
            f.write(_LAYOUT_C)
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = {k: int(v) for k, v in (line.split() for line in subprocess.check_output([exe], text=True).splitlines())}
    S, T = plan.PlanPointsIn, plan.PlanTrace
    want = {"size": ctypes.sizeof(S), **{n: getattr(S, n).offset for n, _ in S._fields_},
            "trace_size": ctypes.sizeof(T), "raw_r": T.raw_r.offset, "bspline_degree": T.bspline_degree.offset,
            "point_count": plan.POINT_COUNT, "bspline_degree_code": plan.BSPLINE_DEGREE,
            "too_many_points": plan.TOO_MANY_POINTS}
    assert got == want
    assert plan.STATUS_NAMES[plan.POINT_COUNT] == "POINT_COUNT" and plan.STATUS_NAMES[plan.BSPLINE_DEGREE] == "BSPLINE_DEGREE"
    assert (bso.POINT_COUNT, bso.BSPLINE_DEGREE) == (plan.POINT_COUNT, plan.BSPLINE_DEGREE)


# ------------------------------------------------------------------------------------------------- GPU
METHODS = ("TENSION2", "TENSION")
SHARED = [n for n, _, _ in plan._TRACE if n not in ("raw_r", "bspline_degree")]


@pytest.fixture(scope="module")
def world():
    dmap = sharedmap.DistanceMap()
    return (dmap,) + sharedmap.make_plan_points(64, dmap=dmap)


@pytest.fixture(scope="module", params=METHODS)
def setup(request, world):
    dmap, ref_x, ref_y, start, target = world
    pl = plan.Planner(dmap.dist, dmap.res, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=64,
                      params=plan.default_params(request.param))
    run = pl.plan_points(ref_x, ref_y, start, target, trace=True)
    yield request.param, pl, run
    pl.close()


def _same_row(a, b, i, j):
    return (a.status[i] == b.status[j] and a.n[i] == b.n[j] and np.array_equal(a.path[i], b.path[j])
            and np.array_equal(a.cost[i], b.cost[j]) and np.array_equal(a.iters[i], b.iters[j]))


@pytest.mark.gpu
def test_samples_match_oracle_bitwise(world, setup):
    _, ref_x, ref_y, _, _ = world
    _, _, run = setup
    T = run.trace
    assert np.mean(run.status == plan.OK) > 0.8, run.status_names()
    for b in range(64):
        o = bso.b_spline(ref_x[b], ref_y[b], R_MAX)
        r = o["r"]
        assert (T["raw_r"][b], T["bspline_degree"][b]) == (r, o["degree"]) and o["status"] == po.OK, b
        assert np.array_equal(T["raw_spline"][b, 4, :r], o["x"]) and np.array_equal(T["raw_spline"][b, 8, :r], o["y"]), b


@pytest.mark.gpu
def test_composition_equals_plan_on_the_samples(world, setup):
    _, _, _, start, target = world
    _, pl, run = setup
    T = run.trace
    xs = [T["raw_spline"][b, 4, :T["raw_r"][b]].copy() for b in range(64)]
    ys = [T["raw_spline"][b, 8, :T["raw_r"][b]].copy() for b in range(64)]
    res = pl.plan(xs, ys, start, target, trace=True)
    for k in ("status", "n", "path", "cost", "iters"):
        assert np.array_equal(getattr(res, k), getattr(run, k)), k
    for k in SHARED:
        assert np.array_equal(res.trace[k], T[k], equal_nan=True), k
    assert not res.trace["raw_r"].any() and not res.trace["bspline_degree"].any()  # pqp_plan leaves them untouched


@pytest.mark.gpu
def test_independent_oracle_chain(world, setup):
    dmap, ref_x, ref_y, start, target = world
    method, pl, run = setup
    for b in range(64):
        o = bso.plan(dmap.dist, dmap.res, ref_x[b], ref_y[b], start[b], target[b], r_max=R_MAX, smoothing_method=method,
                     params=pl.params.solver, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX)
        assert o["status"] == run.status[b], (b, o["status"], run.status_names()[b])


@pytest.mark.gpu
def test_every_new_failure_is_reached(world, setup):
    _, ref_x, ref_y, start, target = world
    _, pl, run = setup
    idx = list(range(8))
    xs, ys = [ref_x[i].copy() for i in idx], [ref_y[i].copy() for i in idx]
    m_max = 16
    assert max(len(v) for v in ref_x[:8]) <= m_max
    xs[0], ys[0] = xs[0][:0], ys[0][:0]                            # no points
    xs[1], ys[1] = xs[1][:3], ys[1][:3]                            # 3 points
    xs[2], ys[2] = np.linspace(0, 60, m_max + 4), np.zeros(m_max + 4)  # more points than the row holds
    xs[3], ys[3] = 3.0 * np.arange(4), np.zeros(4)                 # 4 points 3 m apart: degree 5 >= 4
    xs[4], ys[4] = np.array([0.0, 33.0, 66.0, 100.0]), np.zeros(4)  # 100 m of polygon: over r_max samples
    xs[5], ys[5] = np.full(8, 5.0), np.full(8, -3.0)               # all points equal: two equal samples
    res = pl.plan_points(xs, ys, start[idx], target[idx], trace=True, m_max=m_max)
    T = res.trace
    want = [plan.POINT_COUNT, plan.POINT_COUNT, plan.POINT_COUNT, plan.BSPLINE_DEGREE, plan.TOO_MANY_POINTS,
            plan.SPLINE_DEGENERATE]
    assert list(res.status[:6]) == want, res.status_names()
    assert list(T["raw_r"][:6]) == [0, 0, 0, 0, R_MAX + 1, 2] and list(T["bspline_degree"][:6]) == [0, 0, 0, 5, 3, 5]
    for b in (6, 7):
        assert _same_row(res, run, b, b), b
        assert np.array_equal(T["raw_spline"][b], run.trace["raw_spline"][b])
    for b in range(6):
        assert res.n[b] == 0 and not res.path[b].any()


@pytest.mark.gpu
def test_device_call_and_batch_invariance(world, setup):
    import torch
    _, ref_x, ref_y, start, target = world
    _, pl, run = setup
    dev = torch.device("cuda:0")
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    M = int(m.max())
    px, py = np.zeros((64, M)), np.zeros((64, M))
    for b in range(64):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    out = pl.plan_points_device(t(px), t(py), t(m), t(start), t(target), trace=True)
    torch.cuda.synchronize()
    for k in ("status", "n", "path", "cost", "iters"):
        assert np.array_equal(out[k].cpu().numpy(), getattr(run, k)), k
    for k in ("raw_r", "bspline_degree", "raw_spline", "seg_x", "knots", "sol1", "states", "ref_spline"):
        assert np.array_equal(out["trace"][k].cpu().numpy(), run.trace[k]), k
    for b in (0, 17, 63):  # B = 1 equals its row of the batch, bitwise
        one = pl.plan_points([ref_x[b]], [ref_y[b]], start[b:b + 1], target[b:b + 1], trace=True)
        assert _same_row(one, run, 0, b), b
        r = int(run.trace["raw_r"][b])
        assert np.array_equal(one.trace["raw_spline"][0, :, :r], run.trace["raw_spline"][b, :, :r])


@pytest.mark.gpu
def test_launch_count_and_stage_times(world, setup):
    _, ref_x, ref_y, start, target = world
    method, pl, _ = setup
    base = 24 if method == "TENSION" else 23
    raw = sharedmap.make_plan_inputs(8)
    c0 = pl.launch_count
    pl.plan(*raw)
    c1 = pl.launch_count
    pl.plan_points(ref_x[:8], ref_y[:8], start[:8], target[:8])
    c2 = pl.launch_count
    assert c1 - c0 == base and c2 - c1 == base + 2  # bspline_prep_kernel, bspline_eval_kernel
    ms = pl.last_stage_ms
    assert 0 < ms["smoothing"] <= ms["total"]
