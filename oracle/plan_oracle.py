"""plan_oracle.py — CPU restatement of PathOptimizer::solve (path_optimizer.cpp:34-71) for one path, composed from the
stage restatements (bounds_oracle, smoother_oracle, dp_oracle, the C solver oracle). TEST INFRASTRUCTURE: imported
only by tests/, __graft_entry__.smoke() and bench_plan.py's comparison leg; the product path is
path_optimizer_2_b200/csrc/pqp_plan.cu and never calls this.

Restated here (the rest is the stage oracles), relative to /root/reference/:
  chord_length         src/reference_path_smoother/reference_path_smoother.cpp:519-523 (s_list_ of bSpline())
  segment              :47-85 (segmentRawReference)
  tension_epilogue     tension_smoother.cpp:36-41, tension_smoother_2.cpp:57-70
  post_epilogue        reference_path_smoother.cpp:560-577
  process_reference    src/path_optimizer.cpp:73-117, src/tools/tools.cpp:57-126
  instance_block       src/solver/base_solver.cpp:24-34, 216-259; the knot block of include/pqp_base_solver.hpp
Squares are written d * d (correctly rounded; glibc's pow(d, 2) is within an ulp of it). Every stage function takes its
upstream stage's result as arguments, so it can equally be fed the GPU's upstream output (conditional stage parity).
"""
import math

import numpy as np

from . import bounds_oracle as bo
from . import dp_oracle, smoother_oracle

(OK, SPLINE_DEGENERATE, TOO_MANY_POINTS, TENSION_FAILED, DP_VEHICLE_FAR, POST_TOO_SHORT, POST_FAILED, EMPTY_REFERENCE,
 INIT_HEADING, TOO_MANY_KNOTS, BLOCKED_AT_START, PRE_SOLVE_FAILED, SOLVE_FAILED) = range(13)
NFIELDS, NINST = 9, 5
F_S, F_KREF, F_L, F_PSI, F_K, F_B0_LB, F_B0_UB, F_B1_LB, F_B1_UB = range(9)
INFTY = 1e30


def spline_rows(s, x, y):
    """[9][k] rows (abscissa; a, b, c, y of x(s); a, b, c, y of y(s)) of tk::spline::set_points."""
    rows = [np.asarray(s, dtype=np.float64)]
    for v in (x, y):
        a, b, c = bo.natural_spline(s, v)
        rows += [a, b, c, np.asarray(v, dtype=np.float64)]
    return np.stack(rows)


def chord_length(x, y):
    s = [0.0]
    for i in range(1, len(x)):
        dx, dy = float(x[i]) - float(x[i - 1]), float(y[i]) - float(y[i - 1])
        s.append(s[-1] + math.sqrt(dx * dx + dy * dy))
    return np.array(s)


def _increasing(s):
    return bool(np.all(np.diff(s) > 0))


def segment_count(max_s):
    """segmentRawReference's loop (:61-68): the last sample overshoots max_s by up to 1 m; the `> 1` branch after it
    cannot fire."""
    s = [0.0]
    while s[-1] < max_s:
        s.append(s[-1] + 1.0)
    if max_s - s[-1] > 1:  # never true after the loop above; kept literal
        s.append(max_s)
    return len(s)


def _eval(sp, s):
    x, dx, ddx = (float(v) for v in sp.x(s))
    y, dy, ddy = (float(v) for v in sp.y(s))
    return x, dx, ddx, y, dy, ddy


def segment(raw_rows, p):
    """Samples s = 0, 1, ..., p-1 of the raw spline: (x, y, angle, k, s)."""
    sp = bo.Spline2(raw_rows)
    out = np.zeros((5, p))
    for j in range(p):
        s = float(j)
        x, dx, ddx, y, dy, ddy = _eval(sp, s)
        out[:, j] = x, y, math.atan2(dy, dx), (dx * ddy - dy * ddx) / math.pow(dx * dx + dy * dy, 1.5), s
    return tuple(out)


def tension_epilogue(tx, ty, ts):
    """-> (rows, length = result_s.back() + 3)."""
    return spline_rows(ts, tx, ty), float(ts[-1]) + 3.0


def post_epilogue(tension_rows, layer_s, offsets):
    """-> (s, x, y) of the post-smoothed points."""
    sp = bo.Spline2(tension_rows)
    xs, ys, ss = [], [], []
    acc = 0.0
    for i, rs in enumerate(layer_s):
        rx, dx, _, ry, dy, _ = _eval(sp, float(rs))
        d = math.atan2(dy, dx) + math.pi / 2
        xs.append(rx + float(offsets[i]) * math.cos(d))
        ys.append(ry + float(offsets[i]) * math.sin(d))
        if i > 0:
            ex, ey = xs[i] - xs[i - 1], ys[i] - ys[i - 1]
            acc += math.sqrt(ex * ex + ey * ey)
        ss.append(acc)
    return np.array(ss), np.array(xs), np.array(ys)


def process_reference(rows, length, start, target, epsilon=1e-6):
    """processInitState, the 75 degree gate and setReferencePathLength -> (status, l0, psi0, max_s)."""
    if abs(length - 0.0) < epsilon:
        return EMPTY_REFERENCE, 0.0, 0.0, length
    sp = bo.Spline2(rows)
    ix, dx, _, iy, dy, _ = _eval(sp, 0.0)
    ih = math.atan2(dy, dx)
    gx, gy = ix - float(start[0]), iy - float(start[1])
    local_y = -gx * math.sin(start[2]) + gy * math.cos(start[2])
    dist = math.sqrt(gx * gx + gy * gy)
    l0 = dist if local_y < 0.0 else -dist
    psi0 = dp_oracle.constrain_angle(float(start[2]) - ih)
    if abs(psi0) > 75 * math.pi / 180:
        return INIT_HEADING, l0, psi0, length
    ex, dx, _, ey, dy, _ = _eval(sp, length)
    eh = math.atan2(dy, dx)
    tx, ty = float(target[0]) - ex, float(target[1]) - ey
    if tx * math.cos(eh) + ty * math.sin(eh) > 0.0:
        return OK, l0, psi0, length
    return OK, l0, psi0, dp_oracle.get_projection_s(sp, float(target[0]), float(target[1]), length)


def precise_size(s, n, rough, precise_length=30.0):
    if not rough:
        return n
    return int(np.searchsorted(np.asarray(s[:n]), precise_length, side="left"))


def end_heading_rows(constrain, blocked, target_heading, last_heading):
    if constrain and not blocked:
        e = dp_oracle.constrain_angle(target_heading - last_heading)
        if e < 70 * math.pi / 180:  # signed, as base_solver.cpp:256
            return e - 0.087, e + 0.087
    return -INFTY, INFTY


def instance_block(states, curvature, bounds, n_valid, start, target, l0, psi0, *, rough=False, precise_length=30.0,
                   constrain_end_heading=True):
    """Solver input of BaseSolver on the states cut at n_valid: (knots[9][n_valid], inst[5], p)."""
    s, _, _, h = states
    n, total = int(n_valid), len(s)
    p = precise_size(s, n, rough, precise_length)
    knots = np.zeros((NFIELDS, n))
    knots[F_S], knots[F_KREF], knots[F_K] = s[:n], curvature[:n], curvature[:n]
    knots[F_B0_LB], knots[F_B0_UB] = bounds[0, :n], bounds[1, :n]
    knots[F_B1_LB], knots[F_B1_UB] = bounds[2, :n], bounds[3, :n]
    knots[F_B0_LB, p:], knots[F_B0_UB, p:] = bounds[4, p:n], bounds[5, p:n]
    knots[F_B1_LB, p:] = knots[F_B1_UB, p:] = 0.0
    lo, hi = end_heading_rows(constrain_end_heading, n < total, float(target[2]), float(h[n - 1]))
    inst = np.array([l0, psi0, float(start[3]), lo, hi])
    return knots, inst, p


def plan(dist, res, raw_x, raw_y, start, target, *, params, p_max, layers_max, n_max, rough=False,
         precise_length=30.0, constrain_end_heading=True, output_spacing=0.3, dynamic=True):
    """The whole chain for one path -> dict(status, and every stage's result up to the failing one)."""
    from . import oracle as solver_oracle
    out = dict(status=OK)

    def fail(code):
        out["status"] = code
        return out

    raw_x, raw_y = np.asarray(raw_x, dtype=np.float64), np.asarray(raw_y, dtype=np.float64)
    if len(raw_x) < 3:
        return fail(SPLINE_DEGENERATE)
    s_raw = chord_length(raw_x, raw_y)
    if not _increasing(s_raw):
        return fail(SPLINE_DEGENERATE)
    p = segment_count(s_raw[-1])
    out["seg_p"] = p
    if p > p_max:
        return fail(TOO_MANY_POINTS)
    out["raw_spline"] = raw = spline_rows(s_raw, raw_x, raw_y)
    out["seg"] = seg = segment(raw, p)
    ok, tx, ty, _, g = smoother_oracle.osqp_smooth(seg[0], seg[1], seg[2], seg[3], seg[4])
    ts = chord_length(tx, ty)
    out.update(tension_x=tx, tension_y=ty, tension_s=ts, tension_status=g.status, tension_iters=g.iters)
    if not ok:
        return fail(TENSION_FAILED)
    if not _increasing(ts):
        return fail(SPLINE_DEGENERATE)
    t_rows, t_len = tension_epilogue(tx, ty, ts)
    out.update(tension_spline=t_rows, tension_length=t_len)
    d = dp_oracle.graph_search_dp(dist, res, t_rows, t_len, np.asarray(start[:3], dtype=np.float64))
    out["dp"] = d
    if d["n_layers"] > layers_max:
        return fail(TOO_MANY_POINTS)
    if not d["ok"]:
        return fail(DP_VEHICLE_FAR)
    if d["n_out"] < 4:
        return fail(POST_TOO_SHORT)
    okp, off, gp = smoother_oracle.post_smooth(d["layer_s"], d["lower"], d["upper"], d["vehicle_l"])
    out.update(post_offsets=off, post_status=gp.status, post_iters=gp.iters)
    if not okp:
        return fail(POST_FAILED)
    rs, rx, ry = post_epilogue(t_rows, d["layer_s"], off)
    if not _increasing(rs):
        return fail(SPLINE_DEGENERATE)
    out["ref_spline"] = r_rows = spline_rows(rs, rx, ry)
    st, l0, psi0, max_s = process_reference(r_rows, float(rs[-1]), start, target)
    out.update(l0=l0, psi0=psi0, max_s=max_s)
    if st != OK:
        return fail(st)
    s, x, y, h, k = bo.build_states(r_rows, max_s, output_spacing / 2.0, output_spacing, dynamic)
    out.update(states=np.stack([s, x, y, h]), curvature=k, total=len(s))
    if len(s) > n_max:
        return fail(TOO_MANY_KNOTS)
    bnd, n_valid = bo.update_bounds(dist, res, r_rows, s, x, y, h)
    out.update(bounds=bnd, n_valid=n_valid)
    if n_valid < 2:
        return fail(BLOCKED_AT_START)
    knots, inst, pp = instance_block(out["states"], k, bnd, n_valid, start, target, l0, psi0, rough=rough,
                                     precise_length=precise_length, constrain_end_heading=constrain_end_heading)
    out.update(knots=knots, inst=inst, p=pp)
    sv = solver_oracle.OracleSolver(params, knots, inst, n_valid, pp)
    sv.solve()
    out.update(status1=sv.status, iters1=sv.iters)
    if sv.status != 0:
        return fail(PRE_SOLVE_FAILED)
    sol1 = sv.sol()
    out["sol1"] = sol1
    sv.update(sol1[0], sol1[1], sol1[2])
    sv.solve()
    out.update(status2=sv.status, iters2=sv.iters)
    if sv.status != 0:
        return fail(SOLVE_FAILED)
    sol2 = sv.sol()
    xyh = solver_oracle.frenet_to_cartesian(out["states"][1:4, :n_valid], sol2[0], sol2[1])
    d_k = np.concatenate((sol2[3, :n_valid - 1], [0.0]))
    out["path"] = np.stack([xyh[0], xyh[1], xyh[2], sol2[2], d_k, sol2[0], sol2[1]])
    out["n"] = n_valid
    out["cost"] = sv.cost
    return out
