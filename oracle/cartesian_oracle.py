"""cartesian_oracle.py — CPU restatement of TensionSmoother::osqpSmooth, the smoother of --smoothing_method=TENSION
(src/reference_path_smoother/tension_smoother.cpp:49-177), and of PathOptimizer::solve with that smoother. TEST
INFRASTRUCTURE: imported only by tests/ and bench_plan.py's comparison leg; the product path is
path_optimizer_2_b200/csrc/pqp_smoother*.cu* and pqp_plan.cu and never calls this. PARITY UNPINNED like
smoother_oracle.py (no reference-produced vectors; pinned by closed forms in tests/test_cartesian_tension.py).

Variables (3p): x_0..x_{p-1}, y_0.., d_0.. (lateral shift of each point); constraints (3p):
  x_i - cos(theta_i) d_i = x_list_i,  y_i - sin(theta_i) d_i = y_list_i,  theta_i = angle_i + pi/2     (:143-156)
  d_0 = 0, d_{p-1} in [-0.5, 0.5], interior d_i in +-min(clearance_i, 2)                                  (:158-176)
Cost: 1/2 z' P z, q = 0, P from dense blocks (:102-126): w_k [1 -2 1]'[1 -2 1] on x_i..x_{i+2} and on y, i = 0..p-3;
w_dk [-1 3 -3 1]'[-1 3 -3 1] on x_i..x_{i+3} and on y, i = 0..p-4 (the `i != size - 3` rule); P(d_i, d_i) = w_d (no
factor 2). Solved with the generic OSQP restatement (OSQP defaults, eps 1e-3: the reference sets only verbosity and
warm start, :62-63). clearance_i is Map::getObstacleDistance (src/tools/Map.cpp:16-22, bounds_oracle.map_distance).
"""
import numpy as np
import scipy.sparse as sp

from . import bounds_oracle as bo
from . import dp_oracle, osqp_generic, smoother_oracle
from . import plan_oracle as po

W_CURVATURE, W_CURVATURE_RATE, W_DEVIATION = 1.0, 50.0, 0.0  # planning_flags.cpp:51-55
DEFAULT_CLEARANCE = 2.0                                        # tension_smoother.cpp:163


def assemble(x_list, y_list, angle_list, clearance, w_k=W_CURVATURE, w_dk=W_CURVATURE_RATE, w_d=W_DEVIATION):
    """`clearance[i]`: the map's obstacle distance at (x_list[i], y_list[i]) (0 off the map); read for interior points."""
    x_list, y_list, angle_list, clearance = (np.asarray(v, dtype=np.float64) for v in (x_list, y_list, angle_list, clearance))
    p = len(x_list)
    xs, ys, ds = 0, p, 2 * p
    H = np.zeros((3 * p, 3 * p))
    dds = np.outer([1.0, -2.0, 1.0], [1.0, -2.0, 1.0]) * w_k
    ddds = np.outer([-1.0, 3.0, -3.0, 1.0], [-1.0, 3.0, -3.0, 1.0]) * w_dk
    for i in range(p - 2):
        H[xs + i:xs + i + 3, xs + i:xs + i + 3] += dds
        H[ys + i:ys + i + 3, ys + i:ys + i + 3] += dds
        if i != p - 3:
            H[xs + i:xs + i + 4, xs + i:xs + i + 4] += ddds
            H[ys + i:ys + i + 4, ys + i:ys + i + 4] += ddds
    for i in range(p):
        H[ds + i, ds + i] = w_d
    A = np.zeros((3 * p, 3 * p))
    lo, up = np.zeros(3 * p), np.zeros(3 * p)
    for i in range(p):
        theta = angle_list[i] + np.pi / 2
        A[xs + i, xs + i] = A[ys + i, ys + i] = 1.0
        A[xs + i, ds + i] = -np.cos(theta)
        A[ys + i, ds + i] = -np.sin(theta)
        A[ds + i, ds + i] = 1.0
        lo[xs + i] = up[xs + i] = x_list[i]
        lo[ys + i] = up[ys + i] = y_list[i]
    lo[ds], up[ds] = 0.0, 0.0
    lo[ds + p - 1], up[ds + p - 1] = -0.5, 0.5
    for i in range(1, p - 1):
        c = DEFAULT_CLEARANCE if DEFAULT_CLEARANCE < clearance[i] else clearance[i]  # std::min(clearance, 2)
        lo[ds + i], up[ds + i] = -c, c
    return sp.csc_matrix(H), np.zeros(3 * p), sp.csc_matrix(A), lo, up


def osqp_smooth(x_list, y_list, angle_list, clearance, **weights):
    """-> (ok, result_x, result_y, result_s, solver): OSQP defaults, result_s re-accumulated from the smoothed points
    (:85-98)."""
    H, q, A, lo, up = assemble(x_list, y_list, angle_list, clearance, **weights)
    g = osqp_generic.GenericOsqp(H, q, A, lo, up)
    ok = g.solve() == osqp_generic.SOLVED
    x, _, _ = g.solution()
    p = len(x_list)
    rx, ry = x[:p], x[p:2 * p]
    rs = np.concatenate(([0.0], np.cumsum(np.hypot(np.diff(rx), np.diff(ry)))))
    return ok, rx, ry, rs, g


def plan(dist, res, raw_x, raw_y, start, target, *, params, p_max, layers_max, n_max, rough=False,
         precise_length=30.0, constrain_end_heading=True, output_spacing=0.3, dynamic=True):
    """plan_oracle.plan with TensionSmoother in place of TensionSmoother2: the clearance of each segmented point is
    the map's obstacle distance there (tension_smoother.cpp:165-170). Same stage functions and status codes; the
    result dict also carries `tension_clearance`."""
    from . import oracle as solver_oracle
    out = dict(status=po.OK)

    def fail(code):
        out["status"] = code
        return out

    raw_x, raw_y = np.asarray(raw_x, dtype=np.float64), np.asarray(raw_y, dtype=np.float64)
    if len(raw_x) < 3:
        return fail(po.SPLINE_DEGENERATE)
    s_raw = po.chord_length(raw_x, raw_y)
    if not po._increasing(s_raw):
        return fail(po.SPLINE_DEGENERATE)
    p = po.segment_count(s_raw[-1])
    out["seg_p"] = p
    if p > p_max:
        return fail(po.TOO_MANY_POINTS)
    out["raw_spline"] = raw = po.spline_rows(s_raw, raw_x, raw_y)
    out["seg"] = seg = po.segment(raw, p)
    out["tension_clearance"] = clearance = bo.map_distance(dist, res, seg[0], seg[1])
    ok, tx, ty, _, g = osqp_smooth(seg[0], seg[1], seg[2], clearance)
    ts = po.chord_length(tx, ty)
    out.update(tension_x=tx, tension_y=ty, tension_s=ts, tension_status=g.status, tension_iters=g.iters)
    if not ok:
        return fail(po.TENSION_FAILED)
    if not po._increasing(ts):
        return fail(po.SPLINE_DEGENERATE)
    t_rows, t_len = po.tension_epilogue(tx, ty, ts)
    out.update(tension_spline=t_rows, tension_length=t_len)
    d = dp_oracle.graph_search_dp(dist, res, t_rows, t_len, np.asarray(start[:3], dtype=np.float64))
    out["dp"] = d
    if d["n_layers"] > layers_max:
        return fail(po.TOO_MANY_POINTS)
    if not d["ok"]:
        return fail(po.DP_VEHICLE_FAR)
    if d["n_out"] < 4:
        return fail(po.POST_TOO_SHORT)
    okp, off, gp = smoother_oracle.post_smooth(d["layer_s"], d["lower"], d["upper"], d["vehicle_l"])
    out.update(post_offsets=off, post_status=gp.status, post_iters=gp.iters)
    if not okp:
        return fail(po.POST_FAILED)
    rs, rx, ry = po.post_epilogue(t_rows, d["layer_s"], off)
    if not po._increasing(rs):
        return fail(po.SPLINE_DEGENERATE)
    out["ref_spline"] = r_rows = po.spline_rows(rs, rx, ry)
    st, l0, psi0, max_s = po.process_reference(r_rows, float(rs[-1]), start, target)
    out.update(l0=l0, psi0=psi0, max_s=max_s)
    if st != po.OK:
        return fail(st)
    s, x, y, h, k = bo.build_states(r_rows, max_s, output_spacing / 2.0, output_spacing, dynamic)
    out.update(states=np.stack([s, x, y, h]), curvature=k, total=len(s))
    if len(s) > n_max:
        return fail(po.TOO_MANY_KNOTS)
    bnd, n_valid = bo.update_bounds(dist, res, r_rows, s, x, y, h)
    out.update(bounds=bnd, n_valid=n_valid)
    if n_valid < 2:
        return fail(po.BLOCKED_AT_START)
    knots, inst, pp = po.instance_block(out["states"], k, bnd, n_valid, start, target, l0, psi0, rough=rough,
                                        precise_length=precise_length, constrain_end_heading=constrain_end_heading)
    out.update(knots=knots, inst=inst, p=pp)
    sv = solver_oracle.OracleSolver(params, knots, inst, n_valid, pp)
    sv.solve()
    out.update(status1=sv.status, iters1=sv.iters)
    if sv.status != 0:
        return fail(po.PRE_SOLVE_FAILED)
    sol1 = sv.sol()
    out["sol1"] = sol1
    sv.update(sol1[0], sol1[1], sol1[2])
    sv.solve()
    out.update(status2=sv.status, iters2=sv.iters)
    if sv.status != 0:
        return fail(po.SOLVE_FAILED)
    sol2 = sv.sol()
    xyh = solver_oracle.frenet_to_cartesian(out["states"][1:4, :n_valid], sol2[0], sol2[1])
    d_k = np.concatenate((sol2[3, :n_valid - 1], [0.0]))
    out["path"] = np.stack([xyh[0], xyh[1], xyh[2], sol2[2], d_k, sol2[0], sol2[1]])
    out["n"] = n_valid
    out["cost"] = sv.cost
    return out
