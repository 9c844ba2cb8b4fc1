"""bspline_oracle.py — CPU restatement of ReferencePathSmoother::bSpline() (src/reference_path_smoother/
reference_path_smoother.cpp:490-524, distance() of src/tools/tools.cpp:46-48) and of PathOptimizer::solve from the
reference points (path_optimizer.cpp:34-71, reference_path_smoother.cpp:31-45). TEST INFRASTRUCTURE: imported only by
tests/, __graft_entry__.smoke() and bench_plan.py's comparison leg; the product path is
path_optimizer_2_b200/csrc/pqp_plan.cu and never calls this.

The curve is tinyspline's BSpline(m, 2, degree) with its default clamped knots and the reference points as control
points: degree + 1 zeros, interior knots (i - degree) / (m - degree), degree + 1 ones, evaluated with de Boor's
algorithm. Same operations in the same order as pqp_plan_core.cuh, so samples, counts and degrees agree bit for bit;
the span is found here by a linear scan over the same computed knots (the kernel bisects). tinyspline's snapping of a
parameter to a nearby knot is not restated.
"""
import math

import numpy as np

from . import plan_oracle as po

POINT_COUNT, BSPLINE_DEGREE = 13, 14


def polygon_length(x, y):
    """Sequential sum of the point distances, squares written d * d."""
    length = 0.0
    for i in range(len(x) - 1):
        dx, dy = float(x[i]) - float(x[i + 1]), float(y[i]) - float(y[i + 1])
        length += math.sqrt(dx * dx + dy * dy)
    return length


def degree_for(length, m):
    average = length / float(m - 1)
    if average > 10:
        return 3
    if average > 5:
        return 4
    return 5


def abscissae(length, cap):
    """The reference's `while (tmp_t < 1)` loop and its final t = 1; None when there are more than `cap` samples."""
    delta_t = 1.0 / length if length != 0.0 else math.inf  # C: 1.0 / 0.0 = inf
    t, tmp_t = [], 0.0
    while tmp_t < 1:
        if len(t) == cap:
            return None
        t.append(tmp_t)
        tmp_t += delta_t
    if len(t) == cap:
        return None
    t.append(1.0)
    return t


def knot(i, degree, m):
    if i <= degree:
        return 0.0
    if i >= m:
        return 1.0
    return float(i - degree) / float(m - degree)


def span(t, degree, m):
    k = degree
    while k < m - 1 and knot(k + 1, degree, m) <= t:
        k += 1
    return k


def de_boor(px, py, degree, t):
    m = len(px)
    k = span(t, degree, m)
    dx = [float(px[j + k - degree]) for j in range(degree + 1)]
    dy = [float(py[j + k - degree]) for j in range(degree + 1)]
    for r in range(1, degree + 1):
        for j in range(degree, r - 1, -1):
            ua, ub = knot(j + k - degree, degree, m), knot(j + 1 + k - r, degree, m)
            alpha = (t - ua) / (ub - ua)
            dx[j] = (1.0 - alpha) * dx[j - 1] + alpha * dx[j]
            dy[j] = (1.0 - alpha) * dy[j - 1] + alpha * dy[j]
    return dx[degree], dy[degree]


def b_spline(ref_x, ref_y, r_max):
    """bSpline() for one path -> dict(status, degree, r, x, y): status OK, POINT_COUNT (fewer than 4 points),
    BSPLINE_DEGREE (degree >= m) or TOO_MANY_POINTS (more than r_max samples, r = r_max + 1)."""
    m = len(ref_x)
    if m < 4:
        return dict(status=POINT_COUNT, degree=0, r=0, x=np.zeros(0), y=np.zeros(0))
    length = polygon_length(ref_x, ref_y)
    deg = degree_for(length, m)
    if deg >= m:
        return dict(status=BSPLINE_DEGREE, degree=deg, r=0, x=np.zeros(0), y=np.zeros(0))
    t = abscissae(length, r_max)
    if t is None:
        return dict(status=po.TOO_MANY_POINTS, degree=deg, r=r_max + 1, x=np.zeros(0), y=np.zeros(0))
    xy = np.array([de_boor(ref_x, ref_y, deg, tt) for tt in t])
    return dict(status=po.OK, degree=deg, r=len(t), x=xy[:, 0].copy(), y=xy[:, 1].copy(), t=np.array(t))


def plan(dist, res, ref_x, ref_y, start, target, *, r_max, smoothing_method="TENSION2", **kw):
    """PathOptimizer::solve from the reference points: bSpline(), then plan_oracle.plan (cartesian_oracle.plan under
    TENSION) on its samples. The result dict also carries `bspline` (b_spline's dict)."""
    bs = b_spline(ref_x, ref_y, r_max)
    if bs["status"] != po.OK:
        return dict(status=bs["status"], bspline=bs)
    if smoothing_method == "TENSION":
        from . import cartesian_oracle
        out = cartesian_oracle.plan(dist, res, bs["x"], bs["y"], start, target, **kw)
    else:
        out = po.plan(dist, res, bs["x"], bs["y"], start, target, **kw)
    out["bspline"] = bs
    return out
