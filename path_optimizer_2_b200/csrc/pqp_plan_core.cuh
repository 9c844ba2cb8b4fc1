// pqp_plan_core.cuh — the per-path steps that connect the stages of PathOptimizer::solve (include/pqp_plan.h):
// natural spline fits, the 1 m resampling of the raw reference, the two smoother epilogues, processReferencePath's
// start / target decisions and the solver's per-instance block. Plain FP64 scalar code with no CUDA intrinsics, so
// the same source is compiled by nvcc for the kernels (pqp_plan.cu, --fmad=false) and by g++ (-ffp-contract=off) for
// the CPU test driver (tests/emu/plan_driver.cpp). Splines are evaluated with pqp_bounds_core.cuh, as every other
// stage evaluates them. Citations are relative to /root/reference/.
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "pqp_bounds_core.cuh"
#include "pqp_dp_core.cuh"

namespace pqpl {

// status codes (include/pqp_plan.h)
enum {
    kOk = 0, kSplineDegenerate = 1, kTooManyPoints = 2, kTensionFailed = 3, kDpVehicleFar = 4, kPostTooShort = 5,
    kPostFailed = 6, kEmptyReference = 7, kInitHeading = 8, kTooManyKnots = 9, kBlockedAtStart = 10,
    kPreSolveFailed = 11, kSolveFailed = 12, kPointCount = 13, kBsplineDegree = 14,
    kMapIndex = 15
};

constexpr int kSplineRows = 9;  // PQP_SPLINE_ROWS

// Spline rows of one path: [kSplineRows][stride] = abscissa; a, b, c, y of x(s); a, b, c, y of y(s).
PQB_HD pqb::SplineView view(const double *rows, int stride, int k) {
    pqb::SplineView sp;
    sp.sx = rows;
    sp.xa = rows + stride;
    sp.xb = rows + 2 * (size_t)stride;
    sp.xc = rows + 3 * (size_t)stride;
    sp.xy = rows + 4 * (size_t)stride;
    sp.ya = rows + 5 * (size_t)stride;
    sp.yb = rows + 6 * (size_t)stride;
    sp.yc = rows + 7 * (size_t)stride;
    sp.yy = rows + 8 * (size_t)stride;
    sp.k = k;
    return sp;
}

// tk::spline::set_points with the default (natural) boundary (src/tools/spline.cpp:161-249) for one coordinate:
// the band system solved by the Thomas recurrence, then a, c and the reference's right-end entries
// (a[k-1] = 0, c[k-1] = f'(x_{k-1})). Same operations in the same order as oracle/bounds_oracle.natural_spline, so
// the rows agree bit for bit. a[] and b[] hold the recurrence's c' and d' until they are overwritten.
PQB_HD void natural_spline_fit(const double *sx, const double *y, int k, double *a, double *b, double *c) {
    double *cp = a, *dp = b;
    cp[0] = 0.0 / 2.0;  // up[0] / di[0]
    dp[0] = 0.0 / 2.0;  // rhs[0] / di[0]
    for (int i = 1; i < k; ++i) {
        double lo = 0.0, di = 2.0, up = 0.0, rhs = 0.0;
        if (i < k - 1) {
            const double h0 = sx[i] - sx[i - 1], h1 = sx[i + 1] - sx[i];
            lo = h0 / 3.0;
            di = 2.0 / 3.0 * (sx[i + 1] - sx[i - 1]);
            up = h1 / 3.0;
            rhs = (y[i + 1] - y[i]) / h1 - (y[i] - y[i - 1]) / h0;
        }
        const double den = di - lo * cp[i - 1];
        cp[i] = up / den;
        dp[i] = (rhs - lo * dp[i - 1]) / den;
    }
    // b[k-1] = dp[k-1] already in place
    for (int i = k - 2; i >= 0; --i) b[i] = dp[i] - cp[i] * b[i + 1];
    for (int i = 0; i < k - 1; ++i) {
        const double h = sx[i + 1] - sx[i];
        a[i] = (b[i + 1] - b[i]) / (3.0 * h);
        c[i] = (y[i + 1] - y[i]) / h - (2.0 * b[i] + b[i + 1]) * h / 3.0;
    }
    const double hl = sx[k - 1] - sx[k - 2];
    a[k - 1] = 0.0;
    c[k - 1] = 3.0 * a[k - 2] * hl * hl + 2.0 * b[k - 2] * hl + c[k - 2];
}

PQB_HD bool increasing(const double *s, int k) {
    for (int i = 1; i < k; ++i)
        if (!(s[i] > s[i - 1])) return false;
    return true;
}

// ---- bSpline() (reference_path_smoother.cpp:490-524): a clamped B-spline whose control points are the reference
// points, sampled at t = 0, delta_t, 2 delta_t (accumulated), ... below 1, then at t = 1 ----

// Length of the control polygon: the sequential sum of the point distances (tools.cpp:46-48), squares as d * d.
PQB_HD double polygon_length(const double *x, const double *y, int m) {
    double length = 0.0;
    for (int i = 0; i + 1 < m; ++i) {
        const double dx = x[i] - x[i + 1], dy = y[i] - y[i + 1];
        length += sqrt(dx * dx + dy * dy);
    }
    return length;
}

// 3 when the average point spacing is above 10 m, 4 above 5 m, else 5 (strict comparisons: NaN gives 5).
PQB_HD int bspline_degree(double length, int m) {
    const double average = length / (double)(m - 1);
    if (average > 10.0) return 3;
    if (average > 5.0) return 4;
    return 5;
}

// The sample parameters: t = 0, then t += 1 / length while t < 1, then t = 1. Writes at most `cap` values into t[]
// and returns their count, or cap + 1 when there would be more (an infinite length gives delta_t = 0, on which the
// reference loops forever). A NaN length, a zero length or one below 1 m gives the two samples t = 0 and t = 1.
PQB_HD int bspline_abscissae(double length, int cap, double *t) {
    const double delta_t = 1.0 / length;
    double tmp_t = 0.0;
    int count = 0;
    while (tmp_t < 1.0) {
        if (count == cap) return cap + 1;
        t[count++] = tmp_t;
        tmp_t += delta_t;
    }
    if (count == cap) return cap + 1;
    t[count++] = 1.0;
    return count;
}

// Knot i of the clamped uniform vector of m control points: degree + 1 zeros, (i - degree) / (m - degree), degree + 1
// ones. Computed the same way wherever it is compared, so the span choice is a pure function of (t, degree, m).
PQB_HD double bspline_knot(int i, int degree, int m) {
    if (i <= degree) return 0.0;
    if (i >= m) return 1.0;
    return (double)(i - degree) / (double)(m - degree);
}

// The span k in [degree, m - 1] with knot(k) <= t < knot(k + 1); t = 1 falls in the last non-empty span, m - 1.
PQB_HD int bspline_span(double t, int degree, int m) {
    int lo = degree, hi = m - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (bspline_knot(mid, degree, m) <= t) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// de Boor's algorithm at t for degree D (unrolled, so the working points stay in registers). At t = 0 every alpha is
// 0 and at t = 1 every alpha is 1, so the end samples are the first and the last point exactly.
template <int D>
PQB_HD void de_boor(const double *px, const double *py, int m, double t, double &x, double &y) {
    const int k = bspline_span(t, D, m);
    double dx[D + 1], dy[D + 1];
#pragma unroll
    for (int j = 0; j <= D; ++j) {
        dx[j] = px[j + k - D];
        dy[j] = py[j + k - D];
    }
#pragma unroll
    for (int r = 1; r <= D; ++r) {
#pragma unroll
        for (int j = D; j >= r; --j) {
            const double ua = bspline_knot(j + k - D, D, m);
            const double ub = bspline_knot(j + 1 + k - r, D, m);
            const double alpha = (t - ua) / (ub - ua);
            dx[j] = (1.0 - alpha) * dx[j - 1] + alpha * dx[j];
            dy[j] = (1.0 - alpha) * dy[j - 1] + alpha * dy[j];
        }
    }
    x = dx[D];
    y = dy[D];
}

// One sample of the curve of degree 3, 4 or 5 over the m points (px, py).
PQB_HD void bspline_eval(const double *px, const double *py, int m, int degree, double t, double &x, double &y) {
    if (degree == 3) de_boor<3>(px, py, m, t, x, y);
    else if (degree == 4) de_boor<4>(px, py, m, t, x, y);
    else de_boor<5>(px, py, m, t, x, y);
}

// bSpline()'s checks and sample parameters for one path: kPointCount for fewer than 4 points (reference_path_smoother
// .cpp:33-36) or more than the row holds, kBsplineDegree when degree >= m (tinyspline refuses the spline),
// kTooManyPoints when there are more than `cap` samples. r = samples written to t[] (cap + 1 when over capacity, 0 when
// the points were rejected), degree = 0 when the count was rejected.
PQB_HD int bspline_prepare(const double *x, const double *y, int m, int m_max, int cap, double *t, int &r, int &degree) {
    r = 0;
    degree = 0;
    if (m < 4 || m > m_max) return kPointCount;
    const double length = polygon_length(x, y, m);
    degree = bspline_degree(length, m);
    if (degree >= m) return kBsplineDegree;
    r = bspline_abscissae(length, cap, t);
    return r > cap ? kTooManyPoints : kOk;
}

// s_list_ of bSpline() (reference_path_smoother.cpp:519-523): cumulative chord length, squares written as d * d.
PQB_HD void chord_length(const double *x, const double *y, int r, double *s) {
    s[0] = 0.0;
    for (int i = 1; i < r; ++i) {
        const double dx = x[i] - x[i - 1], dy = y[i] - y[i - 1];
        s[i] = s[i - 1] + sqrt(dx * dx + dy * dy);
    }
}

// segmentRawReference's sample count (:61-68): 0, 1, 2, ... while the last is below max_s, so the last sample
// overshoots max_s by up to 1 m (it is extrapolated); the following `max_s - last > 1` branch cannot fire.
// Returns cap + 1 when the count exceeds `cap`.
PQB_HD int segment_count(double max_s, int cap) {
    double last = 0.0;
    int count = 1;
    while (last < max_s) {
        last += 1.0;
        if (++count > cap) return cap + 1;
    }
    return count;
}

// The j-th sample's abscissa: repeated addition of 1.0 from 0 is exact for integers, so it is j itself.
PQB_HD double segment_s(int j) { return (double)j; }

// One sample of segmentRawReference (:71-83): position, heading atan2(dy, dx) and curvature. pow(q, 1.5) is
// written q * sqrt(q), within an ulp of it (as pqp_bounds_core.cuh does for tools.cpp:38-44).
PQB_HD void segment_sample(const pqb::SplineView &sp, double s, double &x, double &y, double &angle, double &k) {
    double dx, ddx, dy, ddy;
    pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, s), s, x, dx, ddx, y, dy, ddy);
    angle = atan2(dy, dx);
    const double q = dx * dx + dy * dy;
    k = (dx * ddy - dy * ddx) / (q * sqrt(q));
}

// postSmooth's epilogue (reference_path_smoother.cpp:560-573): the point of layer i is the tension spline at
// layer_s[i] moved by offsets[i] along the normal heading + pi/2; s re-accumulated from the points.
PQB_HD void post_points(const pqb::SplineView &sp, const double *layer_s, const double *offsets, int n, double *s,
                        double *x, double *y) {
    double acc = 0.0;
    for (int i = 0; i < n; ++i) {
        const double rs = layer_s[i];
        double rx, dx, ddx, ry, dy, ddy;
        pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, rs), rs, rx, dx, ddx, ry, dy, ddy);
        const double dir = atan2(dy, dx) + M_PI_2;
        x[i] = rx + offsets[i] * cos(dir);
        y[i] = ry + offsets[i] * sin(dir);
        if (i > 0) {
            const double ex = x[i] - x[i - 1], ey = y[i] - y[i - 1];
            acc += sqrt(ex * ex + ey * ey);
        }
        s[i] = acc;
    }
}

// A well-formed stand-in for a path that has failed: three collinear points (s = x = 0, 1, 2; y = 0) of length 2,
// so that stages which read a spline unconditionally (the DP reads k and length) still get valid input.
PQB_HD void placeholder_points(double *s, double *x, double *y) {
    for (int i = 0; i < 3; ++i) {
        s[i] = (double)i;
        x[i] = (double)i;
        y[i] = 0.0;
    }
}
constexpr int kPlaceholderK = 3;
constexpr double kPlaceholderLength = 2.0;

// processReferencePath up to buildReferenceFromSpline (path_optimizer.cpp:73-117, tools.cpp:57-126): the zero
// length test, processInitState (l0, psi0), the 75 degree gate and setReferencePathLength. Returns a status;
// max_s = the reference length the states are built to.
PQB_HD int process_reference(const pqb::SplineView &sp, double length, const double *start, const double *target,
                             double epsilon, double &l0, double &psi0, double &max_s) {
    l0 = psi0 = 0.0;
    max_s = length;
    if (fabs(length - 0.0) < epsilon) return kEmptyReference;  // isEqual (tools.cpp:28-30)
    double ix, dx, ddx, iy, dy, ddy;
    pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, 0.0), 0.0, ix, dx, ddx, iy, dy, ddy);
    const double ih = atan2(dy, dx);
    // global2Local(start, init_point).y and distance(start, init_point)
    const double gx = ix - start[0], gy = iy - start[1];
    const double local_y = -gx * sin(start[2]) + gy * cos(start[2]);
    const double dist = sqrt(gx * gx + gy * gy);
    l0 = local_y < 0.0 ? dist : -dist;
    psi0 = pqb::constrain_angle(start[2] - ih);
    if (fabs(psi0) > 75 * M_PI / 180) return kInitHeading;
    // setReferencePathLength: a target beyond the end of the reference keeps the length
    double ex, ey;
    pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, length), length, ex, dx, ddx, ey, dy, ddy);
    const double eh = atan2(dy, dx);
    const double tx = target[0] - ex, ty = target[1] - ey;
    const double local_x = tx * cos(eh) + ty * sin(eh);
    if (local_x > 0.0) return kOk;
    max_s = pqdp::projection_s(sp, target[0], target[1], length);
    return kOk;
}

// BaseSolver's precise_planning_size_ (base_solver.cpp:24-34): lower_bound of the states' s at the length.
PQB_HD int precise_size(const double *s, int n, bool rough, double precise_length) {
    if (!rough) return n;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s[mid] < precise_length) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// The end-heading rows of setConstraints (base_solver.cpp:250-259): only when the path is not blocked, and the
// test is signed (a target heading error below -70 degrees still gets rows).
PQB_HD void end_heading_rows(bool constrain, bool blocked, double target_heading, double last_heading, double &lo,
                             double &hi) {
    lo = -1e30;  // OsqpEigen::INFTY
    hi = 1e30;
    if (constrain && !blocked) {
        const double end_psi = pqb::constrain_angle(target_heading - last_heading);
        if (end_psi < 70 * M_PI / 180) {
            lo = end_psi - 0.087;
            hi = end_psi + 0.087;
        }
    }
}

}  // namespace pqpl
