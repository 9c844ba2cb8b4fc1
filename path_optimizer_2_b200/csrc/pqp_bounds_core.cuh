// pqp_bounds_core.cuh — per-thread work of the clearance-bounds kernel (include/pqp_bounds.h).
// Plain FP64 scalar code with no CUDA intrinsics, so the same source is compiled by nvcc for the
// kernel (pqp_bounds.cu) and by g++ for the CPU test driver (tests/emu/bounds_driver.cpp).
// Citations are relative to /root/reference/.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define PQB_HD __host__ __device__ __forceinline__
#else
#define PQB_HD inline
#endif

namespace pqb {

struct MapView {
    const float *dist;  // [rows * cols]
    int rows, cols;
    double res, inv_res, half_lx, half_ly, cx, cy;
};

// The map of path b under a per-path slot index (the *_mapped calls): &table[index[b]], or NULL when the index is
// outside [0, n_maps). Every map-reading kernel looks its slot up here; the view stays in the table (global memory),
// so a kernel reads its fields where it uses them rather than holding a copy in registers.
PQB_HD const MapView *slot_view(const MapView *table, int n_maps, const int32_t *index, int b) {
    const int32_t i = index[b];
    return i >= 0 && i < n_maps ? table + i : nullptr;
}

struct Params {
    double front_length, rear_length, car_width, safety_margin, epsilon;
};

struct SplineView {
    const double *sx;                   // abscissae
    const double *xa, *xb, *xc, *xy;    // x(s)
    const double *ya, *yb, *yc, *yy;    // y(s)
    int k;
};

// grid_map's isInside: strictly inside the map's rectangle (false for NaN), the test map_distance makes
PQB_HD bool map_inside(const MapView &m, double x, double y) {
    return fabs(x - m.cx) < m.half_lx && fabs(y - m.cy) < m.half_ly;
}

// Map::getObstacleDistance (src/tools/Map.cpp:16-22): 0 outside the map, otherwise grid_map's
// INTER_LINEAR lookup of the float "distance" layer - bilinear between the four cell centres
// around the position (grid_map itself is not in the tree; at the outermost half cell it falls
// back to the nearest cell, which the clamped weights below reproduce).
PQB_HD double map_distance(const MapView &m, double x, double y) {
    const double dx = x - m.cx, dy = y - m.cy;
    if (!(fabs(dx) < m.half_lx && fabs(dy) < m.half_ly)) return 0.0;
    // (position - corner) / resolution as a multiplication: the interpolant is continuous across
    // cell borders, so a last-bit difference in fi, fj cannot change the value beyond rounding
    const double fi = (m.half_lx - dx) * m.inv_res - 0.5;
    const double fj = (m.half_ly - dy) * m.inv_res - 0.5;
    int i0 = (int)floor(fi), j0 = (int)floor(fj);
    i0 = i0 < 0 ? 0 : (i0 > m.rows - 2 ? m.rows - 2 : i0);
    j0 = j0 < 0 ? 0 : (j0 > m.cols - 2 ? m.cols - 2 : j0);
    double ti = fi - i0, tj = fj - j0;
    ti = ti < 0.0 ? 0.0 : (ti > 1.0 ? 1.0 : ti);
    tj = tj < 0.0 ? 0.0 : (tj > 1.0 ? 1.0 : tj);
    const float *r0 = m.dist + (size_t)i0 * m.cols + j0;
    const float *r1 = r0 + m.cols;
    const double d00 = r0[0], d01 = r0[1], d10 = r1[0], d11 = r1[1];
    return d00 * (1.0 - ti) * (1.0 - tj) + d10 * ti * (1.0 - tj) + d01 * (1.0 - ti) * tj + d11 * ti * tj;
}

// Segment index of tk::spline::operator() / deriv (src/tools/spline.cpp:252-258): lower_bound - 1
// clamped at 0, i.e. the last abscissa strictly below s (0 if there is none, also for NaN).
PQB_HD int seg_index(const double *sx, int k, double s) {
    int lo = 0, hi = k;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sx[mid] < s) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1 < 0 ? 0 : lo - 1;
}

// The same index reached by walking from a nearby one (the previous Newton iterate / the previous
// state of the walk): one or two loads instead of a dependent binary-search chain.
PQB_HD int seg_index_from(const double *sx, int k, double s, int hint) {
    int j = hint < 0 ? 0 : (hint > k - 1 ? k - 1 : hint);
    if (sx[j] < s) {
        while (j + 1 < k && sx[j + 1] < s) ++j;
    } else {
        while (j > 0 && !(sx[j] < s)) --j;
    }
    return j;
}

// operator() and deriv(1|2) of one spline at s, given the segment index (spline.cpp:259-330):
// quadratic extrapolation left and right with the reference's own coefficients (incl. its left
// second derivative 2 b0 h).
PQB_HD void spline_eval_at(int idx, const double *sx, const double *a, const double *b, const double *c, const double *y,
                           int k, double s, double &v, double &d1, double &d2) {
    const double h = s - sx[idx];
    if (s < sx[0]) {
        const double b0 = b[0], c0 = c[0];
        v = (b0 * h + c0) * h + y[0];
        d1 = 2.0 * b0 * h + c0;
        d2 = 2.0 * b0 * h;
    } else if (s > sx[k - 1]) {
        v = (b[k - 1] * h + c[k - 1]) * h + y[k - 1];
        d1 = 2.0 * b[k - 1] * h + c[k - 1];
        d2 = 2.0 * b[k - 1];
    } else {
        v = ((a[idx] * h + b[idx]) * h + c[idx]) * h + y[idx];
        d1 = (3.0 * a[idx] * h + 2.0 * b[idx]) * h + c[idx];
        d2 = 6.0 * a[idx] * h + 2.0 * b[idx];
    }
}

// x(s), y(s) and their first two derivatives: the two splines share their abscissae, so one index
PQB_HD void path_eval(const SplineView &sp, int idx, double s, double &x, double &dx, double &ddx, double &y, double &dy,
                      double &ddy) {
    spline_eval_at(idx, sp.sx, sp.xa, sp.xb, sp.xc, sp.xy, sp.k, s, x, dx, ddx);
    spline_eval_at(idx, sp.sx, sp.ya, sp.yb, sp.yc, sp.yy, sp.k, s, y, dy, ddy);
}

PQB_HD double std_min(double a, double b) { return (b < a) ? b : a; }  // std::min, NaN behaviour included

// getDirectionalProjectionByNewton (src/tools/tools.cpp:156-189): foot point of the line through
// (tx, ty) with direction `angle` on the spline; returns its position.
PQB_HD void directional_projection(const SplineView &sp, double tx, double ty, double angle, double max_s,
                                   double hint_s, double &px, double &py) {
    hint_s = std_min(hint_s, max_s);
    double cur_s = hint_s, prev_s = hint_s;
    double sa, ca;
    sincos(angle, &sa, &ca);
    const double v1 = sa, v2 = -ca;
    double x, y, dx, dy, ddx, ddy;
    int idx = seg_index(sp.sx, sp.k, cur_s);
    for (int i = 0; i < 20; ++i) {
        path_eval(sp, idx, cur_s, x, dx, ddx, y, dy, ddy);
        const double p1 = v1 * (x - tx) + v2 * (y - ty);
        const double p2 = v1 * dx + v2 * dy;
        const double j = p1 * p2;
        const double h = p1 * (v1 * ddx + v2 * ddy) + p2 * p2;
        cur_s -= j / h;
        idx = seg_index_from(sp.sx, sp.k, cur_s, idx);
        if (fabs(cur_s - prev_s) < 1e-5) break;
        prev_s = cur_s;
    }
    cur_s = std_min(cur_s, max_s);
    idx = seg_index_from(sp.sx, sp.k, cur_s, idx);
    path_eval(sp, idx, cur_s, px, dx, ddx, py, dy, ddy);
}

PQB_HD double constrain_angle(double a) {  // include/tools/tools.hpp:25-35 (recursion unrolled, bounded)
    for (int i = 0; i < 8 && a > M_PI; ++i) a -= 2 * M_PI;
    for (int i = 0; i < 8 && a < -M_PI; ++i) a += 2 * M_PI;
    return a;
}

// ReferencePathImpl::getClearanceWithDirectionStrict (reference_path_impl.cpp:232-312).
// lb = right bound (<= 0 side), ub = left bound; {0, 0} when the state is too close to an
// obstacle or the corridor is narrower than the car.
PQB_HD void clearance(const MapView &m, const Params &P, double sx, double sy, double heading, double &lb, double &ub) {
    const double delta_s = 0.3, search_radius = 0.5, smaller_ds = 0.05, min_space = 0.2;
    const double left_angle = constrain_angle(heading + M_PI_2);
    const double right_angle = constrain_angle(heading - M_PI_2);
    const int n = (int)(6.0 / delta_s);
    lb = ub = 0.0;
    if (!(map_distance(m, sx, sy) > search_radius)) return;
    double cl, sl, cr, sr;
    sincos(left_angle, &sl, &cl);
    sincos(right_angle, &sr, &cr);
    double right_s = 0.0;
    for (int j = 0; j != n; ++j) {
        right_s += delta_s;
        if (map_distance(m, sx + right_s * cr, sy + right_s * sr) < search_radius) break;
    }
    double left_s = 0.0;
    for (int j = 0; j != n; ++j) {
        left_s += delta_s;
        if (map_distance(m, sx + left_s * cl, sy + left_s * sl) < search_radius) break;
    }
    double right_bound = -(right_s - delta_s);
    double left_bound = left_s - delta_s;
    const int fine = (int)(delta_s / smaller_ds);
    for (int i = 1; i != fine; ++i) {
        left_bound += smaller_ds;
        if (map_distance(m, sx + left_bound * cl, sy + left_bound * sl) < search_radius) {
            left_bound -= smaller_ds;
            break;
        }
    }
    for (int i = 1; i != fine; ++i) {
        right_bound -= smaller_ds;
        // as the reference: the negative bound times the right-hand direction (:288-291)
        if (map_distance(m, sx + right_bound * cr, sy + right_bound * sr) < search_radius) {
            right_bound += smaller_ds;
            break;
        }
    }
    const double diff_radius = P.car_width * 0.5 - search_radius;
    left_bound -= diff_radius;
    right_bound += diff_radius;
    if (left_bound < right_bound) return;
    const double space = left_bound - right_bound;
    const double max_margin = fmax(0.0, (space - min_space) / 2.0);
    const double margin = fmin(P.safety_margin, max_margin);
    ub = left_bound - margin;
    lb = right_bound + margin;
}

// One (state, anchor) task of updateBoundsImproved (reference_path_impl.cpp:183-215):
// anchor 0 = front circle, 1 = rear circle (projected onto the spline along the state's normal,
// bounds shifted by the projection's lateral offset), 2 = the state itself.
PQB_HD void anchor_bounds(const MapView &m, const Params &P, const SplineView &sp, double s, double x, double y,
                          double heading, int anchor, double &lb, double &ub) {
    if (anchor == 2) {
        clearance(m, P, x, y, heading, lb, ub);
        return;
    }
    const double len = anchor == 0 ? P.front_length : P.rear_length;
    double ch, sh;
    sincos(heading, &sh, &ch);
    const double ax = x + len * ch, ay = y + len * sh;
    double px, py;
    directional_projection(sp, ax, ay, heading + M_PI_2, s + 5.0, s + len, px, py);
    clearance(m, P, px, py, heading, lb, ub);
    // global2Local(anchor, projection).y (src/tools/tools.cpp:57-64)
    const double ddx = px - ax, ddy = py - ay;
    const double offset = -ddx * sh + ddy * ch;
    lb += offset;
    ub += offset;
}

// ReferencePathImpl::buildReferenceFromSpline (reference_path_impl.cpp:314-338) for one path:
// writes at most n_max states (rows s, x, y, heading with stride n_max, curvature separately) and
// returns the number of states the reference would emit (count_all) or min(that, n_max).
PQB_HD int build_states(const SplineView &sp, double max_s, double ds_small, double ds_large, bool dynamic, int n_max,
                        bool count_all, double *st, double *curv) {
    const double large_k = 0.2, small_k = 0.08;
    double tmp_s = 0.0;
    int count = 0, idx = 0, cached = -1;
    // coefficients of the current segment stay in registers: the walk crosses a segment border
    // only every few steps, so most steps touch no memory
    double x0 = 0.0, x1 = 0.0, xa = 0.0, xb = 0.0, xc = 0.0, xy = 0.0, ya = 0.0, yb = 0.0, yc = 0.0, yy = 0.0;
    const double s_first = sp.sx[0], s_last = sp.sx[sp.k - 1];
    while (tmp_s <= max_s) {
        if (count >= n_max && !count_all) break;
        double x, y, dx, dy, ddx, ddy;
        // still strictly above the cached segment's start and not above its end: same index
        if (!(cached >= 0 && x0 < tmp_s && !(x1 < tmp_s))) idx = seg_index_from(sp.sx, sp.k, tmp_s, idx);
        if (tmp_s < s_first || tmp_s > s_last) {
            path_eval(sp, idx, tmp_s, x, dx, ddx, y, dy, ddy);  // extrapolation (spline.cpp:262-268)
        } else {
            if (idx != cached) {
                cached = idx;
                x0 = sp.sx[idx];
                x1 = idx + 1 < sp.k ? sp.sx[idx + 1] : HUGE_VAL;
                xa = sp.xa[idx]; xb = sp.xb[idx]; xc = sp.xc[idx]; xy = sp.xy[idx];
                ya = sp.ya[idx]; yb = sp.yb[idx]; yc = sp.yc[idx]; yy = sp.yy[idx];
            }
            const double h = tmp_s - x0;
            x = ((xa * h + xb) * h + xc) * h + xy;
            dx = (3.0 * xa * h + 2.0 * xb) * h + xc;
            ddx = 6.0 * xa * h + 2.0 * xb;
            y = ((ya * h + yb) * h + yc) * h + yy;
            dy = (3.0 * ya * h + 2.0 * yb) * h + yc;
            ddy = 6.0 * ya * h + 2.0 * yb;
        }
        const double h = atan2(dy, dx);                                             // tools.cpp:32-36
        // tools.cpp:38-44: pow(pow(dx, 2) + pow(dy, 2), 1.5), written with products and a square
        // root (each within 1 ulp of the pow form; CUDA's pow itself is only 2-ulp accurate)
        const double sq = dx * dx + dy * dy;
        const double k = (dx * ddy - dy * ddx) / (sq * sqrt(sq));
        if (count < n_max) {
            st[count] = tmp_s;
            st[n_max + count] = x;
            st[2 * n_max + count] = y;
            st[3 * n_max + count] = h;
            curv[count] = k;
        }
        ++count;
        if (dynamic) {
            const double ak = fabs(k);
            const double k_share = ak > large_k ? 1.0 : (ak < small_k ? 0.0 : (ak - small_k) / (large_k - small_k));
            tmp_s += ds_large - k_share * (ds_large - ds_small);
        } else {
            tmp_s += ds_large;
        }
        if (count > (1 << 24)) break;  // a non-positive step would never terminate
    }
    return count;
}

}  // namespace pqb
