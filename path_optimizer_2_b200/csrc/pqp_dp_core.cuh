// pqp_dp_core.cuh — the lattice DP search of the reference's front end (SURVEY.md §8 row f-4),
// ReferencePathSmoother::graphSearchDp + calculateCostAt
// (/root/reference/src/reference_path_smoother/reference_path_smoother.cpp:107-295), as ONE templated
// per-path routine over an execution context: the CUDA kernel (pqp_dp.cu) runs it with one CTA per path
// (nodes sampled in parallel, a layer's 34 x 34 edges spread over 4 lanes per node and min-reduced with the
// reference's first-minimum rule, bounds extended in parallel), the CPU test driver (tests/emu/dp_driver.cpp)
// with a single thread. Plain FP64 scalar code, compiled with contraction off in both builds.
// Citations are relative to /root/reference/.
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "pqp_bounds_core.cuh"

namespace pqdp {

constexpr int kJMax = 64;  // lateral samples per layer the kernel is laid out for (34 at the flag defaults)

struct Params {
    double lateral_range;    // FLAGS_search_lateral_range        10.0  (planning_flags.cpp:38)
    double lateral_spacing;  // FLAGS_search_lateral_spacing      0.6   (:42)
    double lon_spacing;      // FLAGS_search_longitudial_spacing  1.5   (:40)
    double car_width;        // FLAGS_car_width                   2.0   (:10)
};

// Per-path inputs / outputs / scratch (device or host pointers, already offset to this path)
struct PathIO {
    pqb::SplineView sp;
    double length;          // reference->getLength()
    double sx, sy, sh;      // start_state_
    int layers_max;
    // outputs
    int32_t *ok, *n_layers, *n_out, *chosen;
    double *layer_s, *lower, *upper, *vehicle_l, *target_s;
    double *cost;           // [layers_max][J] table (DBL_MAX = not reached)
    int8_t *parent;         // [layers_max][J]  (-1 = none)
    uint8_t *feasible;      // [layers_max][J]
    // scratch
    double *nx, *ny, *dis;  // [layers_max][J]
    double *ref;            // [layers_max][4]: x, y, heading of the reference at the layer, 1 / curvature sign helper
};

// status written to ok[]
enum { kDpOk = 1, kDpVehicleFar = 0, kDpTooManyLayers = -1 };

PQB_HD double heading_of(const pqb::SplineView &sp, double s) {  // tools.cpp:32-36
    double x, dx, ddx, y, dy, ddy;
    pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, s), s, x, dx, ddx, y, dy, ddy);
    return atan2(dy, dx);
}

// getProjectionByNewton (tools.cpp:98-128): returns the .s of the result
PQB_HD double projection_newton(const pqb::SplineView &sp, double tx, double ty, double max_s, double hint_s) {
    hint_s = pqb::std_min(hint_s, max_s);
    double cur = hint_s, prev = hint_s;
    int idx = pqb::seg_index(sp.sx, sp.k, cur);
    for (int i = 0; i < 20; ++i) {
        double x, dx, ddx, y, dy, ddy;
        pqb::path_eval(sp, idx, cur, x, dx, ddx, y, dy, ddy);
        const double j = (x - tx) * dx + (y - ty) * dy;
        const double h = dx * dx + (x - tx) * ddx + dy * dy + (y - ty) * ddy;
        cur -= j / h;
        idx = pqb::seg_index(sp.sx, sp.k, cur);
        if (fabs(cur - prev) < 1e-5) break;
        prev = cur;
    }
    return pqb::std_min(cur, max_s);
}

// getProjection (tools.cpp:66-96): coarse 1 m scan, end point test, Newton; only .s is used by the caller
PQB_HD double projection_s(const pqb::SplineView &sp, double tx, double ty, double max_s) {
    const double start_s = 0.0;
    if (max_s <= start_s) return 0.0;
    double tmp = start_s, min_s = start_s, min_dis = DBL_MAX;
    while (tmp <= max_s) {
        double x, dx, ddx, y, dy, ddy;
        pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, tmp), tmp, x, dx, ddx, y, dy, ddy);
        const double d = sqrt(pow(x - tx, 2) + pow(y - ty, 2));
        if (d < min_dis) {
            min_dis = d;
            min_s = tmp;
        }
        tmp += 1.0;
    }
    double ex, dx, ddx, ey, dy, ddy;
    pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, max_s), max_s, ex, dx, ddx, ey, dy, ddy);
    if (sqrt(pow(ex - tx, 2) + pow(ey - ty, 2)) < min_dis) return max_s;
    return projection_newton(sp, tx, ty, max_s, min_s);
}

using pqb::map_inside;

// The j-th lateral offset by repeated addition, as the reference accumulates cur_l (:185,213)
PQB_HD double lateral_offset(const Params &p, int j) {
    double cl = -p.lateral_range;
    for (int t = 0; t < j; ++t) cl += p.lateral_spacing;
    return cl;
}
PQB_HD int lateral_count(const Params &p) {
    int n = 0;
    double cl = -p.lateral_range;
    while (cl <= p.lateral_range && n < kJMax) {
        ++n;
        cl += p.lateral_spacing;
    }
    return n;
}

// Execution context of the CPU build: one thread, no cross-lane exchange.
struct SerialCtx {
    PQB_HD int tid() const { return 0; }
    PQB_HD int nthreads() const { return 1; }
    PQB_HD void sync() const {}
    static constexpr int kPredLanes = 1;
    // combine (total, pred, dir) over the kPredLanes lanes of a node: nothing to do
    PQB_HD void reduce_pred(double &, int &, double &) const {}
    PQB_HD bool any(bool v) const { return v; }
};

// One path. `Ctx`: tid / nthreads / sync (barrier over the path's threads) / reduce_pred / any.
// `sh` = shared scratch of the path: doubles [6 * kJMax + 8] and ints [8] (CPU: plain arrays).
template <class Ctx>
PQB_HD void dp_search_path(const Ctx &c, const pqb::MapView &map, const Params &prm, const PathIO &io, double *shd, int *shi) {
    const pqb::SplineView &sp = io.sp;
    const int J = lateral_count(prm);
    const double threshold = prm.car_width / 2.0 + 0.2;  // search_threshold (:176)
    double *ls = shd;                       // [kJMax] lateral offsets
    double *pl_x = shd + kJMax, *pl_y = shd + 2 * kJMax, *pl_dir = shd + 3 * kJMax, *pl_cost = shd + 4 * kJMax;  // previous layer
    double *cur_dir = shd + 5 * kJMax;      // [kJMax] directions chosen in the current layer
    // ---- phase 0: layers (:146-158), vehicle offset (:160-170) - serial
    if (c.tid() == 0) {
        double tmp_s = projection_s(sp, io.sx, io.sy, io.length);
        const double search_ds = io.length > 6 ? prm.lon_spacing : 0.5;
        int L = 0;
        bool overflow = false;
        while (tmp_s < io.length) {
            if (L < io.layers_max) io.layer_s[L] = tmp_s;
            else overflow = true;
            ++L;
            tmp_s += search_ds;
        }
        if (L < io.layers_max) io.layer_s[L] = io.length;
        else overflow = true;
        ++L;
        double px, dx, ddx, py, dy, ddy;
        const double vs = io.layer_s[0];
        pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, vs), vs, px, dx, ddx, py, dy, ddy);
        const double ph = atan2(dy, dx);
        const double ex = io.sx - px, ey = io.sy - py;
        const double vl = -ex * sin(ph) + ey * cos(ph);  // global2Local(...).y (tools.cpp:56-63)
        *io.vehicle_l = vl;
        *io.target_s = io.length;
        *io.n_layers = L;
        int status = kDpOk;
        if (overflow) status = kDpTooManyLayers;
        else if (fabs(vl) > prm.lateral_range) status = kDpVehicleFar;
        shi[0] = L;
        shi[1] = status;
        shi[2] = (int)((prm.lateral_range + vl) / prm.lateral_spacing);  // start_lateral_index (:171-172)
        *io.ok = status;
        *io.n_out = 0;
    }
    c.sync();
    const int L = shi[0];
    if (shi[1] != kDpOk) return;
    const int start_j = shi[2];
    for (int j = c.tid(); j < J; j += c.nthreads()) ls[j] = lateral_offset(prm, j);
    // ---- phase 1a: the reference at every layer (:180-184)
    for (int i = c.tid(); i < L; i += c.nthreads()) {
        const double cs = io.layer_s[i];
        double x, dx, ddx, y, dy, ddy;
        pqb::path_eval(sp, pqb::seg_index(sp.sx, sp.k, cs), cs, x, dx, ddx, y, dy, ddy);
        const double k = (dx * ddy - dy * ddx) / pow(pow(dx, 2) + pow(dy, 2), 1.5);  // getCurvature (tools.cpp:38-44)
        io.ref[4 * i + 0] = x;
        io.ref[4 * i + 1] = y;
        io.ref[4 * i + 2] = atan2(dy, dx);
        io.ref[4 * i + 3] = k;
    }
    c.sync();
    // ---- phase 1b: nodes (:185-212)
    for (int idx = c.tid(); idx < L * J; idx += c.nthreads()) {
        const int i = idx / J, j = idx - i * J;
        const double rx = io.ref[4 * i], ry = io.ref[4 * i + 1], rh = io.ref[4 * i + 2], rk = io.ref[4 * i + 3];
        const double rr = 1 / rk;
        const double cl = ls[j];
        const double x = rx + cl * cos(rh + M_PI_2), y = ry + cl * sin(rh + M_PI_2);
        const double d = map_inside(map, x, y) ? pqb::map_distance(map, x, y) : -1.0;
        bool feas = !((rk < 0 && cl < rr) || (rk > 0 && cl > rr) || d < threshold);
        if (i == 0) feas = (j == start_j);
        io.nx[idx] = x;
        io.ny[idx] = y;
        io.dis[idx] = d;
        io.feasible[idx] = feas ? 1 : 0;
        io.cost[idx] = (i == 0 && j == start_j) ? 0.0 : DBL_MAX;
        io.parent[idx] = -1;
    }
    c.sync();
    // ---- phase 2: layer-by-layer cost (:107-140, :234-243)
    for (int j = c.tid(); j < J; j += c.nthreads()) {
        pl_x[j] = io.nx[j];
        pl_y[j] = io.ny[j];
        pl_dir[j] = io.sh;                                 // only the start node's is ever read
        pl_cost[j] = (j == start_j) ? 0.0 : DBL_MAX;       // DBL_MAX: infeasible or not reached
    }
    c.sync();
    int max_layer = 0;
    constexpr int G = Ctx::kPredLanes;
    for (int i = 1; i < L; ++i) {
        const double ds_layer = io.layer_s[i] - io.layer_s[i - 1];
        const double rh = io.ref[4 * i + 2];
        bool found = false;
        // work item w = node j x predecessor lane g; lanes of one node are adjacent threads
        for (int w = c.tid(); w < ((J * G + c.nthreads() - 1) / c.nthreads()) * c.nthreads(); w += c.nthreads()) {
            const int j = w / G, g = w - j * G;
            double best = DBL_MAX, bdir = 0.0;
            int bp = -1;
            const bool live = j < J && io.feasible[i * J + j] != 0;
            if (live) {
                const double x = io.nx[i * J + j], y = io.ny[i * J + j], l = ls[j], d = io.dis[i * J + j];
                double self_cost = 0;
                if (d < 3.0) self_cost += (3.0 - d) / 3.0 * 0.5;         // safe_distance, weight_obstacle (:116-117,121)
                self_cost += fabs(l) / prm.lateral_range * 1.0;           // weight_ref_offset (:122)
                for (int p = g; p < J; p += G) {
                    if (!(pl_cost[p] < DBL_MAX)) continue;                // infeasible, or never reached (cannot win)
                    if (fabs(ls[p] - l) > ds_layer) continue;             // (:127)
                    const double direction = atan2(y - pl_y[p], x - pl_x[p]);
                    const double edge = fabs(pqb::constrain_angle(direction - pl_dir[p])) / M_PI_2 * 16.0 +
                                        fabs(pqb::constrain_angle(direction - rh)) / M_PI_2 * 0.5;  // (:129-130)
                    const double total = self_cost + edge + pl_cost[p];
                    if (total < best) {  // strict: the first minimum in predecessor order wins (:132)
                        best = total;
                        bp = p;
                        bdir = direction;
                    }
                }
            }
            c.reduce_pred(best, bp, bdir);
            if (g == 0 && j < J) {
                if (bp >= 0) {
                    io.cost[i * J + j] = best;
                    io.parent[i * J + j] = (int8_t)bp;
                    found = true;
                }
                cur_dir[j] = bdir;
            }
        }
        const bool layer_ok = c.any(found);
        if (!layer_ok) break;  // (:241)
        max_layer = i;
        c.sync();
        for (int j = c.tid(); j < J; j += c.nthreads()) {
            pl_x[j] = io.nx[i * J + j];
            pl_y[j] = io.ny[i * J + j];
            pl_dir[j] = cur_dir[j];
            pl_cost[j] = io.cost[i * J + j];
        }
        c.sync();
    }
    c.sync();
    // ---- phase 3: retrieve (:246-254) and walk the parents (:256, :291) - serial
    if (c.tid() == 0) {
        int jb = -1;
        double cb = DBL_MAX;
        for (int j = 0; j < J; ++j)
            if (io.cost[max_layer * J + j] < cb) {
                jb = j;
                cb = io.cost[max_layer * J + j];
            }
        int n_out = 0;
        if (jb >= 0) {
            n_out = max_layer + 1;
            int j = jb;
            for (int i = max_layer; i >= 0; --i) {
                io.chosen[i] = j;
                if (i > 0) j = io.parent[i * J + j];
            }
        }
        *io.n_out = n_out;
        shi[3] = n_out;
    }
    c.sync();
    const int n_out = shi[3];
    // ---- phase 3b: bounds of the chosen nodes (:257-290), one thread per kept layer
    for (int i = c.tid(); i < n_out; i += c.nthreads()) {
        if (i == 0) {
            io.lower[0] = -10;
            io.upper[0] = 10;
            continue;
        }
        const int j = io.chosen[i];
        // rough bounds (:214-229): the ends of the run of feasible samples around j
        int ju = j, jl = j;
        if (io.feasible[i * J + j]) {
            while (ju + 1 < J && io.feasible[i * J + ju + 1]) ++ju;
            while (jl - 1 >= 0 && io.feasible[i * J + jl - 1]) --jl;
        }
        const double check_s = 0.2, check_limit = 6.0;
        double ub = check_s + ls[ju], lb = -check_s + ls[jl];
        const double rx = io.ref[4 * i], ry = io.ref[4 * i + 1], rh = io.ref[4 * i + 2];
        const double ca = cos(rh + M_PI_2), sa = sin(rh + M_PI_2);
        while (ub < check_limit) {
            const double x = rx + ub * ca, y = ry + ub * sa;
            if (map_inside(map, x, y) && pqb::map_distance(map, x, y) > threshold) {
                ub += check_s;
            } else {
                ub -= check_s;
                break;
            }
        }
        while (lb > -check_limit) {
            const double x = rx + lb * ca, y = ry + lb * sa;
            if (map_inside(map, x, y) && pqb::map_distance(map, x, y) > threshold) {
                lb -= check_s;
            } else {
                lb += check_s;
                break;
            }
        }
        io.lower[i] = lb;
        io.upper[i] = ub;
    }
}

}  // namespace pqdp
