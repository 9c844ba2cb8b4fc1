// pqp_path_optimizer.hpp — drop-in replacement for the reference's PathOptimizer on top of include/pqp_plan.h.
//
// Mirrors the reference's include/path_optimizer_2/path_optimizer.hpp:24-57 and src/path_optimizer.cpp:
//   PathOptimizer(const State &start_state, const State &end_state, const grid_map::GridMap &map)   :24-31
//   bool solve(const std::vector<State> &reference_points, std::vector<SlState> *final_path)       :33-71
//   const ReferencePath &getReferencePath() const                                                  :163-165
// The whole of solve (smoothing, processReferencePath, both solves) is one pqp_plan_points call with B = 1. Same
// bool behaviour (false unless the plan ends PQP_PLAN_OK; nothing throws), same output fields (x, y, heading, k,
// d_k, l, d_heading; s, v and a stay 0, base_solver.cpp:263-288). What final_path and the reference path hold after
// a failure follows the reference's control flow, stage by stage (the table in INTEGRATION.md §6).
//
// The class is a template over the reference's own State, SlState and VehicleStateBound, so this header neither
// needs nor copies the reference's headers; INTEGRATION.md §6 shows the binding. There is no CPU path: without an
// H100 the constructor's handle creation fails and solve returns false with that reason.
//
// The demo constructs a PathOptimizer per tick with that tick's map (demo.cpp:196). Creating a plan handle costs
// 14-58 ms, so the constructor borrows one from a process-wide pool (PlanHandlePool) and hands it the
// map; the destructor gives it back. A handle is used by one optimizer at a time.
#ifndef PQP_PATH_OPTIMIZER_HPP_
#define PQP_PATH_OPTIMIZER_HPP_

#include <cstddef>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "pqp_base_solver.hpp"
#include "pqp_plan.h"
#include "pqp_reference_path.hpp"

namespace pqp {
namespace dropin {

// What a PathOptimizerT is built with besides its states and map. The binding fills `params` from the reference's
// gflags (INTEGRATION.md §6); the capacities are those of the borrowed plan handle (pqp_plan_create).
struct PathOptimizerOptions {
    pqp_plan_params params;
    int32_t r_max = 256;      // reference points and bSpline() samples
    int32_t p_max = 256;      // resampled points of the smoother QP
    int32_t layers_max = 160; // DP layers
    int32_t n_max = 511;      // reference states (knots of the path QP)
    int device = 0;           // CUDA device ordinal
    PathOptimizerOptions() {
        std::memset(&params, 0, sizeof(params));  // the pool compares the bytes, padding included
        pqp_plan_default_params(&params);
    }
};

struct PlanHandleKey {
    pqp_plan_params params;
    int32_t r_max, p_max, layers_max, n_max;
    int device;
    size_t cells;  // map cells the handle holds: any map up to this size can be set on it
};

inline void destroyPlanHandle(pqp_plan_handle *h) { pqp_plan_destroy(h); }

// Process-wide pool of B = 1 plan handles, keyed by device, the bytes of pqp_plan_params, the four capacities and
// a map cell capacity of at least the requested map's. Idle handles are kept (at most kMaxIdle) until clear().
class PlanHandlePool : public IdlePool<PlanHandleKey, pqp_plan_handle> {
 public:
    static PlanHandlePool &instance() {
        static PlanHandlePool *pool = new PlanHandlePool;  // never destroyed: no CUDA calls during static teardown
        return *pool;
    }
    // an idle handle that can hold a map of `cells` cells, or nullptr
    pqp_plan_handle *acquire(const PathOptimizerOptions &o, size_t cells) {
        return take([&](const PlanHandleKey &k) {
            return k.device == o.device && k.r_max == o.r_max && k.p_max == o.p_max && k.layers_max == o.layers_max &&
                   k.n_max == o.n_max && k.cells >= cells && std::memcmp(&k.params, &o.params, sizeof(o.params)) == 0;
        });
    }
    // a new handle holding `map`, lent to the caller; nullptr with `error` set when the library refuses it
    pqp_plan_handle *create(const PathOptimizerOptions &o, const pqp_bounds_map &map, std::string *error) {
        pqp_plan_handle *h = nullptr;
        if (pqp_plan_create(&map, &o.params, o.r_max, o.p_max, o.layers_max, o.n_max, 1, o.device, &h) != PQP_OK) {
            if (error) *error = pqp_plan_last_error(nullptr);
            return nullptr;
        }
        PlanHandleKey key;
        std::memset(&key, 0, sizeof(key));
        key.params = o.params;
        key.r_max = o.r_max;
        key.p_max = o.p_max;
        key.layers_max = o.layers_max;
        key.n_max = o.n_max;
        key.device = o.device;
        key.cells = static_cast<size_t>(map.rows) * static_cast<size_t>(map.cols);
        return add(key, h);
    }

    // a plan handle with the default capacities and the 701 x 710 demo map takes 20 MiB of device memory
    // (bench_path_optimizer.py, DESIGN.md §7), so four idle ones hold 0.1 % of an 80 GB H100
    static constexpr size_t kMaxIdle = 4;

 private:
    PlanHandlePool() : IdlePool(kMaxIdle, destroyPlanHandle) {}
};

// PathOptimizer::getReferencePath's content (ReferencePath: x_s_ / y_s_, max_s_, reference_states_, bounds_,
// blocked_bound_), filled from the plan's trace.
template <class StateT, class VehicleStateBoundT>
struct ReferencePathViewT {
    SplineRows x_s, y_s;  // the final reference spline (tk::spline m_x, m_a, m_b, m_c, m_y)
    double length = 0.0;  // getLength()
    std::vector<StateT> reference_states;
    std::vector<VehicleStateBoundT> bounds;
    std::shared_ptr<VehicleStateBoundT> blocked;  // isBlocked()
};

template <class StateT, class SlStateT, class VehicleStateBoundT>
class PathOptimizerT {
 public:
    typedef ReferencePathViewT<StateT, VehicleStateBoundT> ReferencePathView;

    // `distance`: the map's float "distance" layer, row-major rows x cols (pqp_bounds.h, INTEGRATION.md §4)
    PathOptimizerT(const StateT &start_state, const StateT &end_state, const float *distance, int rows, int cols,
                   double resolution, double center_x, double center_y,
                   const PathOptimizerOptions &options = PathOptimizerOptions())
        : start_(start_state), end_(end_state), opt_(options) {
        const pqp_bounds_map m = {rows, cols, resolution, center_x, center_y, distance};
        handle_ = PlanHandlePool::instance().acquire(opt_, cells(rows, cols));
        if (!handle_) handle_ = PlanHandlePool::instance().create(opt_, m, &error_);  // created holding this map
        else if (pqp_plan_set_map(handle_, &m) != PQP_OK) refuse();
    }
    // `image`: an occupancy image, obstacle where a pixel is <= obstacle_max (0 = demo.cpp's zero pixels); its
    // exact Euclidean distance transform, the demo's cv::distanceTransform times the resolution, runs on the GPU
    PathOptimizerT(const StateT &start_state, const StateT &end_state, const unsigned char *image, int rows, int cols,
                   double resolution, double center_x, double center_y, int obstacle_max,
                   const PathOptimizerOptions &options = PathOptimizerOptions())
        : start_(start_state), end_(end_state), opt_(options) {
        handle_ = PlanHandlePool::instance().acquire(opt_, cells(rows, cols));
        if (!handle_) {  // a handle needs a distance layer to be created: a zero one of this size, replaced below
            const std::vector<float> zero(cells(rows, cols), 0.0f);
            const pqp_bounds_map m = {rows, cols, resolution, center_x, center_y, zero.data()};
            handle_ = PlanHandlePool::instance().create(opt_, m, &error_);
        }
        const pqp_occupancy_map occ = {rows, cols, resolution, center_x, center_y, image, obstacle_max};
        if (handle_ && pqp_plan_set_occupancy(handle_, &occ) != PQP_OK) refuse();
    }
    PathOptimizerT(const PathOptimizerT &) = delete;
    PathOptimizerT &operator=(const PathOptimizerT &) = delete;
    ~PathOptimizerT() {
        if (handle_) PlanHandlePool::instance().release(handle_);
    }

    // path_optimizer.cpp:33-71. Reads .x / .y of the points, x, y, heading, k of the start state and x, y, heading
    // of the target. final_path and the reference path after a failure: see lastStatus() and INTEGRATION.md §6.
    bool solve(const std::vector<StateT> &reference_points, std::vector<SlStateT> *final_path) {
        if (!handle_) return false;  // error_ holds the constructor's reason
        if (!final_path) {
            error_ = "final_path is null";
            return false;
        }
        if (reference_points.empty()) {  // :35-38, returns before the reference path is cleared
            status_ = PQP_PLAN_POINT_COUNT;
            error_ = "empty input";
            return false;
        }
        if (reference_points.size() > static_cast<size_t>(opt_.r_max)) {
            status_ = PQP_PLAN_POINT_COUNT;
            error_ = "more reference points than r_max = " + std::to_string(opt_.r_max);
            view_ = ReferencePathView();
            return false;
        }
        const int32_t m = static_cast<int32_t>(reference_points.size());
        const size_t L = static_cast<size_t>(opt_.layers_max), N = static_cast<size_t>(opt_.n_max);
        px_.resize(m);
        py_.resize(m);
        for (int32_t i = 0; i < m; ++i) {
            px_[i] = reference_points[i].x;
            py_[i] = reference_points[i].y;
        }
        const double start[4] = {start_.x, start_.y, start_.heading, start_.k};
        const double target[3] = {end_.x, end_.y, end_.heading};
        path_.resize(PQP_PLAN_PATH_ROWS * N);
        ref_spline_.resize(PQP_SPLINE_ROWS * L);
        states_.resize(PQP_STATE_ROWS * N);
        curvature_.resize(N);
        bounds_.resize(PQP_BOUND_ROWS * N);
        sol1_.resize(4 * N);
        pqp_plan_trace tr;
        std::memset(&tr, 0, sizeof(tr));  // only the fields below are copied back
        tr.dp_n_out = &k_;
        tr.ref_spline = ref_spline_.data();
        tr.max_s = &max_s_;
        tr.states = states_.data();
        tr.curvature = curvature_.data();
        tr.total = &total_;
        tr.bounds = bounds_.data();
        tr.n_valid = &n_valid_;
        tr.sol1 = sol1_.data();
        int32_t status = 0, n = 0, iters[2] = {0, 0};
        double cost = 0.0;
        const pqp_plan_points_in in = {1, m, px_.data(), py_.data(), &m, start, target};
        const pqp_plan_out out = {&status, &n, path_.data(), &cost, iters, &tr};
        if (pqp_plan_points(handle_, &in, &out) != PQP_OK || pqp_plan_last_stage_ms(handle_, stage_ms_) != PQP_OK) {
            error_ = pqp_plan_last_error(handle_);
            return false;
        }
        status_ = status;
        error_.clear();
        fillView();
        if (status == PQP_PLAN_OK) {
            final_path->clear();
            for (int32_t i = 0; i < n; ++i) {
                SlStateT pt;
                pt.x = path_[i];
                pt.y = path_[N + i];
                pt.heading = path_[2 * N + i];
                pt.k = path_[3 * N + i];
                pt.d_k = path_[4 * N + i];
                pt.l = path_[5 * N + i];
                pt.d_heading = path_[6 * N + i];
                final_path->push_back(pt);
            }
            return true;
        }
        error_ = std::string("plan failed: ") + statusName(status);
        if (status == PQP_PLAN_PRE_SOLVE_FAILED) {
            final_path->clear();  // optimizePath clears it before the first solve (:126)
        } else if (status == PQP_PLAN_SOLVE_FAILED) {
            // the first solve had written final_path before the re-solve failed (:142-157)
            getOptimizedPath(view_.reference_states, sol1_.data(), N, view_.reference_states.size(), final_path);
        }
        return false;
    }

    // PQP_PLAN_* of the last plan, -1 before the first
    int lastStatus() const { return status_; }
    const std::string &lastError() const { return error_; }
    // device times of the last plan, ms, indexed by PQP_PLAN_STAGE_*: the TimeRecorder stages of solve (:41-69)
    const float *lastStageMs() const { return stage_ms_; }
    const ReferencePathView &getReferencePath() const { return view_; }

    static const char *statusName(int status) {
        static const char *const names[] = {"OK", "SPLINE_DEGENERATE", "TOO_MANY_POINTS", "TENSION_FAILED",
                                            "DP_VEHICLE_FAR", "POST_TOO_SHORT", "POST_FAILED", "EMPTY_REFERENCE",
                                            "INIT_HEADING", "TOO_MANY_KNOTS", "BLOCKED_AT_START", "PRE_SOLVE_FAILED",
                                            "SOLVE_FAILED", "POINT_COUNT", "BSPLINE_DEGREE", "MAP_INDEX"};
        return status >= 0 && status < 16 ? names[status] : "unknown status";
    }

 private:
    static size_t cells(int rows, int cols) {
        return rows > 0 && cols > 0 ? static_cast<size_t>(rows) * static_cast<size_t>(cols) : 0;
    }
    void refuse() {  // a map the handle refused: give the handle back, solve reports the reason
        error_ = pqp_plan_last_error(handle_);
        PlanHandlePool::instance().release(handle_);
        handle_ = nullptr;
    }

    // The reference path as the reference leaves it after the stage the plan ended in. A smoothing failure leaves
    // it cleared (path_optimizer.cpp:44-53); processReferencePath's first two exits keep the smoothed spline and its
    // length (:100-108); after them the states and bounds are built, cut at the first blocked state.
    void fillView() {
        view_ = ReferencePathView();
        const int st = status_;
        const bool smoothed = st == PQP_PLAN_OK || (st >= PQP_PLAN_EMPTY_REFERENCE && st <= PQP_PLAN_SOLVE_FAILED);
        if (!smoothed) return;
        const size_t L = static_cast<size_t>(opt_.layers_max), N = static_cast<size_t>(opt_.n_max);
        const size_t k = static_cast<size_t>(k_);
        const double *r = ref_spline_.data();
        view_.x_s = SplineRows{{r, r + k}, {r + L, r + L + k}, {r + 2 * L, r + 2 * L + k}, {r + 3 * L, r + 3 * L + k},
                               {r + 4 * L, r + 4 * L + k}};
        view_.y_s = SplineRows{{r, r + k}, {r + 5 * L, r + 5 * L + k}, {r + 6 * L, r + 6 * L + k},
                               {r + 7 * L, r + 7 * L + k}, {r + 8 * L, r + 8 * L + k}};
        if (st == PQP_PLAN_EMPTY_REFERENCE || st == PQP_PLAN_INIT_HEADING) {
            view_.length = r[k - 1];  // the smoother's length; setReferencePathLength has not run
            return;
        }
        view_.length = max_s_;
        // more states than n_max: the plan keeps the first n_max and computes no bounds (DESIGN.md §9)
        const size_t total = static_cast<size_t>(total_) < N ? static_cast<size_t>(total_) : N;
        const size_t n_valid = st == PQP_PLAN_TOO_MANY_KNOTS ? total : static_cast<size_t>(n_valid_);
        for (size_t i = 0; i < n_valid; ++i) view_.reference_states.push_back(state(i));
        if (st == PQP_PLAN_TOO_MANY_KNOTS) return;
        // updateBoundsImproved (reference_path_impl.cpp:177-230): the blocked state's bound is kept aside
        const size_t filled = n_valid < total ? n_valid + 1 : total;
        const pqp_bounds_params &bp = opt_.params.bounds;
        for (size_t i = 0; i < filled; ++i) {
            const StateT s = i < n_valid ? view_.reference_states[i] : state(i);
            const double *b = bounds_.data();
            VehicleStateBoundT vb;
            set(&vb.front, b[i], b[N + i], s.x + bp.front_length * std::cos(s.heading),
                s.y + bp.front_length * std::sin(s.heading), s.heading);
            set(&vb.rear, b[2 * N + i], b[3 * N + i], s.x + bp.rear_length * std::cos(s.heading),
                s.y + bp.rear_length * std::sin(s.heading), s.heading);
            set(&vb.center, b[4 * N + i], b[5 * N + i], s.x, s.y, s.heading);
            if (i == n_valid) view_.blocked.reset(new VehicleStateBoundT(vb));
            else view_.bounds.push_back(vb);
        }
    }
    StateT state(size_t i) const {
        const size_t N = static_cast<size_t>(opt_.n_max);
        StateT s;
        s.s = states_[i];
        s.x = states_[N + i];
        s.y = states_[2 * N + i];
        s.heading = states_[3 * N + i];
        s.k = curvature_[i];
        return s;
    }
    template <class SingleBoundT>
    static void set(SingleBoundT *sb, double lb, double ub, double x, double y, double heading) {
        sb->ub = ub;
        sb->lb = lb;
        sb->x = x;
        sb->y = y;
        sb->heading = heading;
    }

    const StateT start_, end_;
    const PathOptimizerOptions opt_;
    pqp_plan_handle *handle_ = nullptr;
    int status_ = -1;
    std::string error_;
    float stage_ms_[PQP_PLAN_NSTAGES] = {0, 0, 0, 0};
    ReferencePathView view_;
    // host buffers of the plan call and of the trace fields the view and a failed re-solve read
    std::vector<double> px_, py_, path_, ref_spline_, states_, curvature_, bounds_, sol1_;
    int32_t k_ = 0, total_ = 0, n_valid_ = 0;
    double max_s_ = 0.0;
};

}  // namespace dropin
}  // namespace pqp
#endif  // PQP_PATH_OPTIMIZER_HPP_
