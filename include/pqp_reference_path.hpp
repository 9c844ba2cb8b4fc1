// pqp_reference_path.hpp — drop-in bodies for the two ReferencePathImpl methods that feed the
// solver, on top of include/pqp_bounds.h (SURVEY.md §8 rows f-1, f-2):
//
//   bool ReferencePathImpl::buildReferenceFromSpline(double delta_s_smaller, double delta_s_larger)
//        /root/reference/src/data_struct/reference_path_impl.cpp:314-338
//   void ReferencePathImpl::updateBoundsImproved(const Map &map)              ...:177-230
//
// Same outputs with the same meaning: reference_states_ (x, y, heading, k, s per state), bounds_
// (front / rear / center .ub = left, .lb = right, plus the circle's x, y, heading as
// VehicleStateBound::SingleBound::set stores them, data_struct.hpp:82-88), blocked_bound_ and the
// truncation of reference_states_ at the first blocked state. Templates over the reference's own
// State / VehicleStateBound types, so this header neither needs nor copies the reference's headers;
// the two member functions of ReferencePathImpl become one-line forwards (INTEGRATION.md §4).
// Nothing throws; errors come back as `false` with lastError(). There is no CPU path: without an
// H100 the constructor's handle creation fails and both calls return false.
#ifndef PQP_REFERENCE_PATH_HPP_
#define PQP_REFERENCE_PATH_HPP_

#include <cmath>
#include <cstddef>
#include <memory>
#include <string>
#include <vector>

#include "pqp_bounds.h"

namespace pqp {
namespace dropin {

// tk::spline's private members m_x, m_a, m_b, m_c, m_y (include/tools/spline.h:85-88), as the
// one-line accessor of INTEGRATION.md hands them out.
struct SplineRows {
    std::vector<double> x, a, b, c, y;
};

template <class StateT, class VehicleStateBoundT>
class ReferenceFrontEndT {
 public:
    // `distance`: the map's float "distance" layer, row-major rows x cols (pqp_bounds.h)
    ReferenceFrontEndT(const float *distance, int rows, int cols, double resolution, double center_x, double center_y,
                       const pqp_bounds_params *params = nullptr, int device = 0) {
        pqp_bounds_map m = {rows, cols, resolution, center_x, center_y, distance};
        const int rc = pqp_bounds_create(&m, params, device, &handle_);
        if (rc != PQP_OK) {
            const char *e = pqp_bounds_last_error(nullptr);
            error_ = e ? e : "pqp_bounds_create failed";
            handle_ = nullptr;
        }
        pqp_bounds_default_params(&params_);
        if (params) params_ = *params;
    }
    ~ReferenceFrontEndT() { pqp_bounds_destroy(handle_); }
    ReferenceFrontEndT(const ReferenceFrontEndT &) = delete;
    ReferenceFrontEndT &operator=(const ReferenceFrontEndT &) = delete;

    const std::string &lastError() const { return error_; }

    // Replace the map (ReferencePath::updateBounds(const Map &) takes one per call): a float distance layer, or an
    // occupancy image (obstacle where a pixel is <= obstacle_max; 0 = demo.cpp's zero pixels) whose exact Euclidean
    // distance transform runs on the GPU. rows * cols may not exceed the constructor's. Synchronous; false with
    // lastError() on a refused map, which leaves the current one in place.
    bool setMap(const float *distance, int rows, int cols, double resolution, double center_x, double center_y) {
        if (!handle_) return false;
        pqp_bounds_map m = {rows, cols, resolution, center_x, center_y, distance};
        return pqp_bounds_set_map(handle_, &m) == PQP_OK || fail();
    }
    bool setOccupancy(const unsigned char *cells, int rows, int cols, double resolution, double center_x,
                      double center_y, int obstacle_max = 0) {
        if (!handle_) return false;
        pqp_occupancy_map m = {rows, cols, resolution, center_x, center_y, cells, obstacle_max};
        return pqp_bounds_set_occupancy(handle_, &m) == PQP_OK || fail();
    }

    // buildReferenceFromSpline (reference_path_impl.cpp:314-338). `dynamic_segmentation` is
    // FLAGS_enable_dynamic_segmentation. Returns false for a zero-length reference (:316-319).
    bool buildReferenceFromSpline(const SplineRows &x_s, const SplineRows &y_s, double max_s, double delta_s_smaller,
                                  double delta_s_larger, bool dynamic_segmentation, std::vector<StateT> *reference_states) {
        if (!handle_ || !reference_states) return false;
        if (std::fabs(max_s) < params_.epsilon) return false;
        int k = 0;
        if (!pack(x_s, y_s, &k)) return false;
        // upper bound on the number of states: every step is at least delta_s_smaller
        const int n_max = static_cast<int>(max_s / delta_s_smaller) + 2;
        std::vector<double> states(4 * static_cast<std::size_t>(n_max)), curv(n_max);
        int32_t n = 0, total = 0;
        pqp_states_in in = {1, n_max, k, spline_.data(), &k, &max_s, delta_s_smaller, delta_s_larger,
                            dynamic_segmentation ? 1 : 0};
        pqp_states_out out = {states.data(), curv.data(), &n, &total, nullptr};
        if (pqp_bounds_build_states(handle_, &in, &out) != PQP_OK) return fail();
        reference_states->clear();
        reference_states->reserve(n);
        for (int i = 0; i < n; ++i) {
            StateT st;
            st.s = states[i];
            st.x = states[n_max + i];
            st.y = states[2 * static_cast<std::size_t>(n_max) + i];
            st.heading = states[3 * static_cast<std::size_t>(n_max) + i];
            st.k = curv[i];
            reference_states->push_back(st);
        }
        return true;
    }

    // updateBoundsImproved (reference_path_impl.cpp:177-230): fills `bounds` for the states before
    // the first blocked one, stores the blocked state's bound in `blocked_bound` and cuts
    // `reference_states` there.
    bool updateBoundsImproved(const SplineRows &x_s, const SplineRows &y_s, std::vector<StateT> *reference_states,
                              std::vector<VehicleStateBoundT> *bounds,
                              std::shared_ptr<VehicleStateBoundT> *blocked_bound) {
        if (!handle_ || !reference_states || !bounds) return false;
        if (reference_states->empty()) return false;  // "Empty reference, updateBounds fail!" (:178-181)
        int k = 0;
        if (!pack(x_s, y_s, &k)) return false;
        const int n = static_cast<int>(reference_states->size());
        std::vector<double> states(4 * static_cast<std::size_t>(n)), b(6 * static_cast<std::size_t>(n));
        for (int i = 0; i < n; ++i) {
            const StateT &st = (*reference_states)[i];
            states[i] = st.s;
            states[n + i] = st.x;
            states[2 * static_cast<std::size_t>(n) + i] = st.y;
            states[3 * static_cast<std::size_t>(n) + i] = st.heading;
        }
        int32_t n_valid = 0;
        pqp_bounds_in in = {1, n, k, states.data(), &n, spline_.data(), &k};
        pqp_bounds_out out = {b.data(), &n_valid, nullptr};
        if (pqp_bounds_compute(handle_, &in, &out) != PQP_OK) return fail();
        bounds->clear();
        const int filled = n_valid < n ? n_valid + 1 : n;  // the blocked state's bound is kept aside
        for (int i = 0; i < filled; ++i) {
            const StateT &st = (*reference_states)[i];
            VehicleStateBoundT vb;
            set(&vb.front, b[i], b[n + i], st.x + params_.front_length * std::cos(st.heading),
                st.y + params_.front_length * std::sin(st.heading), st.heading);
            set(&vb.rear, b[2 * static_cast<std::size_t>(n) + i], b[3 * static_cast<std::size_t>(n) + i],
                st.x + params_.rear_length * std::cos(st.heading), st.y + params_.rear_length * std::sin(st.heading),
                st.heading);
            set(&vb.center, b[4 * static_cast<std::size_t>(n) + i], b[5 * static_cast<std::size_t>(n) + i], st.x, st.y,
                st.heading);
            if (i == n_valid) {
                if (blocked_bound) blocked_bound->reset(new VehicleStateBoundT(vb));
            } else {
                bounds->push_back(vb);
            }
        }
        if (reference_states->size() != bounds->size()) reference_states->resize(bounds->size());
        return true;
    }

 private:
    template <class SingleBoundT>
    static void set(SingleBoundT *sb, double lb, double ub, double x, double y, double heading) {
        sb->ub = ub;
        sb->lb = lb;
        sb->x = x;
        sb->y = y;
        sb->heading = heading;
    }
    bool pack(const SplineRows &xs, const SplineRows &ys, int *k) {
        const std::size_t m = xs.x.size();
        if (m < 3 || ys.x.size() != m || xs.a.size() != m || xs.b.size() != m || xs.c.size() != m || xs.y.size() != m ||
            ys.a.size() != m || ys.b.size() != m || ys.c.size() != m || ys.y.size() != m) {
            error_ = "spline rows must hold >= 3 points and equal lengths";
            return false;
        }
        spline_.resize(9 * m);
        const std::vector<double> *rows[9] = {&xs.x, &xs.a, &xs.b, &xs.c, &xs.y, &ys.a, &ys.b, &ys.c, &ys.y};
        for (int r = 0; r < 9; ++r)
            for (std::size_t i = 0; i < m; ++i) spline_[r * m + i] = (*rows[r])[i];
        *k = static_cast<int>(m);
        return true;
    }
    bool fail() {
        const char *e = pqp_bounds_last_error(handle_);
        error_ = e ? e : "pqp_bounds call failed";
        return false;
    }

    pqp_bounds_handle *handle_ = nullptr;
    pqp_bounds_params params_;
    std::vector<double> spline_;
    std::string error_;
};

}  // namespace dropin
}  // namespace pqp
#endif
