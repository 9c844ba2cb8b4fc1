// pqp_base_solver.hpp — drop-in replacement for the reference's BaseSolver on top of the C ABI.
//
// Mirrors /root/reference/include/solver/base_solver.hpp:20-71 and
// /root/reference/src/solver/base_solver.cpp:
//   BaseSolver(const ReferencePath&, const VehicleState&, const std::vector<SlState>&)   :15-39
//   virtual bool solve(std::vector<SlState>*)                                            :56-95
//   virtual bool updateProblemFormulationAndSolve(const std::vector<SlState>&,
//                                                 std::vector<SlState>*)                 :97-117
// Same constructor arguments, same argument meaning, same bool error behaviour (false unless
// the solver reports SOLVED; nothing throws), same output fields filled
// (x, y, heading, k, d_k, l, d_heading; s/v/a left at 0 — base_solver.cpp:268-285), and it is
// safe under the caller's in-place aliasing of the second call (path_optimizer.cpp:153).
//
// The class is a template over the reference's own types so this header does not need (or
// copy) the reference's headers. Inside the reference tree one line binds it:
//
//   namespace PathOptimizationNS {
//   using BaseSolver = pqp::dropin::BaseSolverT<ReferencePath, VehicleState, SlState>;
//   }
//
// (see INTEGRATION.md). The host side only packs plain arrays; assembly of P/A/l/u, the OSQP
// iteration and the warm state live on the GPU behind include/pqp.h. There is no CPU path:
// without an H100 the constructor's handle creation fails and both calls return false.
// Handles (device buffers, streams) come from a process-wide pool, so constructing a solver per
// plan - as the reference's caller does at 30 Hz - costs no allocation after the first plan.
#ifndef PQP_BASE_SOLVER_HPP_
#define PQP_BASE_SOLVER_HPP_

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "pqp.h"

namespace pqp {
namespace dropin {

// The gflags the reference's solver reads (SURVEY.md §5). Defaults = planning_flags.cpp.
struct SolverFlags {
    bool rough_constraints_far_away = false;  // planning_flags.cpp:112
    double precise_planning_length = 30.0;    // :114
    bool constraint_end_heading = true;       // :98
    int device = 0;                           // CUDA device ordinal
};

inline double constrainAngle(double angle) {  // include/tools/tools.hpp:24-35
    while (angle > M_PI) angle -= 2 * M_PI;
    while (angle < -M_PI) angle += 2 * M_PI;
    return angle;
}

// Largest problem the CUDA library holds (512 stages: 16 per lane of one warp). The
// reference itself has no cap (base_solver.cpp:15-39): at its 0.15-0.3 m knot spacing 511 knots are
// 77-153 m of path; beyond that the drop-in reports failure with an explicit error text.
constexpr size_t kMaxKnots = 511;

// Capacity a handle is created with for an n-knot plan: the largest n served by the same kernel
// instantiation (32 C - 1 knots for C = 1, 2, 4, 8, 16 stages per lane), made even so that an
// instance's knot block stays 16-byte aligned for the TMA staging copy. Plans of similar length
// therefore share a handle.
inline int32_t handleCapacity(size_t n) {
    size_t c = 1;
    while (32 * c < n + 1) c *= 2;
    const size_t cap = 32 * c - 1;
    return static_cast<int32_t>(n < cap ? cap - 1 : cap);
}

// Borrow / return bookkeeping of a process-wide pool of library handles. A handle is lent to one object at a
// time; returned handles stay idle (at most max_idle, the oldest idle one is destroyed first) until clear().
// The pool that derives from this decides which stored key fits a request and how a handle is made. Thread-safe.
template <class Key, class Handle>
class IdlePool {
 public:
    typedef void (*DestroyFn)(Handle *);
    IdlePool(size_t max_idle, DestroyFn destroy) : max_idle_(max_idle), destroy_(destroy) {}
    IdlePool(const IdlePool &) = delete;
    IdlePool &operator=(const IdlePool &) = delete;
    void release(Handle *h) {
        Handle *victim = nullptr;
        {
            std::lock_guard<std::mutex> lock(mutex_);
            size_t idle = 0;
            for (auto &e : entries_) {
                if (e.handle == h) e.busy = false;
                if (!e.busy) ++idle;
            }
            if (idle > max_idle_) {  // drop the oldest idle handle
                for (size_t i = 0; i < entries_.size(); ++i) {
                    if (!entries_[i].busy && entries_[i].handle != h) {
                        victim = entries_[i].handle;
                        entries_.erase(entries_.begin() + static_cast<std::ptrdiff_t>(i));
                        break;
                    }
                }
            }
        }
        if (victim) destroy_(victim);
    }
    // destroy every idle handle (call before cudaDeviceReset / at shutdown if desired)
    void clear() {
        std::vector<Handle *> idle;
        {
            std::lock_guard<std::mutex> lock(mutex_);
            for (size_t i = entries_.size(); i-- > 0;) {
                if (!entries_[i].busy) {
                    idle.push_back(entries_[i].handle);
                    entries_.erase(entries_.begin() + static_cast<std::ptrdiff_t>(i));
                }
            }
        }
        for (Handle *h : idle) destroy_(h);
    }
    size_t creates() const { return creates_; }
    size_t hits() const { return hits_; }

 protected:
    // lend the first idle handle whose key satisfies fits(key), or nullptr
    template <class Fits>
    Handle *take(Fits fits) {
        std::lock_guard<std::mutex> lock(mutex_);
        for (auto &e : entries_) {
            if (!e.busy && fits(e.key)) {
                e.busy = true;
                ++hits_;
                return e.handle;
            }
        }
        return nullptr;
    }
    // record a handle just created for `key`, lent to the caller
    Handle *add(const Key &key, Handle *h) {
        std::lock_guard<std::mutex> lock(mutex_);
        Entry e;
        e.key = key;
        e.handle = h;
        e.busy = true;
        entries_.push_back(e);
        ++creates_;
        return h;
    }

 private:
    struct Entry {
        Key key;
        Handle *handle;
        bool busy;
    };
    const size_t max_idle_;
    const DestroyFn destroy_;
    std::mutex mutex_;
    std::vector<Entry> entries_;
    size_t creates_ = 0, hits_ = 0;
};

struct SolverHandleKey {
    pqp_params params;
    int32_t n_max;
    int device;
};

inline void destroySolverHandle(pqp_handle *h) { pqp_destroy(h); }

// Process-wide pool of solver handles. The reference constructs a BaseSolver per plan at 30 Hz
// (path_optimizer.cpp:138); a pqp_handle owns device buffers, streams and events, so creating one
// per plan would put a few milliseconds of cudaMalloc / cudaFree (device-synchronising) around a
// 0.3 ms solve. BaseSolverT borrows a handle of matching (device, capacity, params) and gives it
// back in its destructor; idle handles are kept (at most 8) until clear(). A handle is used
// by one solver object at a time, which is the threading contract of the reference (one call at a
// time per solver); the pool itself is thread-safe.
class HandlePool : public IdlePool<SolverHandleKey, pqp_handle> {
 public:
    static HandlePool &instance() {
        static HandlePool *pool = new HandlePool;  // never destroyed: no CUDA calls during static teardown
        return *pool;
    }
    pqp_handle *acquire(const pqp_params &params, int32_t n_max, int device, std::string *error) {
        pqp_handle *h = take([&](const SolverHandleKey &k) {
            return k.n_max == n_max && k.device == device && std::memcmp(&k.params, &params, sizeof(params)) == 0;
        });
        if (h) return h;
        if (pqp_create(&params, n_max, 1, device, &h) != PQP_OK) {
            if (error) *error = pqp_last_error(nullptr);
            return nullptr;
        }
        SolverHandleKey key;
        key.params = params;
        key.n_max = n_max;
        key.device = device;
        return add(key, h);
    }

 private:
    HandlePool() : IdlePool(8, destroySolverHandle) {}
};

// BaseSolver::getOptimizedPath (base_solver.cpp:263-288): the Cartesian path of a solution sol[f * stride + i]
// (f = 0: l, 1: psi, 2: kappa, 3: d_k) over the first n reference states; s, v and a stay 0.
template <class StateT, class SlStateT>
void getOptimizedPath(const std::vector<StateT> &ref_states, const double *sol, size_t stride, size_t n,
                      std::vector<SlStateT> *optimized_path) {
    optimized_path->clear();
    for (size_t i = 0; i != n; ++i) {
        SlStateT pt;
        const double angle = ref_states[i].heading;
        const double l = sol[i], psi = sol[stride + i];
        pt.heading = constrainAngle(angle + psi);
        pt.d_heading = psi;
        pt.l = l;
        const double new_angle = constrainAngle(angle + M_PI_2);
        pt.x = ref_states[i].x + l * std::cos(new_angle);
        pt.y = ref_states[i].y + l * std::sin(new_angle);
        pt.k = sol[2 * stride + i];
        if (i < n - 1) pt.d_k = sol[3 * stride + i];
        optimized_path->push_back(pt);
    }
}

template <class ReferencePathT, class VehicleStateT, class SlStateT>
class BaseSolverT {
 public:
    BaseSolverT() = delete;
    BaseSolverT(const ReferencePathT &reference_path, const VehicleStateT &vehicle_state,
                const std::vector<SlStateT> &input_path, const SolverFlags &flags = SolverFlags(),
                const pqp_params *params = nullptr)
        : n_(input_path.size()),
          reference_path_(reference_path),
          vehicle_state_(vehicle_state),
          input_path_(input_path),
          flags_(flags) {
        // base_solver.cpp:22-37
        precise_planning_size_ = n_;
        if (flags_.rough_constraints_far_away) {
            auto it = std::lower_bound(input_path.begin(), input_path.end(), flags_.precise_planning_length,
                                       [](const SlStateT &state, double s) { return state.s < s; });
            precise_planning_size_ = static_cast<size_t>(std::distance(input_path.begin(), it));
        }
        if (params) params_ = *params;
        else pqp_default_params(&params_);
        if (n_ >= 2 && n_ <= kMaxKnots) {
            n_max_ = handleCapacity(n_);
            handle_ = HandlePool::instance().acquire(params_, n_max_, flags_.device, &error_);
        } else {
            // the reference underflows for n < 2 (:23) and has no upper limit; see kMaxKnots
            error_ = "number of knots must be in [2, 511]";
        }
    }
    BaseSolverT(const BaseSolverT &) = delete;
    BaseSolverT &operator=(const BaseSolverT &) = delete;
    virtual ~BaseSolverT() {
        if (handle_) HandlePool::instance().release(handle_);
    }

    // base_solver.cpp:56-95
    virtual bool solve(std::vector<SlStateT> *optimized_path) {
        if (!handle_ || !optimized_path) return false;
        pack(input_path_);
        return run(false, optimized_path);
    }

    // base_solver.cpp:97-117. input_path and *optimized_path may be the same vector.
    virtual bool updateProblemFormulationAndSolve(const std::vector<SlStateT> &input_path,
                                                  std::vector<SlStateT> *optimized_path) {
        if (!handle_ || !optimized_path || input_path.size() != n_) return false;
        input_path_ = input_path;  // copy first: the output may alias the input (:100 vs :266)
        pack(input_path_);
        return run(true, optimized_path);
    }

    int lastStatus() const { return status_; }
    int lastIterations() const { return iters_; }
    double lastCost() const { return cost_; }
    const std::string &lastError() const { return error_; }
    // device times of the last call, ms, indexed by PQP_STAGE_* (pqp.h): what the reference's
    // TimeRecorder prints for its solve stages (base_solver.cpp:57-93)
    const float *lastStageMs() const { return stage_ms_; }

 private:
    // flat POD pack of everything setConstraints reads (base_solver.cpp:150-261)
    void pack(const std::vector<SlStateT> &lin) {
        const auto &ref_states = reference_path_.getReferenceStates();
        const auto &bounds = reference_path_.getBounds();
        const size_t n = n_, p = precise_planning_size_, st = static_cast<size_t>(n_max_);  // field stride
        knots_.assign(PQP_NFIELDS * st, 0.0);
        for (size_t i = 0; i < n; ++i) {
            knots_[PQP_F_S * st + i] = ref_states[i].s;
            knots_[PQP_F_KREF * st + i] = ref_states[i].k;
            knots_[PQP_F_L * st + i] = lin[i].l;
            knots_[PQP_F_PSI * st + i] = lin[i].d_heading;
            knots_[PQP_F_K * st + i] = lin[i].k;
            if (i < p) {
                knots_[PQP_F_B0_LB * st + i] = bounds[i].front.lb;
                knots_[PQP_F_B0_UB * st + i] = bounds[i].front.ub;
                knots_[PQP_F_B1_LB * st + i] = bounds[i].rear.lb;
                knots_[PQP_F_B1_UB * st + i] = bounds[i].rear.ub;
            } else {
                knots_[PQP_F_B0_LB * st + i] = bounds[i].center.lb;
                knots_[PQP_F_B0_UB * st + i] = bounds[i].center.ub;
            }
        }
        const auto init_error = vehicle_state_.getInitError();
        inst_[PQP_I_L0] = init_error[0];
        inst_[PQP_I_PSI0] = init_error[1];
        inst_[PQP_I_K0] = vehicle_state_.getStartState().k;
        inst_[PQP_I_EPSI_LO] = -1e30;  // OsqpEigen::INFTY (:252-253)
        inst_[PQP_I_EPSI_HI] = 1e30;
        if (flags_.constraint_end_heading && reference_path_.isBlocked() == nullptr) {
            const double end_psi = constrainAngle(vehicle_state_.getTargetState().heading - ref_states.back().heading);
            if (end_psi < 70 * M_PI / 180) {  // signed test, as in the reference (:256)
                inst_[PQP_I_EPSI_LO] = end_psi - 0.087;
                inst_[PQP_I_EPSI_HI] = end_psi + 0.087;
            }
        }
    }

    bool run(bool warm, std::vector<SlStateT> *optimized_path) {
        const int32_t n = static_cast<int32_t>(n_), p = static_cast<int32_t>(precise_planning_size_);
        sol_.assign(4 * static_cast<size_t>(n_max_), 0.0);
        pqp_batch_in in;
        in.batch = 1;
        in.n_max = n_max_;
        in.knots = knots_.data();
        in.inst = inst_;
        in.n = &n;
        in.p = &p;
        pqp_batch_out out = {};
        out.sol = sol_.data();
        out.cost = &cost_;
        out.status = &status_;
        out.iters = &iters_;
        const int rc = warm ? pqp_resolve(handle_, &in, &out) : pqp_solve(handle_, &in, &out);
        if (rc != PQP_OK) {
            error_ = pqp_last_error(handle_);
            return false;
        }
        pqp_last_stage_ms(handle_, stage_ms_);
        if (status_ != PQP_SOLVED) return false;  // osqp-eigen: solve() fails unless OSQP_SOLVED
        getOptimizedPath(reference_path_.getReferenceStates(), sol_.data(), static_cast<size_t>(n_max_), n_,
                         optimized_path);
        return true;
    }

    // base_solver.cpp:263-288
    void get_optimized_path(std::vector<SlStateT> *optimized_path) const {
        optimized_path->clear();
        const auto &ref_states = reference_path_.getReferenceStates();
        const size_t n = n_, st = static_cast<size_t>(n_max_);
        for (size_t i = 0; i != n; ++i) {
            SlStateT pt;
            const double angle = ref_states[i].heading;
            const double l = sol_[i], psi = sol_[st + i];
            pt.heading = constrainAngle(angle + psi);
            pt.d_heading = psi;
            pt.l = l;
            const double new_angle = constrainAngle(angle + M_PI_2);
            pt.x = ref_states[i].x + l * std::cos(new_angle);
            pt.y = ref_states[i].y + l * std::sin(new_angle);
            pt.k = sol_[2 * st + i];
            if (i < n - 1) pt.d_k = sol_[3 * st + i];
            optimized_path->push_back(pt);
        }
    }

 protected:
    const size_t n_;
    size_t precise_planning_size_{};
    const ReferencePathT &reference_path_;
    const VehicleStateT &vehicle_state_;
    std::vector<SlStateT> input_path_;
    SolverFlags flags_;
    pqp_params params_{};
    pqp_handle *handle_ = nullptr;
    int32_t n_max_ = 0;  // capacity of the borrowed handle = field stride of knots_ / sol_
    float stage_ms_[PQP_NSTAGES] = {0, 0, 0, 0, 0};
    std::vector<double> knots_, sol_;
    double inst_[PQP_NINST] = {0, 0, 0, 0, 0};
    double cost_ = 0.0;
    int32_t status_ = PQP_UNSOLVED, iters_ = 0;
    std::string error_;
};

}  // namespace dropin
}  // namespace pqp
#endif  // PQP_BASE_SOLVER_HPP_
