// pqp_plan.cu — include/pqp_plan.h: PathOptimizer::solve for a batch, device-resident on one stream.
// The stage kernels are the existing ones, called through their C ABIs; the glue kernels here run the per-path code
// of pqp_plan_core.cuh (shared with the CPU test driver). Built with --fmad=false: the glue is threshold and argmin
// decisions (the 1 m projection grid, the 75 and 70 degree tests, the resampling loop counts) and spline fits whose
// rows must equal the host restatement's bit for bit, so every operation rounds separately as in the host code.
//
// Masking: a path that has failed keeps status != OK and every later stage still receives well-formed input for it:
// the smoother QPs and the solver skip it by their size fields (p = 0, n = 0), and the DP, which reads the spline
// unconditionally, gets a three-point placeholder line.
#include <cuda_runtime.h>

#include <new>
#include <optional>
#include <string>

#include "../../include/pqp_plan.h"
#include "pqp_bounds_internal.h"
#include "pqp_host_handle.h"
#include "pqp_plan_core.cuh"
#include "pqp_plan_trace.h"
#include "pqp_smoother_internal.h"

namespace {

thread_local std::string g_plan_create_error;
constexpr int kThreads = 128;

// Launches of the stage handles' entry points per plan call that their own ABIs do not count: tension QP, DP,
// post QP, reference states, bounds (n_valid initialisation + clearance kernel).
constexpr int kStageLaunches = 6;

inline unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

struct Dims {
    int B, R, P, L, N, in_r;
};

// per-path maps of a mapped plan call: path b reads table[map_index[b]]; map_index NULL: the shared map
struct Slots {
    const pqb::MapView *table;
    const int32_t *map_index;
    int n_maps;
};

// a mapped call's bad index is the path's status whatever else is wrong with it
__device__ int map_index_status(const Slots &m, int b, int st) {
    return m.map_index && !pqb::slot_view(m.table, m.n_maps, m.map_index, b) ? pqpl::kMapIndex : st;
}

// bSpline() up to its sample parameters (pqp_plan_points), one thread per path: the point-count and degree checks,
// the control polygon's length and degree, and the t accumulation into the path's row of t_all (at most R values)
__global__ void bspline_prep_kernel(Dims d, Slots slots, int m_max, const double *__restrict__ px,
                                    const double *__restrict__ py, const int32_t *__restrict__ m, double *t_all,
                                    int32_t *raw_r, int32_t *degree, int32_t *status) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    int r = 0, deg = 0, st = map_index_status(slots, b, pqpl::kOk);
    if (st == pqpl::kOk)
        st = pqpl::bspline_prepare(px + (size_t)b * m_max, py + (size_t)b * m_max, m[b], m_max, d.R,
                                   t_all + (size_t)b * d.R, r, deg);
    status[b] = st;
    raw_r[b] = r;
    degree[b] = deg;
}

// bSpline()'s samples (pqp_plan_points): de Boor at each parameter, one thread per (path, sample), into the [B][R]
// rows the raw prep reads
__global__ void bspline_eval_kernel(Dims d, int m_max, const double *__restrict__ px, const double *__restrict__ py,
                                    const int32_t *__restrict__ m, const double *__restrict__ t_all,
                                    const int32_t *__restrict__ raw_r, const int32_t *__restrict__ degree,
                                    const int32_t *__restrict__ status, double *out_x, double *out_y) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)d.B * d.R) return;
    const int b = (int)(t / d.R), j = (int)(t % d.R);
    if (status[b] != pqpl::kOk || j >= raw_r[b]) return;
    const size_t o = (size_t)b * d.R + j;
    double x, y;
    pqpl::bspline_eval(px + (size_t)b * m_max, py + (size_t)b * m_max, m[b], degree[b], t_all[o], x, y);
    out_x[o] = x;
    out_y[o] = y;
}

// raw samples -> s_list_ (chord length) into the raw spline rows, sample count of segmentRawReference. `prior`
// (pqp_plan_points: the B-spline stage's status, possibly `status` itself) keeps an earlier failure; NULL under pqp_plan.
// (pqp_plan_mapped: the map index is checked here, or by bspline_prep_kernel under pqp_plan_points_mapped)
__global__ void raw_prep_kernel(Dims d, Slots slots, const double *__restrict__ raw_x, const double *__restrict__ raw_y,
                                const int32_t *__restrict__ r, const double *__restrict__ start, const int32_t *prior,
                                double *raw_rows, int32_t *raw_k, int32_t *seg_p, int32_t *status, double *start3) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    start3[3 * b] = start[4 * b];
    start3[3 * b + 1] = start[4 * b + 1];
    start3[3 * b + 2] = start[4 * b + 2];
    double *rows = raw_rows + (size_t)b * pqpl::kSplineRows * d.R;
    double *sx = rows, *x = rows + 4 * (size_t)d.R, *y = rows + 8 * (size_t)d.R;
    int st = prior ? prior[b] : map_index_status(slots, b, pqpl::kOk), p = 0;
    const int rb = st == pqpl::kOk ? r[b] : 0;  // a path that failed before its samples has none to read
    if (st == pqpl::kOk && (rb < 3 || rb > d.R)) {
        st = pqpl::kSplineDegenerate;
    } else if (st == pqpl::kOk) {
        for (int i = 0; i < rb; ++i) {
            x[i] = raw_x[(size_t)b * d.in_r + i];
            y[i] = raw_y[(size_t)b * d.in_r + i];
        }
        pqpl::chord_length(x, y, rb, sx);
        if (!pqpl::increasing(sx, rb)) {
            st = pqpl::kSplineDegenerate;
        } else {
            p = pqpl::segment_count(sx[rb - 1], d.P);
            if (p > d.P) st = pqpl::kTooManyPoints;
        }
    }
    status[b] = st;
    raw_k[b] = st == pqpl::kOk ? rb : 0;
    seg_p[b] = st == pqpl::kOk ? p : 0;  // the tension kernel skips p < 3
}

// one thread per (path, coordinate): natural spline fit of rows 4 (x) or 8 (y) over row 0; k < 3 is skipped
__global__ void fit_kernel(int B, int stride, double *rows_all, const int32_t *__restrict__ k) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * B) return;
    const int b = t >> 1, coord = t & 1;
    const int kb = k[b];
    if (kb < 3 || kb > stride) return;
    double *rows = rows_all + (size_t)b * pqpl::kSplineRows * stride;
    double *base = rows + (size_t)(1 + 4 * coord) * stride;  // a, b, c, y of this coordinate
    pqpl::natural_spline_fit(rows, base + 3 * (size_t)stride, kb, base, base + stride, base + 2 * (size_t)stride);
}

// one thread per (path, output sample) of segmentRawReference
__global__ void segment_kernel(Dims d, const double *__restrict__ raw_rows, const int32_t *__restrict__ raw_k,
                               const int32_t *__restrict__ seg_p, double *sx_, double *sy_, double *sa_, double *sk_,
                               double *ss_) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)d.B * d.P) return;
    const int b = (int)(t / d.P), j = (int)(t % d.P);
    if (j >= seg_p[b]) return;
    const pqb::SplineView sp = pqpl::view(raw_rows + (size_t)b * pqpl::kSplineRows * d.R, d.R, raw_k[b]);
    const double s = pqpl::segment_s(j);
    double x, y, a, k;
    pqpl::segment_sample(sp, s, x, y, a, k);
    const size_t o = (size_t)b * d.P + j;
    sx_[o] = x;
    sy_[o] = y;
    sa_[o] = a;
    sk_[o] = k;
    ss_[o] = s;
}

// TENSION only: Map::getObstacleDistance at each resampled point (tension_smoother.cpp:166-168), the clearance of the
// Cartesian tension QP; one thread per (path, point), paths without points (seg_p = 0) skipped
__global__ void clearance_kernel(Dims d, const pqb::MapView map, Slots slots, const int32_t *__restrict__ seg_p,
                                 const double *__restrict__ sx_, const double *__restrict__ sy_, double *clearance) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)d.B * d.P) return;
    const int b = (int)(t / d.P), j = (int)(t % d.P);
    if (j >= seg_p[b]) return;
    const size_t o = (size_t)b * d.P + j;
    if (slots.map_index) {
        const pqb::MapView *m = pqb::slot_view(slots.table, slots.n_maps, slots.map_index, b);
        if (m) clearance[o] = pqb::map_distance(*m, sx_[o], sy_[o]);
    } else {
        clearance[o] = pqb::map_distance(map, sx_[o], sy_[o]);
    }
}

__device__ void write_placeholder(double *rows, int stride, int32_t *k, double *length) {
    pqpl::placeholder_points(rows, rows + 4 * (size_t)stride, rows + 8 * (size_t)stride);
    *k = pqpl::kPlaceholderK;
    *length = pqpl::kPlaceholderLength;
}

// TensionSmoother::smooth after the QP (tension_smoother.cpp:32-41): the result points become the spline rows,
// length = result_s.back() + 3
__global__ void tension_epilogue_kernel(Dims d, const int32_t *__restrict__ seg_p, const double *__restrict__ tx,
                                        const double *__restrict__ ty, const double *__restrict__ ts,
                                        const int32_t *__restrict__ tstatus, int32_t *status, double *rows_all,
                                        int32_t *tk, double *tlen) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    double *rows = rows_all + (size_t)b * pqpl::kSplineRows * d.P;
    int st = status[b];
    if (st == pqpl::kOk && tstatus[b] != PQP_SOLVED) st = pqpl::kTensionFailed;
    const int p = seg_p[b];
    if (st == pqpl::kOk) {
        const size_t o = (size_t)b * d.P;
        for (int i = 0; i < p; ++i) {
            rows[i] = ts[o + i];
            rows[4 * (size_t)d.P + i] = tx[o + i];
            rows[8 * (size_t)d.P + i] = ty[o + i];
        }
        if (!pqpl::increasing(rows, p)) st = pqpl::kSplineDegenerate;
    }
    status[b] = st;
    if (st == pqpl::kOk) {
        tk[b] = p;
        tlen[b] = rows[p - 1] + 3.0;
    } else {
        write_placeholder(rows, d.P, tk + b, tlen + b);
    }
}

// graphSearchDp's outcome -> status, and postSmooth's size test (reference_path_smoother.cpp:527-531)
__global__ void post_prep_kernel(int B, const int32_t *__restrict__ dp_status, const int32_t *__restrict__ n_out,
                                 int32_t *status, int32_t *post_p) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int st = status[b];
    if (st == pqpl::kOk) {
        if (dp_status[b] == PQP_DP_VEHICLE_FAR) st = pqpl::kDpVehicleFar;
        else if (dp_status[b] != PQP_DP_OK) st = pqpl::kTooManyPoints;
        else if (n_out[b] < 4) st = pqpl::kPostTooShort;
    }
    status[b] = st;
    post_p[b] = st == pqpl::kOk ? n_out[b] : 0;  // the post kernel skips p < 2
}

// postSmooth after the QP (:560-577): points, arc length, the new reference spline, length = s.back()
__global__ void post_epilogue_kernel(Dims d, const double *__restrict__ t_rows, const int32_t *__restrict__ tk,
                                     const double *__restrict__ layer_s, const double *__restrict__ offsets,
                                     const int32_t *__restrict__ post_p, const int32_t *__restrict__ pstatus,
                                     int32_t *status, double *rows_all, int32_t *rk, double *rlen) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    double *rows = rows_all + (size_t)b * pqpl::kSplineRows * d.L;
    int st = status[b];
    if (st == pqpl::kOk && pstatus[b] != PQP_SOLVED) st = pqpl::kPostFailed;
    const int n = post_p[b];
    if (st == pqpl::kOk) {
        const pqb::SplineView sp = pqpl::view(t_rows + (size_t)b * pqpl::kSplineRows * d.P, d.P, tk[b]);
        pqpl::post_points(sp, layer_s + (size_t)b * d.L, offsets + (size_t)b * d.L, n, rows, rows + 4 * (size_t)d.L,
                          rows + 8 * (size_t)d.L);
        if (!pqpl::increasing(rows, n)) st = pqpl::kSplineDegenerate;
    }
    status[b] = st;
    if (st == pqpl::kOk) {
        rk[b] = n;
        rlen[b] = rows[n - 1];
    } else {
        write_placeholder(rows, d.L, rk + b, rlen + b);
    }
}

// processReferencePath up to buildReferenceFromSpline; failed paths get max_s < 0 (no states)
__global__ void process_kernel(Dims d, double epsilon, const double *__restrict__ r_rows, const int32_t *__restrict__ rk,
                               const double *__restrict__ rlen, const double *__restrict__ start,
                               const double *__restrict__ target, int32_t *status, double *max_s, double *inst) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    int st = status[b];
    double l0 = 0.0, psi0 = 0.0, ms = -1.0;
    if (st == pqpl::kOk) {
        const pqb::SplineView sp = pqpl::view(r_rows + (size_t)b * pqpl::kSplineRows * d.L, d.L, rk[b]);
        st = pqpl::process_reference(sp, rlen[b], start + 4 * b, target + 3 * b, epsilon, l0, psi0, ms);
        if (st != pqpl::kOk) ms = -1.0;
    }
    status[b] = st;
    max_s[b] = ms;
    inst[b * PQP_NINST + PQP_I_L0] = l0;
    inst[b * PQP_NINST + PQP_I_PSI0] = psi0;
}

// states beyond n_max are reported, not truncated; failed paths get no states for the bounds kernel
__global__ void states_check_kernel(int B, int N, const int32_t *__restrict__ total, int32_t *status, int32_t *n_states) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int st = status[b];
    if (st == pqpl::kOk && total[b] > N) st = pqpl::kTooManyKnots;
    status[b] = st;
    if (st != pqpl::kOk) n_states[b] = 0;
}

struct InstArgs {
    int B, N, rough, constrain_end;
    double precise_length;
    const double *states, *bounds, *start, *target;
    const int32_t *n_states, *n_valid;
    int32_t *status, *n1, *p;
    double *knots, *inst, *ref_xyh;
};

// BaseSolver's per-instance block (base_solver.cpp:25-34, 216-259) on the states cut at n_valid
__global__ void inst_kernel(const InstArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    int st = a.status[b];
    const int nv = a.n_valid[b];
    if (st == pqpl::kOk && nv < 2) st = pqpl::kBlockedAtStart;
    a.status[b] = st;
    const int N = a.N;
    const double *sts = a.states + (size_t)b * PQP_STATE_ROWS * N;
    double *in = a.inst + (size_t)b * PQP_NINST;
    in[PQP_I_K0] = a.start[4 * b + 3];
    double lo = -1e30, hi = 1e30;
    int p = 0;
    if (st == pqpl::kOk) {
        p = pqpl::precise_size(sts, nv, a.rough != 0, a.precise_length);
        pqpl::end_heading_rows(a.constrain_end != 0, nv < a.n_states[b], a.target[3 * b + 2], sts[3 * N + nv - 1], lo, hi);
        // rough knots (i >= p) take the centre bounds in the first clearance row (base_solver.cpp:242-246)
        double *kb = a.knots + (size_t)b * PQP_NFIELDS * N;
        const double *bd = a.bounds + (size_t)b * PQP_BOUND_ROWS * N;
        for (int i = p; i < nv; ++i) {
            kb[(size_t)PQP_F_B0_LB * N + i] = bd[4 * (size_t)N + i];
            kb[(size_t)PQP_F_B0_UB * N + i] = bd[5 * (size_t)N + i];
        }
        double *rx = a.ref_xyh + (size_t)b * 3 * N;
        for (int i = 0; i < nv; ++i) {
            rx[i] = sts[N + i];
            rx[N + i] = sts[2 * (size_t)N + i];
            rx[2 * (size_t)N + i] = sts[3 * (size_t)N + i];
        }
    }
    in[PQP_I_EPSI_LO] = lo;
    in[PQP_I_EPSI_HI] = hi;
    a.p[b] = p;
    a.n1[b] = st == pqpl::kOk ? nv : 0;  // the solver skips n outside [2, n_max]
}

__global__ void between_kernel(int B, const int32_t *__restrict__ status1, const int32_t *__restrict__ n1, int32_t *status,
                               int32_t *n2) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int st = status[b];
    if (st == pqpl::kOk && status1[b] != PQP_SOLVED) st = pqpl::kPreSolveFailed;
    status[b] = st;
    n2[b] = st == pqpl::kOk ? n1[b] : 0;
}

struct FinalArgs {
    int B, N;
    const int32_t *status, *status2, *n2, *iters1, *iters2;
    const double *sol2, *xyh, *cost2;
    int32_t *out_status, *out_n, *out_iters;
    double *out_path, *out_cost;
};

// getOptimizedPath's rows (base_solver.cpp:263-288) and the per-path outputs; one thread per (path, knot)
__global__ void final_kernel(const FinalArgs a) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)a.B * a.N) return;
    const int b = (int)(t / a.N), i = (int)(t % a.N);
    int st = a.status[b];
    if (st == pqpl::kOk && a.status2[b] != PQP_SOLVED) st = pqpl::kSolveFailed;
    const int n = st == pqpl::kOk ? a.n2[b] : 0;
    const int N = a.N;
    double *row = a.out_path + (size_t)b * PQP_PLAN_PATH_ROWS * N;
    const double *sol = a.sol2 + (size_t)b * 4 * N;
    const double *xyh = a.xyh + (size_t)b * 3 * N;
    const bool on = i < n;
    row[i] = on ? xyh[i] : 0.0;
    row[N + i] = on ? xyh[N + i] : 0.0;
    row[2 * (size_t)N + i] = on ? xyh[2 * (size_t)N + i] : 0.0;
    row[3 * (size_t)N + i] = on ? sol[2 * (size_t)N + i] : 0.0;
    row[4 * (size_t)N + i] = (on && i < n - 1) ? sol[3 * (size_t)N + i] : 0.0;
    row[5 * (size_t)N + i] = on ? sol[i] : 0.0;
    row[6 * (size_t)N + i] = on ? sol[N + i] : 0.0;
    if (i == 0) {
        a.out_status[b] = st;
        a.out_n[b] = n;
        a.out_cost[b] = st == pqpl::kOk ? a.cost2[b] : 0.0;
        a.out_iters[2 * b] = a.iters1[b];
        a.out_iters[2 * b + 1] = a.iters2[b];
    }
}

}  // namespace

struct pqp_plan_handle {
    int device = 0, R = 0, P = 0, L = 0, N = 0, batch_max = 0;
    pqp_plan_params prm{};
    pqp_bounds_handle *bounds = nullptr;
    pqp_dp_handle *dp = nullptr;
    pqp_smoother_handle *tension = nullptr, *post = nullptr;  // p_max = P, resp. L (the DP's layer stride)
    pqp_handle *solver = nullptr;
    cudaStream_t stream = nullptr;  // of the host-pointer call
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool timed = false;
    long long launches = 0;
    // inputs of the host-pointer call
    double *in_x = nullptr, *in_y = nullptr, *in_start = nullptr, *in_target = nullptr;
    int32_t *in_r = nullptr;
    // outputs of the host-pointer call
    int32_t *o_status = nullptr, *o_n = nullptr, *o_iters = nullptr;
    double *o_path = nullptr, *o_cost = nullptr;
    // stages
    int32_t *status = nullptr, *raw_k = nullptr, *seg_p = nullptr, *t_status = nullptr, *t_iters = nullptr, *tk = nullptr;
    double *start3 = nullptr, *raw_rows = nullptr, *seg[5] = {}, *t_x = nullptr, *t_y = nullptr, *t_s = nullptr,
           *t_rows = nullptr, *t_len = nullptr;
    int32_t *dp_status = nullptr, *dp_nl = nullptr, *dp_nout = nullptr, *dp_chosen = nullptr;
    double *dp_ls = nullptr, *dp_lo = nullptr, *dp_up = nullptr, *dp_vl = nullptr, *dp_ts = nullptr;
    int32_t *post_p = nullptr, *post_status = nullptr, *post_iters = nullptr, *rk = nullptr;
    double *post_off = nullptr, *r_rows = nullptr, *r_len = nullptr, *max_s = nullptr;
    double *t_clear = nullptr;  // [B][P] clearance of the Cartesian tension QP (TENSION only)
    // pqp_plan_points: the host call's staged points, the sample parameters, samples and degree per path (the samples
    // themselves go to in_x / in_y)
    double *pt_x = nullptr, *pt_y = nullptr, *bs_t = nullptr;
    int32_t *pt_m = nullptr, *raw_r = nullptr, *bs_deg = nullptr;
    int32_t *in_map_index = nullptr;  // [B] the host mapped calls' slot per path
    double *states = nullptr, *curv = nullptr, *bnd = nullptr, *knots = nullptr, *knots2 = nullptr, *inst = nullptr,
           *ref_xyh = nullptr, *xyh = nullptr;
    int32_t *n_states = nullptr, *total = nullptr, *n_valid = nullptr, *n1 = nullptr, *n2 = nullptr, *p = nullptr;
    double *sol1 = nullptr, *sol2 = nullptr, *cost1 = nullptr, *cost2 = nullptr;
    double *full[6] = {};  // x, y, z of the first solve, then of the second: written only when traced
    int32_t *status1 = nullptr, *iters1 = nullptr, *status2 = nullptr, *iters2 = nullptr;
    std::string err;
    pqp::Resources res;  // last member: releasing clears the members above
};

namespace {

using pqp::fail;

#define PQL_SUB(h, call, errfn, sub)                                                              \
    do {                                                                                          \
        const int rc_ = (call);                                                                   \
        if (rc_ != PQP_OK) return fail((h)->err, rc_, std::string(#call) + ": " + errfn(sub));   \
    } while (0)

// a stage handle's create inside pqp_plan_create: its error is the plan's create error
#define PQL_SUB_CREATE(call, errfn)                                                                \
    do {                                                                                           \
        const int rc_ = (call);                                                                    \
        if (rc_ != PQP_OK) return fail(g_plan_create_error, rc_, std::string("pqp_plan_create: ") + errfn(nullptr)); \
    } while (0)

#define PQL_LAUNCH(h)                              \
    do {                                           \
        PQP_CUDA((h)->err, cudaGetLastError());    \
        (h)->launches++;                           \
    } while (0)

int validate(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out) return fail(h->err, PQP_E_INVALID, "null batch");
    if (!in->raw_x || !in->raw_y || !in->r || !in->start || !in->target) return fail(h->err, PQP_E_INVALID, "null input buffer");
    if (!out->status || !out->n || !out->path || !out->cost || !out->iters) return fail(h->err, PQP_E_INVALID, "null output buffer");
    if (in->batch < 1 || in->batch > h->batch_max) return fail(h->err, PQP_E_INVALID, "batch out of range");
    if (in->r_max < 3 || in->r_max > h->R) return fail(h->err, PQP_E_INVALID, "r_max must be in [3, the handle's r_max]");
    return PQP_OK;
}

int validate_points(pqp_plan_handle *h, const pqp_plan_points_in *in, const pqp_plan_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out) return fail(h->err, PQP_E_INVALID, "null batch");
    if (!in->ref_x || !in->ref_y || !in->m || !in->start || !in->target) return fail(h->err, PQP_E_INVALID, "null input buffer");
    if (!out->status || !out->n || !out->path || !out->cost || !out->iters) return fail(h->err, PQP_E_INVALID, "null output buffer");
    if (in->batch < 1 || in->batch > h->batch_max) return fail(h->err, PQP_E_INVALID, "batch out of range");
    if (in->m_max < 1 || in->m_max > h->R) return fail(h->err, PQP_E_INVALID, "m_max must be in [1, the handle's r_max]");
    return PQP_OK;
}

int copy_out(pqp_plan_handle *h, void *dst, const void *src, size_t bytes, cudaStream_t s) {
    if (dst) PQP_CUDA(h->err, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s));
    return PQP_OK;
}

int copy_trace(pqp_plan_handle *h, const pqp_plan_trace *t, int B, bool points, cudaStream_t s) {
    if (!t) return PQP_OK;
    // the handle's buffer behind each trace member; NULL where the call has none (tension_clearance under TENSION2,
    // the B-spline fields outside pqp_plan_points)
    pqp_plan_trace src{};
    src.raw_spline = h->raw_rows;
    src.seg_p = h->seg_p;
    src.seg_x = h->seg[0];
    src.seg_y = h->seg[1];
    src.seg_angle = h->seg[2];
    src.seg_k = h->seg[3];
    src.seg_s = h->seg[4];
    src.tension_x = h->t_x;
    src.tension_y = h->t_y;
    src.tension_s = h->t_s;
    src.tension_status = h->t_status;
    src.tension_iters = h->t_iters;
    src.tension_spline = h->t_rows;
    src.tension_length = h->t_len;
    src.dp_status = h->dp_status;
    src.dp_n_out = h->dp_nout;
    src.dp_layer_s = h->dp_ls;
    src.dp_lower = h->dp_lo;
    src.dp_upper = h->dp_up;
    src.dp_chosen = h->dp_chosen;
    src.dp_vehicle_l = h->dp_vl;
    src.post_offsets = h->post_off;
    src.post_status = h->post_status;
    src.post_iters = h->post_iters;
    src.ref_spline = h->r_rows;
    src.max_s = h->max_s;
    src.states = h->states;
    src.curvature = h->curv;
    src.total = h->total;
    src.bounds = h->bnd;
    src.n_valid = h->n_valid;
    src.knots = h->knots;
    src.inst = h->inst;
    src.p = h->p;
    src.sol1 = h->sol1;
    src.status1 = h->status1;
    src.iters1 = h->iters1;
    src.x_full1 = h->full[0];
    src.y_full1 = h->full[1];
    src.z_full1 = h->full[2];
    src.x_full2 = h->full[3];
    src.y_full2 = h->full[4];
    src.z_full2 = h->full[5];
    src.tension_clearance = h->t_clear;
    src.raw_r = points ? h->raw_r : nullptr;
    src.bspline_degree = points ? h->bs_deg : nullptr;
    for (const pqpl::TraceField &f : pqpl::trace_fields(h->P, h->L, h->N, h->R)) {
        const void *from = pqpl::trace_get(src, f);
        if (!from) continue;
        const int rc = copy_out(h, pqpl::trace_get(*t, f), from, (size_t)B * f.per_path, s);
        if (rc != PQP_OK) return rc;
    }
    return PQP_OK;
}

// the host calls' outputs from the handle's staging buffers; waits for the call to finish
int copy_results(pqp_plan_handle *h, const pqp_plan_out *out, int batch, cudaStream_t s) {
    const size_t B = batch, N = h->N;
    PQP_CUDA(h->err, cudaMemcpyAsync(out->status, h->o_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->n, h->o_n, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->iters, h->o_iters, B * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->cost, h->o_cost, B * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(out->path, h->o_path, B * PQP_PLAN_PATH_ROWS * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQP_CUDA(h->err, cudaStreamSynchronize(s));
    return PQP_OK;
}

// `pts` (pqp_plan_points, device pointers): bSpline() first writes the samples of those points into `in`'s raw_x,
// raw_y and r (the handle's in_x, in_y and raw_r) and its status into h->status
// `map_index` (device, [B]) or NULL: the mapped calls' slot per path; the kernels and stage calls that read a map get it
int run(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out, cudaStream_t s,
        const pqp_plan_points_in *pts = nullptr, const int32_t *map_index = nullptr) {
    const int B = in->batch;
    const Dims d{B, h->R, h->P, h->L, h->N, in->r_max};
    const Slots slots{pqb::handle_table(h->bounds), map_index, pqb::handle_map_count(h->bounds)};
    const pqp_plan_trace *tr = out->trace;
    h->timed = true;
    PQP_CUDA(h->err, cudaEventRecord(h->ev[0], s));
    // ---- reference path smoothing (ReferencePathSmoother::solve) ----
    if (pts) {
        bspline_prep_kernel<<<blocks_for(B), kThreads, 0, s>>>(d, slots, pts->m_max, pts->ref_x, pts->ref_y, pts->m, h->bs_t,
                                                                h->raw_r, h->bs_deg, h->status);
        PQL_LAUNCH(h);
        bspline_eval_kernel<<<blocks_for((long long)B * h->R), kThreads, 0, s>>>(
            d, pts->m_max, pts->ref_x, pts->ref_y, pts->m, h->bs_t, h->raw_r, h->bs_deg, h->status, h->in_x, h->in_y);
        PQL_LAUNCH(h);
    }
    raw_prep_kernel<<<blocks_for(B), kThreads, 0, s>>>(d, slots, in->raw_x, in->raw_y, in->r, in->start,
                                                        pts ? h->status : nullptr, h->raw_rows, h->raw_k, h->seg_p,
                                                        h->status, h->start3);
    PQL_LAUNCH(h);
    fit_kernel<<<blocks_for(2LL * B), kThreads, 0, s>>>(B, h->R, h->raw_rows, h->raw_k);
    PQL_LAUNCH(h);
    segment_kernel<<<blocks_for((long long)B * h->P), kThreads, 0, s>>>(d, h->raw_rows, h->raw_k, h->seg_p, h->seg[0],
                                                                         h->seg[1], h->seg[2], h->seg[3], h->seg[4]);
    PQL_LAUNCH(h);
    if (h->prm.smoothing_method == PQP_PLAN_SMOOTH_TENSION) {
        clearance_kernel<<<blocks_for((long long)B * h->P), kThreads, 0, s>>>(d, *pqb::handle_map(h->bounds), slots, h->seg_p,
                                                                               h->seg[0], h->seg[1], h->t_clear);
        PQL_LAUNCH(h);
        pqp_cartesian_tension_in ci = {B, h->P, h->seg_p, h->seg[0], h->seg[1], h->seg[2], h->t_clear};
        pqp_tension_out to = {h->t_x, h->t_y, h->t_s, h->t_status, h->t_iters, nullptr};
        PQL_SUB(h, pqp_cartesian_tension_smooth_device(h->tension, &ci, &to, s), pqp_smoother_last_error, h->tension);
    } else {
        pqp_tension_in ti = {B, h->P, h->seg_p, h->seg[0], h->seg[1], h->seg[2], h->seg[3], h->seg[4]};
        pqp_tension_out to = {h->t_x, h->t_y, h->t_s, h->t_status, h->t_iters, nullptr};
        PQL_SUB(h, pqp_tension_smooth_device(h->tension, &ti, &to, s), pqp_smoother_last_error, h->tension);
    }
    tension_epilogue_kernel<<<blocks_for(B), kThreads, 0, s>>>(d, h->seg_p, h->t_x, h->t_y, h->t_s, h->t_status, h->status,
                                                                h->t_rows, h->tk, h->t_len);
    PQL_LAUNCH(h);
    fit_kernel<<<blocks_for(2LL * B), kThreads, 0, s>>>(B, h->P, h->t_rows, h->tk);
    PQL_LAUNCH(h);
    {
        pqp_dp_in di = {B, h->P, h->t_rows, h->tk, h->t_len, h->start3};
        pqp_dp_out dout = {h->dp_status, h->dp_nl, h->dp_nout, h->dp_ls, h->dp_lo, h->dp_up, h->dp_chosen,
                           h->dp_vl, h->dp_ts, nullptr, nullptr, nullptr};
        if (map_index)
            PQL_SUB(h, pqp_dp_search_mapped_device(h->dp, &di, map_index, &dout, s), pqp_dp_last_error, h->dp);
        else
            PQL_SUB(h, pqp_dp_search_device(h->dp, &di, &dout, s), pqp_dp_last_error, h->dp);
    }
    post_prep_kernel<<<blocks_for(B), kThreads, 0, s>>>(B, h->dp_status, h->dp_nout, h->status, h->post_p);
    PQL_LAUNCH(h);
    {
        pqp_post_in pi = {B, h->L, h->post_p, h->dp_ls, h->dp_lo, h->dp_up, h->dp_vl};
        pqp_post_out po = {h->post_off, h->post_status, h->post_iters, nullptr};
        PQL_SUB(h, pqp_post_smooth_device(h->post, &pi, &po, s), pqp_smoother_last_error, h->post);
    }
    post_epilogue_kernel<<<blocks_for(B), kThreads, 0, s>>>(d, h->t_rows, h->tk, h->dp_ls, h->post_off, h->post_p,
                                                             h->post_status, h->status, h->r_rows, h->rk, h->r_len);
    PQL_LAUNCH(h);
    fit_kernel<<<blocks_for(2LL * B), kThreads, 0, s>>>(B, h->L, h->r_rows, h->rk);
    PQL_LAUNCH(h);
    PQP_CUDA(h->err, cudaEventRecord(h->ev[1], s));
    // ---- processReferencePath ----
    process_kernel<<<blocks_for(B), kThreads, 0, s>>>(d, h->prm.bounds.epsilon, h->r_rows, h->rk, h->r_len, in->start,
                                                       in->target, h->status, h->max_s, h->inst);
    PQL_LAUNCH(h);
    {
        pqp_states_in si = {B, h->N, h->L, h->r_rows, h->rk, h->max_s, h->prm.output_spacing / 2.0, h->prm.output_spacing,
                            h->prm.dynamic_segmentation};
        pqp_states_out so = {h->states, h->curv, h->n_states, h->total, h->knots};
        PQL_SUB(h, pqp_bounds_build_states_device(h->bounds, &si, &so, s), pqp_bounds_last_error, h->bounds);
    }
    states_check_kernel<<<blocks_for(B), kThreads, 0, s>>>(B, h->N, h->total, h->status, h->n_states);
    PQL_LAUNCH(h);
    {
        pqp_bounds_in bi = {B, h->N, h->L, h->states, h->n_states, h->r_rows, h->rk};
        pqp_bounds_out bo = {h->bnd, h->n_valid, h->knots};
        if (map_index)
            PQL_SUB(h, pqp_bounds_compute_mapped_device(h->bounds, &bi, map_index, &bo, s), pqp_bounds_last_error,
                    h->bounds);
        else
            PQL_SUB(h, pqp_bounds_compute_device(h->bounds, &bi, &bo, s), pqp_bounds_last_error, h->bounds);
    }
    {
        InstArgs a;
        a.B = B;
        a.N = h->N;
        a.rough = h->prm.rough_constraints_far_away;
        a.constrain_end = h->prm.constraint_end_heading;
        a.precise_length = h->prm.precise_planning_length;
        a.states = h->states;
        a.bounds = h->bnd;
        a.start = in->start;
        a.target = in->target;
        a.n_states = h->n_states;
        a.n_valid = h->n_valid;
        a.status = h->status;
        a.n1 = h->n1;
        a.p = h->p;
        a.knots = h->knots;
        a.inst = h->inst;
        a.ref_xyh = h->ref_xyh;
        inst_kernel<<<blocks_for(B), kThreads, 0, s>>>(a);
        PQL_LAUNCH(h);
    }
    PQP_CUDA(h->err, cudaEventRecord(h->ev[2], s));
    // ---- optimizePath: solve, updateProblemFormulationAndSolve, getOptimizedPath ----
    const size_t kb = (size_t)B * PQP_NFIELDS * h->N * sizeof(double);
    PQP_CUDA(h->err, cudaMemcpyAsync(h->knots2, h->knots, kb, cudaMemcpyDeviceToDevice, s));
    {
        pqp_batch_in bi = {B, h->N, h->knots, h->inst, h->n1, h->p};
        pqp_batch_out bo = {h->sol1, h->cost1, h->status1, h->iters1, (tr && tr->x_full1) ? h->full[0] : nullptr,
                            (tr && tr->y_full1) ? h->full[1] : nullptr, (tr && tr->z_full1) ? h->full[2] : nullptr,
                            nullptr};
        PQL_SUB(h, pqp_solve_device(h->solver, &bi, &bo, s), pqp_last_error, h->solver);
    }
    between_kernel<<<blocks_for(B), kThreads, 0, s>>>(B, h->status1, h->n1, h->status, h->n2);
    PQL_LAUNCH(h);
    PQL_SUB(h, pqp_relinearise_device(h->solver, B, h->sol1, h->knots2, s), pqp_last_error, h->solver);
    {
        pqp_batch_in bi = {B, h->N, h->knots2, h->inst, h->n2, h->p};
        pqp_batch_out bo = {h->sol2, h->cost2, h->status2, h->iters2, (tr && tr->x_full2) ? h->full[3] : nullptr,
                            (tr && tr->y_full2) ? h->full[4] : nullptr, (tr && tr->z_full2) ? h->full[5] : nullptr,
                            nullptr};
        PQL_SUB(h, pqp_resolve_device(h->solver, &bi, &bo, s), pqp_last_error, h->solver);
    }
    PQL_SUB(h, pqp_frenet_to_cartesian_device(h->solver, B, h->n2, h->ref_xyh, h->sol2, h->xyh, s), pqp_last_error,
            h->solver);
    {
        FinalArgs a;
        a.B = B;
        a.N = h->N;
        a.status = h->status;
        a.status2 = h->status2;
        a.n2 = h->n2;
        a.iters1 = h->iters1;
        a.iters2 = h->iters2;
        a.sol2 = h->sol2;
        a.xyh = h->xyh;
        a.cost2 = h->cost2;
        a.out_status = out->status;
        a.out_n = out->n;
        a.out_iters = out->iters;
        a.out_path = out->path;
        a.out_cost = out->cost;
        final_kernel<<<blocks_for((long long)B * h->N), kThreads, 0, s>>>(a);
        PQL_LAUNCH(h);
    }
    PQP_CUDA(h->err, cudaEventRecord(h->ev[3], s));
    h->launches += kStageLaunches;
    return copy_trace(h, tr, B, pts != nullptr, s);
}

// pqp_plan_points(_device) on device points: the samples go to the handle's [B][R] sample storage
int run_points(pqp_plan_handle *h, const pqp_plan_points_in *pts, const pqp_plan_out *out, cudaStream_t s,
               const int32_t *map_index = nullptr) {
    const pqp_plan_in din = {pts->batch, h->R, h->in_x, h->in_y, h->raw_r, pts->start, pts->target};
    return run(h, &din, out, s, pts, map_index);
}

// every pqp_plan* and pqp_plan_points* entry point: `pts` for the points forms (`in` is then NULL), `mapped` for the
// mapped forms (path b on slot map_index[b]), `stream` empty for the host forms, which stage the inputs into the
// handle's buffers, run on the handle's stream, copy the outputs back and wait
int plan(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_points_in *pts, bool mapped,
         const int32_t *map_index, const pqp_plan_out *out, std::optional<cudaStream_t> stream) {
    int rc = pts ? validate_points(h, pts, out) : validate(h, in, out);
    if (rc != PQP_OK) return rc;
    if (mapped && !map_index) return fail(h->err, PQP_E_INVALID, "null map_index");
    pqp::DeviceGuard guard_(h->device);
    if (stream) return pts ? run_points(h, pts, out, *stream, map_index) : run(h, in, out, *stream, nullptr, map_index);
    cudaStream_t s = h->stream;
    const int batch = pts ? pts->batch : in->batch;
    const size_t B = batch;
    if (pts) {
        const size_t M = pts->m_max;
        PQP_CUDA(h->err, cudaMemcpyAsync(h->pt_x, pts->ref_x, B * M * sizeof(double), cudaMemcpyHostToDevice, s));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->pt_y, pts->ref_y, B * M * sizeof(double), cudaMemcpyHostToDevice, s));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->pt_m, pts->m, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    } else {
        const size_t R = in->r_max;
        PQP_CUDA(h->err, cudaMemcpyAsync(h->in_x, in->raw_x, B * R * sizeof(double), cudaMemcpyHostToDevice, s));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->in_y, in->raw_y, B * R * sizeof(double), cudaMemcpyHostToDevice, s));
        PQP_CUDA(h->err, cudaMemcpyAsync(h->in_r, in->r, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    }
    const double *start = pts ? pts->start : in->start, *target = pts ? pts->target : in->target;
    PQP_CUDA(h->err, cudaMemcpyAsync(h->in_start, start, B * 4 * sizeof(double), cudaMemcpyHostToDevice, s));
    PQP_CUDA(h->err, cudaMemcpyAsync(h->in_target, target, B * 3 * sizeof(double), cudaMemcpyHostToDevice, s));
    if (mapped)
        PQP_CUDA(h->err, cudaMemcpyAsync(h->in_map_index, map_index, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    const int32_t *dmap_index = mapped ? h->in_map_index : nullptr;
    const pqp_plan_out dout = {h->o_status, h->o_n, h->o_path, h->o_cost, h->o_iters, out->trace};
    if (pts) {
        const pqp_plan_points_in din = {batch, pts->m_max, h->pt_x, h->pt_y, h->pt_m, h->in_start, h->in_target};
        rc = run_points(h, &din, &dout, s, dmap_index);
    } else {
        const pqp_plan_in din = {batch, in->r_max, h->in_x, h->in_y, h->in_r, h->in_start, h->in_target};
        rc = run(h, &din, &dout, s, nullptr, dmap_index);
    }
    if (rc != PQP_OK) return rc;
    return copy_results(h, out, batch, s);
}

// a map call of the plan forwarded to its bounds handle: the bounds handle's reason in h->err, `n` more kernel launches
// on success; `sync`: a host form, which waits for the plan stream
#define PQL_MAP(h, call, n, sync)                                                             \
    do {                                                                                      \
        if (!(h)) return PQP_E_INVALID;                                                       \
        PQL_SUB(h, call, pqp_bounds_last_error, (h)->bounds);                                 \
        (h)->launches += (n);                                                                 \
        if (sync) {                                                                           \
            pqp::DeviceGuard guard_((h)->device);                                             \
            PQP_CUDA((h)->err, cudaStreamSynchronize((h)->stream));                           \
        }                                                                                     \
        return PQP_OK;                                                                        \
    } while (0)

// column pass, row pass and the table entries, PQP_MAP_TABLE_CHUNK per launch
long long occupancy_slots_launches(const pqp_occupancy_stack *st) {
    return 2 + (st->count + PQP_MAP_TABLE_CHUNK - 1) / PQP_MAP_TABLE_CHUNK;
}

}  // namespace

extern "C" {

void pqp_plan_default_params(pqp_plan_params *p) {
    if (!p) return;
    *p = pqp_plan_params{};
    pqp_default_params(&p->solver);
    pqp_bounds_default_params(&p->bounds);
    pqp_dp_default_params(&p->dp);
    pqp_smoother_default_params(&p->smoother);
    p->output_spacing = 0.3;
    p->precise_planning_length = 30.0;
    p->dynamic_segmentation = 1;
    p->rough_constraints_far_away = 0;
    p->constraint_end_heading = 1;
    p->smoothing_method = PQP_PLAN_SMOOTH_TENSION2;
}

const char *pqp_plan_last_error(const pqp_plan_handle *h) { return h ? h->err.c_str() : g_plan_create_error.c_str(); }

int pqp_plan_create(const pqp_bounds_map *map, const pqp_plan_params *params, int32_t r_max, int32_t p_max,
                    int32_t layers_max, int32_t n_max, int32_t batch_max, int32_t device, pqp_plan_handle **out) {
    return pqp_plan_create_maps(map, map ? 1 : 0, params, r_max, p_max, layers_max, n_max, batch_max, device, out);
}

int pqp_plan_create_maps(const pqp_bounds_map *maps, int32_t n_maps, const pqp_plan_params *params, int32_t r_max,
                         int32_t p_max, int32_t layers_max, int32_t n_max, int32_t batch_max, int32_t device,
                         pqp_plan_handle **out) {
    if (!out) return PQP_E_INVALID;
    *out = nullptr;
    if (!maps || n_maps < 1) return fail(g_plan_create_error, PQP_E_INVALID, "pqp_plan_create: a map is required");
    if (r_max < 3 || p_max < 4 || layers_max < 4 || n_max < 2 || n_max > 511 || batch_max < 1)
        return fail(g_plan_create_error, PQP_E_INVALID,
                    "pqp_plan_create: r_max >= 3, p_max >= 4, layers_max >= 4, 2 <= n_max <= 511, batch_max >= 1");
    pqp_plan_params dflt;
    pqp_plan_default_params(&dflt);
    const pqp_plan_params &prm = params ? *params : dflt;
    if (!(prm.output_spacing > 0))
        return fail(g_plan_create_error, PQP_E_INVALID, "pqp_plan_create: output_spacing must be positive");
    if (prm.smoothing_method != PQP_PLAN_SMOOTH_TENSION2 && prm.smoothing_method != PQP_PLAN_SMOOTH_TENSION)
        return fail(g_plan_create_error, PQP_E_INVALID,
                    "pqp_plan_create: smoothing_method must be PQP_PLAN_SMOOTH_TENSION2 (0) or PQP_PLAN_SMOOTH_TENSION (1)");
    pqp_plan_handle *h = new (std::nothrow) pqp_plan_handle;
    if (!h) return fail(g_plan_create_error, PQP_E_INVALID, "out of host memory");
    h->prm = prm;
    h->device = h->res.device = device;
    h->R = r_max;
    h->P = p_max;
    h->L = layers_max;
    h->N = n_max;
    h->batch_max = batch_max;
    std::string &err = g_plan_create_error;
    pqp::DeviceGuard guard_(device);
    const int rc = [&]() -> int {
        PQL_SUB_CREATE(pqp_bounds_create_maps(maps, n_maps, &h->prm.bounds, device, &h->bounds), pqp_bounds_last_error);
        PQL_SUB_CREATE(pqp_dp_create(h->bounds, &h->prm.dp, layers_max, batch_max, &h->dp), pqp_dp_last_error);
        PQL_SUB_CREATE(pqp_smoother_create(&h->prm.smoother, p_max, batch_max, device, &h->tension), pqp_smoother_last_error);
        PQL_SUB_CREATE(pqp_smoother_create(&h->prm.smoother, layers_max, batch_max, device, &h->post), pqp_smoother_last_error);
        if (h->prm.smoothing_method == PQP_PLAN_SMOOTH_TENSION)
            if (const char *why = pqs::cartesian_unavailable(h->tension))
                return fail(err, PQP_E_INVALID, std::string("pqp_plan_create: smoothing_method TENSION: ") + why);
        PQL_SUB_CREATE(pqp_create(&h->prm.solver, n_max, batch_max, device, &h->solver), pqp_last_error);
        pqp::Resources &r = h->res;
        const size_t B = batch_max, R = r_max, P = p_max, L = layers_max, N = n_max, S = PQP_SPLINE_ROWS;
        PQP_CUDA(err, r.stream(h->stream));
        for (int i = 0; i < 4; ++i) PQP_CUDA(err, r.event(h->ev[i]));
        PQP_CUDA(err, r.alloc(h->in_x, B * R));
        PQP_CUDA(err, r.alloc(h->in_y, B * R));
        PQP_CUDA(err, r.alloc(h->in_start, B * 4));
        PQP_CUDA(err, r.alloc(h->in_target, B * 3));
        PQP_CUDA(err, r.alloc(h->in_r, B));
        PQP_CUDA(err, r.alloc(h->o_status, B));
        PQP_CUDA(err, r.alloc(h->o_n, B));
        PQP_CUDA(err, r.alloc(h->o_iters, B * 2));
        PQP_CUDA(err, r.alloc(h->o_path, B * PQP_PLAN_PATH_ROWS * N));
        PQP_CUDA(err, r.alloc(h->o_cost, B));
        PQP_CUDA(err, r.alloc(h->status, B));
        PQP_CUDA(err, r.alloc(h->raw_k, B));
        PQP_CUDA(err, r.alloc(h->seg_p, B));
        PQP_CUDA(err, r.alloc(h->t_status, B));
        PQP_CUDA(err, r.alloc(h->t_iters, B));
        PQP_CUDA(err, r.alloc(h->tk, B));
        PQP_CUDA(err, r.alloc(h->start3, B * 3));
        PQP_CUDA(err, r.alloc(h->raw_rows, B * S * R));
        for (int i = 0; i < 5; ++i) PQP_CUDA(err, r.alloc(h->seg[i], B * P));
        PQP_CUDA(err, r.alloc(h->t_x, B * P));
        PQP_CUDA(err, r.alloc(h->t_y, B * P));
        PQP_CUDA(err, r.alloc(h->t_s, B * P));
        PQP_CUDA(err, r.alloc(h->t_rows, B * S * P));
        PQP_CUDA(err, r.alloc(h->t_len, B));
        PQP_CUDA(err, r.alloc(h->dp_status, B));
        PQP_CUDA(err, r.alloc(h->dp_nl, B));
        PQP_CUDA(err, r.alloc(h->dp_nout, B));
        PQP_CUDA(err, r.alloc(h->dp_chosen, B * L));
        PQP_CUDA(err, r.alloc(h->dp_ls, B * L));
        PQP_CUDA(err, r.alloc(h->dp_lo, B * L));
        PQP_CUDA(err, r.alloc(h->dp_up, B * L));
        PQP_CUDA(err, r.alloc(h->dp_vl, B));
        PQP_CUDA(err, r.alloc(h->dp_ts, B));
        PQP_CUDA(err, r.alloc(h->post_p, B));
        PQP_CUDA(err, r.alloc(h->post_status, B));
        PQP_CUDA(err, r.alloc(h->post_iters, B));
        PQP_CUDA(err, r.alloc(h->rk, B));
        PQP_CUDA(err, r.alloc(h->post_off, B * L));
        PQP_CUDA(err, r.alloc(h->r_rows, B * S * L));
        PQP_CUDA(err, r.alloc(h->r_len, B));
        PQP_CUDA(err, r.alloc(h->max_s, B));
        PQP_CUDA(err, r.alloc(h->states, B * PQP_STATE_ROWS * N));
        PQP_CUDA(err, r.alloc(h->curv, B * N));
        PQP_CUDA(err, r.alloc(h->bnd, B * PQP_BOUND_ROWS * N));
        PQP_CUDA(err, r.alloc(h->knots, B * PQP_NFIELDS * N));
        PQP_CUDA(err, r.alloc(h->knots2, B * PQP_NFIELDS * N));
        PQP_CUDA(err, r.alloc(h->inst, B * PQP_NINST));
        PQP_CUDA(err, r.alloc(h->ref_xyh, B * 3 * N));
        PQP_CUDA(err, r.alloc(h->xyh, B * 3 * N));
        PQP_CUDA(err, r.alloc(h->n_states, B));
        PQP_CUDA(err, r.alloc(h->total, B));
        PQP_CUDA(err, r.alloc(h->n_valid, B));
        PQP_CUDA(err, r.alloc(h->n1, B));
        PQP_CUDA(err, r.alloc(h->n2, B));
        PQP_CUDA(err, r.alloc(h->p, B));
        PQP_CUDA(err, r.alloc(h->sol1, B * 4 * N));
        PQP_CUDA(err, r.alloc(h->sol2, B * 4 * N));
        PQP_CUDA(err, r.alloc(h->cost1, B));
        PQP_CUDA(err, r.alloc(h->cost2, B));
        PQP_CUDA(err, r.alloc(h->status1, B));
        PQP_CUDA(err, r.alloc(h->iters1, B));
        PQP_CUDA(err, r.alloc(h->status2, B));
        PQP_CUDA(err, r.alloc(h->iters2, B));
        for (int i = 0; i < 6; ++i)
            PQP_CUDA(err, r.alloc(h->full[i], B * pqp::per_instance(i % 3 == 0 ? &pqp_batch_out::x_full : &pqp_batch_out::y_full, N)));
        if (h->prm.smoothing_method == PQP_PLAN_SMOOTH_TENSION) PQP_CUDA(err, r.alloc(h->t_clear, B * P));
        PQP_CUDA(err, r.alloc(h->pt_x, B * R));
        PQP_CUDA(err, r.alloc(h->pt_y, B * R));
        PQP_CUDA(err, r.alloc(h->pt_m, B));
        PQP_CUDA(err, r.alloc(h->bs_t, B * R));
        PQP_CUDA(err, r.alloc(h->raw_r, B));
        PQP_CUDA(err, r.alloc(h->bs_deg, B));
        PQP_CUDA(err, r.alloc(h->in_map_index, B));
        // spline rows are zero beyond each path's k, so every row read past the end of a fit is defined
        PQP_CUDA(err, cudaMemset(h->raw_rows, 0, B * S * R * sizeof(double)));
        PQP_CUDA(err, cudaMemset(h->t_rows, 0, B * S * P * sizeof(double)));
        PQP_CUDA(err, cudaMemset(h->r_rows, 0, B * S * L * sizeof(double)));
        PQP_CUDA(err, cudaMemset(h->knots, 0, B * PQP_NFIELDS * N * sizeof(double)));
        PQP_CUDA(err, cudaMemset(h->ref_xyh, 0, B * 3 * N * sizeof(double)));
        PQP_CUDA(err, cudaDeviceSynchronize());
        return PQP_OK;
    }();
    if (rc != PQP_OK) {
        const std::string msg = err;
        pqp_plan_destroy(h);
        err = msg;
        return rc;
    }
    *out = h;
    return PQP_OK;
}

void pqp_plan_destroy(pqp_plan_handle *h) {
    if (!h) return;
    pqp::DeviceGuard guard_(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->solver) pqp_destroy(h->solver);
    if (h->post) pqp_smoother_destroy(h->post);
    if (h->tension) pqp_smoother_destroy(h->tension);
    if (h->dp) pqp_dp_destroy(h->dp);
    if (h->bounds) pqp_bounds_destroy(h->bounds);
    delete h;
}

int pqp_plan_device(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out, void *stream) {
    return plan(h, in, nullptr, false, nullptr, out, static_cast<cudaStream_t>(stream));
}

int pqp_plan(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out) {
    return plan(h, in, nullptr, false, nullptr, out, std::nullopt);
}

int pqp_plan_points_device(pqp_plan_handle *h, const pqp_plan_points_in *in, const pqp_plan_out *out, void *stream) {
    return plan(h, nullptr, in, false, nullptr, out, static_cast<cudaStream_t>(stream));
}

int pqp_plan_points(pqp_plan_handle *h, const pqp_plan_points_in *in, const pqp_plan_out *out) {
    return plan(h, nullptr, in, false, nullptr, out, std::nullopt);
}

int pqp_plan_mapped_device(pqp_plan_handle *h, const pqp_plan_in *in, const int32_t *map_index, const pqp_plan_out *out,
                           void *stream) {
    return plan(h, in, nullptr, true, map_index, out, static_cast<cudaStream_t>(stream));
}

int pqp_plan_mapped(pqp_plan_handle *h, const pqp_plan_in *in, const int32_t *map_index, const pqp_plan_out *out) {
    return plan(h, in, nullptr, true, map_index, out, std::nullopt);
}

int pqp_plan_points_mapped_device(pqp_plan_handle *h, const pqp_plan_points_in *in, const int32_t *map_index,
                                  const pqp_plan_out *out, void *stream) {
    return plan(h, nullptr, in, true, map_index, out, static_cast<cudaStream_t>(stream));
}

int pqp_plan_points_mapped(pqp_plan_handle *h, const pqp_plan_points_in *in, const int32_t *map_index,
                           const pqp_plan_out *out) {
    return plan(h, nullptr, in, true, map_index, out, std::nullopt);
}

int pqp_plan_set_map_device(pqp_plan_handle *h, const pqp_bounds_map *map, void *stream) {
    PQL_MAP(h, pqp_bounds_set_map_device(h->bounds, map, stream), 1, false);  // the slot's table entry
}

int pqp_plan_set_map(pqp_plan_handle *h, const pqp_bounds_map *map) {
    PQL_MAP(h, pqp_bounds_set_map_device(h->bounds, map, h->stream), 1, true);
}

int pqp_plan_set_map_slot_device(pqp_plan_handle *h, int32_t slot, const pqp_bounds_map *map, void *stream) {
    PQL_MAP(h, pqp_bounds_set_map_slot_device(h->bounds, slot, map, stream), 1, false);
}

int pqp_plan_set_map_slot(pqp_plan_handle *h, int32_t slot, const pqp_bounds_map *map) {
    PQL_MAP(h, pqp_bounds_set_map_slot_device(h->bounds, slot, map, h->stream), 1, true);
}

int pqp_plan_set_occupancy_device(pqp_plan_handle *h, const pqp_occupancy_map *occ, void *stream) {
    PQL_MAP(h, pqp_bounds_set_occupancy_device(h->bounds, occ, stream), 2, false);  // column and row pass
}

int pqp_plan_set_occupancy(pqp_plan_handle *h, const pqp_occupancy_map *occ) {
    PQL_MAP(h, pqp_bounds_set_occupancy(h->bounds, occ), 2, false);
}

int pqp_plan_set_occupancy_slots_device(pqp_plan_handle *h, int32_t first_slot, const pqp_occupancy_stack *stack,
                                        void *stream) {
    PQL_MAP(h, pqp_bounds_set_occupancy_slots_device(h->bounds, first_slot, stack, stream),
            occupancy_slots_launches(stack), false);
}

int pqp_plan_set_occupancy_slots(pqp_plan_handle *h, int32_t first_slot, const pqp_occupancy_stack *stack) {
    PQL_MAP(h, pqp_bounds_set_occupancy_slots(h->bounds, first_slot, stack), occupancy_slots_launches(stack), false);
}

int pqp_plan_set_occupancy_boxes_device(pqp_plan_handle *h, int32_t first_slot, const pqp_occupancy_stack *base,
                                        int32_t shared_base, const pqp_obstacle_boxes *boxes, void *stream) {
    PQL_MAP(h, pqp_bounds_set_occupancy_boxes_device(h->bounds, first_slot, base, shared_base, boxes, stream),
            occupancy_slots_launches(base), false);
}

int pqp_plan_set_occupancy_boxes(pqp_plan_handle *h, int32_t first_slot, const pqp_occupancy_stack *base,
                                 int32_t shared_base, const pqp_obstacle_boxes *boxes) {
    PQL_MAP(h, pqp_bounds_set_occupancy_boxes(h->bounds, first_slot, base, shared_base, boxes),
            occupancy_slots_launches(base), false);
}

int pqp_plan_get_map(pqp_plan_handle *h, pqp_bounds_map *meta, float *distance) {
    PQL_MAP(h, pqp_bounds_get_map(h->bounds, meta, distance), 0, false);
}

int pqp_plan_get_map_slot(pqp_plan_handle *h, int32_t slot, pqp_bounds_map *meta, float *distance) {
    PQL_MAP(h, pqp_bounds_get_map_slot(h->bounds, slot, meta, distance), 0, false);
}

int32_t pqp_plan_map_count(const pqp_plan_handle *h) { return h ? pqp_bounds_map_count(h->bounds) : 0; }

int pqp_plan_collision_check(pqp_plan_handle *h, const pqp_collision_in *in, const pqp_collision_out *out) {
    PQL_MAP(h, pqp_bounds_collision_check(h->bounds, in, out), 1, false);
}

int pqp_plan_collision_check_device(pqp_plan_handle *h, const pqp_collision_in *in, const pqp_collision_out *out,
                                    void *stream) {
    PQL_MAP(h, pqp_bounds_collision_check_device(h->bounds, in, out, stream), 1, false);
}

int pqp_plan_collision_check_mapped(pqp_plan_handle *h, const pqp_collision_in *in, const int32_t *map_index,
                                    const pqp_collision_out *out) {
    PQL_MAP(h, pqp_bounds_collision_check_mapped(h->bounds, in, map_index, out), 1, false);
}

int pqp_plan_collision_check_mapped_device(pqp_plan_handle *h, const pqp_collision_in *in, const int32_t *map_index,
                                           const pqp_collision_out *out, void *stream) {
    PQL_MAP(h, pqp_bounds_collision_check_mapped_device(h->bounds, in, map_index, out, stream), 1, false);
}

int pqp_plan_last_stage_ms(pqp_plan_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    if (!h->timed) return fail(h->err, PQP_E_STATE, "no plan has run yet");
    pqp::DeviceGuard guard_(h->device);
    PQP_CUDA(h->err, cudaEventSynchronize(h->ev[3]));
    PQP_CUDA(h->err, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_SMOOTHING], h->ev[0], h->ev[1]));
    PQP_CUDA(h->err, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_SEGMENTATION], h->ev[1], h->ev[2]));
    PQP_CUDA(h->err, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_OPTIMISATION], h->ev[2], h->ev[3]));
    PQP_CUDA(h->err, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_TOTAL], h->ev[0], h->ev[3]));
    return PQP_OK;
}

int pqp_plan_launch_count(pqp_plan_handle *h, int64_t *count) {
    if (!h || !count) return PQP_E_INVALID;
    int64_t solver = 0;
    const int rc = pqp_launch_count(h->solver, &solver);
    if (rc != PQP_OK) return fail(h->err, rc, pqp_last_error(h->solver));
    *count = h->launches + solver;
    return PQP_OK;
}

}  // extern "C"
