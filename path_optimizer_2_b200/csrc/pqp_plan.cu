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
#include <string>

#include "../../include/pqp_plan.h"
#include "pqp_bounds_internal.h"
#include "pqp_device_guard.h"
#include "pqp_plan_core.cuh"
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

// raw samples -> s_list_ (chord length) into the raw spline rows, sample count of segmentRawReference
__global__ void raw_prep_kernel(Dims d, const double *__restrict__ raw_x, const double *__restrict__ raw_y,
                                const int32_t *__restrict__ r, const double *__restrict__ start, double *raw_rows,
                                int32_t *raw_k, int32_t *seg_p, int32_t *status, double *start3) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.B) return;
    start3[3 * b] = start[4 * b];
    start3[3 * b + 1] = start[4 * b + 1];
    start3[3 * b + 2] = start[4 * b + 2];
    double *rows = raw_rows + (size_t)b * pqpl::kSplineRows * d.R;
    double *sx = rows, *x = rows + 4 * (size_t)d.R, *y = rows + 8 * (size_t)d.R;
    const int rb = r[b];
    int st = pqpl::kOk, p = 0;
    if (rb < 3 || rb > d.R) {
        st = pqpl::kSplineDegenerate;
    } else {
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
__global__ void clearance_kernel(Dims d, const pqb::MapView map, const int32_t *__restrict__ seg_p,
                                 const double *__restrict__ sx_, const double *__restrict__ sy_, double *clearance) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)d.B * d.P) return;
    const int b = (int)(t / d.P), j = (int)(t % d.P);
    if (j >= seg_p[b]) return;
    const size_t o = (size_t)b * d.P + j;
    clearance[o] = pqb::map_distance(map, sx_[o], sy_[o]);
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

template <typename T>
cudaError_t dalloc(T **p, size_t n) {
    return cudaMalloc(reinterpret_cast<void **>(p), (n ? n : 1) * sizeof(T));
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
    double *states = nullptr, *curv = nullptr, *bnd = nullptr, *knots = nullptr, *knots2 = nullptr, *inst = nullptr,
           *ref_xyh = nullptr, *xyh = nullptr;
    int32_t *n_states = nullptr, *total = nullptr, *n_valid = nullptr, *n1 = nullptr, *n2 = nullptr, *p = nullptr;
    double *sol1 = nullptr, *sol2 = nullptr, *cost1 = nullptr, *cost2 = nullptr;
    double *full[6] = {};  // x, y, z of the first solve, then of the second: written only when traced
    int32_t *status1 = nullptr, *iters1 = nullptr, *status2 = nullptr, *iters2 = nullptr;
    std::string err;
};

namespace {

int pfail(pqp_plan_handle *h, int code, const std::string &msg) {
    if (h) h->err = msg;
    else g_plan_create_error = msg;
    return code;
}

#define PQL_CUDA(h, call)                                                  \
    do {                                                                   \
        cudaError_t e_ = (call);                                           \
        if (e_ != cudaSuccess) {                                           \
            (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_); \
            return PQP_E_CUDA;                                             \
        }                                                                  \
    } while (0)

#define PQL_SUB(h, call, errfn, sub)                                                          \
    do {                                                                                      \
        const int rc_ = (call);                                                               \
        if (rc_ != PQP_OK) return pfail((h), rc_, std::string(#call) + ": " + errfn(sub));   \
    } while (0)

#define PQL_LAUNCH(h)                              \
    do {                                           \
        PQL_CUDA(h, cudaGetLastError());           \
        (h)->launches++;                           \
    } while (0)

int validate(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out) {
    if (!h) return PQP_E_INVALID;
    if (!in || !out) return pfail(h, PQP_E_INVALID, "null batch");
    if (!in->raw_x || !in->raw_y || !in->r || !in->start || !in->target) return pfail(h, PQP_E_INVALID, "null input buffer");
    if (!out->status || !out->n || !out->path || !out->cost || !out->iters) return pfail(h, PQP_E_INVALID, "null output buffer");
    if (in->batch < 1 || in->batch > h->batch_max) return pfail(h, PQP_E_INVALID, "batch out of range");
    if (in->r_max < 3 || in->r_max > h->R) return pfail(h, PQP_E_INVALID, "r_max must be in [3, the handle's r_max]");
    return PQP_OK;
}

int copy_out(pqp_plan_handle *h, void *dst, const void *src, size_t bytes, cudaStream_t s) {
    if (dst) PQL_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s));
    return PQP_OK;
}

int copy_trace(pqp_plan_handle *h, const pqp_plan_trace *t, int B, cudaStream_t s) {
    if (!t) return PQP_OK;
    const size_t b = B, d = sizeof(double), i4 = sizeof(int32_t), P = h->P, L = h->L, N = h->N, R = h->R;
    int rc = PQP_OK;
#define PQL_T(dst, src, bytes) \
    if ((rc = copy_out(h, (dst), (src), (bytes), s)) != PQP_OK) return rc
    PQL_T(t->raw_spline, h->raw_rows, b * PQP_SPLINE_ROWS * R * d);
    PQL_T(t->seg_p, h->seg_p, b * i4);
    PQL_T(t->seg_x, h->seg[0], b * P * d);
    PQL_T(t->seg_y, h->seg[1], b * P * d);
    PQL_T(t->seg_angle, h->seg[2], b * P * d);
    PQL_T(t->seg_k, h->seg[3], b * P * d);
    PQL_T(t->seg_s, h->seg[4], b * P * d);
    PQL_T(t->tension_x, h->t_x, b * P * d);
    PQL_T(t->tension_y, h->t_y, b * P * d);
    PQL_T(t->tension_s, h->t_s, b * P * d);
    PQL_T(t->tension_status, h->t_status, b * i4);
    PQL_T(t->tension_iters, h->t_iters, b * i4);
    PQL_T(t->tension_spline, h->t_rows, b * PQP_SPLINE_ROWS * P * d);
    PQL_T(t->tension_length, h->t_len, b * d);
    PQL_T(t->dp_status, h->dp_status, b * i4);
    PQL_T(t->dp_n_out, h->dp_nout, b * i4);
    PQL_T(t->dp_layer_s, h->dp_ls, b * L * d);
    PQL_T(t->dp_lower, h->dp_lo, b * L * d);
    PQL_T(t->dp_upper, h->dp_up, b * L * d);
    PQL_T(t->dp_chosen, h->dp_chosen, b * L * i4);
    PQL_T(t->dp_vehicle_l, h->dp_vl, b * d);
    PQL_T(t->post_offsets, h->post_off, b * L * d);
    PQL_T(t->post_status, h->post_status, b * i4);
    PQL_T(t->post_iters, h->post_iters, b * i4);
    PQL_T(t->ref_spline, h->r_rows, b * PQP_SPLINE_ROWS * L * d);
    PQL_T(t->max_s, h->max_s, b * d);
    PQL_T(t->states, h->states, b * PQP_STATE_ROWS * N * d);
    PQL_T(t->curvature, h->curv, b * N * d);
    PQL_T(t->total, h->total, b * i4);
    PQL_T(t->bounds, h->bnd, b * PQP_BOUND_ROWS * N * d);
    PQL_T(t->n_valid, h->n_valid, b * i4);
    PQL_T(t->knots, h->knots, b * PQP_NFIELDS * N * d);
    PQL_T(t->inst, h->inst, b * PQP_NINST * d);
    PQL_T(t->p, h->p, b * i4);
    PQL_T(t->sol1, h->sol1, b * 4 * N * d);
    PQL_T(t->status1, h->status1, b * i4);
    PQL_T(t->iters1, h->iters1, b * i4);
    const size_t nv = 6 * N - 1, m = 6 * N + 2;  // pqp_batch_out's x_full / y_full / z_full strides
    PQL_T(t->x_full1, h->full[0], b * nv * d);
    PQL_T(t->y_full1, h->full[1], b * m * d);
    PQL_T(t->z_full1, h->full[2], b * m * d);
    PQL_T(t->x_full2, h->full[3], b * nv * d);
    PQL_T(t->y_full2, h->full[4], b * m * d);
    PQL_T(t->z_full2, h->full[5], b * m * d);
    if (h->t_clear) PQL_T(t->tension_clearance, h->t_clear, b * P * d);
#undef PQL_T
    return PQP_OK;
}

int run(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out, cudaStream_t s) {
    const int B = in->batch;
    const Dims d{B, h->R, h->P, h->L, h->N, in->r_max};
    const pqp_plan_trace *tr = out->trace;
    h->timed = true;
    PQL_CUDA(h, cudaEventRecord(h->ev[0], s));
    // ---- reference path smoothing (ReferencePathSmoother::solve) ----
    raw_prep_kernel<<<blocks_for(B), kThreads, 0, s>>>(d, in->raw_x, in->raw_y, in->r, in->start, h->raw_rows, h->raw_k,
                                                        h->seg_p, h->status, h->start3);
    PQL_LAUNCH(h);
    fit_kernel<<<blocks_for(2LL * B), kThreads, 0, s>>>(B, h->R, h->raw_rows, h->raw_k);
    PQL_LAUNCH(h);
    segment_kernel<<<blocks_for((long long)B * h->P), kThreads, 0, s>>>(d, h->raw_rows, h->raw_k, h->seg_p, h->seg[0],
                                                                         h->seg[1], h->seg[2], h->seg[3], h->seg[4]);
    PQL_LAUNCH(h);
    if (h->prm.smoothing_method == PQP_PLAN_SMOOTH_TENSION) {
        clearance_kernel<<<blocks_for((long long)B * h->P), kThreads, 0, s>>>(d, *pqb::handle_map(h->bounds), h->seg_p,
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
    PQL_CUDA(h, cudaEventRecord(h->ev[1], s));
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
    PQL_CUDA(h, cudaEventRecord(h->ev[2], s));
    // ---- optimizePath: solve, updateProblemFormulationAndSolve, getOptimizedPath ----
    const size_t kb = (size_t)B * PQP_NFIELDS * h->N * sizeof(double);
    PQL_CUDA(h, cudaMemcpyAsync(h->knots2, h->knots, kb, cudaMemcpyDeviceToDevice, s));
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
    PQL_CUDA(h, cudaEventRecord(h->ev[3], s));
    h->launches += kStageLaunches;
    return copy_trace(h, tr, B, s);
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
    if (!out) return PQP_E_INVALID;
    *out = nullptr;
    if (!map) return pfail(nullptr, PQP_E_INVALID, "pqp_plan_create: a map is required");
    if (r_max < 3 || p_max < 4 || layers_max < 4 || n_max < 2 || n_max > 511 || batch_max < 1)
        return pfail(nullptr, PQP_E_INVALID,
                     "pqp_plan_create: r_max >= 3, p_max >= 4, layers_max >= 4, 2 <= n_max <= 511, batch_max >= 1");
    pqp_plan_params dflt;
    pqp_plan_default_params(&dflt);
    pqp_plan_handle *h = new (std::nothrow) pqp_plan_handle;
    if (!h) return pfail(nullptr, PQP_E_INVALID, "out of host memory");
    h->prm = params ? *params : dflt;
    if (!(h->prm.output_spacing > 0)) {
        delete h;
        return pfail(nullptr, PQP_E_INVALID, "pqp_plan_create: output_spacing must be positive");
    }
    if (h->prm.smoothing_method != PQP_PLAN_SMOOTH_TENSION2 && h->prm.smoothing_method != PQP_PLAN_SMOOTH_TENSION) {
        delete h;
        return pfail(nullptr, PQP_E_INVALID,
                     "pqp_plan_create: smoothing_method must be PQP_PLAN_SMOOTH_TENSION2 (0) or PQP_PLAN_SMOOTH_TENSION (1)");
    }
    h->device = device;
    h->R = r_max;
    h->P = p_max;
    h->L = layers_max;
    h->N = n_max;
    h->batch_max = batch_max;
    int rc = pqp_bounds_create(map, &h->prm.bounds, device, &h->bounds);
    if (rc == PQP_OK) {
        rc = pqp_dp_create(h->bounds, &h->prm.dp, layers_max, batch_max, &h->dp);
        if (rc != PQP_OK) g_plan_create_error = std::string("pqp_plan_create: ") + pqp_dp_last_error(nullptr);
    } else {
        g_plan_create_error = std::string("pqp_plan_create: ") + pqp_bounds_last_error(nullptr);
    }
    if (rc == PQP_OK) {
        rc = pqp_smoother_create(&h->prm.smoother, p_max, batch_max, device, &h->tension);
        if (rc == PQP_OK) rc = pqp_smoother_create(&h->prm.smoother, layers_max, batch_max, device, &h->post);
        if (rc != PQP_OK) g_plan_create_error = std::string("pqp_plan_create: ") + pqp_smoother_last_error(nullptr);
    }
    if (rc == PQP_OK && h->prm.smoothing_method == PQP_PLAN_SMOOTH_TENSION) {
        if (const char *why = pqs::cartesian_unavailable(h->tension)) {
            rc = PQP_E_INVALID;
            g_plan_create_error = std::string("pqp_plan_create: smoothing_method TENSION: ") + why;
        }
    }
    if (rc == PQP_OK) {
        rc = pqp_create(&h->prm.solver, n_max, batch_max, device, &h->solver);
        if (rc != PQP_OK) g_plan_create_error = std::string("pqp_plan_create: ") + pqp_last_error(nullptr);
    }
    if (rc != PQP_OK) {
        const std::string msg = g_plan_create_error;
        pqp_plan_destroy(h);
        g_plan_create_error = msg;
        return rc;
    }
    pqp::DeviceGuard guard_(device);
    const size_t B = batch_max, R = r_max, P = p_max, L = layers_max, N = n_max, S = PQP_SPLINE_ROWS;
    cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = cudaEventCreate(&h->ev[i]);
    if (e == cudaSuccess) e = dalloc(&h->in_x, B * R);
    if (e == cudaSuccess) e = dalloc(&h->in_y, B * R);
    if (e == cudaSuccess) e = dalloc(&h->in_start, B * 4);
    if (e == cudaSuccess) e = dalloc(&h->in_target, B * 3);
    if (e == cudaSuccess) e = dalloc(&h->in_r, B);
    if (e == cudaSuccess) e = dalloc(&h->o_status, B);
    if (e == cudaSuccess) e = dalloc(&h->o_n, B);
    if (e == cudaSuccess) e = dalloc(&h->o_iters, B * 2);
    if (e == cudaSuccess) e = dalloc(&h->o_path, B * PQP_PLAN_PATH_ROWS * N);
    if (e == cudaSuccess) e = dalloc(&h->o_cost, B);
    if (e == cudaSuccess) e = dalloc(&h->status, B);
    if (e == cudaSuccess) e = dalloc(&h->raw_k, B);
    if (e == cudaSuccess) e = dalloc(&h->seg_p, B);
    if (e == cudaSuccess) e = dalloc(&h->t_status, B);
    if (e == cudaSuccess) e = dalloc(&h->t_iters, B);
    if (e == cudaSuccess) e = dalloc(&h->tk, B);
    if (e == cudaSuccess) e = dalloc(&h->start3, B * 3);
    if (e == cudaSuccess) e = dalloc(&h->raw_rows, B * S * R);
    for (int i = 0; i < 5 && e == cudaSuccess; ++i) e = dalloc(&h->seg[i], B * P);
    if (e == cudaSuccess) e = dalloc(&h->t_x, B * P);
    if (e == cudaSuccess) e = dalloc(&h->t_y, B * P);
    if (e == cudaSuccess) e = dalloc(&h->t_s, B * P);
    if (e == cudaSuccess) e = dalloc(&h->t_rows, B * S * P);
    if (e == cudaSuccess) e = dalloc(&h->t_len, B);
    if (e == cudaSuccess) e = dalloc(&h->dp_status, B);
    if (e == cudaSuccess) e = dalloc(&h->dp_nl, B);
    if (e == cudaSuccess) e = dalloc(&h->dp_nout, B);
    if (e == cudaSuccess) e = dalloc(&h->dp_chosen, B * L);
    if (e == cudaSuccess) e = dalloc(&h->dp_ls, B * L);
    if (e == cudaSuccess) e = dalloc(&h->dp_lo, B * L);
    if (e == cudaSuccess) e = dalloc(&h->dp_up, B * L);
    if (e == cudaSuccess) e = dalloc(&h->dp_vl, B);
    if (e == cudaSuccess) e = dalloc(&h->dp_ts, B);
    if (e == cudaSuccess) e = dalloc(&h->post_p, B);
    if (e == cudaSuccess) e = dalloc(&h->post_status, B);
    if (e == cudaSuccess) e = dalloc(&h->post_iters, B);
    if (e == cudaSuccess) e = dalloc(&h->rk, B);
    if (e == cudaSuccess) e = dalloc(&h->post_off, B * L);
    if (e == cudaSuccess) e = dalloc(&h->r_rows, B * S * L);
    if (e == cudaSuccess) e = dalloc(&h->r_len, B);
    if (e == cudaSuccess) e = dalloc(&h->max_s, B);
    if (e == cudaSuccess) e = dalloc(&h->states, B * PQP_STATE_ROWS * N);
    if (e == cudaSuccess) e = dalloc(&h->curv, B * N);
    if (e == cudaSuccess) e = dalloc(&h->bnd, B * PQP_BOUND_ROWS * N);
    if (e == cudaSuccess) e = dalloc(&h->knots, B * PQP_NFIELDS * N);
    if (e == cudaSuccess) e = dalloc(&h->knots2, B * PQP_NFIELDS * N);
    if (e == cudaSuccess) e = dalloc(&h->inst, B * PQP_NINST);
    if (e == cudaSuccess) e = dalloc(&h->ref_xyh, B * 3 * N);
    if (e == cudaSuccess) e = dalloc(&h->xyh, B * 3 * N);
    if (e == cudaSuccess) e = dalloc(&h->n_states, B);
    if (e == cudaSuccess) e = dalloc(&h->total, B);
    if (e == cudaSuccess) e = dalloc(&h->n_valid, B);
    if (e == cudaSuccess) e = dalloc(&h->n1, B);
    if (e == cudaSuccess) e = dalloc(&h->n2, B);
    if (e == cudaSuccess) e = dalloc(&h->p, B);
    if (e == cudaSuccess) e = dalloc(&h->sol1, B * 4 * N);
    if (e == cudaSuccess) e = dalloc(&h->sol2, B * 4 * N);
    if (e == cudaSuccess) e = dalloc(&h->cost1, B);
    if (e == cudaSuccess) e = dalloc(&h->cost2, B);
    if (e == cudaSuccess) e = dalloc(&h->status1, B);
    if (e == cudaSuccess) e = dalloc(&h->iters1, B);
    if (e == cudaSuccess) e = dalloc(&h->status2, B);
    if (e == cudaSuccess) e = dalloc(&h->iters2, B);
    for (int i = 0; i < 6 && e == cudaSuccess; ++i) e = dalloc(&h->full[i], B * (i % 3 == 0 ? 6 * N - 1 : 6 * N + 2));
    if (e == cudaSuccess && h->prm.smoothing_method == PQP_PLAN_SMOOTH_TENSION) e = dalloc(&h->t_clear, B * P);
    // spline rows are zero beyond each path's k, so every row read past the end of a fit is defined
    if (e == cudaSuccess) e = cudaMemset(h->raw_rows, 0, B * S * R * sizeof(double));
    if (e == cudaSuccess) e = cudaMemset(h->t_rows, 0, B * S * P * sizeof(double));
    if (e == cudaSuccess) e = cudaMemset(h->r_rows, 0, B * S * L * sizeof(double));
    if (e == cudaSuccess) e = cudaMemset(h->knots, 0, B * PQP_NFIELDS * N * sizeof(double));
    if (e == cudaSuccess) e = cudaMemset(h->ref_xyh, 0, B * 3 * N * sizeof(double));
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        const std::string msg = std::string("pqp_plan_create: ") + cudaGetErrorString(e);
        pqp_plan_destroy(h);
        g_plan_create_error = msg;
        return PQP_E_CUDA;
    }
    *out = h;
    return PQP_OK;
}

void pqp_plan_destroy(pqp_plan_handle *h) {
    if (!h) return;
    {
        pqp::DeviceGuard guard_(h->device);
        if (h->stream) cudaStreamSynchronize(h->stream);
        void *bufs[] = {h->in_x, h->in_y, h->in_start, h->in_target, h->in_r, h->o_status, h->o_n, h->o_iters, h->o_path,
                        h->o_cost, h->status, h->raw_k, h->seg_p, h->t_status, h->t_iters, h->tk, h->start3, h->raw_rows,
                        h->seg[0], h->seg[1], h->seg[2], h->seg[3], h->seg[4], h->t_x, h->t_y, h->t_s, h->t_rows, h->t_len,
                        h->dp_status, h->dp_nl, h->dp_nout, h->dp_chosen, h->dp_ls, h->dp_lo, h->dp_up, h->dp_vl, h->dp_ts,
                        h->post_p, h->post_status, h->post_iters, h->rk, h->post_off, h->r_rows, h->r_len, h->max_s,
                        h->states, h->curv, h->bnd, h->knots, h->knots2, h->inst, h->ref_xyh, h->xyh, h->n_states,
                        h->total, h->n_valid, h->n1, h->n2, h->p, h->sol1, h->sol2, h->cost1, h->cost2, h->status1,
                        h->iters1, h->status2, h->iters2, h->full[0], h->full[1], h->full[2], h->full[3], h->full[4],
                        h->full[5], h->t_clear};
        for (void *p : bufs) cudaFree(p);
        for (cudaEvent_t ev : h->ev)
            if (ev) cudaEventDestroy(ev);
        if (h->stream) cudaStreamDestroy(h->stream);
    }
    if (h->solver) pqp_destroy(h->solver);
    if (h->post) pqp_smoother_destroy(h->post);
    if (h->tension) pqp_smoother_destroy(h->tension);
    if (h->dp) pqp_dp_destroy(h->dp);
    if (h->bounds) pqp_bounds_destroy(h->bounds);
    delete h;
}

int pqp_plan_device(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out, void *stream) {
    int rc = validate(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    return run(h, in, out, static_cast<cudaStream_t>(stream));
}

int pqp_plan(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out) {
    int rc = validate(h, in, out);
    if (rc != PQP_OK) return rc;
    pqp::DeviceGuard guard_(h->device);
    cudaStream_t s = h->stream;
    const size_t B = in->batch, R = in->r_max, N = h->N;
    PQL_CUDA(h, cudaMemcpyAsync(h->in_x, in->raw_x, B * R * sizeof(double), cudaMemcpyHostToDevice, s));
    PQL_CUDA(h, cudaMemcpyAsync(h->in_y, in->raw_y, B * R * sizeof(double), cudaMemcpyHostToDevice, s));
    PQL_CUDA(h, cudaMemcpyAsync(h->in_r, in->r, B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    PQL_CUDA(h, cudaMemcpyAsync(h->in_start, in->start, B * 4 * sizeof(double), cudaMemcpyHostToDevice, s));
    PQL_CUDA(h, cudaMemcpyAsync(h->in_target, in->target, B * 3 * sizeof(double), cudaMemcpyHostToDevice, s));
    const pqp_plan_in din = {in->batch, in->r_max, h->in_x, h->in_y, h->in_r, h->in_start, h->in_target};
    const pqp_plan_out dout = {h->o_status, h->o_n, h->o_path, h->o_cost, h->o_iters, out->trace};
    rc = run(h, &din, &dout, s);
    if (rc != PQP_OK) return rc;
    PQL_CUDA(h, cudaMemcpyAsync(out->status, h->o_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQL_CUDA(h, cudaMemcpyAsync(out->n, h->o_n, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQL_CUDA(h, cudaMemcpyAsync(out->iters, h->o_iters, B * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    PQL_CUDA(h, cudaMemcpyAsync(out->cost, h->o_cost, B * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQL_CUDA(h, cudaMemcpyAsync(out->path, h->o_path, B * PQP_PLAN_PATH_ROWS * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    PQL_CUDA(h, cudaStreamSynchronize(s));
    return PQP_OK;
}

int pqp_plan_last_stage_ms(pqp_plan_handle *h, float *ms) {
    if (!h || !ms) return PQP_E_INVALID;
    if (!h->timed) return pfail(h, PQP_E_STATE, "no plan has run yet");
    pqp::DeviceGuard guard_(h->device);
    PQL_CUDA(h, cudaEventSynchronize(h->ev[3]));
    PQL_CUDA(h, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_SMOOTHING], h->ev[0], h->ev[1]));
    PQL_CUDA(h, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_SEGMENTATION], h->ev[1], h->ev[2]));
    PQL_CUDA(h, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_OPTIMISATION], h->ev[2], h->ev[3]));
    PQL_CUDA(h, cudaEventElapsedTime(&ms[PQP_PLAN_STAGE_TOTAL], h->ev[0], h->ev[3]));
    return PQP_OK;
}

int pqp_plan_launch_count(pqp_plan_handle *h, int64_t *count) {
    if (!h || !count) return PQP_E_INVALID;
    int64_t solver = 0;
    const int rc = pqp_launch_count(h->solver, &solver);
    if (rc != PQP_OK) return pfail(h, rc, pqp_last_error(h->solver));
    *count = h->launches + solver;
    return PQP_OK;
}

}  // extern "C"
