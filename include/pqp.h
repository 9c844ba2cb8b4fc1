/*
 * pqp.h — C ABI of the batched path-QP solver (H100 / sm_90a).
 *
 * This is the drop-in boundary for the solve path of LiJiangnanBit/path_optimizer_2:
 *
 *   reference interface being replaced                       | entry point here
 *   ---------------------------------------------------------+----------------------------
 *   BaseSolver::BaseSolver            base_solver.cpp:15-39   | pqp_create (+ host packer)
 *   OsqpEigen settings                base_solver.cpp:59-62   | pqp_params / pqp_default_params
 *   BaseSolver::solve                 base_solver.cpp:56-95   | pqp_solve / pqp_solve_device
 *     setCost / setConstraints        base_solver.cpp:119-261 |   (assembled inside the kernel)
 *     OsqpEigen initSolver + solve    base_solver.cpp:87-88   |   (ADMM inside the kernel)
 *   BaseSolver::updateProblem...Solve base_solver.cpp:97-117  | pqp_resolve / pqp_resolve_device
 *   BaseSolver::getOptimizedPath      base_solver.cpp:263-288 | pqp_frenet_to_cartesian
 *   ~BaseSolver (OSQP workspace)      base_solver.hpp:62      | pqp_destroy
 *
 * Plain C: pointers, sizes, POD structs. No C++ / torch types cross this boundary and
 * nothing here throws. Every function returns 0 on success or a negative PQP_E_* code;
 * pqp_last_error() gives the text. There is NO CPU fallback: without a CUDA device
 * pqp_create fails with PQP_E_NO_DEVICE.
 *
 * Problem (SURVEY.md Appendix A): n knots, p "precise" knots (p == n unless the
 * reference's rough_constraints_far_away flag is on),
 *   variables  nv = 3n + (n-1) + (p+n)     [l,psi,kappa]*n, u*(n-1), slacks
 *   rows       m  = 3n + n + 2p + (n-p) + 2
 */
#ifndef PQP_H_
#define PQP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PQP_VERSION 1

/* per-instance solver status (mirrors the OSQP status the reference sees through osqp-eigen) */
enum {
    PQP_SOLVED = 0,
    PQP_MAX_ITER_REACHED = 1,
    PQP_PRIMAL_INFEASIBLE = 2,
    PQP_DUAL_INFEASIBLE = 3,
    PQP_SOLVED_INACCURATE = 4,
    PQP_PRIMAL_INFEASIBLE_INACCURATE = 5,
    PQP_DUAL_INFEASIBLE_INACCURATE = 6,
    PQP_NUMERICAL_ERROR = 7,
    PQP_UNSOLVED = 10
};

/* API error codes (function return values) */
enum {
    PQP_OK = 0,
    PQP_E_INVALID = -1,    /* bad argument (null pointer, n < 2, n > n_max, batch > batch_max ...) */
    PQP_E_NO_DEVICE = -2,  /* no CUDA device / wrong architecture */
    PQP_E_CUDA = -3,       /* a CUDA runtime call failed; see pqp_last_error */
    PQP_E_STATE = -4       /* resolve called before solve, etc. */
};

/* Field order inside one instance's knot block (doubles, each field n_max long). */
enum {
    PQP_F_S = 0,      /* reference arc length s_i                      (base_solver.cpp:174)        */
    PQP_F_KREF = 1,   /* reference curvature k_ref,i                   (base_solver.cpp:182)        */
    PQP_F_L = 2,      /* linearisation point l_i      = input_path[i].l          (:166-171)         */
    PQP_F_PSI = 3,    /* linearisation point psi_i    = input_path[i].d_heading                     */
    PQP_F_K = 4,      /* linearisation point k_i      = input_path[i].k                             */
    PQP_F_B0_LB = 5,  /* row-0 clearance: front.lb (i<p) or center.lb (i>=p)  (:236,243)            */
    PQP_F_B0_UB = 6,  /*                  front.ub        center.ub                                 */
    PQP_F_B1_LB = 7,  /* row-1 clearance: rear.lb  (i<p), ignored for i>=p    (:237)                */
    PQP_F_B1_UB = 8,
    PQP_NFIELDS = 9
};

/* Per-instance scalar block (doubles). */
enum {
    PQP_I_L0 = 0,        /* vehicle_state.getInitError()[0]      (base_solver.cpp:217) */
    PQP_I_PSI0 = 1,      /* vehicle_state.getInitError()[1]                            */
    PQP_I_K0 = 2,        /* vehicle_state.getStartState().k      (:218)                */
    PQP_I_EPSI_LO = 3,   /* end-heading row lower bound (-1e30 when unconstrained, :252-259) */
    PQP_I_EPSI_HI = 4,
    PQP_NINST = 5
};

/* Problem constants + OSQP settings. Defaults = reference flag defaults
 * (planning_flags.cpp:16-22,95) + hard-coded weights (base_solver.cpp:123-126) +
 * OSQP 0.6.x defaults with the reference's eps override (base_solver.cpp:61-62). */
typedef struct pqp_params {
    /* vehicle / formulation */
    double front_length;            /* 3.9   */
    double rear_length;             /* -1.0  */
    double wheel_base;              /* 2.5   */
    double max_steering_angle;      /* 35 deg in rad */
    double expected_safety_margin;  /* 0.6   */
    double weight_l;                /* 0     */
    double weight_kappa;            /* 20    */
    double weight_dkappa;           /* 100   */
    double weight_slack;            /* 10    */
    double end_l_lb;                /* -1.0  (base_solver.cpp:250) */
    double end_l_ub;                /* +1.0  */
    /* OSQP settings */
    double rho;                     /* 0.1   */
    double sigma;                   /* 1e-6  */
    double alpha;                   /* 1.6   */
    double eps_abs;                 /* 2e-3  */
    double eps_rel;                 /* 2e-3  */
    double eps_prim_inf;            /* 1e-4  */
    double eps_dual_inf;            /* 1e-4  */
    double adaptive_rho_tolerance;  /* 5     */
    int32_t max_iter;               /* 4000  */
    int32_t check_termination;      /* 25    */
    int32_t scaling;                /* 10 Ruiz passes */
    int32_t adaptive_rho;           /* 1     */
    int32_t adaptive_rho_interval;  /* 25: fixed; OSQP's default 0 = wall-clock rule, not reproducible */
    int32_t reserved;               /* option bits, default 0: 1 = (unused),
                                       2 = iterate in FP64 (whole kernel in double precision),
                                       4 = do not re-solve suspected-infeasible instances in FP64,
                                       8 = persistent FP32 launch (one-warp CTAs that take instances from a
                                           work counter; host calls stream their copies under one launch): the
                                           default for n_max >= 128,
                                       16 = one CTA per instance even where the persistent launch is the default,
                                       32 = ADMM step in increment form (dx solve, carried row values): the FP32
                                            kernel then follows an FP64 OSQP iteration count for count; the
                                            default for n_max >= 64 (bit 32 forces it below as well),
                                       64 = textbook form everywhere,
                                       128 = cold-only handle: no warm state is kept or written back
                                             (pqp_resolve* returns PQP_E_STATE); for batches that are only
                                             ever solved once (BASELINE configs[2]/[3]) this removes 18 KB
                                             per instance of HBM write traffic */
} pqp_params;

/* Batch input. All pointers are HOST pointers for pqp_solve/pqp_resolve and DEVICE
 * pointers for the *_device variants. Layout is instance-major so that one instance's
 * knot block is one contiguous 9*n_max*8-byte span (one TMA bulk copy per instance):
 *   knots[(b*PQP_NFIELDS + f)*n_max + i], inst[b*PQP_NINST + j], n[b], p[b].
 * n_max must equal the handle's n_max. Entries i >= n[b] are ignored. */
typedef struct pqp_batch_in {
    int32_t batch;
    int32_t n_max;
    const double *knots;
    const double *inst;
    const int32_t *n;
    const int32_t *p;   /* may be NULL: p[b] = n[b] */
} pqp_batch_in;

/* Batch output (caller-owned). sol is mandatory, the rest may be NULL.
 *   sol[(b*4 + f)*n_max + i], f = 0:l 1:psi 2:kappa 3:u(=d_k, i<n-1)   (base_solver.cpp:270-281)
 *   cost[b] = 0.5 x'Px, status[b] = PQP_* status, iters[b] = ADMM iterations
 * Debug/parity outputs in the reference's own index order (Appendix A.1/A.3):
 *   x_full[b*nv_max + j], y_full[b*m_max + r], z_full[b*m_max + r],
 *   nv_max = 6*n_max - 1, m_max = 6*n_max + 2. */
typedef struct pqp_batch_out {
    double *sol;
    double *cost;
    int32_t *status;
    int32_t *iters;
    double *x_full;
    double *y_full;
    double *z_full;
    double *info;      /* optional [b*PQP_NINFO + k]: see PQP_INFO_* */
} pqp_batch_out;

enum {
    PQP_INFO_PRI_RES = 0,
    PQP_INFO_DUA_RES = 1,
    PQP_INFO_RHO = 2,
    PQP_INFO_RHO_UPDATES = 3,
    PQP_NINFO = 4
};

typedef struct pqp_handle pqp_handle;

/* Fill *params with the defaults listed above. */
int pqp_default_params(pqp_params *params);

/* Create a solver bound to CUDA device `device` able to hold `batch_max` instances of up
 * to `n_max` knots (2 <= n_max <= 511; the reference itself has no cap, see INTEGRATION.md). Owns device buffers for inputs, outputs and the
 * per-instance warm state (scaled x, z, y and rho; the OSQP workspace of
 * base_solver.hpp:62). Returns PQP_E_INVALID, before looking for a device, for params that
 * OSQP's settings validation refuses (rho, sigma <= 0; alpha outside (0, 2); eps_abs or
 * eps_rel < 0, or both 0; eps_prim_inf, eps_dual_inf <= 0; adaptive_rho not 0 or 1;
 * adaptive_rho_tolerance < 1; max_iter <= 0; negative check_termination, scaling or
 * adaptive_rho_interval), for any non-finite double, for a negative weight, for
 * wheel_base <= 0 and for max_steering_angle outside (0, pi/2). */
int pqp_create(const pqp_params *params, int32_t n_max, int32_t batch_max, int32_t device,
               pqp_handle **out);
int pqp_destroy(pqp_handle *h);

/* Cold solve of in->batch instances (BaseSolver::solve). Host buffers; H2D, kernel, D2H. */
int pqp_solve(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out);

/* Warm re-solve (BaseSolver::updateProblemFormulationAndSolve): `in` carries the new
 * linearisation point in its L/PSI/K fields (the reference passes the previous result,
 * path_optimizer.cpp:153). If in == NULL the previous solution held on the device is
 * used as the new linearisation point (no H2D). Warm x,z,y,rho persist per instance. */
int pqp_resolve(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out);

/* Same, with DEVICE pointers and the caller's stream (a cudaStream_t passed as void*,
 * NULL = default stream). Asynchronous: no host synchronisation inside. Two differences from the
 * host-pointer calls follow from that: (1) n[] and p[] cannot be validated on the host - an instance
 * whose n is outside [2, n_max] is skipped by the kernel with status PQP_NUMERICAL_ERROR; (2) there
 * is no FP64 re-solve of suspected-infeasible instances (that needs the statuses on the host): an
 * infeasible instance the FP32 certificate cannot resolve ends as PQP_MAX_ITER_REACHED here and as
 * PQP_PRIMAL_INFEASIBLE through pqp_solve (cold solves only: pqp_resolve never escalates, the FP64 re-solve
 * would start cold). Both mean `false` to the reference's caller
 * (base_solver.cpp:88). After a host-pointer call escalated an instance, its warm slot holds the FP64
 * run's iterates and rho (cast to FP32), i.e. a later pqp_resolve warm-starts from the run that was returned. */
int pqp_solve_device(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out,
                     void *stream);
int pqp_resolve_device(pqp_handle *h, const pqp_batch_in *in, const pqp_batch_out *out,
                       void *stream);

/* The caller's step between solve and updateProblemFormulationAndSolve (path_optimizer.cpp:153
 * passes the first result back as the new input path): copy sol[b][0..2][i] (l, psi, kappa) into
 * the linearisation fields PQP_F_L, PQP_F_PSI, PQP_F_K of knots[b][PQP_NFIELDS][n_max]. Device
 * pointers, asynchronous on `stream`. (pqp_resolve with in = NULL does the same internally.) */
int pqp_relinearise_device(pqp_handle *h, int32_t batch, const double *sol, double *knots, void *stream);

/* Receding-horizon bookkeeping between two pqp_resolve_device calls (the caller side of
 * path_optimizer.cpp:153 when the plan is re-issued every tick, BASELINE configs[4]), one launch,
 * device pointers, asynchronous on `stream`: knots[b][f][i] = ext_knots[b][f][tick + i] from an
 * extended reference ext_knots[b][PQP_NFIELDS][ext_len], except the linearisation fields L, PSI, K,
 * which take the previous solution shifted by one knot (sol[b][0..2][min(i + 1, n_max - 1)]);
 * inst[b][L0, PSI0, K0] = the previous solution at knot 1. `sol` is the buffer of the last solve. */
int pqp_advance_window_device(pqp_handle *h, int32_t batch, int32_t ext_len, int32_t tick,
                              const double *ext_knots, const double *sol, double *knots, double *inst,
                              void *stream);

/* BaseSolver::getOptimizedPath (base_solver.cpp:263-288) for a batch, FP64, on device
 * pointers: ref_xyh[(b*3+f)*n_max+i] f=0:x 1:y 2:heading of the reference states;
 * sol as produced above; out_xyh same layout as ref_xyh (x, y, heading of the result). */
int pqp_frenet_to_cartesian_device(pqp_handle *h, int32_t batch, const int32_t *n,
                                   const double *ref_xyh, const double *sol,
                                   double *out_xyh, void *stream);
int pqp_frenet_to_cartesian(pqp_handle *h, int32_t batch, const int32_t *n,
                            const double *ref_xyh, const double *sol, double *out_xyh);

/* Device time (ms) of the last host-pointer solve/resolve, first copy to last copy (CUDA
 * events on the handle's streams; the call is a chunked H2D / kernel / D2H pipeline), and the
 * number of kernel launches the handle has issued so far. */
int pqp_last_kernel_ms(pqp_handle *h, float *ms);
int pqp_launch_count(pqp_handle *h, int64_t *count);

/* Per-stage device times (ms, CUDA events) of the last host-pointer solve/resolve: the counterpart of
 * the TimeRecorder stages BaseSolver::solve logs (base_solver.cpp:57-93: "Set cost", "Set
 * constraints", "Set solver", "OSQP Solve", "Retrive path"). Cost, constraints, solver set-up and
 * the ADMM loop are ONE kernel here, so the stages are: host-to-device copy, kernel, device-to-host
 * copy, FP64 re-solve of suspected-infeasible instances, whole call. ms[PQP_NSTAGES]. The three
 * pipeline stages are only defined for single-stream calls (batches below the chunking threshold,
 * i.e. the B = 1 drop-in); chunked / streamed calls overlap them and report -1 there. */
enum {
    PQP_STAGE_H2D = 0,
    PQP_STAGE_KERNEL = 1,
    PQP_STAGE_D2H = 2,
    PQP_STAGE_ESCALATION = 3,
    PQP_STAGE_TOTAL = 4,
    PQP_NSTAGES = 5
};
int pqp_last_stage_ms(pqp_handle *h, float *ms);

/* Device-side properties, for occupancy reporting: SM count, resident warps per SM of
 * the solve kernel, dynamic shared memory per warp in bytes (the whole per-QP state: 72 x 32 x C
 * values for C stages per lane, plus the input-staging barrier). */
int pqp_kernel_info(pqp_handle *h, int32_t *sm_count, int32_t *warps_per_sm,
                    int32_t *smem_per_warp);

const char *pqp_last_error(const pqp_handle *h); /* h may be NULL: last create error */
int pqp_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PQP_H_ */
