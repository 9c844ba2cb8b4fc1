/*
 * pqp_plan.h — C ABI of the whole plan: PathOptimizer::solve for a batch of paths on the GPU.
 *
 * reference interface replaced:
 *   PathOptimizer::solve                         src/path_optimizer.cpp:34-71
 *     ReferencePathSmoother::solve               src/reference_path_smoother/reference_path_smoother.cpp:17-45
 *       segmentRawReference + s_list_             :47-85, :519-523
 *       TensionSmoother2::osqpSmooth + spline     tension_smoother_2.cpp:20-72, tension_smoother.cpp:36-41
 *       or TensionSmoother::osqpSmooth (TENSION)  tension_smoother.cpp:20-177, clearance Map.cpp:16-22
 *       graphSearchDp, postSmooth                 reference_path_smoother.cpp:142-295, :526-580
 *     processReferencePath                        src/path_optimizer.cpp:73-122, src/tools/tools.cpp:57-126
 *     optimizePath (solve, re-solve, path)        src/path_optimizer.cpp:124-161, src/solver/base_solver.cpp
 * from the bSpline() samples of each path to its final path, device-resident on one stream. The stage
 * kernels are those of pqp_smoother.h, pqp_dp.h, pqp_bounds.h and pqp.h; this handle adds the steps that
 * connect them (natural spline fits, the 1 m resampling, the two smoother epilogues, the start / target
 * decisions and the solver's per-instance block) and reports per path which stage failed.
 *
 * bSpline() itself (tinyspline) and its "fewer than 4 reference points" check stay with the caller. There is
 * no CPU fallback. Every function returns a PQP_* code from pqp.h and never throws.
 */
#ifndef PQP_PLAN_H
#define PQP_PLAN_H

#include <stdint.h>

#include "pqp.h"
#include "pqp_bounds.h"
#include "pqp_dp.h"
#include "pqp_smoother.h"

#ifdef __cplusplus
extern "C" {
#endif

/* status[b]: the first stage that failed. Each code is one `return false` of the reference, except
 * SPLINE_DEGENERATE and the capacity codes, where the reference asserts or grows its vectors. */
enum {
    PQP_PLAN_OK = 0,
    PQP_PLAN_SPLINE_DEGENERATE = 1, /* fewer than 3 samples, or abscissae (arc lengths) not increasing */
    PQP_PLAN_TOO_MANY_POINTS = 2,   /* resampled list longer than p_max, or more DP layers than layers_max */
    PQP_PLAN_TENSION_FAILED = 3,    /* tension QP (either method) not solved (tension_smoother.cpp:32-35) */
    PQP_PLAN_DP_VEHICLE_FAR = 4,    /* graphSearchDp: |vehicle offset| > lateral range */
    PQP_PLAN_POST_TOO_SHORT = 5,    /* postSmooth: fewer than 4 DP layers kept */
    PQP_PLAN_POST_FAILED = 6,       /* post-smooth QP not solved */
    PQP_PLAN_EMPTY_REFERENCE = 7,   /* processReferencePath: smoothed length is 0 */
    PQP_PLAN_INIT_HEADING = 8,      /* |start heading error| > 75 deg */
    PQP_PLAN_TOO_MANY_KNOTS = 9,    /* more reference states than n_max (reported, never truncated) */
    PQP_PLAN_BLOCKED_AT_START = 10, /* fewer than 2 states before the first blocked one */
    PQP_PLAN_PRE_SOLVE_FAILED = 11, /* first solve not PQP_SOLVED (path_optimizer.cpp:142-146) */
    PQP_PLAN_SOLVE_FAILED = 12      /* re-solve not PQP_SOLVED (:153-157) */
};

#define PQP_PLAN_PATH_ROWS 7 /* x, y, heading, k, d_k, l, d_heading: the SlState fields getOptimizedPath sets */

/* pqp_plan_last_stage_ms: the TimeRecorder stages of PathOptimizer::solve (path_optimizer.cpp:41-69) */
enum {
    PQP_PLAN_STAGE_SMOOTHING = 0,    /* segmentation, tension QP, DP, post-smooth QP, reference spline */
    PQP_PLAN_STAGE_SEGMENTATION = 1, /* processReferencePath: start / target, reference states, bounds */
    PQP_PLAN_STAGE_OPTIMISATION = 2, /* both solves and the final path */
    PQP_PLAN_STAGE_TOTAL = 3,
    PQP_PLAN_NSTAGES = 4
};

typedef struct pqp_plan_params {
    pqp_params solver;
    pqp_bounds_params bounds;
    pqp_dp_params dp;
    pqp_smoother_params smoother;
    double output_spacing;            /* 0.3: states at (spacing / 2, spacing), path_optimizer.cpp:119 */
    double precise_planning_length;   /* 30 */
    int32_t dynamic_segmentation;     /* 1 */
    int32_t rough_constraints_far_away; /* 0: p[b] = n[b]; 1: p[b] = states with s < precise_planning_length */
    int32_t constraint_end_heading;   /* 1 */
    int32_t smoothing_method;         /* PQP_PLAN_SMOOTH_*: the reference's --smoothing_method (0 = TENSION2);
                                         any other value makes pqp_plan_create fail with PQP_E_INVALID */
} pqp_plan_params;

/* pqp_plan_params.smoothing_method (planning_flags.cpp:27-32, reference_path_smoother.cpp:17-29) */
enum {
    PQP_PLAN_SMOOTH_TENSION2 = 0, /* TensionSmoother2: Frenet-style QP over x, y, heading, curvature (default) */
    PQP_PLAN_SMOOTH_TENSION = 1   /* TensionSmoother: Cartesian QP over x, y and a lateral shift bounded by the map's
                                     obstacle distance at each resampled point (one more kernel per call; p_max <= 877
                                     on an H100, checked by pqp_plan_create) */
};

/* Inputs. Host pointers for pqp_plan, device pointers for pqp_plan_device. */
typedef struct pqp_plan_in {
    int32_t batch, r_max;   /* r_max: row stride of raw_x / raw_y, <= the handle's r_max */
    const double *raw_x;    /* [b][r_max] x_list_ of bSpline() */
    const double *raw_y;    /* [b][r_max] y_list_ */
    const int32_t *r;       /* [b] samples per path */
    const double *start;    /* [b][4] x, y, heading, k of the start state */
    const double *target;   /* [b][3] x, y, heading of the target state */
} pqp_plan_in;

/* Intermediate results per stage; every pointer is optional (NULL = not written). Same memory space as the
 * call's buffers. P = p_max, L = layers_max, N = n_max, R = r_max of the handle. A path that failed before a
 * stage has unspecified entries for that stage. */
typedef struct pqp_plan_trace {
    double *raw_spline;      /* [b][PQP_SPLINE_ROWS][R] fit of the raw samples (row 0 = s_list_) */
    int32_t *seg_p;          /* [b] resampled points */
    double *seg_x, *seg_y, *seg_angle, *seg_k, *seg_s; /* [b][P] segmentRawReference's lists */
    double *tension_x, *tension_y, *tension_s;          /* [b][P] */
    int32_t *tension_status, *tension_iters;            /* [b] */
    double *tension_spline;  /* [b][PQP_SPLINE_ROWS][P] */
    double *tension_length;  /* [b] result_s.back() + 3 */
    int32_t *dp_status, *dp_n_out;                      /* [b] PQP_DP_*, kept layers */
    double *dp_layer_s, *dp_lower, *dp_upper;           /* [b][L] */
    int32_t *dp_chosen;                                 /* [b][L] */
    double *dp_vehicle_l;                               /* [b] */
    double *post_offsets;                               /* [b][L] */
    int32_t *post_status, *post_iters;                  /* [b] */
    double *ref_spline;      /* [b][PQP_SPLINE_ROWS][L] final reference spline (k = dp_n_out) */
    double *max_s;           /* [b] reference length after setReferencePathLength */
    double *states;          /* [b][PQP_STATE_ROWS][N] */
    double *curvature;       /* [b][N] */
    int32_t *total;          /* [b] states buildReferenceFromSpline emits (no n_max cap) */
    double *bounds;          /* [b][PQP_BOUND_ROWS][N] */
    int32_t *n_valid;        /* [b] */
    double *knots;           /* [b][PQP_NFIELDS][N] as passed to the first solve */
    double *inst;            /* [b][PQP_NINST]: l0, psi0 (written by processInitState), k0, end-heading rows */
    int32_t *p;              /* [b] precise knots */
    double *sol1;            /* [b][4][N] first solution */
    int32_t *status1, *iters1;
    double *x_full1, *y_full1, *z_full1; /* as pqp_batch_out, first solve */
    double *x_full2, *y_full2, *z_full2; /* second solve */
    double *tension_clearance; /* [b][P] obstacle distance at the seg_x / seg_y points (TENSION only; untouched
                                  under TENSION2) */
} pqp_plan_trace;

typedef struct pqp_plan_out {
    int32_t *status;        /* [b] PQP_PLAN_* */
    int32_t *n;             /* [b] knots of the final path (0 unless OK) */
    double *path;           /* [b][PQP_PLAN_PATH_ROWS][n_max] (entries i >= n[b] are 0) */
    double *cost;           /* [b] cost of the second solve */
    int32_t *iters;         /* [b][2] ADMM iterations of the two solves */
    pqp_plan_trace *trace;  /* optional (host struct; its pointers as above) */
} pqp_plan_out;

typedef struct pqp_plan_handle pqp_plan_handle;

void pqp_plan_default_params(pqp_plan_params *p);
/* One map (copied), 1 <= batch_max, r_max >= 3, p_max >= 4, layers_max >= 4, 2 <= n_max <= 511. All device
 * memory is allocated here; the plan calls allocate nothing. */
int pqp_plan_create(const pqp_bounds_map *map, const pqp_plan_params *params, int32_t r_max, int32_t p_max,
                    int32_t layers_max, int32_t n_max, int32_t batch_max, int32_t device, pqp_plan_handle **out);
void pqp_plan_destroy(pqp_plan_handle *h);
/* Host buffers; synchronous. */
int pqp_plan(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out);
/* Device buffers; asynchronous on `stream` (a cudaStream_t passed as void*): no host synchronisation, no
 * allocation. Solves are FP32 without the FP64 re-solve (pqp.h, *_device): an infeasible instance the FP32
 * certificate cannot resolve ends as PQP_PLAN_PRE_SOLVE_FAILED. pqp_plan uses this same path. */
int pqp_plan_device(pqp_plan_handle *h, const pqp_plan_in *in, const pqp_plan_out *out, void *stream);
/* ms[PQP_PLAN_NSTAGES] of the last call (CUDA events; waits for that call to finish). */
int pqp_plan_last_stage_ms(pqp_plan_handle *h, float *ms);
/* Kernel launches issued by the handle so far: the glue kernels plus those of every stage handle it owns. */
int pqp_plan_launch_count(pqp_plan_handle *h, int64_t *count);
const char *pqp_plan_last_error(const pqp_plan_handle *h); /* h may be NULL: last create error */

#ifdef __cplusplus
}
#endif
#endif /* PQP_PLAN_H */
