/*
 * pqp_smoother.h — C ABI of the reference-line smoother QPs (SURVEY.md §8 row f-3), batched on the GPU.
 *
 * reference interfaces replaced (both build a QP and hand it to OSQP with default settings, eps 1e-3):
 *   TensionSmoother2::osqpSmooth            src/reference_path_smoother/tension_smoother_2.cpp:20-72
 *     (setHessianMatrix :74-96, setConstraintMatrix :98-142, setGradient :143-157)
 *   TensionSmoother::osqpSmooth             src/reference_path_smoother/tension_smoother.cpp:49-100
 *     (setHessianMatrix :102-126, setConstraintMatrix :128-177) - the smoother of --smoothing_method=TENSION
 *   ReferencePathSmoother::postSmooth (QP)  src/reference_path_smoother/reference_path_smoother.cpp:526-558
 *     (setPostHessianMatrix :584-597, setPostConstraintMatrix :599-636)
 * for a batch of paths: one warp per QP runs OSQP's algorithm (Ruiz scaling, rho vector, relaxed ADMM step on the
 * reduced banded system, unscaled termination test, certificates, adaptive rho) in FP64. Outputs are what the
 * reference reads from OSQP's solution: the smoothed points + re-accumulated arc length, resp. the lateral offset per
 * DP layer. No CPU fallback.
 */
#ifndef PQP_SMOOTHER_H
#define PQP_SMOOTHER_H

#include <stdint.h>

#include "pqp.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pqp_smoother_params {
    /* TensionSmoother2 weights (planning_flags.cpp:57-61) */
    double tension_deviation_weight;       /* 0.005 */
    double tension_curvature_weight;       /* 1     */
    double tension_curvature_rate_weight;  /* 10    */
    /* postSmooth weights (reference_path_smoother.cpp:590-592) */
    double post_weight_x, post_weight_dx, post_weight_ddx; /* 1, 100, 1000 */
    /* OSQP settings: the library defaults (the reference sets only verbosity and warm start) */
    double rho, sigma, alpha;              /* 0.1, 1e-6, 1.6 */
    double eps_abs, eps_rel;               /* 1e-3, 1e-3 */
    double eps_prim_inf, eps_dual_inf;     /* 1e-4, 1e-4 */
    double adaptive_rho_tolerance;         /* 5 */
    int32_t max_iter, check_termination, scaling, adaptive_rho; /* 4000, 25, 10, 1 */
    int32_t adaptive_rho_interval;         /* 25: fixed (OSQP's default 0 derives it from wall-clock time) */
    int32_t reserved;
    /* TensionSmoother weights (planning_flags.cpp:51-55) */
    double cartesian_curvature_weight;       /* 1  */
    double cartesian_curvature_rate_weight;  /* 50 */
    double cartesian_deviation_weight;       /* 0  */
} pqp_smoother_params;

/* TensionSmoother2::osqpSmooth for a batch. Lists are [b][p_max] (the raw reference resampled at 1 m by
 * segmentRawReference, :46-84: x, y, heading, curvature, arc length), p[b] >= 3 points each. */
typedef struct pqp_tension_in {
    int32_t batch, p_max;
    const int32_t *p;
    const double *x, *y, *angle, *k, *s;
} pqp_tension_in;
typedef struct pqp_tension_out {
    double *x, *y, *s;   /* [b][p_max] result_x_list, result_y_list, result_s_list */
    int32_t *status;     /* [b] PQP_* solver status (the reference fails unless PQP_SOLVED) */
    int32_t *iters;      /* [b] */
    double *x_full;      /* optional [b][4 p_max]: the whole primal vector in the reference's index order
                            (x block, y block, theta block, k block; 4 p - 1 entries) */
} pqp_tension_out;

/* TensionSmoother::osqpSmooth for a batch: per path the resampled points (x, y, heading as for pqp_tension_in) and
 * clearance[b][i] = Map::getObstacleDistance(x_i, y_i) (0 off the map; read for interior points only), p[b] >= 3.
 * Lists are [b][p_max]. The QP has 3 p variables (x, y and the lateral shift d of each point); d_i stays within
 * +-min(clearance_i, 2), d_0 = 0, |d_{p-1}| <= 0.5. Written into a pqp_tension_out whose optional x_full is
 * [b][3 p_max]: x block, y block, d block. The band of this QP is wider than TENSION2's: a handle serves it up to
 * p_max = 877 on an H100 (227 KB of shared memory per block); beyond that these two calls return PQP_E_INVALID
 * and the handle's other calls still work. */
typedef struct pqp_cartesian_tension_in {
    int32_t batch, p_max;
    const int32_t *p;
    const double *x, *y, *angle, *clearance;
} pqp_cartesian_tension_in;

/* postSmooth's QP for a batch: per path the kept DP layers (include/pqp_dp.h outputs: layer_s, lower, upper,
 * vehicle_l), p[b] >= 4 layers. offsets[b][i] = QPSolution(i), the lateral offset of layer i. */
typedef struct pqp_post_in {
    int32_t batch, p_max;
    const int32_t *p;
    const double *layer_s, *lower, *upper;  /* [b][p_max] */
    const double *vehicle_l;                /* [b] */
} pqp_post_in;
typedef struct pqp_post_out {
    double *offsets;     /* [b][p_max] */
    int32_t *status, *iters;
    double *x_full;      /* optional [b][3 p_max]: x block, dx block, ddx block */
} pqp_post_out;

typedef struct pqp_smoother_handle pqp_smoother_handle;

void pqp_smoother_default_params(pqp_smoother_params *p);
int pqp_smoother_create(const pqp_smoother_params *params, int32_t p_max, int32_t batch_max, int32_t device,
                        pqp_smoother_handle **out);
void pqp_smoother_destroy(pqp_smoother_handle *h);
/* Host buffers (H2D, one kernel, D2H; synchronous). */
int pqp_tension_smooth(pqp_smoother_handle *h, const pqp_tension_in *in, const pqp_tension_out *out);
int pqp_post_smooth(pqp_smoother_handle *h, const pqp_post_in *in, const pqp_post_out *out);
int pqp_cartesian_tension_smooth(pqp_smoother_handle *h, const pqp_cartesian_tension_in *in, const pqp_tension_out *out);
/* Device buffers, asynchronous on `stream` (a cudaStream_t passed as void*). */
int pqp_tension_smooth_device(pqp_smoother_handle *h, const pqp_tension_in *in, const pqp_tension_out *out, void *stream);
int pqp_post_smooth_device(pqp_smoother_handle *h, const pqp_post_in *in, const pqp_post_out *out, void *stream);
int pqp_cartesian_tension_smooth_device(pqp_smoother_handle *h, const pqp_cartesian_tension_in *in,
                                        const pqp_tension_out *out, void *stream);
int pqp_smoother_last_kernel_ms(pqp_smoother_handle *h, float *ms);
const char *pqp_smoother_last_error(const pqp_smoother_handle *h); /* h may be NULL: last create error */

#ifdef __cplusplus
}
#endif
#endif /* PQP_SMOOTHER_H */
