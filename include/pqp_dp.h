/*
 * pqp_dp.h — C ABI of the lattice DP search of the reference's front end (SURVEY.md §8 row f-4).
 *
 * reference interface replaced:
 *   ReferencePathSmoother::graphSearchDp   src/reference_path_smoother/reference_path_smoother.cpp:142-295
 *   ReferencePathSmoother::calculateCostAt :107-140
 * for a BATCH of reference paths over one shared obstacle map (BASELINE configs[1]): per path, layers every
 * 1.5 m along the smoothed reference, 34 lateral samples per layer (-10 .. 9.8 m, 0.6 m apart), feasibility
 * from the distance map and the curvature centre, a layered min-plus search with the reference's cost terms
 * and first-minimum tie rule, then the chosen corridor's lateral bounds per layer (what postSmooth consumes:
 * layers_s_list_, layers_bounds_, vehicle_l_wrt_smoothed_ref_, :526-636).
 *
 * The map lives in a pqp_bounds_handle (include/pqp_bounds.h); a pqp_dp_handle adds the search's scratch.
 * Index outputs (chosen, parent) are exact; costs are FP64 sums of atan2 / sin / cos terms and agree with a
 * libm evaluation to a few ulp. No CPU fallback.
 */
#ifndef PQP_DP_H
#define PQP_DP_H

#include <stdint.h>

#include "pqp_bounds.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pqp_dp_params {
    double lateral_range;        /* 10.0  FLAGS_search_lateral_range        (planning_flags.cpp:38) */
    double lateral_spacing;      /* 0.6   FLAGS_search_lateral_spacing      (:42) */
    double longitudinal_spacing; /* 1.5   FLAGS_search_longitudial_spacing  (:40) */
    double car_width;            /* 2.0   FLAGS_car_width                   (:10) */
} pqp_dp_params;

#define PQP_DP_LATERAL_MAX 64 /* lateral samples per layer the kernel is laid out for (34 at the defaults) */

/* status per path */
enum {
    PQP_DP_OK = 1,              /* graphSearchDp returned true */
    PQP_DP_VEHICLE_FAR = 0,     /* |vehicle offset| > lateral range: the reference returns false (:167-170) */
    PQP_DP_TOO_MANY_LAYERS = -1, /* more layers than the handle's layers_max: nothing searched */
    PQP_DP_MAP_INDEX = -2        /* pqp_dp_search_mapped*: map index outside [0, n_maps); no map read, n_layers =
                                    n_out = 0 and the other outputs of the path unspecified */
};

typedef struct pqp_dp_in {
    int32_t batch, k_max;
    const double *spline;  /* [b][PQP_SPLINE_ROWS][k_max]: the smoothed reference x(s), y(s) (same abscissae) */
    const int32_t *k;      /* [b] spline points */
    const double *length;  /* [b] reference->getLength() (may exceed the last abscissa: TensionSmoother adds 3 m) */
    const double *start;   /* [b][3]: start_state_ x, y, heading */
} pqp_dp_in;

/* layers_max = the handle's; lateral = pqp_dp_lateral_count(). Tables are optional (may be NULL). */
typedef struct pqp_dp_out {
    int32_t *status;     /* [b] PQP_DP_* */
    int32_t *n_layers;   /* [b] layers sampled (layers_s_list_ before the resize) */
    int32_t *n_out;      /* [b] layers kept = max layer reached + 1 (size of layers_bounds_) */
    double *layer_s;     /* [b][layers_max] */
    double *lower;       /* [b][layers_max] layers_bounds_[i].first  */
    double *upper;       /* [b][layers_max] layers_bounds_[i].second */
    int32_t *chosen;     /* [b][layers_max] lateral index of the chosen node per kept layer */
    double *vehicle_l;   /* [b] vehicle_l_wrt_smoothed_ref_ */
    double *target_s;    /* [b] target_s_ */
    double *cost;        /* optional [b][layers_max][lateral]: DpPoint::cost (DBL_MAX = not reached) */
    int8_t *parent;      /* optional [b][layers_max][lateral]: lateral index of DpPoint::parent, -1 = none */
    uint8_t *feasible;   /* optional [b][layers_max][lateral]: DpPoint::is_feasible */
} pqp_dp_out;

typedef struct pqp_dp_handle pqp_dp_handle;

void pqp_dp_default_params(pqp_dp_params *p);
/* `map_owner` supplies the distance layer and the device; it must outlive the DP handle. */
int pqp_dp_create(pqp_bounds_handle *map_owner, const pqp_dp_params *params, int32_t layers_max, int32_t batch_max,
                  pqp_dp_handle **out);
void pqp_dp_destroy(pqp_dp_handle *h);
int32_t pqp_dp_lateral_count(const pqp_dp_handle *h);
/* Host buffers in and out (H2D, one kernel, D2H; synchronous). */
int pqp_dp_search(pqp_dp_handle *h, const pqp_dp_in *in, const pqp_dp_out *out);
/* Device buffers; asynchronous on `stream` (a cudaStream_t passed as void*). Optional tables that are NULL are
 * kept in the handle's own scratch. */
int pqp_dp_search_device(pqp_dp_handle *h, const pqp_dp_in *in, const pqp_dp_out *out, void *stream);
/* As pqp_dp_search(_device), path b on map slot map_index[b] of the map owner (pqp_bounds_create_maps);
 * map_index [batch] in the memory space of the other buffers. */
int pqp_dp_search_mapped(pqp_dp_handle *h, const pqp_dp_in *in, const int32_t *map_index, const pqp_dp_out *out);
int pqp_dp_search_mapped_device(pqp_dp_handle *h, const pqp_dp_in *in, const int32_t *map_index, const pqp_dp_out *out,
                                void *stream);
int pqp_dp_last_kernel_ms(pqp_dp_handle *h, float *ms);
const char *pqp_dp_last_error(const pqp_dp_handle *h); /* h may be NULL: last create error */

#ifdef __cplusplus
}
#endif
#endif /* PQP_DP_H */
