/* pqp_bounds.h — C ABI of the clearance-bounds front end (SURVEY.md §8 row f-1, "next").
 *
 * Replaces, for a batch of reference paths over one obstacle map (or one map per path, pqp_bounds_create_maps):
 *   ReferencePathImpl::updateBoundsImproved        src/data_struct/reference_path_impl.cpp:177-230
 *   ReferencePathImpl::getClearanceWithDirectionStrict                             ...:232-312
 *   getDirectionalProjectionByNewton               src/tools/tools.cpp:156-189
 *   tk::spline::operator() / deriv                 src/tools/spline.cpp:252-330
 *   Map::getObstacleDistance                       src/tools/Map.cpp:16-22 (grid_map bilinear lookup)
 *
 * One CUDA thread per (path, knot, anchor in {front, rear, centre}); FP64 arithmetic like the
 * reference; the float distance layer of the map stays resident in HBM/L2 for the life of the
 * handle. Output feeds pqp_solve directly (bounds can be written into the solver's knot block).
 * Plain pointers and sizes only; every function returns a PQP_* code from pqp.h and never throws.
 * There is no CPU fallback.
 */
#ifndef PQP_BOUNDS_H
#define PQP_BOUNDS_H

#include <stdint.h>

#include "pqp.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The map's "distance" layer as grid_map holds it (demo.cpp:98-113): float, rows x cols,
 * row-major [i * cols + j]; cell (i, j) is centred at
 *   (center_x + length_x / 2 - (i + 1/2) resolution, center_y + length_y / 2 - (j + 1/2) resolution)
 * with length_x = rows * resolution, length_y = cols * resolution. Host pointer; copied at create (and replaceable
 * later, pqp_bounds_set_map below). */
typedef struct pqp_bounds_map {
    int32_t rows, cols;
    double resolution;
    double center_x, center_y;
    const float *distance;
} pqp_bounds_map;

/* The gflags the reference's bounds code reads (src/config/planning_flags.cpp). The search
 * constants hard-coded in reference_path_impl.cpp:237-277 (0.5 m radius, 0.3 m / 0.05 m steps,
 * 6 m range, 0.2 m minimum space) and tools.cpp:166 (20 Newton steps, 1e-5) are hard-coded here too. */
typedef struct pqp_bounds_params {
    double front_length;   /* 3.9  */
    double rear_length;    /* -1.0 */
    double car_width;      /* 2.0  */
    double safety_margin;  /* 0.3  */
    double epsilon;        /* 1e-6: isEqual() tolerance of the "path is blocked" test */
} pqp_bounds_params;

#define PQP_SPLINE_ROWS 9 /* abscissa; a, b, c, y of x(s); a, b, c, y of y(s)  (tk::spline m_x, m_a, m_b, m_c, m_y) */
#define PQP_STATE_ROWS 4  /* s, x, y, heading of a reference state */
#define PQP_BOUND_ROWS 6  /* front lb, front ub, rear lb, rear ub, centre lb, centre ub */

typedef struct pqp_bounds_in {
    int32_t batch, n_max, k_max;
    const double *states;   /* [b][PQP_STATE_ROWS][n_max]  reference_states_ */
    const int32_t *n;       /* [b] number of reference states */
    const double *spline;   /* [b][PQP_SPLINE_ROWS][k_max]  x_s_, y_s_ (same abscissae) */
    const int32_t *k;       /* [b] number of spline points (>= 3) */
} pqp_bounds_in;

typedef struct pqp_bounds_out {
    double *bounds;      /* [b][PQP_BOUND_ROWS][n_max]; entries at i >= n_valid[b] are unspecified */
    int32_t *n_valid;    /* [b] index of the first blocked state (= n[b] when none): the size
                            reference_states_ is cut to (reference_path_impl.cpp:222-229) */
    double *knots;       /* optional: solver knot block [b][PQP_NFIELDS][n_max]; receives the
                            front bounds in PQP_F_B0_LB/UB and the rear bounds in PQP_F_B1_LB/UB */
} pqp_bounds_out;

/* ReferencePathImpl::buildReferenceFromSpline (reference_path_impl.cpp:314-338; SURVEY.md §8 f-2):
 * walk each spline from s = 0 to max_s with the curvature-dependent step (delta_s_larger where
 * |k| < 0.08, delta_s_smaller where |k| > 0.2, linear in between; fixed delta_s_larger when
 * dynamic_segmentation = 0) and emit x, y, heading (tools.cpp:32-36), curvature (:38-44), s. */
typedef struct pqp_states_in {
    int32_t batch, n_max, k_max;
    const double *spline;   /* [b][PQP_SPLINE_ROWS][k_max] */
    const int32_t *k;       /* [b] */
    const double *max_s;    /* [b] max_s_ of the reference path */
    double delta_s_smaller; /* 0.15 (path_optimizer.cpp: buildReferenceFromSpline(0.15, 0.3)) */
    double delta_s_larger;  /* 0.3 */
    int32_t dynamic_segmentation; /* FLAGS_enable_dynamic_segmentation (default true) */
} pqp_states_in;

typedef struct pqp_states_out {
    double *states;     /* [b][PQP_STATE_ROWS][n_max]: s, x, y, heading */
    double *curvature;  /* [b][n_max] */
    int32_t *n;         /* [b] states written = min(total, n_max) */
    int32_t *total;     /* optional [b]: states the reference would emit (no n_max cap) */
    double *knots;      /* optional solver knot block [b][PQP_NFIELDS][n_max]: receives PQP_F_S,
                           PQP_F_KREF and the first linearisation point of path_optimizer.cpp:128-137
                           (PQP_F_L = PQP_F_PSI = 0, PQP_F_K = curvature) */
} pqp_states_out;

typedef struct pqp_bounds_handle pqp_bounds_handle;

void pqp_bounds_default_params(pqp_bounds_params *p);
int pqp_bounds_create(const pqp_bounds_map *map, const pqp_bounds_params *params, int32_t device,
                      pqp_bounds_handle **out);
void pqp_bounds_destroy(pqp_bounds_handle *h);
/* Host buffers in, host buffers out (H2D, kernel, D2H; synchronous). */
int pqp_bounds_compute(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out);
/* Device buffers; asynchronous on `stream` (a cudaStream_t passed as void*). */
int pqp_bounds_compute_device(pqp_bounds_handle *h, const pqp_bounds_in *in, const pqp_bounds_out *out,
                              void *stream);
/* buildReferenceFromSpline for a batch: host buffers (synchronous) / device buffers (async). */
int pqp_bounds_build_states(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out);
int pqp_bounds_build_states_device(pqp_bounds_handle *h, const pqp_states_in *in, const pqp_states_out *out,
                                   void *stream);
int pqp_bounds_last_kernel_ms(pqp_bounds_handle *h, float *ms);
const char *pqp_bounds_last_error(pqp_bounds_handle *h);

/* An occupancy image, from which the set_occupancy calls compute the distance layer on the GPU. cells is
 * uint8, rows x cols, row-major, in the cell convention of pqp_bounds_map; cell k is an obstacle when
 * cells[k] <= obstacle_max (0: obstacles are the zero pixels, as demo.cpp:98-113 measures them; 127: what
 * sharedmap.DistanceMap thresholds). */
typedef struct pqp_occupancy_map {
    int32_t rows, cols;
    double resolution;
    double center_x, center_y;
    const uint8_t *cells;     /* [rows * cols]: host pointer for pqp_bounds_set_occupancy, device pointer for
                                 pqp_bounds_set_occupancy_device */
    int32_t obstacle_max;
} pqp_occupancy_map;

/* Replacing the map of a live handle (a receding-horizon host gets a new map every tick). No call
 * allocates. rows, cols, resolution and the centre may all change; the map must have rows, cols >= 2,
 * rows * cols no more than the cells the handle was created with, a finite resolution > 0, finite centres
 * and non-NULL pointers. A refused map returns PQP_E_INVALID with last_error set and leaves the handle's map
 * (metadata and layer) untouched.
 *
 * The *_device calls are ordered on `stream`: work already enqueued there sees the old map, work enqueued
 * after it the new one. Across streams the caller orders, as for every other *_device call. The host calls
 * run on the handle's own stream and return when the new map is in place.
 *
 * set_map: the float distance layer as pqp_bounds_create takes it, copied.
 * set_occupancy: the exact Euclidean distance transform of the image, on the GPU:
 *     d2(i, j) = min over obstacle cells (i', j') of (i - i')^2 + (j - j')^2   (exact, integer)
 *     layer    = (float)sqrt((double)d2) * (float)resolution
 *   i.e. scipy.ndimage.distance_transform_edt(cells > obstacle_max).astype(float32) * float32(resolution) bit
 *   for bit; obstacle cells are 0; an image with no obstacle at all gives (float)2^64 * (float)resolution per
 *   cell, as OpenCV's precise transform does. rows, cols <= 16384. Two kernel launches, in place in the
 *   distance layer; the host call first copies the image into a staging buffer allocated at create (1 byte
 *   per cell).
 * get_map: the current metadata (meta->distance is set to NULL) and, when distance is not NULL, a copy of the
 *   layer into distance[rows * cols]; waits for all work on the device first. */
int pqp_bounds_set_map(pqp_bounds_handle *h, const pqp_bounds_map *map);
int pqp_bounds_set_map_device(pqp_bounds_handle *h, const pqp_bounds_map *map, void *stream);
int pqp_bounds_set_occupancy(pqp_bounds_handle *h, const pqp_occupancy_map *occ);
int pqp_bounds_set_occupancy_device(pqp_bounds_handle *h, const pqp_occupancy_map *occ, void *stream);
int pqp_bounds_get_map(pqp_bounds_handle *h, pqp_bounds_map *meta, float *distance);

/* Per-path maps: a handle holds n_maps map slots (1 <= n_maps <= PQP_MAX_MAP_SLOTS), each with the capacity of the
 * largest of the maps it was created with; the *_mapped calls plan path b on slot map_index[b]. A handle made by
 * pqp_bounds_create has one slot, and every call above acts on slot 0. Memory: 5 bytes per cell per slot (the float
 * layer and the 1-byte occupancy staging), plus the staging of the host set_occupancy_boxes call: PQP_MAX_BOXES *
 * PQP_BOX_FIELDS doubles (2.5 MiB) and 4 bytes per slot; all allocated at create, a failed allocation returns
 * PQP_E_CUDA.
 *
 * The map-reading kernels index a device table of the slots' metadata. Slot updates write their entries with a
 * kernel launch on the update's stream, so they keep the ordering of the calls above: work enqueued before an update
 * sees the old slot, work enqueued after the new one, and no update waits for the host. Launches per update:
 *   set_map_slot(_device), and pqp_bounds_set_map(_device):        1 (the table entry; the layer is a copy)
 *   pqp_bounds_set_occupancy(_device):                             2 (the entry is written by the column pass)
 *   set_occupancy_slots(_device):   2 + ceil(count / PQP_MAP_TABLE_CHUNK) (column pass, row pass, table entries)
 *   set_occupancy_boxes(_device):   the same (the boxes are stamped inside the column pass)
 *
 * A slot update is refused (PQP_E_INVALID, every slot untouched) for a slot outside [0, n_maps) or anything
 * pqp_bounds_set_map / pqp_bounds_set_occupancy refuse. */
#define PQP_MAX_MAP_SLOTS 65535
#define PQP_MAP_TABLE_CHUNK 1024 /* table entries one table-write launch carries in its parameters */

/* count occupancy images of one size, [count][rows][cols] uint8 (host pointer for set_occupancy_slots, device
 * pointer for set_occupancy_slots_device), each with its own centre; resolution and obstacle_max are shared. */
typedef struct pqp_occupancy_stack {
    int32_t count, rows, cols;
    double resolution;
    const double *center_x;   /* [count], host */
    const double *center_y;   /* [count], host */
    const uint8_t *cells;     /* [count][rows][cols] */
    int32_t obstacle_max;
} pqp_occupancy_stack;

int pqp_bounds_create_maps(const pqp_bounds_map *maps, int32_t n_maps, const pqp_bounds_params *params,
                           int32_t device, pqp_bounds_handle **out);
int pqp_bounds_set_map_slot(pqp_bounds_handle *h, int32_t slot, const pqp_bounds_map *map);
int pqp_bounds_set_map_slot_device(pqp_bounds_handle *h, int32_t slot, const pqp_bounds_map *map, void *stream);
/* The images go into slots first_slot .. first_slot + count - 1: the exact distance transform of each, as
 * pqp_bounds_set_occupancy computes it for one image. The column pass runs on grid (ceil(cols / 128), count), the row
 * pass on grid (rows, count). The host call copies the stack into the slots' staging and returns when done. */
int pqp_bounds_set_occupancy_slots(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *stack);
int pqp_bounds_set_occupancy_slots_device(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *stack,
                                          void *stream);
/* Obstacle boxes per slot on a static occupancy image (a tick of tracked vehicles and pedestrians on a fixed map).
 *
 * A box is PQP_BOX_FIELDS doubles x, y, heading, length, width in the map's world frame (the frame of the paths),
 * placed like the car of the collision check: centred at (x, y), its length along the heading. Cell (i, j) of a slot
 * is an obstacle when its base image byte is <= obstacle_max (as in pqp_bounds_set_occupancy), or when its centre
 * lies inside or on the boundary of any box of that slot:
 *     px = cx + (half_lx - (i + 0.5) res)     py = cy + (half_ly - (j + 0.5) res)     (the pqp_bounds_map convention,
 *                                              half_lx = 0.5 * rows * res, half_ly = 0.5 * cols * res)
 *     dx = px - x   dy = py - y   c = cos(heading)   s = sin(heading)
 *     u  = dx c + dy s              v = dy c - dx s
 *     inside  <=>  |u| <= 0.5 length  &&  |v| <= 0.5 width
 * Every product and sum rounds on its own (no fused multiply-add); c and s are computed in FP64 on the device. So a
 * box with a NaN field or a negative length or width stamps nothing, a box of zero size stamps only a cell whose
 * centre it hits exactly, and a box partly or wholly off the map stamps the cells it covers, or none. The slot's layer
 * is then the exact distance transform of the combined obstacles, as pqp_bounds_set_occupancy documents it (scipy's
 * distance_transform_edt bit for bit). The base image is read and never written.
 *
 * base: count, rows, cols, resolution, obstacle_max and the per-slot centres as in pqp_bounds_set_occupancy_slots, into
 *   slots first_slot .. first_slot + count - 1. shared_base = 1: base->cells is one [rows][cols] image every slot starts
 *   from; 0: count images [count][rows][cols].
 * boxes: slot first_slot + s gets boxes->boxes[s][0 .. k[s] - 1].
 * The host form takes host pointers, stages the image(s) and the boxes into buffers allocated at create and returns
 * when done; the device form takes device pointers (base->cells, k and boxes; the centres stay host arrays) and is
 * asynchronous on `stream`, with the ordering of set_occupancy_slots_device and no host synchronisation. The device
 * form clamps k[s] to [0, k_max]; the host form refuses a k[s] outside it.
 * Refused with PQP_E_INVALID, every slot untouched: anything set_occupancy_slots refuses, shared_base not 0 or 1, a
 * NULL boxes, k_max < 0, count * k_max > PQP_MAX_BOXES, k_max > 0 with a NULL k or boxes->boxes, and (host form) a
 * k[s] outside [0, k_max]. */
#define PQP_BOX_FIELDS 5      /* x, y, heading, length, width */
#define PQP_MAX_BOXES 65536   /* count * k_max per call, every form */
typedef struct pqp_obstacle_boxes {
    int32_t k_max;            /* row stride of boxes, >= 0; k and boxes may be NULL when 0 */
    const int32_t *k;         /* [count]: boxes of slot first_slot + s */
    const double *boxes;      /* [count][k_max][PQP_BOX_FIELDS] */
} pqp_obstacle_boxes;
int pqp_bounds_set_occupancy_boxes(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *base,
                                   int32_t shared_base, const pqp_obstacle_boxes *boxes);
int pqp_bounds_set_occupancy_boxes_device(pqp_bounds_handle *h, int32_t first_slot, const pqp_occupancy_stack *base,
                                          int32_t shared_base, const pqp_obstacle_boxes *boxes, void *stream);
/* As pqp_bounds_get_map for one slot. */
int pqp_bounds_get_map_slot(pqp_bounds_handle *h, int32_t slot, pqp_bounds_map *meta, float *distance);
int32_t pqp_bounds_map_count(const pqp_bounds_handle *h);
/* As pqp_bounds_compute(_device), path b on slot map_index[b] (map_index [batch] in the memory space of the other
 * buffers). A path whose index is outside [0, n_maps) reads no map and gets n_valid = 0. */
int pqp_bounds_compute_mapped(pqp_bounds_handle *h, const pqp_bounds_in *in, const int32_t *map_index,
                              const pqp_bounds_out *out);
int pqp_bounds_compute_mapped_device(pqp_bounds_handle *h, const pqp_bounds_in *in, const int32_t *map_index,
                                     const pqp_bounds_out *out, void *stream);

/* Footprint collision check of a batch of poses against the map (CollisionChecker, src/tools/collision_checker.cpp:
 * 17-59, with CarGeometry(car_width, |rear_length|, front_length), src/tools/car_geometry.cpp:10-73, from the handle's
 * pqp_bounds_params). A pose is free under isSingleStateCollisionFreeImproved: the car's bounding circle, placed with
 * local2Global (tools.cpp:50-55), must have its centre strictly inside the map; if its interpolated obstacle distance
 * is not below its radius the pose is free, otherwise it is free only if each of the six footprint circles (rr, rl,
 * fr, fl, fm, rm) has its centre inside the map and a distance not below its radius. The comparisons are the
 * reference's: a NaN distance is not below a radius, and a pose the bounding circle clears is free even where a small
 * circle's distance is below its radius. Nothing here changes a plan: a caller enqueues the check after a plan call on
 * the same stream with the same map_index, e.g. on pqp_plan_out.path with row_stride PQP_PLAN_PATH_ROWS. */
typedef struct pqp_collision_in {
    int32_t batch, n_max;
    int32_t row_stride;   /* rows per path: PQP_PLAN_PATH_ROWS for pqp_plan_out.path, PQP_STATE_ROWS for states */
    const double *poses;  /* [b][row_stride][n_max]; rows 0, 1, 2 = x, y, heading. Reference states:
                             states + n_max with row_stride PQP_STATE_ROWS */
    const int32_t *n;     /* [b], clamped to [0, n_max] as the bounds kernel clamps it */
} pqp_collision_in;

typedef struct pqp_collision_out {
    int32_t *first_hit;   /* [b]: index of the first pose that is not free, n[b] when all are (0 for n[b] = 0); -1 for
                             a mapped call's index outside [0, n_maps) */
    uint8_t *state_free;  /* optional [b][n_max]: the per-pose verdict (0 at i >= n[b]) */
    double *clearance;    /* optional [b][n_max]: min over the six circles of d_i - r_i (the exact test's margin; it can
                             be negative on a pose the bounding-circle shortcut passes; 0 at i >= n[b]) */
} pqp_collision_out;

/* One kernel launch per call, one CTA per path; pqp_bounds_last_kernel_ms reports it. The host form copies exactly the
 * ((batch - 1) * row_stride + 3) * n_max doubles of poses the check reads, so states + n_max is a valid argument, and
 * returns when the outputs are in place; the *_device forms take device buffers and are asynchronous on `stream`.
 * The mapped forms check path b on slot map_index[b] (map_index [batch] in the memory space of the other buffers); a
 * path whose index is outside [0, n_maps) reads no map. Refused with PQP_E_INVALID: batch <= 0, n_max <= 0,
 * row_stride < 3, a NULL poses, n or first_hit, a NULL map_index in a mapped form. */
int pqp_bounds_collision_check(pqp_bounds_handle *h, const pqp_collision_in *in, const pqp_collision_out *out);
int pqp_bounds_collision_check_device(pqp_bounds_handle *h, const pqp_collision_in *in, const pqp_collision_out *out,
                                      void *stream);
int pqp_bounds_collision_check_mapped(pqp_bounds_handle *h, const pqp_collision_in *in, const int32_t *map_index,
                                      const pqp_collision_out *out);
int pqp_bounds_collision_check_mapped_device(pqp_bounds_handle *h, const pqp_collision_in *in,
                                             const int32_t *map_index, const pqp_collision_out *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif
