/*
 * pqp_plan_multi.h — the whole plan (pqp_plan.h) over the GPUs of one box, behind the C ABI.
 *
 * One pqp_plan_handle per device, each created by pqp_plan_create_maps with the same params and capacities and its own
 * copy of every map slot; the batch is sharded in contiguous blocks exactly as pqp_multi.h shards it: per =
 * ceil(batch / n_devices), device index i plans paths [i * per, min(batch, (i + 1) * per)) (an empty shard when
 * batch < n_devices). Every plan is independent of the others, so there is no collective: results land in the caller's
 * host buffers, or on the home device (devices[0]) by peer copies. Built on the public single-device plan ABI only.
 *
 * Memory: every device holds every slot, as pqp_plan_create_maps allocates it (a float32 distance layer and the uint8
 * staging of the host-form occupancy update: 5 B per cell per slot, 2.55 GB for 1024 demo-sized slots), and each
 * device other than the home one 1 B per cell per slot more: the staging that the device-form occupancy update
 * peer-copies the images into, plus PQP_MAX_BOXES * PQP_BOX_FIELDS doubles (2.5 MiB) and 4 B per slot: the staging
 * the device-form box update peer-copies the boxes into. A device's plan handle holds ceil(batch_max / n_devices)
 * paths.
 *
 * The footprint collision check is not sharded (about 0.3 ms per 1024 paths against about 13 ms for the plan on an
 * H100): the home device holds every slot, so run pqp_plan_collision_check*_device on pqp_plan_multi_handle(m, 0) over
 * the gathered paths.
 *
 * There is no CPU fallback. Every function returns a PQP_* code from pqp.h and never throws.
 */
#ifndef PQP_PLAN_MULTI_H
#define PQP_PLAN_MULTI_H

#include <stdint.h>

#include "pqp_plan.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the per-device plan handles of one multi-device plan (the function pqp_plan_multi is its samples-form call) */
typedef struct pqp_plan_multi_t pqp_plan_multi_t;

/* n_devices handles (devices[i], or 0..n_devices-1 when devices == NULL; devices[0] is the home device) with n_maps
 * slots each, as pqp_plan_create_maps. A device may appear more than once: two handles on one GPU. PQP_E_INVALID for
 * a NULL out, params or maps, n_maps < 1, n_devices < 1, batch_max < 1, or capacities pqp_plan_create_maps refuses
 * (r_max >= 3, p_max >= 4, layers_max >= 4, 2 <= n_max <= 511), all checked before any device is looked up;
 * PQP_E_NO_DEVICE when a device index is not visible. */
int pqp_plan_multi_create_maps(const pqp_bounds_map *maps, int32_t n_maps, const pqp_plan_params *params,
                               int32_t r_max, int32_t p_max, int32_t layers_max, int32_t n_max, int32_t batch_max,
                               int32_t n_devices, const int32_t *devices, pqp_plan_multi_t **out);
int pqp_plan_multi_destroy(pqp_plan_multi_t *m);

/* Host buffers, synchronous: pqp_plan_points(_mapped) / pqp_plan(_mapped) with every shard on its device's own host
 * thread. Every output and every trace field lands where the single-device call on the whole batch puts it.
 * map_index == NULL: the unmapped call (slot 0). */
int pqp_plan_multi_points(pqp_plan_multi_t *m, const pqp_plan_points_in *in, const int32_t *map_index,
                          const pqp_plan_out *out);
int pqp_plan_multi(pqp_plan_multi_t *m, const pqp_plan_in *in, const int32_t *map_index, const pqp_plan_out *out);

/* Device buffers on the home device, asynchronous on `stream` (a cudaStream_t of the home device): no host
 * synchronisation, no allocation. The home shard runs on the caller's buffers and stream; every other device waits
 * on `stream`, peer-copies its input slice (and map_index slice) into staging allocated at create, plans on its own
 * stream and peer-copies status, n, path, cost and iters back into `out`; `stream` then waits for every device.
 * out->trace must be NULL (PQP_E_INVALID otherwise): a traced shard would need staging for every trace field; the
 * host forms take a trace. */
int pqp_plan_multi_points_device(pqp_plan_multi_t *m, const pqp_plan_points_in *in, const int32_t *map_index,
                                 const pqp_plan_out *out, void *stream);
int pqp_plan_multi_device(pqp_plan_multi_t *m, const pqp_plan_in *in, const int32_t *map_index, const pqp_plan_out *out,
                          void *stream);

/* Map slots, on every device. The host forms return when every device has its copy (the occupancy transforms run
 * concurrently, one host thread per device). The device form takes its image stack on the home device and is ordered
 * on `stream`: the uint8 images are peer-copied to every other device and transformed there, and `stream` waits for
 * every device's transform. Once `stream` has passed the call (e.g. after a cudaStreamSynchronize of it) the stack
 * may be released and the new slots are in place on every device, for any later call, host forms included. A device
 * form enqueued after an update sees the new slots on every device, one enqueued before sees the old ones. The host
 * calls run on each handle's own stream, as the single-device host calls do: they see a device-form update once
 * `stream` has passed it. An update that a handle would refuse (a slot out of range, a map larger than a slot, ...)
 * is refused before anything is enqueued on any device. */
int pqp_plan_multi_set_map_slot(pqp_plan_multi_t *m, int32_t slot, const pqp_bounds_map *map);
int pqp_plan_multi_set_occupancy_slots(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *stack);
int pqp_plan_multi_set_occupancy_slots_device(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *stack,
                                              void *stream);
/* pqp_plan_set_occupancy_boxes(_device) on every device, as the occupancy_slots forms above: the home handle first
 * (its refusal refuses the call on every device); the device form peer-copies the base image(s), k and the boxes to
 * every other device, and `stream` waits for every device. PQP_MAX_BOXES caps every form alike, so a call a single
 * plan handle accepts is accepted here. */
int pqp_plan_multi_set_occupancy_boxes(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *base,
                                       int32_t shared_base, const pqp_obstacle_boxes *boxes);
int pqp_plan_multi_set_occupancy_boxes_device(pqp_plan_multi_t *m, int32_t first_slot, const pqp_occupancy_stack *base,
                                              int32_t shared_base, const pqp_obstacle_boxes *boxes, void *stream);
/* as pqp_plan_get_map_slot on device index i's handle */
int pqp_plan_multi_get_map_slot(pqp_plan_multi_t *m, int32_t device_index, int32_t slot, pqp_bounds_map *meta,
                                float *distance);

/* shard of device index i in the last plan call */
int pqp_plan_multi_shard(pqp_plan_multi_t *m, int32_t device_index, int32_t *first, int32_t *count);
/* the plan handle behind device index i (pqp_plan_last_stage_ms, pqp_plan_launch_count, the collision check) */
int pqp_plan_multi_handle(pqp_plan_multi_t *m, int32_t device_index, pqp_plan_handle **h);
/* m may be NULL: last create error. A device handle's error reads "device <d>: <that handle's message>". */
const char *pqp_plan_multi_last_error(const pqp_plan_multi_t *m);

#ifdef __cplusplus
}
#endif
#endif /* PQP_PLAN_MULTI_H */
