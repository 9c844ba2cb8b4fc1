"""ctypes binding of include/pqp_plan_multi.h: the whole plan (`plan.Planner`) over the GPUs of one box. `MultiPlanner`
owns one plan handle per device, each with its own copy of every map slot, and shards each batch in contiguous blocks
(device i plans paths [i * per, min(B, (i + 1) * per)), per = ceil(B / len(devices))). Results come back as
`plan.PlanResult` (host calls) or as tensors on the home device, devices[0] (device calls), exactly where a single
`Planner` puts them. No CPU path."""
import ctypes as C

import numpy as np

from . import bounds
from . import plan as _plan  # `plan` is also a MultiPlanner method
from .solver import PqpError

EXPORTED_SYMBOLS = ["pqp_plan_multi_create_maps", "pqp_plan_multi_destroy", "pqp_plan_multi_points", "pqp_plan_multi",
                    "pqp_plan_multi_points_device", "pqp_plan_multi_device", "pqp_plan_multi_set_map_slot",
                    "pqp_plan_multi_set_occupancy_slots", "pqp_plan_multi_set_occupancy_slots_device",
                    "pqp_plan_multi_get_map_slot", "pqp_plan_multi_shard", "pqp_plan_multi_handle",
                    "pqp_plan_multi_last_error", "pqp_plan_multi_set_occupancy_boxes",
                    "pqp_plan_multi_set_occupancy_boxes_device"]


def _lib():
    L = _plan._lib()
    if not getattr(L, "_plan_multi_declared", False):
        vp, i32 = C.c_void_p, C.c_int32
        pin, ppts, pout = C.POINTER(_plan.PlanIn), C.POINTER(_plan.PlanPointsIn), C.POINTER(_plan.PlanOut)
        L.pqp_plan_multi_create_maps.argtypes = [C.POINTER(bounds.BoundsMap), i32, C.POINTER(_plan.PlanParams)] + \
            [i32] * 6 + [vp, C.POINTER(vp)]
        L.pqp_plan_multi_destroy.argtypes = [vp]
        L.pqp_plan_multi_points.argtypes = [vp, ppts, vp, pout]
        L.pqp_plan_multi.argtypes = [vp, pin, vp, pout]
        L.pqp_plan_multi_points_device.argtypes = [vp, ppts, vp, pout, vp]
        L.pqp_plan_multi_device.argtypes = [vp, pin, vp, pout, vp]
        L.pqp_plan_multi_set_map_slot.argtypes = [vp, i32, C.POINTER(bounds.BoundsMap)]
        bounds.declare_stack_updates(L, "pqp_plan_multi_")
        L.pqp_plan_multi_get_map_slot.argtypes = [vp, i32, i32, C.POINTER(bounds.BoundsMap), vp]
        L.pqp_plan_multi_shard.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32)]
        L.pqp_plan_multi_handle.argtypes = [vp, i32, C.POINTER(vp)]
        L.pqp_plan_multi_last_error.argtypes = [vp]
        L.pqp_plan_multi_last_error.restype = C.c_char_p
        L._plan_multi_declared = True
    return L


class MultiPlanner:
    """Batched PathOptimizer::solve over `devices` (devices[0] is the home device; a device may be listed twice), with
    one map slot per float32 layer in `dists` on every device, as `plan.Planner.from_maps`. `batch_max` is the largest
    batch of one call; each device's handle holds ceil(batch_max / len(devices)) paths."""

    def __init__(self, dists, resolutions, *, centers=None, r_max, p_max, layers_max=64, n_max=256, batch_max,
                 params=None, devices):
        self.L = _lib()
        self.params = params if params is not None else _plan.default_params()
        self.r_max, self.p_max, self.layers_max, self.n_max = int(r_max), int(p_max), int(layers_max), int(n_max)
        self.batch_max = int(batch_max)
        self.devices = [int(d) for d in devices]
        self.device = self.devices[0]
        arr, self._layers = bounds.map_list(dists, resolutions, centers)
        dv = (C.c_int32 * len(self.devices))(*self.devices)
        h = C.c_void_p()
        rc = self.L.pqp_plan_multi_create_maps(arr, len(self._layers), C.byref(self.params), self.r_max, self.p_max,
                                               self.layers_max, self.n_max, self.batch_max, len(self.devices), dv,
                                               C.byref(h))
        if rc:
            raise PqpError(rc, (self.L.pqp_plan_multi_last_error(None) or b"").decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.pqp_plan_multi_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise PqpError(rc, (self.L.pqp_plan_multi_last_error(self.h) or b"").decode())

    # the buffer handling of a Planner call; the entry points below take the map index (NULL: unmapped) in one place
    dims = _plan.Planner.dims
    _host_call = _plan.Planner._host_call
    _device_call = _plan.Planner._device_call

    def plan(self, raw_x, raw_y, start, target, trace=False, map_index=None) -> _plan.PlanResult:
        """As `plan.Planner.plan`, every shard on its own device and host thread."""
        fn = self.L.pqp_plan_multi
        return self._host_call(lambda h, i, o: fn(h, i, None, o), _plan.PlanIn, raw_x, raw_y, start, target, trace,
                               self.r_max, mapped_fn=fn, map_index=map_index)

    def plan_points(self, ref_x, ref_y, start, target, trace=False, m_max=None, map_index=None) -> _plan.PlanResult:
        """As `plan.Planner.plan_points`, every shard on its own device and host thread."""
        m_max = self.r_max if m_max is None else int(m_max)
        fn = self.L.pqp_plan_multi_points
        return self._host_call(lambda h, i, o: fn(h, i, None, o), _plan.PlanPointsIn, ref_x, ref_y, start, target,
                               trace, m_max, clip=True, mapped_fn=fn, map_index=map_index)

    def plan_device(self, raw_x, raw_y, r, start, target, *, stream=None, map_index=None):
        """As `plan.Planner.plan_device` on tensors of the home device (no trace): asynchronous on `stream` (default:
        the current stream of the home device)."""
        fn = self.L.pqp_plan_multi_device
        return self._device_call(lambda h, i, o, s: fn(h, i, None, o, s), _plan.PlanIn, raw_x, raw_y, r, start, target,
                                 False, stream, fn, map_index)

    def plan_points_device(self, ref_x, ref_y, m, start, target, *, stream=None, map_index=None):
        """As `plan.Planner.plan_points_device` on tensors of the home device (no trace): asynchronous on `stream`
        (default: the current stream of the home device)."""
        fn = self.L.pqp_plan_multi_points_device
        return self._device_call(lambda h, i, o, s: fn(h, i, None, o, s), _plan.PlanPointsIn, ref_x, ref_y, m, start,
                                 target, False, stream, fn, map_index)

    def set_map_slot(self, dist, resolution, center=(0.0, 0.0), *, slot=0):
        """Slot `slot` on every device := a float32 distance layer [rows, cols] (host, synchronous)."""
        m, _keep = bounds.distance_map(dist, resolution, center)
        self._check(self.L.pqp_plan_multi_set_map_slot(self.h, int(slot), C.byref(m)))

    def set_occupancy_slots(self, imgs, resolution, centers=None, obstacle_max=0, *, first_slot=0):
        """As `plan.Planner.set_occupancy_slots` on every device, the transforms concurrently (host, synchronous)."""
        self._check(bounds.occupancy_call(self.L.pqp_plan_multi_set_occupancy_slots, self.h, imgs, resolution, centers,
                                          obstacle_max, first_slot))

    def set_occupancy_slots_device(self, imgs, resolution, centers=None, obstacle_max=0, *, first_slot=0, stream=None):
        """As `set_occupancy_slots` from a torch uint8 tensor [count, rows, cols] on the home device, ordered on `stream`
        (default: the current stream of the home device): the images are peer-copied to every other device and
        transformed there. Plans enqueued before see the old slots on every device, plans enqueued after the new ones;
        the tensor may be released once `stream` has passed the call."""
        self._check(bounds.occupancy_call_device(self.L.pqp_plan_multi_set_occupancy_slots_device, self.h, imgs,
                                                 resolution, centers, obstacle_max, first_slot,
                                                 stream=_plan._stream(stream, imgs.device)))

    def set_occupancy_boxes(self, base, resolution, boxes, k=None, centers=None, obstacle_max=0, *, first_slot=0):
        """As `plan.Planner.set_occupancy_boxes` on every device, the updates concurrently (host, synchronous)."""
        self._check(bounds.occupancy_call(self.L.pqp_plan_multi_set_occupancy_boxes, self.h, base, resolution, centers,
                                          obstacle_max, first_slot, boxes, k))

    def set_occupancy_boxes_device(self, base, resolution, boxes, k, centers=None, obstacle_max=0, *, first_slot=0,
                                   stream=None):
        """As `plan.Planner.set_occupancy_boxes_device` from tensors on the home device, ordered on `stream` (default:
        the current stream of the home device): the base image(s), k and the boxes are peer-copied to every other
        device and stamped there, as `set_occupancy_slots_device` does with its images."""
        self._check(bounds.occupancy_call_device(self.L.pqp_plan_multi_set_occupancy_boxes_device, self.h, base,
                                                 resolution, centers, obstacle_max, first_slot, boxes, k,
                                                 stream=_plan._stream(stream, base.device)))

    def get_map_slot(self, device_index, slot=0):
        """-> (float32 distance layer, resolution, (center_x, center_y)) of `slot` on device index `device_index`."""
        meta = bounds.BoundsMap()
        self._check(self.L.pqp_plan_multi_get_map_slot(self.h, int(device_index), int(slot), C.byref(meta), None))
        dist = np.empty((meta.rows, meta.cols), dtype=np.float32)
        self._check(self.L.pqp_plan_multi_get_map_slot(self.h, int(device_index), int(slot), C.byref(meta),
                                                       dist.ctypes.data))
        return dist, meta.resolution, (meta.center_x, meta.center_y)

    def shard(self, i):
        """(first path, path count) of device index i in the last plan call."""
        first, count = C.c_int32(), C.c_int32()
        self._check(self.L.pqp_plan_multi_shard(self.h, int(i), C.byref(first), C.byref(count)))
        return first.value, count.value

    def handle(self, i):
        """The pqp_plan_handle of device index i (a c_void_p for the pqp_plan_* calls: stage times, launch count,
        the collision check on the home handle, index 0)."""
        h = C.c_void_p()
        self._check(self.L.pqp_plan_multi_handle(self.h, int(i), C.byref(h)))
        return h

    def last_stage_ms(self, i):
        """pqp_plan_last_stage_ms of device index i's handle: its shard's stage times in the last plan call."""
        ms = (C.c_float * len(_plan.STAGES))()
        self._check_plan(i, self.L.pqp_plan_last_stage_ms(self.handle(i), ms))
        return dict(zip(_plan.STAGES, (float(v) for v in ms)))

    def launch_count(self, i):
        """pqp_plan_launch_count of device index i's handle."""
        c = C.c_int64(0)
        self._check_plan(i, self.L.pqp_plan_launch_count(self.handle(i), C.byref(c)))
        return c.value

    def _check_plan(self, i, rc):
        if rc:
            raise PqpError(rc, "device %d: %s" % (self.devices[i],
                                                  (self.L.pqp_plan_last_error(self.handle(i)) or b"").decode()))
