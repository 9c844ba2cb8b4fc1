"""ctypes binding of the clearance-bounds entry points (include/pqp_bounds.h).

`PathBounds` is the batched stand-in for `ReferencePathImpl::updateBoundsImproved`
(reference_path_impl.cpp:177-230): one handle owns the device copy of the map's distance layer;
`compute()` takes the splines and reference states of a batch of paths and returns the
front / rear / centre clearance bounds per state plus the index the reference would cut each
path at. There is no CPU path: without the CUDA library or an H100, construction raises.
"""
import ctypes as C

import numpy as np

from . import abi
from .solver import PqpError, load_library

SPLINE_ROWS, STATE_ROWS, BOUND_ROWS = 9, 4, 6

EXPORTED_SYMBOLS = [
    "pqp_bounds_default_params", "pqp_bounds_create", "pqp_bounds_destroy", "pqp_bounds_compute",
    "pqp_bounds_compute_device", "pqp_bounds_build_states", "pqp_bounds_build_states_device",
    "pqp_bounds_last_kernel_ms", "pqp_bounds_last_error", "pqp_bounds_set_map", "pqp_bounds_set_map_device",
    "pqp_bounds_set_occupancy", "pqp_bounds_set_occupancy_device", "pqp_bounds_get_map",
    "pqp_bounds_create_maps", "pqp_bounds_set_map_slot", "pqp_bounds_set_map_slot_device",
    "pqp_bounds_set_occupancy_slots", "pqp_bounds_set_occupancy_slots_device", "pqp_bounds_get_map_slot",
    "pqp_bounds_map_count", "pqp_bounds_compute_mapped", "pqp_bounds_compute_mapped_device",
    "pqp_bounds_collision_check", "pqp_bounds_collision_check_device", "pqp_bounds_collision_check_mapped",
    "pqp_bounds_collision_check_mapped_device", "pqp_bounds_set_occupancy_boxes", "pqp_bounds_set_occupancy_boxes_device",
]
MAX_MAP_SLOTS = 65535
MAP_TABLE_CHUNK = 1024  # table entries per table-write launch of a slot update
BOX_FIELDS = 5  # x, y, heading, length, width of an obstacle box
MAX_BOXES = 65536  # count * k_max of one set_occupancy_boxes call


class BoundsMap(C.Structure):
    _fields_ = [("rows", C.c_int32), ("cols", C.c_int32), ("resolution", C.c_double),
                ("center_x", C.c_double), ("center_y", C.c_double), ("distance", C.c_void_p)]


class OccupancyMap(C.Structure):
    """pqp_occupancy_map: uint8 image [rows, cols]; a cell is an obstacle when its value <= obstacle_max."""
    _fields_ = [("rows", C.c_int32), ("cols", C.c_int32), ("resolution", C.c_double),
                ("center_x", C.c_double), ("center_y", C.c_double), ("cells", C.c_void_p),
                ("obstacle_max", C.c_int32)]


class OccupancyStack(C.Structure):
    """pqp_occupancy_stack: `count` uint8 images [count, rows, cols] with one centre each (host arrays)."""
    _fields_ = [("count", C.c_int32), ("rows", C.c_int32), ("cols", C.c_int32), ("resolution", C.c_double),
                ("center_x", C.c_void_p), ("center_y", C.c_void_p), ("cells", C.c_void_p), ("obstacle_max", C.c_int32)]


class ObstacleBoxes(C.Structure):
    """pqp_obstacle_boxes: k [count] boxes per slot out of boxes [count, k_max, BOX_FIELDS]."""
    _fields_ = [("k_max", C.c_int32), ("k", C.c_void_p), ("boxes", C.c_void_p)]


def pack_boxes(boxes, k, count):
    """(float64 [count, k_max, BOX_FIELDS], int32 [count]) from `boxes` [count, k_max, BOX_FIELDS] with `k` (None: all
    k_max), or from a list of `count` arrays [k_s, BOX_FIELDS]."""
    if isinstance(boxes, (list, tuple)):
        assert k is None and len(boxes) == count, "a list of boxes takes no k and has one entry per slot"
        per = [np.asarray(b, dtype=np.float64).reshape(-1, BOX_FIELDS) for b in boxes]
        k = np.array([len(b) for b in per], dtype=np.int32)
        packed = np.zeros((count, int(k.max(initial=0)), BOX_FIELDS))
        for s, b in enumerate(per):
            packed[s, :len(b)] = b
        return packed, k
    packed = np.ascontiguousarray(boxes, dtype=np.float64)
    assert packed.ndim == 3 and packed.shape[0] == count and packed.shape[2] == BOX_FIELDS
    k = np.full(count, packed.shape[1], np.int32) if k is None else np.ascontiguousarray(k, dtype=np.int32)
    assert k.shape == (count,)
    return packed, k


def box_base(shape, count=None):
    """(count, shared_base, (rows, cols)) of a base image shape: [rows, cols] shared by `count` slots, or [count, rows,
    cols]."""
    if len(shape) == 2:
        assert count is not None, "a shared base image needs the slot count (from the boxes)"
        return int(count), 1, tuple(int(v) for v in shape)
    assert len(shape) == 3
    return int(shape[0]), 0, tuple(int(v) for v in shape[1:])


def occupancy_stack(cells_ptr, shape, resolution, centers, obstacle_max):
    """(OccupancyStack, the float64 centre arrays it points at) for an image stack of `shape` (count, rows, cols) at
    `cells_ptr`; `centers` is [count, 2] (None: all at the origin)."""
    count, rows, cols = (int(v) for v in shape)
    c = np.zeros((count, 2)) if centers is None else np.asarray(centers, dtype=np.float64).reshape(count, 2)
    cx, cy = np.ascontiguousarray(c[:, 0]), np.ascontiguousarray(c[:, 1])
    return OccupancyStack(count, rows, cols, float(resolution), cx.ctypes.data, cy.ctypes.data, cells_ptr,
                          int(obstacle_max)), (cx, cy)


def map_list(dists, resolutions, centers):
    """(BoundsMap array, the float32 layers it points at) for per-slot layers; `resolutions` is one value or one per
    map, `centers` None or [(x, y)] per map."""
    dists = [np.ascontiguousarray(d, dtype=np.float32) for d in dists]
    n = len(dists)
    res = np.broadcast_to(np.asarray(resolutions, dtype=np.float64), (n,))
    cen = np.zeros((n, 2)) if centers is None else np.asarray(centers, dtype=np.float64).reshape(n, 2)
    arr = (BoundsMap * n)(*(BoundsMap(d.shape[0], d.shape[1], float(r), float(c[0]), float(c[1]), d.ctypes.data)
                            for d, r, c in zip(dists, res, cen)))
    return arr, dists


def index_array(map_index, batch):
    idx = np.ascontiguousarray(map_index, dtype=np.int32)
    assert idx.shape == (batch,)
    return idx


def distance_map(dist, resolution, center):
    """(BoundsMap, the contiguous float32 layer it points at) for a host array."""
    dist = np.ascontiguousarray(dist, dtype=np.float32)
    assert dist.ndim == 2
    return BoundsMap(dist.shape[0], dist.shape[1], float(resolution), float(center[0]), float(center[1]),
                     dist.ctypes.data), dist


def occupancy_map(img, resolution, center, obstacle_max):
    """(OccupancyMap, the contiguous uint8 image it points at) for a host array."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    assert img.ndim == 2
    return OccupancyMap(img.shape[0], img.shape[1], float(resolution), float(center[0]), float(center[1]),
                        img.ctypes.data, int(obstacle_max)), img


class BoundsParams(C.Structure):
    _fields_ = [("front_length", C.c_double), ("rear_length", C.c_double), ("car_width", C.c_double),
                ("safety_margin", C.c_double), ("epsilon", C.c_double)]


class BoundsIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("n_max", C.c_int32), ("k_max", C.c_int32), ("states", C.c_void_p),
                ("n", C.c_void_p), ("spline", C.c_void_p), ("k", C.c_void_p)]


class BoundsOut(C.Structure):
    _fields_ = [("bounds", C.c_void_p), ("n_valid", C.c_void_p), ("knots", C.c_void_p)]


class StatesIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("n_max", C.c_int32), ("k_max", C.c_int32), ("spline", C.c_void_p),
                ("k", C.c_void_p), ("max_s", C.c_void_p), ("delta_s_smaller", C.c_double),
                ("delta_s_larger", C.c_double), ("dynamic_segmentation", C.c_int32)]


class StatesOut(C.Structure):
    _fields_ = [("states", C.c_void_p), ("curvature", C.c_void_p), ("n", C.c_void_p), ("total", C.c_void_p),
                ("knots", C.c_void_p)]


class CollisionIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("n_max", C.c_int32), ("row_stride", C.c_int32), ("poses", C.c_void_p),
                ("n", C.c_void_p)]


class CollisionOut(C.Structure):
    _fields_ = [("first_hit", C.c_void_p), ("state_free", C.c_void_p), ("clearance", C.c_void_p)]


def default_params(**overrides):
    p = BoundsParams(3.9, -1.0, 2.0, 0.3, 1e-6)
    for k, v in overrides.items():
        setattr(p, k, v)
    return p


def _declare(L):
    if getattr(L, "_pqp_bounds_declared", False):
        return L
    vp = C.c_void_p
    L.pqp_bounds_default_params.argtypes = [C.POINTER(BoundsParams)]
    L.pqp_bounds_default_params.restype = None
    L.pqp_bounds_create.argtypes = [C.POINTER(BoundsMap), C.POINTER(BoundsParams), C.c_int32, C.POINTER(vp)]
    L.pqp_bounds_destroy.argtypes = [vp]
    L.pqp_bounds_destroy.restype = None
    L.pqp_bounds_compute.argtypes = [vp, C.POINTER(BoundsIn), C.POINTER(BoundsOut)]
    L.pqp_bounds_compute_device.argtypes = [vp, C.POINTER(BoundsIn), C.POINTER(BoundsOut), vp]
    L.pqp_bounds_build_states.argtypes = [vp, C.POINTER(StatesIn), C.POINTER(StatesOut)]
    L.pqp_bounds_build_states_device.argtypes = [vp, C.POINTER(StatesIn), C.POINTER(StatesOut), vp]
    L.pqp_bounds_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.pqp_bounds_last_error.argtypes = [vp]
    L.pqp_bounds_last_error.restype = C.c_char_p
    L.pqp_bounds_create_maps.argtypes = [C.POINTER(BoundsMap), C.c_int32, C.POINTER(BoundsParams), C.c_int32,
                                         C.POINTER(vp)]
    L.pqp_bounds_compute_mapped.argtypes = [vp, C.POINTER(BoundsIn), vp, C.POINTER(BoundsOut)]
    L.pqp_bounds_compute_mapped_device.argtypes = [vp, C.POINTER(BoundsIn), vp, C.POINTER(BoundsOut), vp]
    declare_map_surface(L, "pqp_bounds_")
    L._pqp_bounds_declared = True
    return L


def declare_map_surface(L, prefix):
    """The map entry points of the ABI `prefix` (pqp_bounds_, pqp_plan_): map and slot updates and reads, the slot
    count and the collision check."""
    vp, i32, bm, om = C.c_void_p, C.c_int32, C.POINTER(BoundsMap), C.POINTER(OccupancyMap)
    cin, cout = C.POINTER(CollisionIn), C.POINTER(CollisionOut)
    for name, argtypes in (
            ("set_map", [vp, bm]), ("set_map_device", [vp, bm, vp]), ("set_occupancy", [vp, om]),
            ("set_occupancy_device", [vp, om, vp]), ("get_map", [vp, bm, vp]), ("set_map_slot", [vp, i32, bm]),
            ("set_map_slot_device", [vp, i32, bm, vp]), ("get_map_slot", [vp, i32, bm, vp]), ("map_count", [vp]),
            ("collision_check", [vp, cin, cout]), ("collision_check_device", [vp, cin, cout, vp]),
            ("collision_check_mapped", [vp, cin, vp, cout]),
            ("collision_check_mapped_device", [vp, cin, vp, cout, vp])):
        getattr(L, prefix + name).argtypes = argtypes
    getattr(L, prefix + "map_count").restype = C.c_int32
    declare_stack_updates(L, prefix)


def declare_stack_updates(L, prefix):
    """The set_occupancy_slots and set_occupancy_boxes entry points of the ABI `prefix` (pqp_bounds_, pqp_plan_,
    pqp_plan_multi_)."""
    vp, i32, st, bx = C.c_void_p, C.c_int32, C.POINTER(OccupancyStack), C.POINTER(ObstacleBoxes)
    getattr(L, prefix + "set_occupancy_slots").argtypes = [vp, i32, st]
    getattr(L, prefix + "set_occupancy_slots_device").argtypes = [vp, i32, st, vp]
    getattr(L, prefix + "set_occupancy_boxes").argtypes = [vp, i32, st, i32, bx]
    getattr(L, prefix + "set_occupancy_boxes_device").argtypes = [vp, i32, st, i32, bx, vp]


def occupancy_call(fn, h, imgs, resolution, centers, obstacle_max, first_slot, boxes=None, k=None):
    """`fn`, a host-form set_occupancy_slots or (with `boxes`) set_occupancy_boxes, on host arrays as
    MapSlots.set_occupancy_slots and MapSlots.set_occupancy_boxes document them."""
    imgs = np.ascontiguousarray(imgs, dtype=np.uint8)
    assert imgs.ndim == 3 or (boxes is not None and imgs.ndim == 2)
    shape, box_args = imgs.shape, ()
    if boxes is not None:
        count, shared, (rows, cols) = box_base(imgs.shape, len(boxes) if imgs.ndim == 2 else None)
        packed, k = pack_boxes(boxes, k, count)
        shape, box_args = (count, rows, cols), (shared, C.byref(ObstacleBoxes(packed.shape[1], k.ctypes.data,
                                                                               packed.ctypes.data)))
    st, _keep = occupancy_stack(imgs.ctypes.data, shape, resolution, centers, obstacle_max)
    return fn(h, int(first_slot), C.byref(st), *box_args)


def occupancy_call_device(fn, h, imgs, resolution, centers, obstacle_max, first_slot, boxes=None, k=None, *, stream):
    """As `occupancy_call` for the device form `fn`, on torch CUDA tensors as MapSlots.set_occupancy_slots_device and
    MapSlots.set_occupancy_boxes_device document them; `stream` a raw cudaStream_t."""
    import torch
    assert imgs.is_cuda and imgs.is_contiguous() and imgs.dtype == torch.uint8
    assert imgs.dim() == 3 or (boxes is not None and imgs.dim() == 2)
    shape, box_args = tuple(imgs.shape), ()
    if boxes is not None:
        assert boxes.is_cuda and boxes.is_contiguous() and boxes.dtype == torch.float64 and boxes.dim() == 3
        assert boxes.shape[2] == BOX_FIELDS
        count, shared, (rows, cols) = box_base(shape, int(boxes.shape[0]))
        assert int(boxes.shape[0]) == count
        assert k.is_cuda and k.is_contiguous() and k.dtype == torch.int32 and tuple(k.shape) == (count,)
        shape, box_args = (count, rows, cols), (shared, C.byref(ObstacleBoxes(int(boxes.shape[1]), k.data_ptr(),
                                                                               boxes.data_ptr())))
    st, _keep = occupancy_stack(imgs.data_ptr(), shape, resolution, centers, obstacle_max)
    return fn(h, int(first_slot), C.byref(st), *box_args, C.c_void_p(stream))


class MapSlots:
    """The map surface of a handle that owns map slots, shared by `PathBounds` and `plan.Planner`: `_abi` is the prefix
    of the handle's C entry points (pqp_bounds_, pqp_plan_), `L` the library and `h` the handle."""
    _abi = None

    def _fn(self, name):
        return getattr(self.L, self._abi + name)

    def _create(self, name, *args):
        """`name` ("create" or "create_maps") with `args` and the out-pointer; raises with the ABI's create error."""
        h = C.c_void_p()
        rc = self._fn(name)(*args, C.byref(h))
        if rc:
            raise PqpError(rc, (self._fn("last_error")(None) or b"").decode())
        self.h = h

    def _create_maps(self, dists, resolutions, centers, *args):
        """from_maps: one slot per float32 layer in `dists`; `args` are the create arguments after the maps."""
        arr, self._layers = map_list(dists, resolutions, centers)
        self.dist = self._layers[0]
        self._create("create_maps", arr, len(self._layers), *args)

    @property
    def n_maps(self):
        return int(self._fn("map_count")(self.h))

    def close(self):
        if getattr(self, "h", None):
            self._fn("destroy")(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise PqpError(rc, (self._fn("last_error")(self.h) or b"").decode())

    def set_map(self, dist, resolution, center=(0.0, 0.0), slot=0):
        """Replace the map (of `slot`) with a float32 distance layer [rows, cols] (host, synchronous); rows * cols may
        not exceed the cells of a slot."""
        m, _keep = distance_map(dist, resolution, center)
        if slot:
            self._check(self._fn("set_map_slot")(self.h, int(slot), C.byref(m)))
        else:
            self._check(self._fn("set_map")(self.h, C.byref(m)))

    def set_occupancy(self, img, resolution, center=(0.0, 0.0), obstacle_max=0, slot=0):
        """Replace the map (of `slot`) with the exact Euclidean distance transform, computed on the GPU, of a uint8
        image [rows, cols] (host, synchronous): cells <= obstacle_max are obstacles (0: the demo's zero pixels)."""
        if slot:
            img = np.ascontiguousarray(img, dtype=np.uint8)
            self.set_occupancy_slots(img[None], resolution, [center], obstacle_max, first_slot=slot)
            return
        m, _keep = occupancy_map(img, resolution, center, obstacle_max)
        self._check(self._fn("set_occupancy")(self.h, C.byref(m)))

    def _raw_stream(self, stream, device):
        """The cudaStream_t a device-form map update runs on: `stream` as given, a raw cudaStream_t (None: 0).
        `plan.Planner` takes a torch stream instead (None: the current stream of `device`)."""
        return 0 if stream is None else stream

    def set_occupancy_slots(self, imgs, resolution, centers=None, obstacle_max=0, *, first_slot=0):
        """The exact distance transforms of a uint8 stack [count, rows, cols] into slots first_slot .. + count - 1,
        in one pair of launches (host, synchronous); `centers` [count, 2] (default: the origin)."""
        self._check(occupancy_call(self._fn("set_occupancy_slots"), self.h, imgs, resolution, centers, obstacle_max,
                                   first_slot))

    def set_occupancy_slots_device(self, imgs, resolution, centers=None, obstacle_max=0, *, first_slot=0, stream=None):
        """As `set_occupancy_slots` from a torch uint8 CUDA tensor [count, rows, cols], asynchronous on `stream` (as
        `_raw_stream` takes it): calls enqueued before see the old slots, calls enqueued after the new ones. The tensor
        must stay alive until the stream has run the transform."""
        self._check(occupancy_call_device(self._fn("set_occupancy_slots_device"), self.h, imgs, resolution, centers,
                                          obstacle_max, first_slot, stream=self._raw_stream(stream, imgs.device)))

    def set_occupancy_boxes(self, base, resolution, boxes, k=None, centers=None, obstacle_max=0, *, first_slot=0):
        """Slots first_slot .. + count - 1 := the exact distance transforms of a static occupancy image plus each slot's
        obstacle boxes, stamped on the GPU (host, synchronous). `base` uint8 [rows, cols] (every slot starts from it) or
        [count, rows, cols]; `boxes` float64 [count, k_max, 5] (x, y, heading, length, width in the map's frame) with
        `k` [count] boxes per slot (None: all k_max), or a list of `count` arrays [k_s, 5]. A cell is an obstacle when
        its base value <= obstacle_max or its centre lies in or on one of its slot's boxes (include/pqp_bounds.h)."""
        self._check(occupancy_call(self._fn("set_occupancy_boxes"), self.h, base, resolution, centers, obstacle_max,
                                   first_slot, boxes, k))

    def set_occupancy_boxes_device(self, base, resolution, boxes, k, centers=None, obstacle_max=0, *, first_slot=0,
                                   stream=None):
        """As `set_occupancy_boxes` from torch CUDA tensors: `base` uint8 [rows, cols] or [count, rows, cols], `boxes`
        float64 [count, k_max, 5], `k` int32 [count] (clamped to [0, k_max] on the device). Asynchronous on `stream` (as
        `_raw_stream` takes it), ordered as `set_occupancy_slots_device`; the tensors must stay alive until the stream
        has run the update."""
        self._check(occupancy_call_device(self._fn("set_occupancy_boxes_device"), self.h, base, resolution, centers,
                                          obstacle_max, first_slot, boxes, k,
                                          stream=self._raw_stream(stream, base.device)))

    def get_map(self, slot=0):
        """-> (float32 distance layer [rows, cols], resolution, (center_x, center_y)) of the current map (of `slot`);
        waits for the device."""
        if slot:
            fn = lambda h_, m_, d_: self._fn("get_map_slot")(h_, int(slot), m_, d_)  # noqa: E731
        else:
            fn = self._fn("get_map")
        meta = BoundsMap()
        self._check(fn(self.h, C.byref(meta), None))
        dist = np.empty((meta.rows, meta.cols), dtype=np.float32)
        self._check(fn(self.h, C.byref(meta), dist.ctypes.data))
        return dist, meta.resolution, (meta.center_x, meta.center_y)

    def check_collision(self, poses, n, *, row_stride=None, map_index=None, clearance=False, per_state=False):
        """CollisionChecker::isSingleStateCollisionFreeImproved for every pose (host, synchronous). `poses` float64
        [B, rows, n_max] with rows 0, 1, 2 = x, y, heading (a plan's `path`, or `states[:, 1:]` of reference states);
        its rows must be n_max elements apart, and `row_stride` (rows from one path to the next) is read from its
        strides unless given. -> dict with first_hit int32 [B] (n[b] when all n[b] poses are free, -1 for a
        `map_index` outside the slots), and when asked state_free uint8 [B, n_max] and clearance float64 [B, n_max]."""
        poses = np.asarray(poses, dtype=np.float64)
        rs = _pose_stride(poses.shape, [s // 8 for s in poses.strides], row_stride)
        if rs is None:
            poses = np.ascontiguousarray(poses)
            rs = _pose_stride(poses.shape, [s // 8 for s in poses.strides], row_stride)
        assert rs is not None, "row_stride disagrees with the layout of poses"
        B, _, n_max = poses.shape
        n = np.ascontiguousarray(n, dtype=np.int32)
        assert n.shape == (B,)
        out = {"first_hit": np.zeros(B, np.int32)}
        if per_state:
            out["state_free"] = np.zeros((B, n_max), np.uint8)
        if clearance:
            out["clearance"] = np.zeros((B, n_max))
        ci = CollisionIn(B, n_max, rs, poses.ctypes.data, n.ctypes.data)
        co = CollisionOut(*(out[k].ctypes.data if k in out else None for k in ("first_hit", "state_free", "clearance")))
        if map_index is None:
            self._check(self._fn("collision_check")(self.h, C.byref(ci), C.byref(co)))
        else:
            idx = index_array(map_index, B)
            self._check(self._fn("collision_check_mapped")(self.h, C.byref(ci), idx.ctypes.data, C.byref(co)))
        return out

    def check_collision_device(self, poses, n, *, row_stride=None, map_index=None, clearance=False, per_state=False,
                               stream=0):
        """As `check_collision` on torch CUDA tensors (poses float64 with rows n_max apart, n and map_index int32 [B]),
        asynchronous on `stream` (a raw cudaStream_t); returns a dict of CUDA tensors. Enqueued after a plan call on
        the same stream, it checks that call's output."""
        import torch
        assert poses.is_cuda and poses.dtype == torch.float64 and poses.dim() == 3
        B, _, n_max = poses.shape
        rs = _pose_stride(poses.shape, poses.stride(), row_stride)
        assert rs is not None, "poses: rows must be n_max elements apart"
        assert n.is_cuda and n.is_contiguous() and n.dtype == torch.int32 and tuple(n.shape) == (B,)
        out = {"first_hit": torch.zeros(B, dtype=torch.int32, device=poses.device)}
        if per_state:
            out["state_free"] = torch.zeros((B, n_max), dtype=torch.uint8, device=poses.device)
        if clearance:
            out["clearance"] = torch.zeros((B, n_max), dtype=torch.float64, device=poses.device)
        ci = CollisionIn(B, n_max, rs, poses.data_ptr(), n.data_ptr())
        co = CollisionOut(*(out[k].data_ptr() if k in out else None for k in ("first_hit", "state_free", "clearance")))
        s = C.c_void_p(stream)
        if map_index is None:
            self._check(self._fn("collision_check_device")(self.h, C.byref(ci), C.byref(co), s))
        else:
            assert map_index.is_cuda and map_index.is_contiguous() and map_index.dtype == torch.int32
            assert tuple(map_index.shape) == (B,)
            self._check(self._fn("collision_check_mapped_device")(self.h, C.byref(ci), map_index.data_ptr(),
                                                                  C.byref(co), s))
        return out


def _pose_stride(shape, strides, row_stride):
    """Rows from one path to the next of a [B, rows, n_max] pose array with element `strides`, or None when its
    rows are not n_max elements apart (or `row_stride` disagrees)."""
    B, rows, n_max = shape
    assert rows >= 3
    if strides[2] != 1 or strides[1] != n_max or strides[0] % n_max:
        return None
    rs = strides[0] // n_max if B > 1 else rows
    return rs if row_stride is None or int(row_stride) == rs else None


class PathBounds(MapSlots):
    """One obstacle map on one GPU; `dist` is the float32 distance layer [rows, cols]."""
    _abi = "pqp_bounds_"

    def __init__(self, dist, resolution, *, center=(0.0, 0.0), params=None, device=0):
        self.L = _declare(load_library())
        self.dist = np.ascontiguousarray(dist, dtype=np.float32)
        self.params = params if params is not None else default_params()
        m = BoundsMap(self.dist.shape[0], self.dist.shape[1], float(resolution), float(center[0]), float(center[1]),
                      self.dist.ctypes.data)
        self._create("create", C.byref(m), C.byref(self.params), int(device))

    @classmethod
    def from_maps(cls, dists, resolutions, *, centers=None, params=None, device=0):
        """One handle with a map slot per float32 layer in `dists` (each slot as large as the largest layer);
        `resolutions` is one value or one per map, `centers` [(x, y)] per map (default: the origin)."""
        self = cls.__new__(cls)
        self.L = _declare(load_library())
        self.params = params if params is not None else default_params()
        self._create_maps(dists, resolutions, centers, C.byref(self.params), int(device))
        return self

    def compute(self, states, n, spline, k, *, knots=None, map_index=None):
        """Host buffers: states[b][4][n_max], n[b], spline[b][9][k_max], k[b] ->
        (bounds[b][6][n_max], n_valid[b]); `knots` (solver block [b][9][n_max]) is filled in place. `map_index` [b]:
        path b on map slot map_index[b] (out of range: n_valid 0)."""
        states = np.ascontiguousarray(states, dtype=np.float64)
        spline = np.ascontiguousarray(spline, dtype=np.float64)
        n = np.ascontiguousarray(n, dtype=np.int32)
        k = np.ascontiguousarray(k, dtype=np.int32)
        B, _, n_max = states.shape
        bounds = np.zeros((B, BOUND_ROWS, n_max))
        n_valid = np.zeros(B, dtype=np.int32)
        if knots is not None:
            assert knots.flags.c_contiguous and knots.dtype == np.float64 and knots.shape == (B, abi.NFIELDS, n_max)
        bi = BoundsIn(B, n_max, spline.shape[2], states.ctypes.data, n.ctypes.data, spline.ctypes.data, k.ctypes.data)
        bo = BoundsOut(bounds.ctypes.data, n_valid.ctypes.data, knots.ctypes.data if knots is not None else None)
        if map_index is None:
            self._check(self.L.pqp_bounds_compute(self.h, C.byref(bi), C.byref(bo)))
        else:
            idx = index_array(map_index, B)
            self._check(self.L.pqp_bounds_compute_mapped(self.h, C.byref(bi), idx.ctypes.data, C.byref(bo)))
        return bounds, n_valid

    def compute_device(self, bin_struct: BoundsIn, bout_struct: BoundsOut, stream=0):
        """Raw device pointers (e.g. torch tensors' data_ptr()), asynchronous on `stream`."""
        self._check(self.L.pqp_bounds_compute_device(self.h, C.byref(bin_struct), C.byref(bout_struct),
                                                     C.c_void_p(stream)))

    def build_states(self, spline, k, max_s, n_max, *, ds_small=0.15, ds_large=0.3, dynamic=True, knots=None):
        """buildReferenceFromSpline for a batch (host buffers): -> (states[b][4][n_max],
        curvature[b][n_max], n[b], total[b]); `knots` (solver block) is filled in place."""
        spline = np.ascontiguousarray(spline, dtype=np.float64)
        k = np.ascontiguousarray(k, dtype=np.int32)
        max_s = np.ascontiguousarray(max_s, dtype=np.float64)
        B = spline.shape[0]
        states, curv = np.zeros((B, STATE_ROWS, n_max)), np.zeros((B, n_max))
        n, total = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        if knots is not None:
            assert knots.flags.c_contiguous and knots.dtype == np.float64 and knots.shape == (B, abi.NFIELDS, n_max)
        si = StatesIn(B, n_max, spline.shape[2], spline.ctypes.data, k.ctypes.data, max_s.ctypes.data, ds_small, ds_large,
                      1 if dynamic else 0)
        so = StatesOut(states.ctypes.data, curv.ctypes.data, n.ctypes.data, total.ctypes.data,
                       knots.ctypes.data if knots is not None else None)
        self._check(self.L.pqp_bounds_build_states(self.h, C.byref(si), C.byref(so)))
        return states, curv, n, total

    def build_states_device(self, sin_struct: StatesIn, sout_struct: StatesOut, stream=0):
        self._check(self.L.pqp_bounds_build_states_device(self.h, C.byref(sin_struct), C.byref(sout_struct),
                                                          C.c_void_p(stream)))

    @property
    def last_kernel_ms(self):
        ms = C.c_float(0)
        self._check(self.L.pqp_bounds_last_kernel_ms(self.h, C.byref(ms)))
        return ms.value
