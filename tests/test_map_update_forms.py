"""Every form of an occupancy-map update (include/pqp_bounds.h, pqp_plan.h, pqp_plan_multi.h) against the others.

CPU: the ctypes argtypes of every map entry point of the bounds, plan and multi-GPU plan ABIs, against a literal table.
GPU: one image into slot 0, a stack from slot 1, boxes on a shared base (ragged k, some 0) and boxes on per-slot bases,
through the bounds, plan and MultiPlanner(devices=[0, 0]) handles in the host and device form: every slot's layer and
metadata bit for bit against the transform and box oracles, the plan handle's launch counts, and the refusals, which
must leave every slot untouched on every handle.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import edt_oracle as eo
from path_optimizer_2_b200 import abi, bounds, plan, plan_multi, solver
from tests import box_oracle as bo

vp, i32 = C.c_void_p, C.c_int32
BM, OM, ST, BX = (C.POINTER(t) for t in (bounds.BoundsMap, bounds.OccupancyMap, bounds.OccupancyStack,
                                         bounds.ObstacleBoxes))
CI, CO = C.POINTER(bounds.CollisionIn), C.POINTER(bounds.CollisionOut)
SURFACE = {
    "set_map": [vp, BM], "set_map_device": [vp, BM, vp], "set_occupancy": [vp, OM], "set_occupancy_device": [vp, OM, vp],
    "get_map": [vp, BM, vp], "set_map_slot": [vp, i32, BM], "set_map_slot_device": [vp, i32, BM, vp],
    "set_occupancy_slots": [vp, i32, ST], "set_occupancy_slots_device": [vp, i32, ST, vp],
    "get_map_slot": [vp, i32, BM, vp], "map_count": [vp], "collision_check": [vp, CI, CO],
    "collision_check_device": [vp, CI, CO, vp], "collision_check_mapped": [vp, CI, vp, CO],
    "collision_check_mapped_device": [vp, CI, vp, CO, vp], "set_occupancy_boxes": [vp, i32, ST, i32, BX],
    "set_occupancy_boxes_device": [vp, i32, ST, i32, BX, vp],
}
MULTI = {
    "set_map_slot": [vp, i32, BM], "set_occupancy_slots": [vp, i32, ST], "set_occupancy_slots_device": [vp, i32, ST, vp],
    "set_occupancy_boxes": [vp, i32, ST, i32, BX], "set_occupancy_boxes_device": [vp, i32, ST, i32, BX, vp],
    "get_map_slot": [vp, i32, i32, BM, vp],
}


def test_map_entry_point_argtypes():
    L = bounds._declare(solver.load_library())
    plan_multi._lib()
    for prefix, table in (("pqp_bounds_", SURFACE), ("pqp_plan_", SURFACE), ("pqp_plan_multi_", MULTI)):
        for name, argtypes in table.items():
            assert list(getattr(L, prefix + name).argtypes) == argtypes, prefix + name
    assert L.pqp_bounds_map_count.restype is C.c_int32 and L.pqp_plan_map_count.restype is C.c_int32


# ------------------------------------------------------------------------------------------------- GPU
N_SLOTS, SHAPE, RES = 4, (37, 29), 0.1
SENTINEL = (np.full(SHAPE, 5.0, np.float32), 1.0, (9.0, -9.0))  # every slot's map before each update


def _scene():
    rng = np.random.default_rng(17)
    per = np.where(rng.random((N_SLOTS,) + SHAPE) < 0.03, 0, 255).astype(np.uint8)
    centers = [(0.0, 0.0), (0.7, -0.4), (-1.1, 0.3), (0.2, 1.5)]
    k = np.array([2, 0, 3, 1], np.int32)
    boxes = np.zeros((N_SLOTS, 3, 5))
    for s in range(N_SLOTS):  # axis-aligned boxes: the predicate's cos / sin are exact
        boxes[s, :, 0] = centers[s][0] + rng.uniform(-1.5, 1.5, 3)
        boxes[s, :, 1] = centers[s][1] + rng.uniform(-1.2, 1.2, 3)
        boxes[s, :, 3:] = rng.uniform(0.3, 1.0, (3, 2))
    return per, centers, k, boxes


def _requests():
    """(name, first slot, count, kwargs of the update, the expected image of each updated slot)."""
    per, centers, k, boxes = _scene()
    shared = per[0]
    stamp = lambda img, s: bo.stamped_image(img, RES, centers[s], boxes[s, :k[s]], 127)  # noqa: E731
    return [
        ("image", 0, 1, dict(imgs=per[:1], centers=centers[:1]), [per[0]]),
        ("stack", 1, 3, dict(imgs=per[1:], centers=centers[1:]), list(per[1:])),
        ("shared boxes", 0, 4, dict(imgs=shared, centers=centers, boxes=boxes, k=k),
         [stamp(shared, s) for s in range(N_SLOTS)]),
        ("per-slot boxes", 1, 3, dict(imgs=per[1:], centers=centers[1:], boxes=boxes[1:], k=k[1:]),
         [stamp(per[s], s) for s in range(1, N_SLOTS)]),
    ]


def _handles():
    maps = [SENTINEL[0]] * N_SLOTS
    kw = dict(r_max=64, p_max=64, layers_max=64, n_max=120, batch_max=2)
    return (bounds.PathBounds.from_maps(maps, 1.0), plan.Planner.from_maps(maps, 1.0, **kw),
            plan_multi.MultiPlanner(maps, 1.0, devices=[0, 0], **kw))


def _reset(h):
    for s in range(N_SLOTS):
        if isinstance(h, plan_multi.MultiPlanner):
            h.set_map_slot(SENTINEL[0], SENTINEL[1], SENTINEL[2], slot=s)
        else:
            h.set_map(SENTINEL[0], SENTINEL[1], SENTINEL[2], slot=s)


def _slots(h):
    """Every slot's (layer, resolution, centre), of every device of a MultiPlanner."""
    if isinstance(h, plan_multi.MultiPlanner):
        return [h.get_map_slot(d, s) for d in range(2) for s in range(N_SLOTS)]
    return [h.get_map(s) for s in range(N_SLOTS)]


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x[0], y[0]) and x[1:] == y[1:] for x, y in zip(a, b))


def _update(h, form, first, kw):
    """One update through `h` in `form`; the one-image request at slot 0 takes set_occupancy where the handle has it."""
    import torch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    imgs, centers, boxes, k = kw["imgs"], kw["centers"], kw.get("boxes"), kw.get("k")
    single = boxes is None and first == 0 and len(imgs) == 1 and not isinstance(h, plan_multi.MultiPlanner)
    if form == "host":
        if single:
            h.set_occupancy(imgs[0], RES, centers[0], obstacle_max=127)
        elif boxes is None:
            h.set_occupancy_slots(imgs, RES, centers, obstacle_max=127, first_slot=first)
        else:
            h.set_occupancy_boxes(imgs, RES, boxes, k, centers, obstacle_max=127, first_slot=first)
        return
    d_imgs = t(imgs)  # the device inputs stay alive until the update has run
    d_boxes = (t(boxes), t(k)) if boxes is not None else ()
    if single and isinstance(h, plan.Planner):
        h.set_occupancy_device(d_imgs[0], RES, centers[0], obstacle_max=127)
    elif single:
        m = bounds.OccupancyMap(*SHAPE, RES, *centers[0], d_imgs.data_ptr(), 127)
        h._check(h.L.pqp_bounds_set_occupancy_device(h.h, C.byref(m), None))
    elif boxes is None:
        h.set_occupancy_slots_device(d_imgs, RES, centers, obstacle_max=127, first_slot=first)
    else:
        h.set_occupancy_boxes_device(d_imgs, RES, *d_boxes, centers, obstacle_max=127, first_slot=first)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_gpu_every_form_gives_the_oracle_slots():
    handles = _handles()
    try:
        for name, first, count, kw, images in _requests():
            want = [(SENTINEL[0], SENTINEL[1], SENTINEL[2])] * N_SLOTS
            for i, img in enumerate(images):
                s = first + i
                want[s] = (eo.transform(img, RES, 127 if "boxes" not in kw else 0)[1], RES, tuple(kw["centers"][i]))
            for h in handles:
                for form in ("host", "device"):
                    _reset(h)
                    c0 = h.launch_count if isinstance(h, plan.Planner) else None
                    _update(h, form, first, kw)
                    got = _slots(h)
                    expect = want * (2 if isinstance(h, plan_multi.MultiPlanner) else 1)
                    assert _same(got, expect), (name, type(h).__name__, form)
                    if c0 is not None:
                        launches = 2 if name == "image" else plan.occupancy_slots_launches(count)
                        assert h.launch_count - c0 == launches, (name, form)
    finally:
        for h in handles:
            h.close()


@pytest.mark.gpu
def test_gpu_refusals_leave_every_slot_untouched():
    import torch
    per, centers, k, boxes = _scene()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    host = dict(img=np.ascontiguousarray(per), k=np.ascontiguousarray(k), boxes=np.ascontiguousarray(boxes))
    dev = {n: t(a) for n, a in host.items()}
    ptr = dict(host={n: a.ctypes.data for n, a in host.items()}, device={n: a.data_ptr() for n, a in dev.items()})
    cx, cy = (np.ascontiguousarray([c[i] for c in centers]) for i in (0, 1))
    nan = np.array([0.0, float("nan"), 0.0, 0.0])
    k_hi = k.copy()
    k_hi[2] = 4

    def st(form, first=1, count=3, r=SHAPE[0], x=cx):
        return first, bounds.OccupancyStack(count, r, SHAPE[1], RES, x.ctypes.data, cy.ctypes.data, ptr[form]["img"], 127)

    def bx(form, k_max=3, kp="k", bp="boxes"):
        return bounds.ObstacleBoxes(k_max, ptr[form][kp] if kp else None, ptr[form][bp] if bp else None)

    # (name, stack args, shared_base, box args ("null": a NULL pqp_obstacle_boxes; None: set_occupancy_slots), host
    # form only)
    refused = [
        ("slot range", dict(first=2), 0, None, False), ("slot range", dict(first=-1), 0, {}, False),
        ("oversize", dict(r=SHAPE[0] + 1), 0, None, False), ("oversize", dict(r=SHAPE[0] + 1), 0, {}, False),
        ("centre", dict(x=nan), 0, None, False), ("centre", dict(x=nan), 0, {}, False),
        ("shared_base", {}, 2, {}, False), ("box cap", {}, 0, dict(k_max=bounds.MAX_BOXES // 3 + 1), False),
        ("null k", {}, 0, dict(kp=None), False), ("null boxes", {}, 0, dict(bp=None), False),
        ("null struct", {}, 0, "null", False), ("host k", {}, 0, dict(kp="k_hi"), True),
    ]
    host["k_hi"] = np.ascontiguousarray(k_hi)
    ptr["host"]["k_hi"] = host["k_hi"].ctypes.data
    handles = _handles()
    try:
        L = handles[0].L
        for h in handles:
            h.set_occupancy_slots(per, RES, centers, obstacle_max=127)
        before = [_slots(h) for h in handles]
        for h, prefix in zip(handles, ("pqp_bounds_", "pqp_plan_", "pqp_plan_multi_")):
            for name, sa, shared, ba, host_only in refused:
                for form in ("host",) if host_only else ("host", "device"):
                    first, s_ = st(form, **sa)
                    suffix = "_device" if form == "device" else ""
                    tail = (C.c_void_p(torch.cuda.current_stream().cuda_stream),) if suffix else ()
                    if ba is None:
                        fn = prefix + "set_occupancy_slots" + suffix
                        rc = getattr(L, fn)(h.h, first, C.byref(s_), *tail)
                    else:
                        fn = prefix + "set_occupancy_boxes" + suffix
                        b_ = None if ba == "null" else C.byref(bx(form, **ba))
                        rc = getattr(L, fn)(h.h, first, C.byref(s_), shared, b_, *tail)
                    assert rc == abi.PQP_E_INVALID, (fn, name)
                    if prefix == "pqp_bounds_":
                        assert L.pqp_bounds_last_error(h.h).decode().startswith(fn + ": "), (fn, name)
            if prefix != "pqp_plan_multi_":  # the one-image call: oversize and a non-finite centre
                for form in ("host", "device"):
                    suffix = "_device" if form == "device" else ""
                    tail = (C.c_void_p(torch.cuda.current_stream().cuda_stream),) if suffix else ()
                    for r, x in ((SHAPE[0] + 1, 0.0), (SHAPE[0], float("inf"))):
                        m = bounds.OccupancyMap(r, SHAPE[1], RES, x, 0.0, ptr[form]["img"], 127)
                        fn = prefix + "set_occupancy" + suffix
                        assert getattr(L, fn)(h.h, C.byref(m), *tail) == abi.PQP_E_INVALID, (fn, r, x)
        torch.cuda.synchronize()
        for h, b in zip(handles, before):
            assert _same(_slots(h), b), type(h).__name__
    finally:
        for h in handles:
            h.close()
