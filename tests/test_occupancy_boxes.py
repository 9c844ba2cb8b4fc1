"""Obstacle boxes stamped into each map slot's occupancy on the GPU (pqp_bounds_set_occupancy_boxes*,
pqp_plan_set_occupancy_boxes*, pqp_plan_multi_set_occupancy_boxes*; include/pqp_bounds.h).

CPU: the kernels' source (tests/emu/boxes_driver.cpp) against the box oracle (tests/box_oracle.py) and the transform oracle bit for bit on the demo
image and the edge cases; the oracle's mask against an independent half-plane test; the C layout of
pqp_obstacle_boxes.
GPU: slot layers against set_occupancy_slots of the oracle-stamped images (shared and per-slot bases, count 1, 3 and
1025, ragged k), plans and the collision check on stamped slots, launch counts, stream order, clamping of k on the
device, refusals, and the multi-GPU handle against a single one.
"""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import edt_oracle as eo
from tests import box_oracle as bo
from path_optimizer_2_b200 import abi, bounds, plan, sharedmap
from tests.emu import boxes_emu
from tests.test_map_slots import _compile_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PNG = os.path.join(ROOT, "tests", "golden", "gridmap.png")
RES = sharedmap.RES
EDGE = 1e-9  # no fixture at a random heading puts a cell centre this close to a box edge


def _png():
    from PIL import Image
    return np.asarray(Image.open(PNG).convert("L")).astype(np.uint8)


def _random_boxes(rng, shape, res, center, k, side=1.8, headings=False, spread=1.0):
    """k boxes of side x side m with centres uniform over the map (times `spread`), heading 0 or random."""
    rows, cols = shape
    hx, hy = 0.5 * rows * res * spread, 0.5 * cols * res * spread
    b = np.zeros((k, 5))
    b[:, 0] = center[0] + rng.uniform(-hx, hx, k)
    b[:, 1] = center[1] + rng.uniform(-hy, hy, k)
    b[:, 2] = rng.uniform(-math.pi, math.pi, k) if headings else 0.0
    b[:, 3] = side
    b[:, 4] = side
    return b


def _clear_of_edges(shape, res, center, boxes):
    return bo.edge_distance(shape, res, center, boxes).min() > EDGE


def _oracle(img, res, center, boxes, obstacle_max):
    return eo.transform(bo.stamped_image(img, res, center, boxes, obstacle_max), res, 0)


# ------------------------------------------------------------------------------------------------- CPU
def _edge_cases():
    """(name, image, resolution, centre, boxes, obstacle_max)."""
    rng = np.random.default_rng(5)
    small = np.where(rng.random((37, 23)) < 0.03, 0, 255).astype(np.uint8)
    free = np.full((37, 23), 255, np.uint8)
    res, c = 0.1, (0.0, 0.0)
    rows, cols = small.shape
    hx, hy = 0.5 * rows * res, 0.5 * cols * res
    px, py = bo.cell_centres(small.shape, res, c)
    qx, qy = bo.cell_centres(small.shape, 0.125, c)  # dyadic: every centre, sum and half below is exact
    cases = [
        ("outside", small, res, c, [[hx + 0.3, 0.0, 0.4, 1.5, 1.0], [0.0, -hy - 0.2, -1.1, 2.0, 1.2],
                                    [hx + 50.0, hy + 50.0, 0.0, 3.0, 3.0], [-hx - 9.0, 0.0, 0.3, 1.0, 1.0]], 0),
        ("whole map", small, res, c, [[0.0, 0.0, 0.0, 2 * hx + 1.0, 2 * hy + 1.0]], 0),
        ("zero size on a centre", free, res, c, [[px[11, 0], py[0, 7], 0.0, 0.0, 0.0],
                                                 [px[3, 0], py[0, 20], 0.9, 0.0, 0.0]], 0),
        # heading 0 (c = 1, s = 0 exactly): the box's edges fall on rows 10 and 14, columns 5 and 8 exactly
        ("closed boundary", free, 0.125, c, [[0.5 * (qx[10, 0] + qx[14, 0]), 0.5 * (qy[0, 5] + qy[0, 8]), 0.0,
                                              qx[10, 0] - qx[14, 0], qy[0, 5] - qy[0, 8]]], 0),
        ("nan and negative", free, res, c, [[np.nan, 0.0, 0.0, 1.0, 1.0], [0.0, np.nan, 0.0, 1.0, 1.0],
                                            [0.0, 0.0, np.nan, 1.0, 1.0], [0.0, 0.0, 0.0, np.nan, 1.0],
                                            [0.0, 0.0, 0.0, 1.0, np.nan], [0.0, 0.0, 0.0, -1.0, 1.0],
                                            [0.0, 0.0, 0.0, 1.0, -0.5], [0.0, 0.0, np.inf, 1.0, 1.0]], 0),
        ("no boxes", small, res, c, np.zeros((0, 5)), 0),
    ]
    # off the origin, rows != cols, both thresholds, random headings away from the edges
    grey = rng.integers(0, 256, (41, 29)).astype(np.uint8)
    for om in (0, 127):
        center = (3.7, -12.25)
        for seed in range(50):
            b = _random_boxes(np.random.default_rng(seed), grey.shape, 0.15, center, 5, side=1.1, headings=True,
                              spread=1.2)
            if _clear_of_edges(grey.shape, 0.15, center, b):
                break
        else:
            raise AssertionError("no fixture clear of the edges")
        cases.append(("off origin om=%d" % om, grey, 0.15, center, b, om))
    return cases


@pytest.mark.parametrize("case", range(len(_edge_cases())))
def test_driver_equals_oracle_on_edge_cases(case):
    name, img, res, center, boxes, om = _edge_cases()[case]
    d2, layer = boxes_emu.transform(img, res, center, boxes, om)
    od2, olayer = _oracle(img, res, center, boxes, om)
    assert np.array_equal(layer, olayer), name
    if name == "whole map":
        assert not layer.any()
    if name in ("nan and negative", "no boxes"):
        assert np.array_equal(layer, eo.transform(img, res, om)[1]), name
    if name == "zero size on a centre":
        obst = bo.stamp_boxes(img, res, center, boxes, om)
        assert obst.sum() == 2 and obst[11, 7] and obst[3, 20]
    if name == "closed boundary":
        obst = bo.stamp_boxes(img, res, center, boxes, om)
        want = np.zeros_like(obst)
        want[10:15, 5:9] = True
        assert np.array_equal(obst, want)
    if bo.stamp_boxes(img, res, center, boxes, om).any():
        assert np.array_equal(d2, od2), name


@pytest.mark.parametrize("headings", (False, True))
def test_driver_equals_oracle_on_demo_image(headings):
    img = _png()
    for seed in range(50):
        b = _random_boxes(np.random.default_rng(100 + seed), img.shape, RES, (0.0, 0.0), 12, headings=headings)
        if not headings or _clear_of_edges(img.shape, RES, (0.0, 0.0), b):
            break
    else:
        raise AssertionError("no fixture clear of the edges")
    d2, layer = boxes_emu.transform(img, RES, (0.0, 0.0), b, 127)
    od2, olayer = _oracle(img, RES, (0.0, 0.0), b, 127)
    assert np.array_equal(layer, olayer) and np.array_equal(d2, od2)
    stamped = bo.stamp_boxes(img, RES, (0.0, 0.0), b, 127) & ~eo.obstacles(img, 127)
    assert stamped.sum() > 100  # some boxes landed on free cells


def _half_planes(shape, res, center, boxes):
    """Inside or on the edge of the box by the sign of the cross product against each edge of its four corners."""
    px, py = bo.cell_centres(shape, res, center)
    px, py = np.broadcast_arrays(px, py)
    out = np.zeros(shape, bool)
    for x, y, h, length, width in np.asarray(boxes, dtype=np.float64).reshape(-1, 5):
        ex, ey = np.array([math.cos(h), math.sin(h)]), np.array([-math.sin(h), math.cos(h)])
        corners = [np.array([x, y]) + sl * 0.5 * length * ex + sw * 0.5 * width * ey
                   for sl, sw in ((1, 1), (-1, 1), (-1, -1), (1, -1))]  # counter-clockwise
        inside = np.ones(shape, bool)
        for a, b in zip(corners, corners[1:] + corners[:1]):
            inside &= (b[0] - a[0]) * (py - a[1]) - (b[1] - a[1]) * (px - a[0]) >= 0
        out |= inside
    return out


def test_oracle_mask_matches_half_planes():
    rng = np.random.default_rng(9)
    shape, res, center = (120, 90), 0.1, (1.5, -2.0)
    free = np.full(shape, 255, np.uint8)
    for trial in range(20):
        b = _random_boxes(rng, shape, res, center, 6, side=rng.uniform(0.2, 4.0), headings=True)
        b[:, 4] *= rng.uniform(0.3, 1.0, len(b))
        mask = bo.stamp_boxes(free, res, center, b)
        hp = _half_planes(shape, res, center, b)
        near = bo.edge_distance(shape, res, center, b) <= EDGE
        assert np.array_equal(mask[~near], hp[~near]), trial
        assert mask.any()
        # the kernels' predicate, compiled for the host, where no cos / sin bit can decide a cell
        assert np.array_equal(boxes_emu.mask(shape, res, center, b)[~near], mask[~near]), trial


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "pqp_bounds.h"
#define F(m) printf("%s %zu\n", #m, offsetof(pqp_obstacle_boxes, m))
int main(void) {
    printf("size %zu\n", sizeof(pqp_obstacle_boxes));
    F(k_max); F(k); F(boxes);
    printf("fields %d\nmax %d\n", PQP_BOX_FIELDS, PQP_MAX_BOXES);
    return 0;
}
"""


def test_obstacle_boxes_layout_matches_ctypes():
    out = _compile_run(_LAYOUT_C, "layout.c", "gcc", "-std=c99")
    got = {k: int(v) for k, v in (line.split() for line in out.splitlines())}
    S = bounds.ObstacleBoxes
    assert got == {"size": ctypes.sizeof(S), **{n: getattr(S, n).offset for n, _ in S._fields_},
                   "fields": bounds.BOX_FIELDS, "max": bounds.MAX_BOXES}


def test_pack_boxes():
    lst = [np.ones((2, 5)), np.zeros((0, 5)), 2 * np.ones((3, 5))]
    packed, k = bounds.pack_boxes(lst, None, 3)
    assert packed.shape == (3, 3, 5) and k.tolist() == [2, 0, 3]
    assert (packed[0, :2] == 1).all() and (packed[2] == 2).all() and not packed[0, 2:].any()
    arr = np.ones((3, 4, 5))
    assert bounds.pack_boxes(arr, None, 3)[1].tolist() == [4, 4, 4]
    assert bounds.box_base((5, 7), 3) == (3, 1, (5, 7)) and bounds.box_base((2, 5, 7)) == (2, 0, (5, 7))


# ------------------------------------------------------------------------------------------------- GPU
def _slot_scene(count, shape, seed, k_max=6, headings=True, res=0.1):
    """A shared base, per-slot bases and ragged boxes (some slots without any) for `count` slots of `shape`; every box
    clear of the cell centres' edge band when at a random heading."""
    rng = np.random.default_rng(seed)
    shared = np.where(rng.random(shape) < 0.02, 0, 255).astype(np.uint8)
    per = np.where(rng.random((count,) + shape) < 0.02, 0, 255).astype(np.uint8)
    centers = [(rng.uniform(-3, 3), rng.uniform(-3, 3)) for _ in range(count)]
    k = rng.integers(0, k_max + 1, count).astype(np.int32)
    k[::4] = 0
    boxes = np.full((count, k_max, 5), np.nan)  # padding past k[s] is never read
    for s in range(count):
        for _ in range(100):
            b = _random_boxes(rng, shape, res, centers[s], int(k[s]), side=rng.uniform(0.3, 1.5), headings=headings,
                              spread=1.1)
            if k[s] == 0 or not headings or _clear_of_edges(shape, res, centers[s], b):
                break
        else:
            raise AssertionError("no fixture clear of the edges")
        boxes[s, :k[s]] = b
    return dict(shared=shared, per=per, centers=centers, k=k, boxes=boxes, res=res)


def _stamped(sc, shared):
    return np.stack([bo.stamped_image(sc["shared"] if shared else sc["per"][s], sc["res"], sc["centers"][s],
                                      sc["boxes"][s, :sc["k"][s]], 127) for s in range(len(sc["k"]))])


def _layers(h, first, count):
    return [h.get_map(first + s) for s in range(count)]


def _assert_same_slots(a, b, tag):
    assert len(a) == len(b)
    for s, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x[0], y[0]) and x[1:] == y[1:], (tag, s)


@pytest.mark.gpu
@pytest.mark.parametrize("count", (1, 3, 1025))
def test_gpu_layers_equal_stamped_images(count):
    import torch
    shape = (40, 31) if count > 3 else (57, 44)
    sc = _slot_scene(count, shape, seed=count)
    n_maps = count + 2
    sentinel = [np.full(shape, 7.0, np.float32)] * n_maps
    got = bounds.PathBounds.from_maps(sentinel, 1.0)
    ref = bounds.PathBounds.from_maps(sentinel, 1.0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    for shared in (True, False):
        base = sc["shared"] if shared else sc["per"]
        imgs = _stamped(sc, shared)
        ref.set_occupancy_slots(imgs, sc["res"], sc["centers"], obstacle_max=0, first_slot=1)
        want = _layers(ref, 1, count)
        for s in (0, count - 1):  # the reference path against the oracle itself
            assert np.array_equal(want[s][0], eo.transform(imgs[s], sc["res"], 0)[1]), s
        got.set_occupancy_boxes(base, sc["res"], sc["boxes"], sc["k"], sc["centers"], obstacle_max=127, first_slot=1)
        _assert_same_slots(_layers(got, 1, count), want, ("host", shared))
        assert np.array_equal(got.get_map(0)[0], sentinel[0]) and np.array_equal(got.get_map(count + 1)[0], sentinel[0])
        got.set_map(sentinel[0], 1.0, slot=1)
        s_ = torch.cuda.current_stream().cuda_stream
        got.set_occupancy_boxes_device(t(base), sc["res"], t(sc["boxes"]), t(sc["k"]), sc["centers"], obstacle_max=127,
                                       first_slot=1, stream=s_)
        torch.cuda.synchronize()
        _assert_same_slots(_layers(got, 1, count), want, ("device", shared))
    # all k = 0 on per-slot bases: set_occupancy_slots exactly
    zero = np.zeros(count, np.int32)
    got.set_occupancy_boxes(sc["per"], sc["res"], sc["boxes"], zero, sc["centers"], obstacle_max=127, first_slot=1)
    ref.set_occupancy_slots(sc["per"], sc["res"], sc["centers"], obstacle_max=127, first_slot=1)
    _assert_same_slots(_layers(got, 1, count), _layers(ref, 1, count), "k = 0")
    got.set_occupancy_boxes(sc["per"], sc["res"], np.zeros((count, 0, 5)), None, sc["centers"], obstacle_max=127,
                            first_slot=1)
    _assert_same_slots(_layers(got, 1, count), _layers(ref, 1, count), "k_max = 0")
    got.close()
    ref.close()


@pytest.mark.gpu
def test_gpu_demo_image_boxes_and_headings():
    """The demo image shared by 3 slots, 12 boxes each, axis-aligned and at random headings, against the oracle."""
    img = _png()
    for headings in (False, True):
        boxes, centers = [], [(0.0, 0.0), (2.5, -4.0), (-7.0, 1.0)]
        for s, c in enumerate(centers):
            for seed in range(50):
                b = _random_boxes(np.random.default_rng(1000 * s + seed), img.shape, RES, c, 12, headings=headings)
                if _clear_of_edges(img.shape, RES, c, b):
                    break
            else:
                raise AssertionError("no fixture clear of the edges")
            boxes.append(b)
        pbn = bounds.PathBounds.from_maps([np.zeros(img.shape, np.float32)] * 3, RES)
        pbn.set_occupancy_boxes(img, RES, boxes, centers=centers, obstacle_max=127)
        for s, c in enumerate(centers):
            got, res, cc = pbn.get_map(s)
            assert np.array_equal(got, _oracle(img, RES, c, boxes[s], 127)[1]) and cc == c, (headings, s)
        pbn.close()


def _plan_scene():
    """The demo map, PER plan-point inputs on it, and a box on every third path's middle point; heading 0, so that
    the slots stamped on the device equal images stamped by numpy whatever its cos / sin."""
    img = _png()
    dmap = sharedmap.DistanceMap()
    pts = sharedmap.make_plan_points(PER, dmap=dmap)
    boxes = []
    for b in range(0, PER, 3):
        m = len(pts[0][b]) // 2
        boxes.append([pts[0][b][m], pts[1][b][m], 0.0, 1.8, 1.8])
    return img, dmap, pts, np.array(boxes)


PER = 24


@pytest.mark.gpu
@pytest.mark.parametrize("method", ("TENSION2", "TENSION"))
def test_gpu_plans_on_stamped_slots(method):
    from tests.test_map_slots import _assert_row
    from tests.test_plan_points import L_MAX, N_MAX, P_MAX, R_MAX
    img, dmap, pts, boxes = _plan_scene()
    zero = np.zeros(img.shape, np.float32)
    kw = dict(r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=2 * PER,
              params=plan.default_params(method))
    a = plan.Planner.from_maps([zero] * 2, RES, **kw)
    b = plan.Planner.from_maps([zero] * 2, RES, **kw)
    a.set_occupancy_boxes(img, RES, [boxes, np.zeros((0, 5))], obstacle_max=127)
    b.set_occupancy_slots(np.stack([bo.stamped_image(img, RES, (0, 0), boxes, 127), img]), RES, obstacle_max=127)
    idx = np.repeat(np.array([0, 1], np.int32), PER)
    inputs = (pts[0] * 2, pts[1] * 2, np.concatenate([pts[2]] * 2), np.concatenate([pts[3]] * 2))
    ra = a.plan_points(*inputs, trace=True, map_index=idx)
    rb = b.plan_points(*inputs, trace=True, map_index=idx)
    for i in range(2 * PER):
        _assert_row(ra, rb, i, i, (method, i))
    assert not np.array_equal(ra.path[:PER], ra.path[PER:])  # the boxes changed some plans
    assert np.mean(ra.status[PER:] == plan.OK) > 0.6
    if method == "TENSION2":
        # a pose inside a stamped box is the first hit of a path whose other poses are free
        for p in range(PER, 2 * PER):
            n = int(ra.n[p])
            if ra.status[p] != plan.OK or n < 40:
                continue
            poses = np.ascontiguousarray(ra.path[p:p + 1, :3, [0, 1, n - 1]])
            far = np.hypot(*(poses[0, :2, 2] - poses[0, :2, 0])) > 12.0
            if far and a.check_collision(poses, [3], map_index=[1])["first_hit"][0] == 3:
                break
        else:
            raise AssertionError("no free path to place a box on")
        box = [poses[0, 0, 2], poses[0, 1, 2], poses[0, 2, 2], 2.0, 2.0]
        a.set_occupancy_boxes(img, RES, [np.zeros((0, 5)), [box]], obstacle_max=127)
        assert a.check_collision(poses, [3], map_index=[1])["first_hit"][0] == 2
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_launch_counts_stream_order_and_clamp():
    import torch
    from tests.test_plan_points import L_MAX, N_MAX, P_MAX, R_MAX
    img, dmap, pts, boxes = _plan_scene()
    zero = np.zeros(img.shape, np.float32)
    kw = dict(r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=PER)
    pl = plan.Planner.from_maps([zero], RES, **kw)
    pl.set_occupancy(img, RES, obstacle_max=127)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    m = np.array([len(v) for v in pts[0]], np.int32)
    px, py = np.zeros((PER, R_MAX)), np.zeros((PER, R_MAX))
    for b in range(PER):
        px[b, :m[b]], py[b, :m[b]] = pts[0][b], pts[1][b]
    args = [t(px), t(py), t(m), t(pts[2]), t(pts[3])]
    d_img, d_boxes, d_k = t(img), t(boxes[None]), t(np.array([len(boxes)], np.int32))
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        first = pl.plan_points_device(*args)
        c0 = pl.launch_count
        pl.set_occupancy_boxes_device(d_img, RES, d_boxes, d_k, obstacle_max=127)
        c1 = pl.launch_count
        second = pl.plan_points_device(*args)
    s.synchronize()
    assert c1 - c0 == plan.occupancy_slots_launches(1) == 3
    old = pl.plan_points(*pts[:4])  # unmapped: slot 0, now stamped
    stamped = plan.Planner(eo.transform(bo.stamped_image(img, RES, (0, 0), boxes, 127), RES, 0)[1], RES, **kw)
    base = plan.Planner(dmap.dist, RES, **kw)
    want_first, want_second = base.plan_points(*pts[:4]), stamped.plan_points(*pts[:4])
    assert np.array_equal(first["path"].cpu().numpy(), want_first.path)
    assert np.array_equal(second["path"].cpu().numpy(), want_second.path)
    assert np.array_equal(old.path, want_second.path) and not np.array_equal(want_first.path, want_second.path)
    stamped.close()
    base.close()
    pl.close()
    # 1025 slots: 2 + 2 table launches; out-of-range k clamped on the device
    small = (24, 20)
    sc = _slot_scene(1025, small, seed=3, k_max=3)
    big = plan.Planner.from_maps([np.zeros(small, np.float32)] * 1025, 0.1, **dict(kw, batch_max=1))
    c0 = big.launch_count
    big.set_occupancy_boxes(sc["shared"], 0.1, sc["boxes"], sc["k"], sc["centers"], obstacle_max=127)
    assert big.launch_count - c0 == plan.occupancy_slots_launches(1025) == 4
    want = _layers(big, 0, 1025)
    k_bad = sc["k"].copy()
    k_bad[sc["k"] == 0] = -5  # -> 0
    k_bad[sc["k"] == 3] = 40  # -> k_max = 3
    big.set_map(np.zeros(small, np.float32), 0.1, slot=5)
    c0 = big.launch_count
    big.set_occupancy_boxes_device(t(sc["shared"]), 0.1, t(sc["boxes"]), t(k_bad), sc["centers"], obstacle_max=127)
    torch.cuda.synchronize()
    assert big.launch_count - c0 == 4
    _assert_same_slots(_layers(big, 0, 1025), want, "clamped k")
    big.close()


@pytest.mark.gpu
def test_gpu_refusals_leave_slots_untouched():
    shape = (30, 26)
    sc = _slot_scene(3, shape, seed=11, k_max=4)
    n_maps = 4
    pbn = bounds.PathBounds.from_maps([np.full(shape, 3.0, np.float32)] * n_maps, 1.0)
    pbn.set_occupancy_boxes(sc["per"], 0.1, sc["boxes"], sc["k"], sc["centers"], obstacle_max=127, first_slot=1)
    before = _layers(pbn, 0, n_maps)
    L = pbn.L
    img = np.ascontiguousarray(sc["per"])
    cx = np.ascontiguousarray([c[0] for c in sc["centers"]])
    cy = np.ascontiguousarray([c[1] for c in sc["centers"]])
    xs = np.ascontiguousarray(sc["boxes"])
    k = np.ascontiguousarray(sc["k"])
    k_hi, k_lo = k.copy(), k.copy()
    k_hi[1], k_lo[2] = 5, -1

    def st(count=3, r=shape[0], c=shape[1], res=0.1, cells=img.ctypes.data, x=cx):
        return bounds.OccupancyStack(count, r, c, res, x.ctypes.data, cy.ctypes.data, cells, 127)

    def bx(k_max=4, kp=k.ctypes.data, bp=xs.ctypes.data):
        return bounds.ObstacleBoxes(k_max, kp, bp)

    nan = np.array([0.0, float("nan"), 0.0])
    refused = [  # (first_slot, stack, shared_base, boxes, host form only)
        (1, st(r=1), 0, bx(), False), (1, st(cells=None), 0, bx(), False), (1, st(res=0.0), 0, bx(), False),
        (1, st(x=nan), 0, bx(), False), (2, st(), 0, bx(), False), (-1, st(), 0, bx(), False),
        (1, st(count=0), 0, bx(), False), (1, st(r=shape[0] + 1), 0, bx(), False),
        (1, st(), 2, bx(), False), (1, st(), -1, bx(), False), (1, st(), 0, None, False),
        (1, st(), 0, bx(k_max=-1), False), (1, st(), 0, bx(k_max=bounds.MAX_BOXES // 3 + 1), False),
        (1, st(), 0, bx(kp=None), False), (1, st(), 0, bx(bp=None), False),
        (1, st(), 0, bx(kp=k_hi.ctypes.data), True), (1, st(), 0, bx(kp=k_lo.ctypes.data), True),
    ]
    for i, (first, s_, shared, b_, host_only) in enumerate(refused):
        pb = ctypes.byref(b_) if b_ is not None else None
        assert L.pqp_bounds_set_occupancy_boxes(pbn.h, first, ctypes.byref(s_), shared, pb) == abi.PQP_E_INVALID, i
        assert L.pqp_bounds_last_error(pbn.h), i
        if not host_only:
            assert L.pqp_bounds_set_occupancy_boxes_device(pbn.h, first, ctypes.byref(s_), shared, pb,
                                                           None) == abi.PQP_E_INVALID, i
            assert L.pqp_bounds_last_error(pbn.h), i
    assert L.pqp_bounds_set_occupancy_boxes(pbn.h, 0, None, 0, ctypes.byref(bx())) == abi.PQP_E_INVALID
    assert L.pqp_bounds_set_occupancy_boxes(None, 0, ctypes.byref(st()), 0, ctypes.byref(bx())) == abi.PQP_E_INVALID
    # the cap counts count * k_max, not the boxes in use: exactly PQP_MAX_BOXES is accepted
    one = bounds.PathBounds.from_maps([np.zeros(shape, np.float32)], 1.0)
    kmax = np.zeros(1, np.int32)
    cap = np.zeros((bounds.MAX_BOXES, 5))
    s1 = bounds.OccupancyStack(1, shape[0], shape[1], 0.1, cx.ctypes.data, cy.ctypes.data, img.ctypes.data, 127)
    assert L.pqp_bounds_set_occupancy_boxes(one.h, 0, ctypes.byref(s1), 1, ctypes.byref(
        bounds.ObstacleBoxes(bounds.MAX_BOXES, kmax.ctypes.data, cap.ctypes.data))) == 0  # PQP_OK
    one.close()
    _assert_same_slots(_layers(pbn, 0, n_maps), before, "after refusals")
    pbn.close()


@pytest.mark.gpu
def test_gpu_multi_planner_matches_planner():
    import torch
    from path_optimizer_2_b200 import plan_multi
    from tests.test_plan_points import L_MAX, N_MAX, P_MAX, R_MAX
    img, dmap, pts, boxes = _plan_scene()
    zero = np.zeros(img.shape, np.float32)
    kw = dict(r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=2 * PER)
    single = plan.Planner.from_maps([zero] * 3, RES, **kw)
    multi = plan_multi.MultiPlanner([zero] * 3, RES, devices=[0, 0], **kw)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    per_slot = [boxes, np.zeros((0, 5)), boxes[::2] + np.array([0.4, -0.3, 0.5, 0.0, 0.0])]
    packed, k = bounds.pack_boxes(per_slot, None, 3)
    centers = [(0.0, 0.0)] * 3
    idx = np.repeat(np.array([0, 2], np.int32), PER)
    inputs = (pts[0] * 2, pts[1] * 2, np.concatenate([pts[2]] * 2), np.concatenate([pts[3]] * 2))
    for form in ("host", "device"):
        for h in (single, multi):
            if h is multi:  # slot 0 reset, so that each form has to write it
                h.set_map_slot(zero, RES, slot=0)
            else:
                h.set_map(zero, RES, slot=0)
            if form == "host":
                h.set_occupancy_boxes(img, RES, per_slot, centers=centers, obstacle_max=127)
            else:
                h.set_occupancy_boxes_device(t(img), RES, t(packed), t(k), centers, obstacle_max=127)
        torch.cuda.synchronize()
        for s in range(3):
            want = single.get_map(s)
            for d in range(2):
                got = multi.get_map_slot(d, s)
                assert np.array_equal(got[0], want[0]) and got[1:] == want[1:], (form, d, s)
        a = single.plan_points(*inputs, map_index=idx)
        b = multi.plan_points(*inputs, map_index=idx)
        for f in ("status", "n", "path", "cost", "iters"):
            assert np.array_equal(getattr(a, f), getattr(b, f)), (form, f)
    multi.close()
    single.close()
