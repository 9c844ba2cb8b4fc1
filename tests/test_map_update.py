"""Replacing a live handle's map (pqp_bounds_set_map*, pqp_bounds_set_occupancy*, pqp_plan_set_*) and the exact
Euclidean distance transform of an occupancy image on the GPU.

CPU: oracle/edt_oracle.py against the brute-force definition, scipy and (where installed) OpenCV; the kernels' source
(pqp_map_core.cuh under g++) against the oracle bit for bit; the C layout of pqp_occupancy_map.
GPU: the transform read back with get_map against the oracle (host and device calls); set_map semantics and refused
maps; a planner after set_occupancy(B) against a fresh planner on B's layer in every output and trace field, under
both smoothing methods and both inputs, and back to A; the update changing blocked paths; the standalone bounds and
DP handles on B; stream order; launch counts; the C++ drop-in's setOccupancy.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import edt_oracle as eo
from path_optimizer_2_b200 import abi, bounds, plan, sharedmap
from tests.emu import map_emu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PNG = os.path.join(ROOT, "tests", "golden", "gridmap.png")
RES = sharedmap.RES


def _png():
    from PIL import Image
    return np.asarray(Image.open(PNG).convert("L")).astype(np.uint8)


def _random_grid(rng, rows, cols, density, obstacle_max):
    """uint8 image whose obstacle cells (value <= obstacle_max) make up about `density` of it."""
    obst = rng.random((rows, cols)) < density
    lo = rng.integers(0, obstacle_max + 1, (rows, cols)) if obstacle_max >= 0 else np.zeros((rows, cols))
    hi = rng.integers(obstacle_max + 1, 256, (rows, cols)) if obstacle_max < 255 else np.zeros((rows, cols))
    return np.where(obst, lo, hi).astype(np.uint8)


def _random_cases(seed=0, count=120, sizes=(2, 41)):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        rows, cols = (int(v) for v in rng.integers(*sizes, 2))
        density = float(rng.choice([0.0, 0.01, 0.05, 0.2, 0.6]))
        om = int(rng.choice([0, 1, 127, 254]))
        out.append((_random_grid(rng, rows, cols, density, om), om))
    return out


def _special_cases():
    """obstacle-free columns and rows, one obstacle in each corner, all obstacles, none, tall and wide grids."""
    cases = []
    free = np.full((37, 23), 255, np.uint8)
    cases.append((free.copy(), 0))                    # no obstacle at all
    cases.append((np.zeros((9, 13), np.uint8), 0))    # all obstacles
    for i, j in ((0, 0), (0, 22), (36, 0), (36, 22)):
        a = free.copy()
        a[i, j] = 0
        cases.append((a, 0))
    a = free.copy()
    a[5, :] = 0                                       # one obstacle row: every other row has no obstacle
    cases.append((a, 0))
    a = free.copy()
    a[:, 7] = 0                                       # one obstacle column: every other column has none
    cases.append((a, 0))
    rng = np.random.default_rng(5)
    cases.append((_random_grid(rng, 3000, 5, 0.002, 0), 0))
    cases.append((_random_grid(rng, 5, 3000, 0.002, 0), 0))
    tall = np.full((3000, 5), 255, np.uint8)
    tall[1500, 2] = 0
    cases.append((tall, 0))
    wide = np.full((5, 3000), 255, np.uint8)
    wide[0, 2999] = 0
    cases.append((wide, 0))
    cases.append((np.array([[0, 255], [255, 255]], np.uint8), 0))
    cases.append((_random_grid(rng, 64, 64, 0.05, 0), 0))
    cases.append((_random_grid(rng, 300, 17, 0.05, 0), 0))
    return cases


def _scipy_layer(img, om, res):
    from scipy.ndimage import distance_transform_edt
    return distance_transform_edt(img > om).astype(np.float32) * np.float32(res)


# ------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_brute_force():
    for img, om in _random_cases(1) + _special_cases()[:9]:
        d2, layer = eo.transform(img, RES, om)
        bd2, blayer = eo.brute_force(img, RES, om)
        if bd2 is None:
            assert np.all(layer == np.float32(2.0 ** 64) * np.float32(RES)), img.shape
        else:
            assert np.array_equal(d2, bd2), (img.shape, om)
        assert np.array_equal(layer, blayer), (img.shape, om)


def test_oracle_matches_scipy():
    cases = [(_png(), 0), (_png(), 127)] + [(img, om) for img, om in _random_cases(2) if (img <= om).any()]
    cases += [c for c in _special_cases() if (c[0] <= c[1]).any()]
    for img, om in cases:
        _, layer = eo.transform(img, RES, om)
        assert np.array_equal(layer, _scipy_layer(img, om, RES)), (img.shape, om)


def test_oracle_against_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    cases = [_png(), _random_grid(rng, 64, 64, 0.1, 0), _random_grid(rng, 300, 17, 0.05, 0)]
    cases += [img for img, om in _random_cases(4, count=40) if om == 0 and (img == 0).any()]
    for img in cases:
        d2, _ = eo.transform(img, 1.0, 0)
        cv = cv2.distanceTransform(img, cv2.DIST_L2, cv2.DIST_MASK_PRECISE)
        assert np.array_equal(np.round(cv.astype(np.float64) ** 2).astype(np.int64), d2), img.shape
        ours = np.sqrt(d2.astype(np.float64)).astype(np.float32)
        assert np.all(np.abs(ours.view(np.int32) - cv.view(np.int32)) <= 1), img.shape  # within 1 ulp
    png = _png()
    assert np.array_equal(eo.transform(png, 1.0, 0)[1], cv2.distanceTransform(png, cv2.DIST_L2, cv2.DIST_MASK_PRECISE))
    free = np.full((20, 30), 255, np.uint8)
    assert np.all(cv2.distanceTransform(free, cv2.DIST_L2, cv2.DIST_MASK_PRECISE) == np.float32(2.0 ** 64))
    assert np.all(eo.transform(free, 1.0, 0)[1] == np.float32(2.0 ** 64))


def test_kernel_source_on_cpu_matches_oracle():
    for img, om in _random_cases(1) + _special_cases() + [(_png(), 0), (_png(), 127)]:
        d2, layer = map_emu.transform(img, RES, om)
        od2, olayer = eo.transform(img, RES, om)
        assert np.array_equal(layer, olayer), (img.shape, om)
        if (img <= om).any():
            assert np.array_equal(d2, od2), (img.shape, om)


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "pqp_bounds.h"
#define F(m) printf("%s %zu\n", #m, offsetof(pqp_occupancy_map, m))
int main(void) {
    printf("size %zu\n", sizeof(pqp_occupancy_map));
    F(rows); F(cols); F(resolution); F(center_x); F(center_y); F(cells); F(obstacle_max);
    return 0;
}
"""


def test_occupancy_layout_matches_ctypes():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(src, "w") as f:
            f.write(_LAYOUT_C)
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = {k: int(v) for k, v in (line.split() for line in subprocess.check_output([exe], text=True).splitlines())}
    S = bounds.OccupancyMap
    assert got == {"size": ctypes.sizeof(S), **{n: getattr(S, n).offset for n, _ in S._fields_}}


# ------------------------------------------------------------------------------------------------- GPU
from tests.test_plan_points import L_MAX, N_MAX, P_MAX, R_MAX  # noqa: E402

B = 32
METHODS = ("TENSION2", "TENSION")


def _cell(x, y, rows, cols):
    return int((rows * RES / 2 - x) / RES), int((cols * RES / 2 - y) / RES)


@pytest.fixture(scope="module")
def world():
    """Map A (the demo image), map B (A with a 1.8 m block on every third path's reference points) and the
    plan inputs of B paths on A, both as samples and as reference points."""
    img_a = _png()
    rows, cols = img_a.shape
    dist_a = eo.transform(img_a, RES, 127)[1]
    dmap = sharedmap.DistanceMap(dist=dist_a)
    raw = sharedmap.make_plan_inputs(B, dmap=dmap)
    pts = sharedmap.make_plan_points(B, dmap=dmap)
    img_b = img_a.copy()
    blocked = list(range(0, B, 3))
    for b in blocked:
        m = len(pts[0][b]) // 2
        i, j = _cell(pts[0][b][m], pts[1][b][m], rows, cols)
        img_b[max(i - 4, 0):i + 5, max(j - 4, 0):j + 5] = 0
    dist_b = eo.transform(img_b, RES, 127)[1]
    return dict(img_a=img_a, img_b=img_b, dist_a=dist_a, dist_b=dist_b, raw=raw, pts=pts, blocked=blocked)


def _planner(dist, method, batch_max=B):
    return plan.Planner(dist, RES, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX, batch_max=batch_max,
                        params=plan.default_params(method))


def _run(pl, w, points):
    return pl.plan_points(*w["pts"], trace=True) if points else pl.plan(*w["raw"], trace=True)


def _assert_same(a, b, tag, trace=True):
    """Outputs, and with `trace` every trace field. Trace entries a stage leaves unspecified keep whatever the
    handle's buffers held, so whole traces are compared only between handles that ran the same calls."""
    for k in ("status", "n", "path", "cost", "iters"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), (tag, k)
    for k in (a.trace if trace else ()):
        assert np.array_equal(a.trace[k], b.trace[k], equal_nan=True), (tag, k)


@pytest.fixture(scope="module", params=METHODS)
def planners(request, world):
    """(method, planner created on A and set to B by set_occupancy before its first plan, the results of a planner
    on A, a fresh planner on B)"""
    method = request.param
    pl = _planner(world["dist_a"], method)
    pl.set_occupancy(world["img_b"], RES, obstacle_max=127)
    on_a_planner = _planner(world["dist_a"], method)
    on_a = {p: _run(on_a_planner, world, p) for p in (False, True)}
    on_a_planner.close()
    fresh = _planner(world["dist_b"], method)
    yield method, pl, on_a, fresh
    pl.close()
    fresh.close()


@pytest.mark.gpu
def test_gpu_transform_matches_oracle():
    import torch
    rng = np.random.default_rng(9)
    big = np.where(rng.random((4096, 4096)) < 0.01, 0, 255).astype(np.uint8)
    pl = _planner(np.zeros((4096, 4096), np.float32), "TENSION2", batch_max=1)
    cases = _random_cases(1, count=60) + _special_cases() + [(_png(), 0), (_png(), 127), (big, 0)]
    for idx, (img, om) in enumerate(cases):
        res = 0.05 + 0.01 * (idx % 7)
        center = (float(idx) * 0.5, -float(idx))
        pl.set_occupancy(img, res, center, obstacle_max=om)
        got, gres, gc = pl.get_map()
        want = eo.transform(img, res, om)[1]
        assert np.array_equal(got, want), (img.shape, om)
        assert gres == res and gc == center
        # the device call on a fresh image gives the same layer
        pl.set_map(np.full(img.shape, -1.0, np.float32), 1.0)
        pl.set_occupancy_device(torch.from_numpy(img).cuda(), res, center, obstacle_max=om)
        dev, _, _ = pl.get_map()
        assert np.array_equal(dev, got), (img.shape, om)
    pl.close()


@pytest.mark.gpu
def test_gpu_set_map_semantics_and_refusals(world):
    L = plan._lib()
    dist_a = world["dist_a"]
    pl = _planner(dist_a, "TENSION2")
    before = _run(pl, world, True)
    rows, cols = dist_a.shape
    # get_map returns what was set, metadata included
    small = np.ascontiguousarray(dist_a[50:650, 100:600]) * np.float32(1.5)
    pl.set_map(small, 0.3, (2.5, -4.0))
    got, res, c = pl.get_map()
    assert np.array_equal(got, small) and res == 0.3 and c == (2.5, -4.0)
    pl.set_map(dist_a, RES)
    # refused maps leave the handle's map untouched
    keep = np.full((rows, cols), 7.0, np.float32)
    img = np.zeros((rows, cols), np.uint8)
    bad_maps = [bounds.BoundsMap(rows, cols + 1, RES, 0.0, 0.0, keep.ctypes.data),
                bounds.BoundsMap(1, cols, RES, 0.0, 0.0, keep.ctypes.data),
                bounds.BoundsMap(rows, 1, RES, 0.0, 0.0, keep.ctypes.data),
                bounds.BoundsMap(rows, cols, 0.0, 0.0, 0.0, keep.ctypes.data),
                bounds.BoundsMap(rows, cols, -0.2, 0.0, 0.0, keep.ctypes.data),
                bounds.BoundsMap(rows, cols, float("nan"), 0.0, 0.0, keep.ctypes.data),
                bounds.BoundsMap(rows, cols, float("inf"), 0.0, 0.0, keep.ctypes.data),
                bounds.BoundsMap(rows, cols, RES, float("nan"), 0.0, keep.ctypes.data),
                bounds.BoundsMap(rows, cols, RES, 0.0, float("inf"), keep.ctypes.data),
                bounds.BoundsMap(rows, cols, RES, 0.0, 0.0, None)]
    bad_occ = [bounds.OccupancyMap(rows + 1, cols, RES, 0.0, 0.0, img.ctypes.data, 0),
               bounds.OccupancyMap(rows, 1, RES, 0.0, 0.0, img.ctypes.data, 0),
               bounds.OccupancyMap(rows, cols, 0.0, 0.0, 0.0, img.ctypes.data, 0),
               bounds.OccupancyMap(rows, cols, float("nan"), 0.0, 0.0, img.ctypes.data, 0),
               bounds.OccupancyMap(rows, cols, RES, 0.0, 0.0, None, 0)]
    for m in bad_maps:
        assert L.pqp_plan_set_map(pl.h, ctypes.byref(m)) == abi.PQP_E_INVALID
        assert L.pqp_plan_set_map_device(pl.h, ctypes.byref(m), None) == abi.PQP_E_INVALID
        assert L.pqp_plan_last_error(pl.h)
    for m in bad_occ:
        assert L.pqp_plan_set_occupancy(pl.h, ctypes.byref(m)) == abi.PQP_E_INVALID
        assert L.pqp_plan_set_occupancy_device(pl.h, ctypes.byref(m), None) == abi.PQP_E_INVALID
    assert L.pqp_plan_set_map(pl.h, None) == abi.PQP_E_INVALID
    assert L.pqp_plan_set_occupancy(pl.h, None) == abi.PQP_E_INVALID
    got, res, c = pl.get_map()
    assert np.array_equal(got, dist_a) and res == RES and c == (0.0, 0.0)
    _assert_same(_run(pl, world, True), before, "after refused maps")
    pl.close()
    # a smaller map or a moved centre gives the bounds of a fresh handle created with that map
    lines = sharedmap.make_lines(8, 120, dmap=sharedmap.DistanceMap(dist=dist_a))
    pbn = bounds.PathBounds(dist_a, RES)
    for sub, center in ((dist_a, (1.3, -2.1)), (dist_a[100:500, 150:650], (0.0, 0.0)),
                        (dist_a[:300, :], (-20.0, 5.0))):
        pbn.set_map(sub, RES, center)
        ref = bounds.PathBounds(sub, RES, center=center)
        a = pbn.compute(lines.states, lines.n, lines.spline, lines.k)
        r = ref.compute(lines.states, lines.n, lines.spline, lines.k)
        assert np.array_equal(a[0], r[0]) and np.array_equal(a[1], r[1]), (sub.shape, center)
        ref.close()
    pbn.close()


@pytest.mark.gpu
def test_gpu_plan_after_set_occupancy_equals_fresh_planner(world, planners):
    method, pl, on_a, fresh = planners
    # the same calls on both handles: every output and every trace field
    for points in (False, True):
        _assert_same(_run(pl, world, points), _run(fresh, world, points), (method, points, "B"))
    # setting A back reproduces A's results
    pl.set_occupancy(world["img_a"], RES, obstacle_max=127)
    for points in (False, True):
        _assert_same(_run(pl, world, points), on_a[points], (method, points, "A again"), trace=False)
    pl.set_map(world["dist_b"], RES)
    for points in (False, True):
        _assert_same(_run(pl, world, points), _run(fresh, world, points), (method, points, "B by set_map"), trace=False)


@pytest.mark.gpu
def test_gpu_update_changes_blocked_paths(world, planners):
    method, pl, on_a, fresh = planners
    on_b = _run(fresh, world, True)
    a = on_a[True]
    assert np.mean(a.status == plan.OK) > 0.7, a.status_names()
    changed = [b for b in range(B) if a.status[b] != on_b.status[b] or not np.array_equal(a.path[b], on_b.path[b])]
    blocked_ok = [b for b in world["blocked"] if a.status[b] == plan.OK]
    assert len(set(changed) & set(blocked_ok)) >= len(blocked_ok) // 2, (method, changed, blocked_ok)
    assert any(on_b.status[b] != plan.OK for b in blocked_ok), (method, on_b.status_names())


@pytest.mark.gpu
def test_gpu_standalone_handles_see_the_new_map(world):
    from oracle import bounds_oracle, dp_oracle
    from path_optimizer_2_b200 import dp
    from tests.test_dp import _compare
    dist_a, dist_b = world["dist_a"], world["dist_b"]
    dmap_b = sharedmap.DistanceMap(dist=dist_b)
    lines = sharedmap.make_lines(16, 120, dmap=sharedmap.DistanceMap(dist=dist_a))
    pbn = bounds.PathBounds(dist_a, RES)
    ds = dp.DpSearch(pbn, layers_max=160, batch_max=16)
    pbn.set_occupancy(world["img_b"], RES, obstacle_max=127)
    got, _, _ = pbn.get_map()
    assert np.array_equal(got, dist_b)
    bnd, nv = pbn.compute(lines.states, lines.n, lines.spline, lines.k)
    for b in range(16):
        ob, onv = bounds_oracle.update_bounds(dmap_b.dist, RES, lines.spline_rows(b), *lines.states[b])
        d = np.abs(ob - bnd[b])
        assert onv == nv[b] and (d > 1e-9).mean() < 5e-3 and d.max() < 0.31, b
    length = np.array([lines.spline_rows(b)[0, lines.k[b] - 1] + 3.0 for b in range(16)])
    start = np.stack([lines.states[:, 1, 2], lines.states[:, 2, 2], lines.states[:, 3, 2]], axis=1)
    r = ds.search(lines.spline, lines.k, length, start)
    for b in range(16):
        _compare(r, b, dp_oracle.graph_search_dp(dist_b, RES, lines.spline_rows(b), length[b], start[b]), 34)
    ds.close()
    pbn.close()


@pytest.mark.gpu
def test_gpu_stream_order_and_launch_counts(world, planners):
    import torch
    method, pl, on_a, fresh = planners
    base = 26 if method == "TENSION" else 25
    pl.set_map(world["dist_a"], RES)
    ref_x, ref_y, start, target = world["pts"]
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((B, int(m.max()))), np.zeros((B, int(m.max())))
    for b in range(B):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    args = [t(px), t(py), t(m), t(start), t(target)]
    img_b = t(world["img_b"])
    s = torch.cuda.Stream(dev)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        c0 = pl.launch_count
        first = pl.plan_points_device(*args, trace=True)
        c1 = pl.launch_count
        pl.set_occupancy_device(img_b, RES, obstacle_max=127)
        c2 = pl.launch_count
        second = pl.plan_points_device(*args, trace=True)
        c3 = pl.launch_count
    s.synchronize()
    assert (c1 - c0, c2 - c1, c3 - c2) == (base, plan.OCCUPANCY_LAUNCHES, base)
    on_b = _run(fresh, world, True)
    assert not np.array_equal(on_a[True].status, on_b.status) or not np.array_equal(on_a[True].path, on_b.path)
    for out, want in ((first, on_a[True]), (second, on_b)):
        for k in ("status", "n", "path", "cost", "iters"):
            assert np.array_equal(out[k].cpu().numpy(), getattr(want, k)), k
    # a host set_occupancy also counts its two launches, and last_stage_ms still reports the last plan call
    c4 = pl.launch_count
    pl.set_occupancy(world["img_a"], RES, obstacle_max=127)
    assert pl.launch_count - c4 == plan.OCCUPANCY_LAUNCHES
    ms = pl.last_stage_ms
    assert 0 < ms["smoothing"] <= ms["total"]
    pl.set_occupancy(world["img_b"], RES, obstacle_max=127)  # leave the fixture's planner on B


def _dropin_build():
    from path_optimizer_2_b200 import solver
    solver.build_library()
    src = os.path.join(ROOT, "tests", "cpp", "map_update_test.cpp")
    exe = os.path.join(ROOT, "tests", "cpp", "map_update_test")
    deps = [src, os.path.join(ROOT, "include", "pqp_reference_path.hpp"), os.path.join(ROOT, "include", "pqp_bounds.h"),
            solver.LIB_PATH]
    if not os.path.exists(exe) or any(os.path.getmtime(d) > os.path.getmtime(exe) for d in deps):
        subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-o", exe, src, solver.LIB_PATH,
                               "-Wl,-rpath," + os.path.dirname(solver.LIB_PATH)])
    return exe


@pytest.mark.gpu
def test_gpu_cpp_dropin_set_occupancy(world, tmp_path):
    exe = _dropin_build()
    lines = sharedmap.make_lines(2, 120, dmap=sharedmap.DistanceMap(dist=world["dist_a"]))
    img_b, rows_n, cols_n = world["img_b"], *world["img_b"].shape
    for b in range(2):
        rows = lines.spline_rows(b)
        p = str(tmp_path / ("mu%d.txt" % b))
        with open(p, "w") as f:
            f.write("%d %d %.17g %d\n" % (rows_n, cols_n, RES, 127))
            np.savetxt(f, world["dist_a"].reshape(1, -1), fmt="%.9g")
            np.savetxt(f, img_b.reshape(1, -1), fmt="%d")
            np.savetxt(f, world["dist_b"].reshape(1, -1), fmt="%.9g")
            f.write("%d\n" % rows.shape[1])
            np.savetxt(f, rows, fmt="%.17g")
            f.write("%.17g\n" % float(rows[0, -1]))
        out = subprocess.run([exe, p], capture_output=True, text=True, check=True).stdout.strip().split("\n")
        assert out[0] == "refused 1"
        head = out[1].split()
        assert head[:2] == ["run", "1"] and int(head[2]) > 0
        n = int(head[2])
        updated, fresh_head, fresh = out[2:2 + n], out[2 + n], out[3 + n:]
        assert fresh_head == out[1] and updated == fresh
