"""Per-path maps: map slots on one handle (pqp_bounds_create_maps, pqp_plan_create_maps), the batched exact distance
transform (set_occupancy_slots*) and the mapped bounds, DP and plan calls.

CPU: the C layout of pqp_occupancy_stack; the slot lookup of pqp_bounds_core.cuh under g++.
GPU: the batched transform against the oracle and a lone set_occupancy, refusals; a mapped plan over six distinct
maps against single-map planners row by row (both smoothing methods, samples and points, host and device); an
all-zero index against the unmapped call; out-of-range indices in the plan, bounds and DP calls; the standalone
bounds and DP mapped calls; stream order; launch counts.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import edt_oracle as eo
from path_optimizer_2_b200 import abi, bounds, dp, plan, sharedmap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PNG = os.path.join(ROOT, "tests", "golden", "gridmap.png")
RES = sharedmap.RES
INT32_MAX = 2 ** 31 - 1


def _png():
    from PIL import Image
    return np.asarray(Image.open(PNG).convert("L")).astype(np.uint8)


# ------------------------------------------------------------------------------------------------- CPU
_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "pqp_bounds.h"
#define F(m) printf("%s %zu\n", #m, offsetof(pqp_occupancy_stack, m))
int main(void) {
    printf("size %zu\n", sizeof(pqp_occupancy_stack));
    F(count); F(rows); F(cols); F(resolution); F(center_x); F(center_y); F(cells); F(obstacle_max);
    return 0;
}
"""

_SLOT_CPP = r"""
#include <stdint.h>
#include <stdio.h>
#include "pqp_bounds_core.cuh"
int main() {
    pqb::MapView table[3] = {};
    const int32_t index[] = {0, 1, 2, -1, 3, 2147483647, -2147483647 - 1};
    for (int b = 0; b < 7; ++b) {
        const pqb::MapView *m = pqb::slot_view(table, 3, index, b);
        printf("%d\n", m ? (int)(m - table) : -1);
    }
    return 0;
}
"""


def _compile_run(src, name, compiler, std):
    with tempfile.TemporaryDirectory() as d:
        path, exe = os.path.join(d, name), os.path.join(d, "a.out")
        with open(path, "w") as f:
            f.write(src)
        subprocess.check_call([compiler, std, "-I", os.path.join(ROOT, "include"), "-I",
                               os.path.join(ROOT, "path_optimizer_2_b200", "csrc"), "-o", exe, path])
        return subprocess.check_output([exe], text=True)


def test_occupancy_stack_layout_matches_ctypes():
    out = _compile_run(_LAYOUT_C, "layout.c", "gcc", "-std=c99")
    got = {k: int(v) for k, v in (line.split() for line in out.splitlines())}
    S = bounds.OccupancyStack
    assert got == {"size": ctypes.sizeof(S), **{n: getattr(S, n).offset for n, _ in S._fields_}}


def test_slot_lookup_on_cpu():
    out = _compile_run(_SLOT_CPP, "slot.cpp", "g++", "-std=c++11")
    assert [int(v) for v in out.split()] == [0, 1, 2, -1, -1, -1, -1]


# ------------------------------------------------------------------------------------------------- GPU
from tests.test_plan_points import L_MAX, N_MAX, P_MAX, R_MAX  # noqa: E402

PER_MAP = 32
METHODS = ("TENSION2", "TENSION")
# trace fields every row has, whatever stage it failed at
ALWAYS = ("seg_p", "raw_r", "bspline_degree")
# The extent of a trace field a path that reached the end has written (entries past it keep whatever the handle's
# buffer held): per field, a function of the row's trace giving the slice; fields not listed are compared whole.
_P = lambda t, i: np.s_[:int(t["seg_p"][i])]  # noqa: E731
_L = lambda t, i: np.s_[:int(t["dp_n_out"][i])]  # noqa: E731
_N = lambda t, i: np.s_[..., :int(t["n_valid"][i])]  # noqa: E731
_S = lambda t, i: np.s_[..., :int(min(t["total"][i], N_MAX))]  # noqa: E731
EXTENT = {"seg_x": _P, "seg_y": _P, "seg_angle": _P, "seg_k": _P, "seg_s": _P, "tension_x": _P, "tension_y": _P,
          "tension_s": _P, "tension_clearance": _P, "dp_layer_s": _L, "dp_lower": _L, "dp_upper": _L, "dp_chosen": _L,
          "post_offsets": _L, "states": _S, "curvature": _S, "bounds": _N, "sol1": _N}
# the solvers' full iterates: their layout depends on n, their padding on the handle's history
SKIP = ("x_full1", "y_full1", "z_full1", "x_full2", "y_full2", "z_full2")


def _cell(x, y, rows, cols, res):
    return int((rows * res / 2 - x) / res), int((cols * res / 2 - y) / res)


def _shift(inputs, c):
    xs, ys, start, target = inputs
    start, target = start.copy(), target.copy()
    start[:, 0] += c[0]
    start[:, 1] += c[1]
    target[:, 0] += c[0]
    target[:, 1] += c[1]
    return [x + c[0] for x in xs], [y + c[1] for y in ys], start, target


@pytest.fixture(scope="module")
def maps():
    """Six maps (image, resolution, centre, layer) and the plan inputs of PER_MAP paths generated on each: the demo
    map; the demo map with 1.8 m blocks on some of its paths; the demo map flipped; a crop with a moved centre and
    another resolution; a random map; an almost empty map."""
    img = _png()
    rows, cols = img.shape
    rng = np.random.default_rng(21)
    imgs = [img, img.copy(), np.ascontiguousarray(img[::-1]), np.ascontiguousarray(img[100:600, 150:700]),
            np.where(rng.random((rows, cols)) < 0.0005, 0, 255).astype(np.uint8), np.full((rows, cols), 255, np.uint8)]
    imgs[5][0, 0] = imgs[5][-1, -1] = 0
    res = [RES, RES, RES, 0.25, RES, RES]
    centers = [(0.0, 0.0)] * 3 + [(3.0, -2.0)] + [(0.0, 0.0)] * 2
    out = []
    for k in range(6):
        dist = eo.transform(imgs[k], res[k], 127)[1]
        dmap = sharedmap.DistanceMap(dist=dist, res=res[k])
        raw = sharedmap.make_plan_inputs(PER_MAP, first=100 * k, dmap=dmap)
        pts = sharedmap.make_plan_points(PER_MAP, first=100 * k, dmap=dmap)
        if k == 1:  # blocks on every third path of this map, in its own image
            for b in range(0, PER_MAP, 3):
                m = len(pts[0][b]) // 2
                i, j = _cell(pts[0][b][m], pts[1][b][m], rows, cols, RES)
                imgs[1][max(i - 4, 0):i + 5, max(j - 4, 0):j + 5] = 0
            dist = eo.transform(imgs[1], RES, 127)[1]
        out.append(dict(img=imgs[k], res=res[k], center=centers[k], dist=dist, raw=_shift(raw, centers[k]),
                        pts=_shift(pts, centers[k])))
    return out


def _interleave(maps, key):
    """The paths of every map in one batch, in shuffled order: (inputs, map_index, (map, path) of each row)."""
    order = [(k, j) for k in range(len(maps)) for j in range(PER_MAP)]
    perm = np.random.default_rng(4).permutation(len(order))
    order = [order[p] for p in perm]
    xs = [maps[k][key][0][j] for k, j in order]
    ys = [maps[k][key][1][j] for k, j in order]
    start = np.stack([maps[k][key][2][j] for k, j in order])
    target = np.stack([maps[k][key][3][j] for k, j in order])
    return (xs, ys, start, target), np.array([k for k, _ in order], np.int32), order


def _device_args(inputs, points):
    import torch
    xs, ys, start, target = inputs
    cnt = np.array([len(v) for v in xs], dtype=np.int32)
    M = R_MAX if not points else int(cnt.max())
    px, py = np.zeros((len(xs), M)), np.zeros((len(xs), M))
    for b in range(len(xs)):
        px[b, :cnt[b]], py[b, :cnt[b]] = xs[b], ys[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    return [t(px), t(py), t(cnt), t(start), t(target)]


def _mapped_planner(maps, method, batch_max):
    return plan.Planner.from_maps([m["dist"] for m in maps], [m["res"] for m in maps],
                                  centers=[m["center"] for m in maps], r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX,
                                  n_max=N_MAX, batch_max=batch_max, params=plan.default_params(method))


def _single_planner(m, method, batch_max=PER_MAP):
    return plan.Planner(m["dist"], m["res"], center=m["center"], r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX,
                        n_max=N_MAX, batch_max=batch_max, params=plan.default_params(method))


def _as_np(out):
    if isinstance(out, dict):
        r = plan.PlanResult(len(out["status"]), N_MAX)
        for k in ("status", "n", "path", "cost", "iters"):
            setattr(r, k, out[k].cpu().numpy())
        if "trace" in out:
            r.trace = {k: v.cpu().numpy() for k, v in out["trace"].items()}
        return r
    return out


def _assert_row(a, b, i, j, tag):
    """Row i of `a` equals row j of `b` in every output and, for a path that reached the end (status OK), every
    trace field; a failed path's later stages are unspecified, so there only the fields every row has."""
    for k in ("status", "n", "path", "cost", "iters"):
        assert np.array_equal(getattr(a, k)[i], getattr(b, k)[j]), (tag, k)
    if a.trace is None:
        return
    fields = [k for k in a.trace if k not in SKIP] if a.status[i] == plan.OK else ALWAYS
    for k in fields:
        ea = EXTENT[k](a.trace, i) if k in EXTENT else np.s_[...]
        eb = EXTENT[k](b.trace, j) if k in EXTENT else np.s_[...]
        assert np.array_equal(a.trace[k][i][ea], b.trace[k][j][eb], equal_nan=True), (tag, k)


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_gpu_mapped_plan_equals_single_map_plans(maps, method):
    import torch
    B = PER_MAP * len(maps)
    for points in (False, True):
        pl = _mapped_planner(maps, method, B)  # fresh, like the single-map planners: same buffer history per row
        assert pl.n_maps == len(maps)
        key = "pts" if points else "raw"
        inputs, idx, order = _interleave(maps, key)
        host_fn = pl.plan_points if points else pl.plan
        host = host_fn(*inputs, trace=True, map_index=idx)
        dev_fn = pl.plan_points_device if points else pl.plan_device
        dev = _as_np(dev_fn(*_device_args(inputs, points), trace=True,
                            map_index=torch.from_numpy(idx).cuda()))
        torch.cuda.synchronize()
        singles = []
        for k, m in enumerate(maps):
            one = _single_planner(m, method)
            fn = one.plan_points if points else one.plan
            singles.append(fn(*m[key], trace=True))
            one.close()
        for b, (k, j) in enumerate(order):
            _assert_row(host, singles[k], b, j, (method, points, "host", b, k))
            _assert_row(dev, singles[k], b, j, (method, points, "device", b, k))
        assert np.mean(host.status == plan.OK) > 0.6, host.status_names()
        pl.close()


@pytest.mark.gpu
def test_gpu_zero_index_equals_unmapped_call(maps):
    m0 = maps[0]
    pl = _mapped_planner(maps, "TENSION2", PER_MAP)
    for points in (False, True):
        key = "pts" if points else "raw"
        fn = pl.plan_points if points else pl.plan
        a = fn(*m0[key], trace=True)
        b = fn(*m0[key], trace=True, map_index=np.zeros(PER_MAP, np.int32))
        for k in ("status", "n", "path", "cost", "iters"):
            assert np.array_equal(getattr(a, k), getattr(b, k)), (points, k)
        for k in a.trace:
            assert np.array_equal(a.trace[k], b.trace[k], equal_nan=True), (points, k)
    pl.close()


@pytest.mark.gpu
def test_gpu_out_of_range_indices(maps):
    m0 = maps[0]
    n_maps = len(maps)
    pl = _mapped_planner(maps, "TENSION", PER_MAP)
    bad = {3: -1, 10: n_maps, 20: INT32_MAX}
    idx = np.zeros(PER_MAP, np.int32)
    for b, v in bad.items():
        idx[b] = v
    for points in (False, True):
        key = "pts" if points else "raw"
        fn = pl.plan_points if points else pl.plan
        good = fn(*m0[key])
        res = fn(*m0[key], map_index=idx)
        for b in range(PER_MAP):
            if b in bad:
                assert res.status[b] == plan.MAP_INDEX and res.n[b] == 0 and not res.path[b].any(), b
                assert res.cost[b] == 0.0
            else:
                for k in ("status", "n", "path", "cost", "iters"):
                    assert np.array_equal(getattr(res, k)[b], getattr(good, k)[b]), (points, b, k)
    pl.close()
    # the standalone mapped calls
    lines = sharedmap.make_lines(PER_MAP, 120, dmap=sharedmap.DistanceMap(dist=m0["dist"]))
    pbn = bounds.PathBounds.from_maps([m["dist"] for m in maps], [m["res"] for m in maps],
                                      centers=[m["center"] for m in maps])
    ds = dp.DpSearch(pbn, layers_max=160, batch_max=PER_MAP)
    bnd, nv = pbn.compute(lines.states, lines.n, lines.spline, lines.k)
    mbnd, mnv = pbn.compute(lines.states, lines.n, lines.spline, lines.k, map_index=idx)
    length = np.array([lines.spline_rows(b)[0, lines.k[b] - 1] + 3.0 for b in range(PER_MAP)])
    start = np.stack([lines.states[:, 1, 2], lines.states[:, 2, 2], lines.states[:, 3, 2]], axis=1)
    r = ds.search(lines.spline, lines.k, length, start)
    mr = ds.search(lines.spline, lines.k, length, start, map_index=idx)
    for b in range(PER_MAP):
        if b in bad:
            assert mnv[b] == 0 and mr.status[b] == dp.DP_MAP_INDEX and mr.n_layers[b] == 0 and mr.n_out[b] == 0, b
        else:
            assert mnv[b] == nv[b] and np.array_equal(mbnd[b, :, :nv[b]], bnd[b, :, :nv[b]]), b
            for k in ("status", "n_layers", "n_out", "layer_s", "lower", "upper", "chosen", "vehicle_l", "target_s",
                      "cost", "parent", "feasible"):
                assert np.array_equal(getattr(mr, k)[b], getattr(r, k)[b]), (b, k)
    ds.close()
    pbn.close()


@pytest.mark.gpu
def test_gpu_standalone_mapped_bounds_and_dp(maps):
    from oracle import bounds_oracle, dp_oracle
    from tests.test_dp import _compare
    n_maps = len(maps)
    pbn = bounds.PathBounds.from_maps([m["dist"] for m in maps], [m["res"] for m in maps],
                                      centers=[m["center"] for m in maps])
    ds = dp.DpSearch(pbn, layers_max=160, batch_max=n_maps * 4)
    per = [sharedmap.make_lines(4, 120, first=100 * k, dmap=sharedmap.DistanceMap(dist=m["dist"], res=m["res"]))
           for k, m in enumerate(maps) if m["center"] == (0.0, 0.0)]
    ks = [k for k, m in enumerate(maps) if m["center"] == (0.0, 0.0)]
    states = np.concatenate([ln.states for ln in per])
    n = np.concatenate([ln.n for ln in per])
    spline = np.concatenate([ln.spline for ln in per])
    k_ = np.concatenate([ln.k for ln in per])
    idx = np.repeat(np.array(ks, np.int32), 4)
    bnd, nv = pbn.compute(states, n, spline, k_, map_index=idx)
    length = np.array([spline[b, 0, k_[b] - 1] + 3.0 for b in range(len(idx))])
    start = np.stack([states[:, 1, 2], states[:, 2, 2], states[:, 3, 2]], axis=1)
    r = ds.search(spline, k_, length, start, map_index=idx)
    for slot in range(n_maps):
        m = maps[slot]
        rows = np.nonzero(idx == slot)[0]
        if not len(rows):
            continue
        one = bounds.PathBounds(m["dist"], m["res"], center=m["center"])
        one_ds = dp.DpSearch(one, layers_max=160, batch_max=len(rows))
        ob, onv = one.compute(states[rows], n[rows], spline[rows], k_[rows])
        orr = one_ds.search(spline[rows], k_[rows], length[rows], start[rows])
        for i, b in enumerate(rows):
            assert onv[i] == nv[b] and np.array_equal(ob[i], bnd[b]), (slot, b)
            nl = int(r.n_layers[b])
            for f in ("status", "n_layers", "n_out"):
                assert getattr(orr, f)[i] == getattr(r, f)[b], (slot, b, f)
            for f in ("layer_s", "lower", "upper", "chosen", "cost", "parent", "feasible"):
                assert np.array_equal(getattr(orr, f)[i][:nl], getattr(r, f)[b][:nl]), (slot, b, f)
            # against the oracles, to the tolerances of their own tests
            sr = spline[b, :, :k_[b]]
            ob2, onv2 = bounds_oracle.update_bounds(m["dist"], m["res"], sr, *states[b])
            d = np.abs(ob2 - bnd[b])
            assert onv2 == nv[b] and (d > 1e-9).mean() < 5e-3 and d.max() < 0.31, (slot, b)
            _compare(r, b, dp_oracle.graph_search_dp(m["dist"], m["res"], sr, length[b], start[b]), 34)
        one_ds.close()
        one.close()
    ds.close()
    pbn.close()


@pytest.mark.gpu
def test_gpu_batched_transform(maps):
    import torch
    rows, cols = maps[0]["img"].shape
    n_maps = 8
    sentinel = [np.full((rows, cols), float(s + 1), np.float32) for s in range(n_maps)]
    pbn = bounds.PathBounds.from_maps(sentinel, 1.0)
    lone = bounds.PathBounds(np.zeros((rows, cols), np.float32), RES)
    rng = np.random.default_rng(8)
    stack = np.stack([maps[0]["img"], maps[1]["img"], maps[2]["img"], maps[4]["img"],
                      np.where(rng.random((rows, cols)) < 0.02, 0, 255).astype(np.uint8)])
    centers = [(0.5 * i, -1.0 * i) for i in range(len(stack))]
    # host call into slots 2 .. 6 of 8: every slot the oracle's layer and a lone set_occupancy's, the rest untouched
    pbn.set_occupancy_slots(stack, 0.15, centers, obstacle_max=127, first_slot=2)
    for s in range(n_maps):
        got, res, c = pbn.get_map(s)
        if 2 <= s < 7:
            i = s - 2
            want = eo.transform(stack[i], 0.15, 127)[1]
            assert np.array_equal(got, want) and res == 0.15 and c == centers[i], s
            lone.set_occupancy(stack[i], 0.15, centers[i], obstacle_max=127)
            assert np.array_equal(lone.get_map()[0], got), s
        else:
            assert np.array_equal(got, sentinel[s]) and res == 1.0 and c == (0.0, 0.0), s
    # the device call, small and special images of one size, into slots 0 .. count - 1
    from tests.test_map_update import _special_cases
    special = [img for img, om in _special_cases() if img.shape == (37, 23)]
    sstack = np.stack(special)
    pbn.set_occupancy_slots_device(torch.from_numpy(sstack).cuda(), 0.1, obstacle_max=0,
                                   stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for i, img in enumerate(special):
        got, res, c = pbn.get_map(i)
        assert np.array_equal(got, eo.transform(img, 0.1, 0)[1]) and res == 0.1 and c == (0.0, 0.0), i
    # refusals leave every slot as it was
    before = [pbn.get_map(s) for s in range(n_maps)]
    L = pbn.L
    img = np.ascontiguousarray(stack[:2])
    cx, cy = np.zeros(2), np.zeros(2)
    nan = np.array([0.0, float("nan")])

    def st(count=2, r=rows, c=cols, res=RES, x=cx, y=cy, cells=img.ctypes.data):
        return bounds.OccupancyStack(count, r, c, res, x.ctypes.data if x is not None else None,
                                     y.ctypes.data if y is not None else None, cells, 0)
    big = 16385
    refused = [(0, st(r=1)), (0, st(c=1)), (0, st(r=rows + 1)), (0, st(count=1, r=big, c=2)),
               (0, st(count=1, r=2, c=big)), (-1, st()), (7, st()), (n_maps, st(count=1)), (0, st(count=0)),
               (0, st(res=float("nan"))), (0, st(res=0.0)), (0, st(x=nan)), (0, st(y=nan)), (0, st(x=None)),
               (0, st(cells=None))]
    small = bounds.PathBounds.from_maps([np.zeros((big, 2), np.float32), np.zeros((2, big), np.float32)], 1.0)
    for first, s_ in refused:
        assert L.pqp_bounds_set_occupancy_slots(pbn.h, first, ctypes.byref(s_)) == abi.PQP_E_INVALID, first
        assert L.pqp_bounds_set_occupancy_slots_device(pbn.h, first, ctypes.byref(s_), None) == abi.PQP_E_INVALID
        assert L.pqp_bounds_last_error(pbn.h)
    for s_ in (st(count=1, r=big, c=2), st(count=1, r=2, c=big)):  # over 16384 on a handle whose slots hold them
        assert L.pqp_bounds_set_occupancy_slots(small.h, 0, ctypes.byref(s_)) == abi.PQP_E_INVALID
    assert L.pqp_bounds_set_occupancy_slots(pbn.h, 0, None) == abi.PQP_E_INVALID
    for s in range(n_maps):
        got = pbn.get_map(s)
        assert np.array_equal(got[0], before[s][0]) and got[1:] == before[s][1:], s
    small.close()
    lone.close()
    pbn.close()


@pytest.mark.gpu
def test_gpu_stream_order_and_launch_counts(maps):
    import torch
    for method, base in (("TENSION2", 25), ("TENSION", 26)):
        pl = _mapped_planner(maps[:3], method, 2 * PER_MAP)
        inputs = (maps[0]["pts"][0] + maps[2]["pts"][0], maps[0]["pts"][1] + maps[2]["pts"][1],
                  np.concatenate([maps[0]["pts"][2], maps[2]["pts"][2]]),
                  np.concatenate([maps[0]["pts"][3], maps[2]["pts"][3]]))
        idx = np.repeat(np.array([0, 2], np.int32), PER_MAP)
        args = _device_args(inputs, True)
        tidx = torch.from_numpy(idx).cuda()
        # the update swaps the images of slots 0 and 2: demo <-> flipped demo
        new = torch.from_numpy(np.stack([maps[2]["img"], maps[1]["img"], maps[0]["img"]])).cuda()
        s = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            c0 = pl.launch_count
            first = pl.plan_points_device(*args, map_index=tidx)
            c1 = pl.launch_count
            pl.set_occupancy_slots_device(new, RES, obstacle_max=127)
            c2 = pl.launch_count
            second = pl.plan_points_device(*args, map_index=tidx)
            c3 = pl.launch_count
        s.synchronize()
        assert (c1 - c0, c2 - c1, c3 - c2) == (base, plan.occupancy_slots_launches(3), base)
        assert plan.occupancy_slots_launches(3) == plan.occupancy_slots_launches(bounds.MAP_TABLE_CHUNK) == 3
        before = pl.plan_points(*inputs, map_index=idx)  # now on the swapped maps
        single = {k: _single_planner(maps[k], method) for k in (0, 2)}
        want_first = [single[k].plan_points(*maps[k]["pts"]) for k in (0, 2)]
        for o, w in ((first, want_first),):
            st_ = o["status"].cpu().numpy()
            assert np.array_equal(st_[:PER_MAP], w[0].status) and np.array_equal(st_[PER_MAP:], w[1].status)
            p = o["path"].cpu().numpy()
            assert np.array_equal(p[:PER_MAP], w[0].path) and np.array_equal(p[PER_MAP:], w[1].path)
        # after the update the paths of slot 0 run on the flipped map, those of slot 2 on the demo map
        swapped = [plan.Planner(maps[2]["dist"], RES, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX,
                                batch_max=PER_MAP, params=plan.default_params(method)).plan_points(*maps[0]["pts"]),
                   single[0].plan_points(*maps[2]["pts"])]
        sp = second["path"].cpu().numpy()
        ss = second["status"].cpu().numpy()
        assert np.array_equal(ss[:PER_MAP], swapped[0].status) and np.array_equal(ss[PER_MAP:], swapped[1].status)
        assert np.array_equal(sp[:PER_MAP], swapped[0].path) and np.array_equal(sp[PER_MAP:], swapped[1].path)
        assert np.array_equal(before.path, sp)
        assert not np.array_equal(sp, first["path"].cpu().numpy())
        # slot updates and the unmapped calls: documented counts
        c4 = pl.launch_count
        pl.set_map(maps[0]["dist"], RES, slot=1)
        c5 = pl.launch_count
        pl.set_occupancy(maps[0]["img"], RES, obstacle_max=127)
        c6 = pl.launch_count
        pl.plan_points(*maps[0]["pts"], map_index=np.zeros(PER_MAP, np.int32))
        c7 = pl.launch_count
        pl.plan(*maps[0]["raw"], map_index=np.zeros(PER_MAP, np.int32))
        c8 = pl.launch_count
        assert (c5 - c4, c6 - c5, c7 - c6, c8 - c7) == (plan.SET_MAP_LAUNCHES, plan.OCCUPANCY_LAUNCHES, base,
                                                        base - 2)
        for one in single.values():
            one.close()
        pl.close()
