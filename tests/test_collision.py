"""Footprint collision check (pqp_bounds_collision_check*, pqp_plan_collision_check*; include/pqp_bounds.h): the
reference's CollisionChecker::isSingleStateCollisionFreeImproved over a batch of poses, path b on map slot
map_index[b].

CPU: the oracle's circle table against closed form; wall sweeps on a layer linear in y; the bounding-circle shortcut;
the kernel's per-state source (pqp_collision_core.cuh under g++) against the oracle; the C layout of the structs; the
kernel's register report.
GPU: 1024 final paths of plans from reference points (both smoothing methods, host and device forms) against the
oracle; reference states passed as states + n_max; mapped calls against single-map handles; stream order after
set_occupancy_device; n clamping and refusals; launch counts.
"""
import ctypes
import math
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import collision_oracle as co
from path_optimizer_2_b200 import abi, bounds, plan, sharedmap, solver
from tests.emu import collision_emu as ce

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PNG = os.path.join(ROOT, "tests", "golden", "gridmap.png")
SMALL, LARGE, BOUND = math.sqrt(0.5), math.sqrt(6.1025) / 2, math.sqrt(7.0025)


# ------------------------------------------------------------------------------------------------- CPU
def test_circle_table_at_default_flags():
    want_b = (1.45, 0.0, BOUND)
    want = [(-0.5, -0.5, SMALL), (-0.5, 0.5, SMALL), (3.4, -0.5, SMALL), (3.4, 0.5, SMALL), (1.45 + 0.725, 0.0, LARGE),
            (1.45 - 0.725, 0.0, LARGE)]
    b, circles = co.car_geometry()
    assert b == pytest.approx(want_b, abs=1e-15)
    for got, w in zip(circles, want):
        assert got == pytest.approx(w, abs=1e-15)
    fp = ce.footprint()  # what the kernel receives, computed by the library's host code
    assert np.array_equal(fp, np.array([[c[k] for c in [b] + circles] for k in range(3)]))


def _wall_layer(w, rows=400, cols=400, res=0.1):
    """A layer whose value is w - y at every cell centre: a wall at y = w on the +y side, exact under bilinear
    interpolation (up to float32 rounding)."""
    y = cols * res / 2 - (np.arange(cols) + 0.5) * res
    return np.ascontiguousarray(np.broadcast_to((w - y)[None, :], (rows, cols)), dtype=np.float32), res


def _flip(heading, walls, free_fn):
    verdict = np.array([bool(free_fn(*_wall_layer(w), 0.0, 0.0, heading)) for w in walls])
    assert not verdict[0] and verdict[-1]
    k = int(np.argmax(verdict))
    assert verdict[k:].all()
    return walls[k]


@pytest.mark.parametrize("how", ("oracle", "kernel source"))
def test_wall_sweep(how):
    def improved(dist, res, x, y, h):
        if how == "oracle":
            return co.state_free_improved(dist, res, x, y, h)[0]
        return ce.check(dist, res, np.array([[[x], [y], [h]]]), [1])[1][0, 0]

    step = 1e-3
    walls = np.arange(0.9, 1.6, step)
    # heading 0: fm / rm need the wall sqrt(6.1025) / 2 away (rl / fl only 0.5 + sqrt(0.5) ~ 1.2071)
    assert abs(_flip(0.0, walls, improved) - LARGE) <= step
    # heading pi/2: the exact test flips where fr / fl touch (3.4 + sqrt(0.5) ~ 4.1071; fm needs 3.4102) ...
    walls = np.arange(3.8, 4.4, step)
    exact = lambda d, r, x, y, h: co.state_free_exact(d, r, x, y, h)  # noqa: E731
    assert abs(_flip(math.pi / 2, walls, exact) - (3.4 + SMALL)) <= step
    # ... but the bounding circle (centre 1.45 ahead, radius sqrt(7.0025)) clears the wall first, at 4.0962: the
    # reference's shortcut passes the front corner circles' last 11 mm
    assert abs(_flip(math.pi / 2, walls, improved) - (1.45 + BOUND)) <= step


def test_bounding_circle_shortcut():
    res, rows, cols = 0.1, 200, 200
    dist = np.full((rows, cols), 50.0, np.float32)
    # one low 2 x 2 block of cells around the fr centre (3.4, -0.5) of the pose (0, 0, 0)
    i = int((rows * res / 2 - 3.4) / res)
    j = int((cols * res / 2 + 0.5) / res)
    dist[i - 1:i + 2, j - 1:j + 2] = 0.0
    free, clear = co.state_free_improved(dist, res, 0.0, 0.0, 0.0)
    assert free and clear < 0
    assert not co.state_free_exact(dist, res, 0.0, 0.0, 0.0)
    hit, sf, c = ce.check(dist, res, np.zeros((1, 3, 1)), [1])
    assert hit[0] == 1 and sf[0, 0] == 1 and c[0, 0] == pytest.approx(float(clear), abs=1e-12) and c[0, 0] < 0


def test_kernel_source_matches_oracle_on_gridmap():
    d = sharedmap.DistanceMap()
    rng = np.random.default_rng(5)
    B, N = 96, 160
    hx, hy = d.dist.shape[0] * d.res / 2, d.dist.shape[1] * d.res / 2
    poses = np.stack([rng.uniform(-1.1 * hx, 1.1 * hx, (B, N)), rng.uniform(-1.1 * hy, 1.1 * hy, (B, N)),
                      rng.uniform(-4.0, 4.0, (B, N))], axis=1)
    poses[:, 2, ::13] = np.nan
    poses[::7, 0, 5] = np.nan
    n = rng.integers(-3, N + 5, B)
    for center in ((0.0, 0.0), (3.0, -2.5)):
        h1, f1, c1 = ce.check(d.dist, d.res, poses, n, center=center)
        h2, f2, c2 = co.check(d.dist, d.res, poses, n, center=center)
        assert np.array_equal(h1, h2) and np.array_equal(f1, f2)
        assert np.allclose(c1, c2, rtol=0, atol=1e-12, equal_nan=True)
        assert 0.05 < f1.mean() < 0.95


_LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "pqp_bounds.h"
#define F(T, m) printf("%s.%s %zu\n", #T, #m, offsetof(T, m))
int main(void) {
    printf("in %zu\nout %zu\n", sizeof(pqp_collision_in), sizeof(pqp_collision_out));
    F(pqp_collision_in, batch); F(pqp_collision_in, n_max); F(pqp_collision_in, row_stride);
    F(pqp_collision_in, poses); F(pqp_collision_in, n);
    F(pqp_collision_out, first_hit); F(pqp_collision_out, state_free); F(pqp_collision_out, clearance);
    return 0;
}
"""


def test_collision_structs_layout_matches_ctypes():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "a.out")
        with open(src, "w") as f:
            f.write(_LAYOUT_C)
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = dict(line.split() for line in subprocess.check_output([exe], text=True).splitlines())
    want = {"in": ctypes.sizeof(bounds.CollisionIn), "out": ctypes.sizeof(bounds.CollisionOut)}
    for T, name in ((bounds.CollisionIn, "pqp_collision_in"), (bounds.CollisionOut, "pqp_collision_out")):
        want.update({"%s.%s" % (name, f): getattr(T, f).offset for f, _ in T._fields_})
    assert {k: int(v) for k, v in got.items()} == want


def test_collision_kernel_does_not_spill():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                            "607,177", "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-c",
                            os.path.join(ROOT, "path_optimizer_2_b200", "csrc", "pqp_bounds.cu"), "-o",
                            os.path.join(d, "b.o")], capture_output=True, text=True, check=True)
    lines = r.stderr.splitlines()
    k = next(i for i, ln in enumerate(lines) if "Function properties for" in ln and "collision_check_kernel" in ln)
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", lines[k + 1])
    assert m and m.groups() == ("0", "0"), lines[k:k + 3]


# ------------------------------------------------------------------------------------------------- GPU
R, P, L, N = 64, 64, 64, 255


def _png():
    from PIL import Image
    return np.asarray(Image.open(PNG).convert("L")).astype(np.uint8)


def _points_device(B, dmap):
    import torch
    ref_x, ref_y, start, target = sharedmap.make_plan_points(B, dmap=dmap)
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    return (ref_x, ref_y, start, target), [t(px), t(py), t(m), t(start), t(target)]


def _compare_to_oracle(dist, res, path, n, got, tag, center=(0.0, 0.0)):
    """got (first_hit, state_free, clearance) against the oracle; a state whose oracle margin (any circle's d - r,
    the bounding circle's included) is within 1e-9 m of 0 may take either verdict. Returns how many such states."""
    hit, free, clear = got
    oh, of, oc = co.check(dist, res, path, n, center=center)
    n_c = np.clip(n, 0, path.shape[2])
    valid = np.arange(path.shape[2])[None, :] < n_c[:, None]
    mg = co.margins(dist, res, path[:, 0], path[:, 1], path[:, 2], center=center)
    near = valid & np.any(np.abs(mg) < 1e-9, axis=0)
    assert np.array_equal(free[~near], of[~near]), tag
    assert np.allclose(clear, oc, rtol=0, atol=1e-9, equal_nan=True), (tag, np.nanmax(np.abs(clear - oc)))
    for b in np.nonzero(hit != oh)[0]:
        assert near[b, :max(hit[b], oh[b]) + 1].any(), (tag, b, hit[b], oh[b])
    return int(near.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("method", ("TENSION2", "TENSION"))
def test_gpu_plan_output_against_oracle(method):
    import torch
    dmap = sharedmap.DistanceMap()
    B = 1024
    pl = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=B,
                      params=plan.default_params(method))
    host_in, d_in = _points_device(B, dmap)
    out = pl.plan_points_device(*d_in)
    dev = pl.check_collision_device(out["path"], out["n"], clearance=True, per_state=True,
                                    stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    path, n, status = out["path"].cpu().numpy(), out["n"].cpu().numpy(), out["status"].cpu().numpy()
    got_dev = tuple(dev[k].cpu().numpy() for k in ("first_hit", "state_free", "clearance"))
    host = pl.check_collision(path, n, clearance=True, per_state=True)
    got_host = tuple(host[k] for k in ("first_hit", "state_free", "clearance"))
    for k in range(3):
        assert np.array_equal(got_host[k], got_dev[k]), k
    near = _compare_to_oracle(dmap.dist, dmap.res, path, n, got_dev, method)
    ok = status == plan.OK
    flagged = int(np.sum(ok & (got_dev[0] < n)))
    print("%s: %d PLAN_OK paths, %d flagged by the check, %d states within 1e-9 m of a circle's radius"
          % (method, ok.sum(), flagged, near))
    assert ok.mean() > 0.5 and np.all(got_dev[0][n == 0] == 0)
    # the host plan output checked through the host form of the same handle
    pr = pl.plan_points(*host_in)
    assert np.array_equal(pr.path, path)
    pl.close()


@pytest.mark.gpu
def test_gpu_reference_states_layout():
    import torch
    dmap = sharedmap.DistanceMap()
    rng = np.random.default_rng(2)
    B, n_max = 33, 200
    lines = sharedmap.make_lines(B, n_max, dmap=dmap)
    states = np.ascontiguousarray(lines.states)  # [B][4][n_max]: s, x, y, heading
    states[:, 3] += rng.normal(0, 0.3, (B, n_max))
    n = lines.n
    pbn = bounds.PathBounds(dmap.dist, dmap.res)
    packed = np.ascontiguousarray(states[:, 1:])
    want = pbn.check_collision(packed, n, clearance=True, per_state=True)
    view = states[:, 1:]  # states + n_max with row_stride 4
    got = pbn.check_collision(view, n, row_stride=4, clearance=True, per_state=True)
    ts = torch.from_numpy(states).cuda()
    tn = torch.from_numpy(np.ascontiguousarray(n, dtype=np.int32)).cuda()
    dv = pbn.check_collision_device(ts[:, 1:], tn, clearance=True, per_state=True)
    torch.cuda.synchronize()
    for k in want:
        assert np.array_equal(want[k], got[k]) and np.array_equal(want[k], dv[k].cpu().numpy()), k
    _compare_to_oracle(dmap.dist, dmap.res, packed, n, tuple(want[k] for k in ("first_hit", "state_free", "clearance")),
                       "states")
    assert want["state_free"].any() and (want["first_hit"] < n).any()
    pbn.close()


def _six_maps():
    """(layers, resolutions, centres): the demo map, flipped, with random blocks, a crop with another resolution and
    centre, random obstacles, almost empty."""
    from oracle import edt_oracle as eo
    img = _png()
    rows, cols = img.shape
    rng = np.random.default_rng(9)
    blocked = img.copy()
    for i, j in zip(rng.integers(0, rows - 9, 40), rng.integers(0, cols - 9, 40)):
        blocked[i:i + 9, j:j + 9] = 0
    empty = np.full((rows, cols), 255, np.uint8)
    empty[0, 0] = 0
    imgs = [img, np.ascontiguousarray(img[::-1]), blocked, np.ascontiguousarray(img[100:600, 150:700]),
            np.where(rng.random((rows, cols)) < 0.002, 0, 255).astype(np.uint8), empty]
    res = [0.2, 0.2, 0.2, 0.25, 0.2, 0.2]
    centers = [(0.0, 0.0), (0.0, 0.0), (0.0, 0.0), (3.0, -2.0), (0.0, 0.0), (0.0, 0.0)]
    return [eo.transform(im, r, 127)[1] for im, r in zip(imgs, res)], res, centers


def _random_poses(B, n_max, seed, half=70.0):
    rng = np.random.default_rng(seed)
    poses = np.stack([rng.uniform(-half, half, (B, 1)) + np.cumsum(rng.uniform(0, 0.3, (B, n_max)), axis=1) - 20,
                      rng.uniform(-half, half, (B, 1)) + rng.normal(0, 0.05, (B, n_max)).cumsum(axis=1),
                      rng.uniform(-0.3, 0.3, (B, n_max))], axis=1)
    return poses, rng.integers(0, n_max + 1, B).astype(np.int32)


@pytest.mark.gpu
def test_gpu_mapped_calls():
    dists, res, centers = _six_maps()
    pbn = bounds.PathBounds.from_maps(dists, res, centers=centers)
    per = 24
    B = per * len(dists)
    poses, n = _random_poses(B, 150, 3)
    idx = np.random.default_rng(4).permutation(np.repeat(np.arange(len(dists), dtype=np.int32), per))
    got = pbn.check_collision(poses, n, map_index=idx, clearance=True, per_state=True)
    for k in range(len(dists)):
        rows = np.nonzero(idx == k)[0]
        one = bounds.PathBounds(dists[k], res[k], center=centers[k])
        want = one.check_collision(poses[rows], n[rows], clearance=True, per_state=True)
        for f in want:
            assert np.array_equal(want[f], got[f][rows]), (k, f)
        _compare_to_oracle(dists[k], res[k], poses[rows], n[rows],
                           tuple(want[f] for f in ("first_hit", "state_free", "clearance")), k, center=centers[k])
        one.close()
    assert len(set(got["first_hit"].tolist())) > 3
    # an all-zero index is the unmapped call
    z = pbn.check_collision(poses, n, map_index=np.zeros(B, np.int32), clearance=True, per_state=True)
    u = pbn.check_collision(poses, n, clearance=True, per_state=True)
    for f in u:
        assert np.array_equal(z[f], u[f]), f
    # an index outside the slots: -1, no map read, no other path changed
    bad = idx.copy()
    bad[[0, 7, 50]] = [-1, len(dists), 2 ** 31 - 1]
    r = pbn.check_collision(poses, n, map_index=bad, clearance=True, per_state=True)
    assert list(r["first_hit"][[0, 7, 50]]) == [-1, -1, -1]
    assert not r["state_free"][[0, 7, 50]].any() and not r["clearance"][[0, 7, 50]].any()
    keep = np.setdiff1d(np.arange(B), [0, 7, 50])
    for f in got:
        assert np.array_equal(r[f][keep], got[f][keep]), f
    pbn.close()


@pytest.mark.gpu
def test_gpu_stream_order_after_set_occupancy():
    import torch
    dmap = sharedmap.DistanceMap()
    empty = np.full(dmap.dist.shape, 255, np.uint8)
    empty[0, 0] = 0
    pl = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=64)
    pl.set_occupancy(empty, dmap.res, obstacle_max=127)
    poses, n = _random_poses(64, 120, 6, half=50.0)
    tp, tn = torch.from_numpy(poses).cuda(), torch.from_numpy(n).cuda()
    img = torch.from_numpy(_png()).cuda()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        before = pl.check_collision_device(tp, tn, per_state=True, stream=s.cuda_stream)
        pl.set_occupancy_device(img, dmap.res, obstacle_max=127, stream=s)
        after = pl.check_collision_device(tp, tn, per_state=True, stream=s.cuda_stream)
    s.synchronize()
    fresh = bounds.PathBounds(dmap.dist, dmap.res)
    want = fresh.check_collision(poses, n, per_state=True)
    assert np.array_equal(after["first_hit"].cpu().numpy(), want["first_hit"])
    assert np.array_equal(after["state_free"].cpu().numpy(), want["state_free"])
    assert not np.array_equal(before["first_hit"].cpu().numpy(), want["first_hit"])
    fresh.close()
    pl.close()


@pytest.mark.gpu
def test_gpu_n_clamping_and_refusals():
    dmap = sharedmap.DistanceMap()
    pbn = bounds.PathBounds(dmap.dist, dmap.res)
    poses, _ = _random_poses(4, 80, 8, half=40.0)
    full = pbn.check_collision(poses, np.full(4, 80, np.int32), per_state=True, clearance=True)
    r = pbn.check_collision(poses, np.array([0, -5, 200, 80], np.int32), per_state=True, clearance=True)
    assert list(r["first_hit"][:2]) == [0, 0] and not r["state_free"][:2].any() and not r["clearance"][:2].any()
    for f in r:
        assert np.array_equal(r[f][2:], full[f][2:]), f
    assert (full["first_hit"] < 80).any() and full["state_free"].any()
    pl = plan.Planner(dmap.dist, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=4)
    Lb = pbn.L
    pp = np.ascontiguousarray(poses)
    nn = np.full(4, 80, np.int32)
    hit = np.zeros(4, np.int32)
    idx = np.zeros(4, np.int32)
    good_in = lambda **kw: bounds.CollisionIn(*[kw.get(k, v) for k, v in (  # noqa: E731
        ("batch", 4), ("n_max", 80), ("row_stride", 3), ("poses", pp.ctypes.data), ("n", nn.ctypes.data))])
    good_out = bounds.CollisionOut(hit.ctypes.data, None, None)
    cases = [(good_in(batch=0), good_out, "batch"), (good_in(n_max=0), good_out, "n_max"),
             (good_in(row_stride=2), good_out, "row_stride"), (good_in(poses=None), good_out, "poses"),
             (good_in(n=None), good_out, "first_hit"), (good_in(), bounds.CollisionOut(None, None, None), "first_hit")]
    for prefix, h in (("pqp_bounds_", pbn.h), ("pqp_plan_", pl.h)):
        err = getattr(Lb, prefix + "last_error")
        for ci, cout, word in cases:
            for fn, args in (("collision_check", ()), ("collision_check_device", (None,)),
                             ("collision_check_mapped", None), ("collision_check_mapped_device", None)):
                f = getattr(Lb, prefix + fn)
                if args is None:
                    rc = f(h, ctypes.byref(ci), idx.ctypes.data, ctypes.byref(cout), *(
                        (None,) if fn.endswith("device") else ()))
                else:
                    rc = f(h, ctypes.byref(ci), ctypes.byref(cout), *args)
                assert rc == abi.PQP_E_INVALID, (prefix, fn, word)
                assert word in err(h).decode(), (prefix, fn, err(h))
        for fn, args in (("collision_check_mapped", ()), ("collision_check_mapped_device", (None,))):
            rc = getattr(Lb, prefix + fn)(h, ctypes.byref(good_in()), None, ctypes.byref(good_out), *args)
            assert rc == abi.PQP_E_INVALID and b"null map_index" in err(h), (prefix, fn)
        assert getattr(Lb, prefix + "collision_check")(h, None, ctypes.byref(good_out)) == abi.PQP_E_INVALID
    pl.close()
    pbn.close()


@pytest.mark.gpu
def test_gpu_launch_counts():
    import torch
    dmap = sharedmap.DistanceMap()
    B = 32
    host_in, d_in = _points_device(B, dmap)
    raw = sharedmap.make_plan_inputs(B, dmap=dmap)
    for method, base in (("TENSION2", 23), ("TENSION", 24)):
        pl = plan.Planner.from_maps([dmap.dist, dmap.dist], dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N,
                                    batch_max=B, params=plan.default_params(method))
        idx = torch.zeros(B, dtype=torch.int32, device="cuda")
        counts = [pl.launch_count]
        pl.plan(*raw)
        counts.append(pl.launch_count)
        out = pl.plan_points_device(*d_in, map_index=idx)
        counts.append(pl.launch_count)
        pl.check_collision_device(out["path"], out["n"], map_index=idx)
        counts.append(pl.launch_count)
        pl.check_collision_device(out["path"], out["n"])
        counts.append(pl.launch_count)
        torch.cuda.synchronize()
        pr = pl.plan_points(*host_in)
        counts.append(pl.launch_count)
        pl.check_collision(pr.path, pr.n, clearance=True)
        counts.append(pl.launch_count)
        pl.check_collision(pr.path, pr.n, map_index=np.ones(B, np.int32), per_state=True)
        counts.append(pl.launch_count)
        assert list(np.diff(counts)) == [base, base + 2, 1, 1, base + 2, 1, 1], (method, counts)
        assert plan.COLLISION_LAUNCHES == 1
        pl.close()
    pbn = bounds.PathBounds(dmap.dist, dmap.res)
    poses, n = _random_poses(8, 50, 1)
    pbn.check_collision(poses, n)
    assert pbn.last_kernel_ms > 0
    pbn.close()
