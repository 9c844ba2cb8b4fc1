"""The C++ drop-in for the reference's PathOptimizer (include/pqp_path_optimizer.hpp), driven like the demo drives it:
one object per plan, constructed with that plan's map (tests/cpp/path_optimizer_test.cpp).

CPU: it compiles with -Wall against the stub boundary types and links the C ABI library; with no GPU the
constructor records the library's error, solve returns false, a pre-filled final_path stays as it was, the reference
path view is empty and the handle pool holds no handle.
GPU: solve's result, final_path and the view equal Planner.plan_points' outputs and trace bit for bit (same library,
B = 1 equals its row of a batch), under both smoothing methods; each failure row leaves final_path and the view as the
reference's control flow does; per-tick construction on alternating maps creates one plan handle; the occupancy
constructor equals the distance constructor on that image's transform."""
import math
import os
import subprocess

import numpy as np
import pytest

from path_optimizer_2_b200 import plan, sharedmap, solver

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "path_optimizer_test")
PNG = os.path.join(ROOT, "tests", "golden", "gridmap.png")
RES = sharedmap.RES
CAPS = dict(r_max=256, p_max=256, layers_max=160, n_max=511)  # PathOptimizerOptions' defaults
N = CAPS["n_max"]
MARKER = -7.0  # what the program pre-fills final_path with


def _build():
    solver.build_library()
    src = os.path.join(ROOT, "tests", "cpp", "path_optimizer_test.cpp")
    deps = [src, solver.LIB_PATH, os.path.join(ROOT, "tests", "cpp", "ref_stub.hpp")] + [
        os.path.join(ROOT, "include", h) for h in ("pqp_path_optimizer.hpp", "pqp_base_solver.hpp",
                                                   "pqp_reference_path.hpp", "pqp_plan.h")]
    if not os.path.exists(BIN) or any(os.path.getmtime(d) > os.path.getmtime(BIN) for d in deps):
        subprocess.check_call(["g++", "-std=c++11", "-O1", "-Wall", "-o", BIN, src, solver.LIB_PATH,
                               "-Wl,-rpath," + os.path.dirname(solver.LIB_PATH)])
    return BIN


def _png():
    from PIL import Image
    return np.asarray(Image.open(PNG).convert("L")).astype(np.uint8)


def write_script(d, params, maps, cases):
    """maps: ("dist", layer) or ("occ", image, obstacle_max); cases: (map index, xs, ys, start[4], target[3])."""
    lines = []
    if params is not None:
        p = os.path.join(d, "params.bin")
        with open(p, "wb") as f:
            f.write(bytes(params))
        lines.append("params " + p)
    for i, m in enumerate(maps):
        p = os.path.join(d, "map%d.bin" % i)
        if m[0] == "dist":
            np.ascontiguousarray(m[1], dtype=np.float32).tofile(p)
            lines.append("dist %d %d %.17g 0 0 %s" % (m[1].shape + (RES, p)))
        else:
            np.ascontiguousarray(m[1], dtype=np.uint8).tofile(p)
            lines.append("occ %d %d %.17g 0 0 %d %s" % (m[1].shape + (RES, m[2], p)))
    for mi, xs, ys, st, tg in cases:
        vals = list(xs) + list(ys) + list(st) + list(tg)
        lines.append("case %d %d " % (mi, len(xs)) + " ".join("%.17g" % v for v in vals))
    path = os.path.join(d, "script.txt")
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return path


def _rows(lines, width):
    a = np.array([[float(v) for v in ln.split()] for ln in lines], dtype=np.float64)
    return a.reshape(len(lines), width)


def parse(out):
    """-> (list of per-case dicts, pool creates, pool hits)"""
    ln = out.rstrip("\n").split("\n")
    i, cases = 0, []
    while ln[i].startswith("case "):
        t = ln[i].split()
        c = dict(ok=int(t[3]), status=int(t[5]))
        npath = int(t[7])
        c["path"] = _rows(ln[i + 1:i + 1 + npath], 10)
        i += 1 + npath
        t = ln[i].split()
        ns, nb, blk = int(t[3]), int(t[4]), int(t[5])
        c["k"], c["length"] = int(t[1]), float(t[2])
        c["spline"] = [np.array([float(v) for v in r.split()]) for r in ln[i + 1:i + 11]]
        i += 11
        c["states"] = _rows(ln[i:i + ns], 5)
        c["bounds"] = _rows(ln[i + ns:i + ns + nb], 15)
        c["blocked"] = _rows(ln[i + ns + nb:i + ns + nb + blk], 15)[0] if blk else None
        i += ns + nb + blk
        if ln[i].startswith("check "):
            n = int(ln[i].split()[1])
            c["check"] = _rows(ln[i + 1:i + 1 + n], 7)
            i += 1 + n
        assert ln[i].startswith("error"), ln[i]
        c["error"] = ln[i][6:]
        cases.append(c)
        i += 1
    t = ln[i].split()
    assert t[0] == "pool", ln[i]
    return cases, int(t[2]), int(t[4])


def run(script):
    out = subprocess.run([_build(), script], capture_output=True, text=True, check=True).stdout
    return parse(out)


def _wrap(a):
    """constrainAngle (tools.hpp:24-35) for the angles of a path: into [-pi, pi]"""
    a = np.array(a, dtype=np.float64)
    for i in range(a.size):
        while a.flat[i] > math.pi:
            a.flat[i] -= 2 * math.pi
        while a.flat[i] < -math.pi:
            a.flat[i] += 2 * math.pi
    return a


def frenet_path(st, sol, n):
    """getOptimizedPath (base_solver.cpp:263-288) in numpy: st [4][N] s, x, y, heading; sol [4][N] l, psi, k, d_k."""
    h, l, psi = st[3, :n], sol[0, :n], sol[1, :n]
    ang = _wrap(h + math.pi / 2)
    dk = np.append(sol[3, :n - 1], 0.0)
    return np.stack([st[1, :n] + l * np.cos(ang), st[2, :n] + l * np.sin(ang), _wrap(h + psi), sol[2, :n], dk, l, psi])


def check_case(c, r, b, params, tag):
    """The drop-in's outputs for path b of Planner result r (traced): final_path and view per the failure table."""
    st, T = int(r.status[b]), r.trace
    assert c["status"] == st and c["ok"] == (st == plan.OK), (tag, c["status"], st, c["error"])
    assert (c["error"] == "") == (st == plan.OK), (tag, c["error"])
    p = c["path"]
    if st == plan.OK:
        n = int(r.n[b])
        assert p.shape == (n, 10) and np.array_equal(p[:, :7].T, r.path[b, :, :n]) and not p[:, 7:].any(), tag
        # the construction a failed re-solve uses, on the second solution: out.path again
        ck = c["check"]
        assert np.allclose(ck[:, :3].T, r.path[b, :3, :n], atol=1e-12, rtol=0), tag
        assert np.array_equal(ck[:, 3:].T, r.path[b, 3:, :n]), tag
    elif st == plan.PRE_SOLVE_FAILED:
        assert p.shape == (0, 10), tag
    elif st == plan.SOLVE_FAILED:
        nv = int(T["n_valid"][b])
        want = frenet_path(T["states"][b], T["sol1"][b], nv)
        assert p.shape == (nv, 10) and np.allclose(p[:, :3].T, want[:3], atol=1e-12, rtol=0), tag
        assert np.array_equal(p[:, 3:7].T, want[3:]), tag
    else:
        assert p.shape == (2, 10) and np.all(p[:, :7] == MARKER), (tag, "final_path touched")
    # the reference path view
    smoothed = st == plan.OK or plan.EMPTY_REFERENCE <= st <= plan.SOLVE_FAILED
    if not smoothed:
        assert c["k"] == 0 and c["length"] == 0.0 and len(c["states"]) == 0 and len(c["bounds"]) == 0, tag
        assert c["blocked"] is None, tag
        return
    k = int(T["dp_n_out"][b])
    rs = T["ref_spline"][b][:, :k]
    assert c["k"] == k, tag
    for got, want in zip(c["spline"], [rs[0], rs[1], rs[2], rs[3], rs[4], rs[0], rs[5], rs[6], rs[7], rs[8]]):
        assert np.array_equal(got, want), tag
    if st in (plan.EMPTY_REFERENCE, plan.INIT_HEADING):
        assert c["length"] == rs[0, k - 1] and len(c["states"]) == 0 and len(c["bounds"]) == 0, tag
        assert c["blocked"] is None, tag
        return
    assert c["length"] == T["max_s"][b], tag
    total = min(int(T["total"][b]), N)
    nv = total if st == plan.TOO_MANY_KNOTS else int(T["n_valid"][b])
    S = T["states"][b]
    want = np.stack([S[1, :nv], S[2, :nv], S[3, :nv], T["curvature"][b, :nv], S[0, :nv]], axis=1)
    assert np.array_equal(c["states"], want), tag
    if st == plan.TOO_MANY_KNOTS:
        assert len(c["bounds"]) == 0 and c["blocked"] is None, tag
        return
    filled = nv + 1 if nv < total else total
    got = np.vstack([c["bounds"]] + ([c["blocked"][None]] if c["blocked"] is not None else []))
    assert (c["blocked"] is not None) == (nv < total) and got.shape == (filled, 15), tag
    Bd = T["bounds"][b]
    for a, (lo, hi) in enumerate(((0, 1), (2, 3), (4, 5))):
        assert np.array_equal(got[:, 5 * a], Bd[lo, :filled]) and np.array_equal(got[:, 5 * a + 1], Bd[hi, :filled]), tag
        assert np.array_equal(got[:, 5 * a + 4], S[3, :filled]), tag
    x, y, h = S[1, :filled], S[2, :filled], S[3, :filled]
    for a, d in ((0, params.bounds.front_length), (1, params.bounds.rear_length), (2, 0.0)):
        assert np.allclose(got[:, 5 * a + 2], x + d * np.cos(h), atol=1e-12, rtol=0), tag
        assert np.allclose(got[:, 5 * a + 3], y + d * np.sin(h), atol=1e-12, rtol=0), tag


def test_path_optimizer_dropin_compiles_and_fails_loudly_without_gpu(tmp_path):
    _build()
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    img = np.full((40, 50), 255, np.uint8)
    img[10:12, 20:30] = 0
    dist = np.full(img.shape, 3.0, np.float32)
    pts = (np.linspace(-3.0, 3.0, 6), np.zeros(6), (-3.0, 0.0, 0.0, 0.0), (3.0, 0.0, 0.0))
    script = write_script(str(tmp_path), plan.default_params(), [("dist", dist), ("occ", img, 0)],
                          [(0,) + pts, (1,) + pts])
    cases, creates, hits = run(script)
    assert len(cases) == 2 and creates == 0 and hits == 0
    for c in cases:
        assert c["ok"] == 0 and c["status"] == -1 and "no CUDA device" in c["error"], c["error"]
        assert c["path"].shape == (2, 10) and np.all(c["path"][:, :7] == MARKER)
        assert c["k"] == 0 and c["length"] == 0.0 and len(c["states"]) == 0 and len(c["bounds"]) == 0
        assert c["blocked"] is None and "check" not in c


# ------------------------------------------------------------------------------------------------------------ GPU
B = 64


@pytest.fixture(scope="module")
def demo():
    from oracle import edt_oracle as eo
    img = _png()
    dist = eo.transform(img, RES, 127)[1]
    pts = sharedmap.make_plan_points(B, dmap=sharedmap.DistanceMap(dist=dist))
    return dict(img=img, dist=dist, pts=pts)


def _planner(dist, params, batch_max=B):
    return plan.Planner(dist, RES, batch_max=batch_max, params=params, **CAPS)


def _cases(pts, idx, mi=0):
    ref_x, ref_y, start, target = pts
    return [(mi, ref_x[b], ref_y[b], start[b], target[b]) for b in idx]


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["TENSION2", "TENSION"])
def test_gpu_parity_with_planner(tmp_path, demo, method):
    params = plan.default_params(method)
    pl = _planner(demo["dist"], params)
    r = pl.plan_points(*demo["pts"], trace=True)
    pl.close()
    assert np.mean(r.status == plan.OK) > 0.7, r.status_names()
    cases, creates, hits = run(write_script(str(tmp_path), params, [("dist", demo["dist"])],
                                            _cases(demo["pts"], range(B))))
    assert len(cases) == B and creates == 1 and hits == B - 1
    for b in range(B):
        check_case(cases[b], r, b, params, (method, b))
    print(method, "statuses:", sorted(set(r.status_names())))


@pytest.mark.gpu
def test_gpu_failure_rows(tmp_path, demo):
    params = plan.default_params()
    ref_x, ref_y, start, target = demo["pts"]
    dist = demo["dist"]
    pl = _planner(dist, params)
    base = pl.plan_points(*demo["pts"], trace=True)
    ok = [b for b in range(B) if base.status[b] == plan.OK]
    b0, b1 = ok[0], ok[1]
    # 3 points (POINT_COUNT) and a start heading 90 degrees off (INIT_HEADING)
    st = start[[b0, b1]].copy()
    st[1, 2] += math.pi / 2
    xs, ys = [ref_x[b0][:3], ref_x[b1]], [ref_y[b0][:3], ref_y[b1]]
    # a pinched map: a dot of 3 x 3 cells on the reference where the front circle of a state reaches it, small enough
    # to pass between the DP's nodes; 3.9 m along the path it blocks the start, further on it cuts the states
    pinch = []
    for b, s_at in ((b0, 3.9), (b1, 20.0), (ok[2], 12.0)):
        T = base.trace
        i = int(np.argmin(np.abs(T["states"][b, 0, :T["total"][b]] - s_at)))
        d = dist.copy()
        ci = int((d.shape[0] * RES / 2 - T["states"][b, 1, i]) / RES)
        cj = int((d.shape[1] * RES / 2 - T["states"][b, 2, i]) / RES)
        d[ci - 1:ci + 2, cj - 1:cj + 2] = 0.0
        pinch.append((b, d))
    maps = [("dist", dist)] + [("dist", d) for _, d in pinch]
    cases = [(0, xs[j], ys[j], st[j], target[[b0, b1]][j]) for j in range(2)]
    cases += [(1 + j, ref_x[b], ref_y[b], start[b], target[b]) for j, (b, _) in enumerate(pinch)]
    got, _, _ = run(write_script(str(tmp_path), params, maps, cases))
    r = pl.plan_points(xs, ys, st, target[[b0, b1]], trace=True)
    assert list(r.status) == [plan.POINT_COUNT, plan.INIT_HEADING], r.status_names()
    for j in range(2):
        check_case(got[j], r, j, params, ("row", j))
    blocked = 0
    for j, (b, d) in enumerate(pinch):
        pl.set_map(d, RES)
        rp = pl.plan_points([ref_x[b]], [ref_y[b]], start[[b]], target[[b]], trace=True)
        check_case(got[2 + j], rp, 0, params, ("pinch", j))
        blocked += got[2 + j]["blocked"] is not None
    assert blocked >= 2 and got[2]["status"] == plan.BLOCKED_AT_START, [g["status"] for g in got]
    pl.close()
    # the first solve capped by the solver's iteration limit: PRE_SOLVE_FAILED clears final_path, the view is complete
    capped = plan.default_params()
    capped.solver.max_iter = 5
    pc = _planner(dist, capped)
    idx = ok[:4]
    rc = pc.plan_points([ref_x[b] for b in idx], [ref_y[b] for b in idx], start[idx], target[idx], trace=True)
    pc.close()
    assert all(s == plan.PRE_SOLVE_FAILED for s in rc.status), rc.status_names()
    got, _, _ = run(write_script(str(tmp_path), capped, [("dist", dist)], _cases(demo["pts"], idx)))
    for j in range(len(idx)):
        check_case(got[j], rc, j, capped, ("capped", j))
        assert len(got[j]["states"]) > 0 and len(got[j]["path"]) == 0


@pytest.mark.gpu
def test_gpu_frenet_path_matches_second_solution(demo):
    """The SOLVE_FAILED construction in numpy (the same arithmetic as the header's getOptimizedPath) against the
    GPU's final path: applied to each solved plan's second solution it reproduces out.path."""
    params = plan.default_params()
    pl = _planner(demo["dist"], params)
    r = pl.plan_points(*demo["pts"], trace=True)
    pl.close()
    for b in np.nonzero(r.status == plan.OK)[0]:
        n = int(r.n[b])
        sol2 = r.path[b, [5, 6, 3, 4]]
        want = frenet_path(r.trace["states"][b], sol2, n)
        assert np.allclose(want[:3], r.path[b, :3, :n], atol=1e-12, rtol=0) and np.array_equal(want[3:], r.path[b, 3:, :n])


@pytest.mark.gpu
def test_gpu_per_tick_pool(tmp_path, demo):
    from oracle import edt_oracle as eo
    from tests.test_map_update import _cell
    params = plan.default_params()
    img_b = demo["img"].copy()
    ref_x, ref_y, start, target = demo["pts"]
    rows, cols = img_b.shape
    ticks = list(range(20))
    for b in ticks[1::2]:  # a block on the reference of every path planned on map B
        m = len(ref_x[b]) // 2
        i, j = _cell(ref_x[b][m], ref_y[b][m], rows, cols)
        img_b[max(i - 4, 0):i + 5, max(j - 4, 0):j + 5] = 0
    dist_b = eo.transform(img_b, RES, 127)[1]
    cases = [(t % 2, ref_x[t], ref_y[t], start[t], target[t]) for t in ticks]
    got, creates, hits = run(write_script(str(tmp_path), params, [("dist", demo["dist"]), ("dist", dist_b)], cases))
    assert creates == 1 and hits == len(ticks) - 1
    on = {}
    for mi, dist in enumerate((demo["dist"], dist_b)):
        pl = _planner(dist, params, batch_max=len(ticks))
        on[mi] = pl.plan_points([ref_x[t] for t in ticks], [ref_y[t] for t in ticks], start[ticks], target[ticks],
                                trace=True)
        pl.close()
    for t in ticks:
        check_case(got[t], on[t % 2], t, params, ("tick", t))
    # the blocks change what is planned on map B
    assert any(on[0].status[t] != on[1].status[t] or not np.array_equal(on[0].path[t], on[1].path[t])
               for t in ticks[1::2])


@pytest.mark.gpu
def test_gpu_occupancy_constructor(tmp_path, demo):
    from oracle import edt_oracle as eo
    params = plan.default_params()
    img = demo["img"]
    idx = list(range(8))
    maps = [("occ", img, 127), ("dist", eo.transform(img, RES, 127)[1])]
    cases = _cases(demo["pts"], idx, 0) + _cases(demo["pts"], idx, 1)
    got, creates, _ = run(write_script(str(tmp_path), params, maps, cases))
    assert creates == 1
    for j in range(len(idx)):
        a, b = got[j], got[len(idx) + j]
        for key in a:
            if isinstance(a[key], list):
                assert all(np.array_equal(u, v) for u, v in zip(a[key], b[key])), (j, key)
            elif isinstance(a[key], np.ndarray):
                assert np.array_equal(a[key], b[key]), (j, key)
            else:
                assert a[key] == b[key], (j, key)
    assert sum(g["ok"] for g in got) > len(idx)
