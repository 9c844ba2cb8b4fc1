"""include/pqp_plan_multi.h: the whole plan over several GPUs (plan_multi.MultiPlanner).

CPU: the declaration against the binding and the library, the create checks before and at the device lookup, and the
trace table the plan copies with (tests/cpp/plan_trace_test.cpp under g++). GPU: MultiPlanner over [0] and [0, 0] (two
handles on one GPU: two shards, staging and peer copies on any box) against a Planner of the same capacities, bit for
bit, host and device forms, every trace field; slot updates on every device and their order on the stream; launch
counts; no leaks. Over distinct devices when the box has them."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import bench_maps
from path_optimizer_2_b200 import abi, bounds, plan, plan_multi, sharedmap, solver

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R, P, L, N = 64, 64, 64, 255


def test_symbols_match_the_header():
    with open(os.path.join(ROOT, "include", "pqp_plan_multi.h")) as f:
        declared = set(re.findall(r"^\s*(?:int|const char \*)\s*(pqp_\w+)\s*\(", f.read(), re.M))
    assert declared == set(plan_multi.EXPORTED_SYMBOLS)
    L_ = plan_multi._lib()
    assert all(hasattr(L_, s) for s in plan_multi.EXPORTED_SYMBOLS)


def test_create_checks():
    L_ = plan_multi._lib()
    dist = np.ones((4, 4), dtype=np.float32)
    m = bounds.BoundsMap(4, 4, 0.1, 0.0, 0.0, dist.ctypes.data)
    pp = plan.default_params()
    out = C.c_void_p()
    dv = (C.c_int32 * 2)(0, 0)
    create = L_.pqp_plan_multi_create_maps
    err = lambda: (L_.pqp_plan_multi_last_error(None) or b"").decode()  # noqa: E731
    assert create(C.byref(m), 1, C.byref(pp), R, P, L, N, 8, 2, dv, None) == abi.PQP_E_INVALID
    assert err() == "pqp_plan_multi_create_maps: out is null"
    for params, n_dev, batch_max in ((None, 2, 8), (pp, 0, 8), (pp, 2, 0)):
        assert create(C.byref(m), 1, C.byref(params) if params else None, R, P, L, N, batch_max, n_dev, dv,
                      C.byref(out)) == abi.PQP_E_INVALID
        assert err() == "pqp_plan_multi_create_maps: params required, n_devices >= 1, batch_max >= 1"
        assert not out.value
    # a device index no box has: the device lookup, on a machine with or without GPUs
    far = (C.c_int32 * 2)(0, 4096)
    assert create(C.byref(m), 1, C.byref(pp), R, P, L, N, 8, 2, far, C.byref(out)) == abi.PQP_E_NO_DEVICE
    assert re.fullmatch(r"pqp_plan_multi_create_maps: device (0|4096) requested, \d+ CUDA devices visible "
                        r"\(there is no CPU fallback\)", err()), err()
    assert not out.value
    # a capacity the plan handle refuses is refused before the device lookup, too
    for r_max, p_max, layers_max, n_max in ((2, P, L, N), (R, 3, L, N), (R, P, 3, N), (R, P, L, 1), (R, P, L, 512)):
        assert create(C.byref(m), 1, C.byref(pp), r_max, p_max, layers_max, n_max, 8, 2, far,
                      C.byref(out)) == abi.PQP_E_INVALID
        assert err() == "pqp_plan_multi_create_maps: r_max >= 3, p_max >= 4, layers_max >= 4, 2 <= n_max <= 511"
        assert not out.value
    with pytest.raises(solver.PqpError) as e:
        plan_multi.MultiPlanner([dist], 0.1, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=8, devices=[4096])
    assert e.value.code == abi.PQP_E_NO_DEVICE


def test_trace_table_sizes(tmp_path):
    """The per-path bytes of every trace member, against the sizes the plan's trace copy restated before the table."""
    exe = str(tmp_path / "plan_trace_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "plan_trace_test.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok %d" % len(plan._TRACE), out.stdout


# ---------------------------------------------------------------------------------------------------------------- GPU

def _same(a, b):
    """bit-identical arrays (numpy or torch)"""
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    b = b.cpu().numpy() if hasattr(b, "cpu") else np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _assert_results(got, want, trace=False):
    for k in ("status", "n", "path", "cost", "iters"):
        g = got[k] if isinstance(got, dict) else getattr(got, k)
        w = want[k] if isinstance(want, dict) else getattr(want, k)
        assert _same(g, w), k
    if trace:
        assert set(got.trace) == set(want.trace)
        bad = [k for k in want.trace if not _same(got.trace[k], want.trace[k])]
        assert not bad, "trace fields differ: %s" % bad


def _blocked(demo, seed, count, res):
    """`count` copies of the demo image with their own random obstacle blocks (bench_maps.py's maps)"""
    return bench_maps._blocked(demo, np.random.default_rng(seed), count, res)


@pytest.fixture(scope="module")
def scene():
    from PIL import Image
    dmap = sharedmap.DistanceMap()
    demo = np.asarray(Image.open(os.path.join(ROOT, "tests", "golden", "gridmap.png")).convert("L")).astype(np.uint8)
    # three slots: the demo map and two blocked variants, their layers from a single-device planner's transform
    pl = plan.Planner.from_maps([dmap.dist] * 3, dmap.res, r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=1)
    pl.set_occupancy_slots(_blocked(demo, 5, 2, dmap.res), dmap.res, obstacle_max=127, first_slot=1)
    layers = [pl.get_map(s)[0] for s in range(3)]
    pl.close()
    B = 1001  # the last of two shards is one path shorter
    pts = sharedmap.make_plan_points(B, dmap=dmap)
    raw = sharedmap.make_plan_inputs(B, dmap=dmap)
    idx = (np.arange(B) % 3).astype(np.int32)
    idx[700] = 3  # outside the slots
    return dict(dmap=dmap, demo=demo, layers=layers, pts=pts, raw=raw, idx=idx, B=B)


def _pair(scene, devices, method, batch_max=None, layers=None):
    layers = scene["layers"] if layers is None else layers
    kw = dict(r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=batch_max or scene["B"],
              params=plan.default_params(method))
    single = plan.Planner.from_maps(layers, scene["dmap"].res, **kw)
    multi = plan_multi.MultiPlanner(layers, scene["dmap"].res, devices=devices, **kw)
    return single, multi


def _device_points(ref_x, ref_y, start, target):
    import torch
    B = len(ref_x)
    m = np.array([len(v) for v in ref_x], dtype=np.int32)
    px, py = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        px[b, :m[b]], py[b, :m[b]] = ref_x[b], ref_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    return [t(px), t(py), t(m), t(start), t(target)]


def _visible():
    import torch
    return torch.cuda.device_count()


@pytest.mark.gpu
@pytest.mark.parametrize("mapped", [False, True], ids=["unmapped", "mapped"])
@pytest.mark.parametrize("method", ["TENSION2", "TENSION"])
@pytest.mark.parametrize("devices", [[0], [0, 0], [0, 1]], ids=["0", "0-0", "0-1"])
def test_matches_a_planner(scene, devices, method, mapped):
    """B = 1001 from reference points: host form with every trace field, device form, against one Planner."""
    import torch
    if max(devices) >= _visible():
        pytest.skip("needs %d distinct GPUs, %d visible" % (max(devices) + 1, _visible()))
    single, multi = _pair(scene, devices, method)
    idx = scene["idx"] if mapped else None
    want = single.plan_points(*scene["pts"], trace=True, map_index=idx)
    got = multi.plan_points(*scene["pts"], trace=True, map_index=idx)
    _assert_results(got, want, trace=True)
    if mapped:
        assert want.status[700] == plan.MAP_INDEX
    assert (want.status == plan.OK).any()
    per = -(-scene["B"] // len(devices))
    assert [multi.shard(i) for i in range(len(devices))] == [(i * per, min(scene["B"] - i * per, per))
                                                              for i in range(len(devices))]
    d_in = _device_points(*scene["pts"])
    d_idx = torch.from_numpy(scene["idx"]).cuda() if mapped else None
    w = single.plan_points_device(*d_in, map_index=d_idx)
    g = multi.plan_points_device(*d_in, map_index=d_idx)
    torch.cuda.synchronize()
    _assert_results(g, w)
    _assert_results(g, want)
    single.close()
    multi.close()


@pytest.mark.gpu
def test_samples_forms_match_a_planner(scene):
    """pqp_plan_multi / pqp_plan_multi_device (from bSpline() samples) on two shards, mapped."""
    import torch
    single, multi = _pair(scene, [0, 0], "TENSION2")
    raw_x, raw_y, start, target = scene["raw"]
    want = single.plan(raw_x, raw_y, start, target, trace=True, map_index=scene["idx"])
    _assert_results(multi.plan(raw_x, raw_y, start, target, trace=True, map_index=scene["idx"]), want, trace=True)
    B = scene["B"]
    r = np.array([len(v) for v in raw_x], dtype=np.int32)
    rx, ry = np.zeros((B, R)), np.zeros((B, R))
    for b in range(B):
        rx[b, :r[b]], ry[b, :r[b]] = raw_x[b], raw_y[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    g = multi.plan_device(t(rx), t(ry), t(r), t(start), t(target), map_index=t(scene["idx"]))
    torch.cuda.synchronize()
    _assert_results(g, want)
    single.close()
    multi.close()


@pytest.mark.gpu
def test_one_path_on_two_shards(scene):
    import torch
    single, multi = _pair(scene, [0, 0], "TENSION2", batch_max=2)
    one = [v[:1] for v in scene["pts"]]
    want = single.plan_points(*one)
    _assert_results(multi.plan_points(*one), want)
    assert multi.shard(0) == (0, 1) and multi.shard(1) == (1, 0)
    g = multi.plan_points_device(*_device_points(*one))
    torch.cuda.synchronize()
    _assert_results(g, want)
    single.close()
    multi.close()


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["host", "device"])
def test_slot_updates_reach_every_device(scene, form):
    import torch
    res = scene["dmap"].res
    single, multi = _pair(scene, [0, 0], "TENSION2")
    single.close()
    imgs = _blocked(scene["demo"], 9, 2, res)
    if form == "host":
        multi.set_occupancy_slots(imgs, res, obstacle_max=127, first_slot=1)
    else:
        multi.set_occupancy_slots_device(torch.from_numpy(imgs).cuda(), res, obstacle_max=127, first_slot=1)
    layers = []
    for s in range(3):
        home = multi.get_map_slot(0, s)
        other = multi.get_map_slot(1, s)
        assert _same(home[0], other[0]) and home[1:] == other[1:], "slot %d" % s
        layers.append(home[0])
    assert not _same(layers[1], scene["layers"][1])
    fresh, unused = _pair(scene, [0], "TENSION2", layers=layers)
    unused.close()
    want = fresh.plan_points(*scene["pts"], map_index=scene["idx"])
    _assert_results(multi.plan_points(*scene["pts"], map_index=scene["idx"]), want)
    # a layer given as such, on every device
    multi.set_map_slot(scene["layers"][0], res, slot=2)
    assert _same(multi.get_map_slot(1, 2)[0], scene["layers"][0])
    # a refused update changes nothing anywhere
    with pytest.raises(solver.PqpError) as e:
        multi.set_occupancy_slots(imgs, res, obstacle_max=127, first_slot=2)
    assert e.value.code == abi.PQP_E_INVALID and str(e.value).startswith("pqp error -1: device 0: ")
    assert _same(multi.get_map_slot(1, 2)[0], scene["layers"][0])
    fresh.close()
    multi.close()


@pytest.mark.gpu
def test_device_update_is_ordered_on_the_stream(scene):
    """plan, update every slot to all-obstacle images, plan: one stream, no host synchronisation in between."""
    import torch
    res = scene["dmap"].res
    single, multi = _pair(scene, [0, 0], "TENSION2")
    d_in = _device_points(*scene["pts"])
    d_idx = torch.from_numpy(scene["idx"]).cuda()
    blocked = torch.zeros((3,) + scene["demo"].shape, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = multi.plan_points_device(*d_in, map_index=d_idx)
    multi.set_occupancy_slots_device(blocked, res, obstacle_max=127)
    after = multi.plan_points_device(*d_in, map_index=d_idx)
    torch.cuda.synchronize()
    _assert_results(before, single.plan_points_device(*d_in, map_index=d_idx))
    single.set_occupancy_slots_device(blocked, res, obstacle_max=127)
    want_after = single.plan_points_device(*d_in, map_index=d_idx)
    torch.cuda.synchronize()
    _assert_results(after, want_after)
    assert not _same(before["status"], after["status"])
    single.close()
    multi.close()


@pytest.mark.gpu
def test_device_update_is_complete_once_the_stream_has_passed_it(scene):
    """device-form update of 64 slots, a synchronisation of the caller's stream alone, then a host-form plan: the
    second shard's handle plans on its own stream and must see its device's transforms finished"""
    import torch
    res, M = scene["dmap"].res, 64
    zero = np.zeros(scene["demo"].shape, np.float32)
    kw = dict(r_max=R, p_max=P, layers_max=L, n_max=N, batch_max=scene["B"], params=plan.default_params("TENSION2"))
    multi = plan_multi.MultiPlanner([zero] * M, res, devices=[0, 0], **kw)
    imgs = torch.from_numpy(_blocked(scene["demo"], 17, M, res)).cuda()
    stream = torch.cuda.current_stream()
    stream.synchronize()
    multi.set_occupancy_slots_device(imgs, res, obstacle_max=127, stream=stream)
    stream.synchronize()
    del imgs  # released once the stream has passed the update
    idx = (np.arange(scene["B"]) % M).astype(np.int32)
    got = multi.plan_points(*scene["pts"], map_index=idx)
    torch.cuda.synchronize()
    layers = [multi.get_map_slot(0, s)[0] for s in range(M)]
    assert all(_same(multi.get_map_slot(1, s)[0], layers[s]) for s in range(M))
    fresh = plan.Planner.from_maps(layers, res, **kw)
    _assert_results(got, fresh.plan_points(*scene["pts"], map_index=idx))
    fresh.close()
    multi.close()


@pytest.mark.gpu
def test_device_form_refuses_a_trace(scene):
    import torch
    single, multi = _pair(scene, [0, 0], "TENSION2", batch_max=4)
    single.close()
    d_in = _device_points(*[v[:4] for v in scene["pts"]])
    outs = [torch.zeros(s, dtype=dt, device="cuda") for s, dt in
            ((4, torch.int32), (4, torch.int32), ((4, 7, N), torch.float64), (4, torch.float64), ((4, 2), torch.int32))]
    tr = plan._trace_struct(plan._trace_arrays(4, multi.dims, lambda shape, dt: torch.zeros(
        shape, dtype={np.float64: torch.float64, np.int32: torch.int32}[dt], device="cuda")), lambda a: a.data_ptr())
    pin = plan.PlanPointsIn(4, R, *(t.data_ptr() for t in d_in))
    pout = plan.PlanOut(*(t.data_ptr() for t in outs), C.pointer(tr))
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert multi.L.pqp_plan_multi_points_device(multi.h, C.byref(pin), None, C.byref(pout), s) == abi.PQP_E_INVALID
    assert "take no trace" in multi.L.pqp_plan_multi_last_error(multi.h).decode()
    torch.cuda.synchronize()
    assert all(not t.any() for t in outs)
    multi.close()


@pytest.mark.gpu
@pytest.mark.parametrize("devices", [[0, 0, 0], [0, 0]])
def test_launch_counts(scene, devices):
    """per-device launches: a single-device call's count for each non-empty shard (B = 2: one shard empty at G = 3)"""
    single, multi = _pair(scene, devices, "TENSION", batch_max=8)
    two = [v[:2] for v in scene["pts"]]
    G = len(devices)
    c0, m0 = single.launch_count, [multi.launch_count(i) for i in range(G)]
    single.plan_points(*two, map_index=scene["idx"][:2])
    multi.plan_points(*two, map_index=scene["idx"][:2])
    per_call = single.launch_count - c0
    deltas = [multi.launch_count(i) - m0[i] for i in range(G)]
    assert deltas == [per_call] * 2 + [0] * (G - 2)
    assert sum(deltas) == per_call * 2
    assert all(multi.last_stage_ms(i)["total"] > 0 for i in range(2))
    single.close()
    multi.close()


@pytest.mark.gpu
def test_rounds_do_not_leak(scene):
    import torch
    from tests.test_handle_lifecycle import _rounds
    pts = [v[:6] for v in scene["pts"]]
    d_in = _device_points(*pts)
    imgs = torch.from_numpy(_blocked(scene["demo"], 2, 2, scene["dmap"].res)).cuda()

    def one_round():
        mp = plan_multi.MultiPlanner(scene["layers"], scene["dmap"].res, r_max=R, p_max=P, layers_max=L, n_max=N,
                                     batch_max=6, devices=[0, 0], params=plan.default_params("TENSION"))
        mp.plan_points(*pts, trace=True)
        mp.set_occupancy_slots_device(imgs, scene["dmap"].res, obstacle_max=127, first_slot=1)
        mp.plan_points_device(*d_in)
        mp.close()

    _rounds(one_round)


@pytest.mark.gpu
def test_all_visible_devices_8192_plans(scene):
    """The scaling workload over every visible device, against one Planner."""
    import torch
    G = _visible()
    if G < 2:
        pytest.skip("needs 2 or more GPUs, 1 visible")
    B = 8192
    pts = sharedmap.make_plan_points(B, dmap=scene["dmap"])
    single, multi = _pair(scene, list(range(G)), "TENSION2", batch_max=B)
    d_in = _device_points(*pts)
    w = single.plan_points_device(*d_in)
    g = multi.plan_points_device(*d_in)
    torch.cuda.synchronize()
    _assert_results(g, w)
    single.close()
    multi.close()
