"""Lifecycle of the six C-ABI handles (solver, bounds, DP, smoother, plan, multi-GPU).

On the CPU: every create argument check that runs before a device is looked up returns its code and leaves its
text in the ABI's last_error(NULL). On the GPU (`-m gpu`): the checks that run after the device lookup, and
create / use / destroy rounds that must not leak device memory, including creates that fail after they have
allocated."""
import ctypes as C

import numpy as np
import pytest

from path_optimizer_2_b200 import abi, bounds, dp, multi, plan, smoother, solver, synthetic

INVALID, NO_DEVICE = abi.PQP_E_INVALID, abi.PQP_E_NO_DEVICE


def _libs():
    """The library with every ABI declared, and each ABI's last_error."""
    L = bounds._declare(solver.load_library())
    dp._lib(), smoother._lib(), multi._lib(), plan._lib()
    return L


def _err(fn):
    return (fn(None) or b"").decode()


def _tiny_map():
    dist = np.ones((4, 4), dtype=np.float32)
    return dist, bounds.BoundsMap(4, 4, 0.1, 0.0, 0.0, dist.ctypes.data)


# (create call, expected code, expected last_error(NULL) or None where the check sets no text)
def _pre_device_cases(L):
    vp = C.c_void_p
    out = vp()
    p = abi.default_params()
    dist, m = _tiny_map()
    pp = plan.default_params()
    spacing = plan.default_params()
    spacing.output_spacing = 0.0
    method = plan.default_params()
    method.smoothing_method = 2
    sp = smoother.default_params()
    return dist, [
        ("solver out", lambda: L.pqp_create(C.byref(p), 120, 8, 0, None), INVALID, L.pqp_last_error, "out is null"),
        ("solver params", lambda: L.pqp_create(None, 120, 8, 0, C.byref(out)), INVALID, L.pqp_last_error, "invalid params"),
        ("solver n_max", lambda: L.pqp_create(C.byref(p), 512, 8, 0, C.byref(out)), INVALID, L.pqp_last_error,
         "n_max must be in [2, 511]"),
        ("solver batch_max", lambda: L.pqp_create(C.byref(p), 120, 0, 0, C.byref(out)), INVALID, L.pqp_last_error,
         "batch_max must be >= 1"),
        ("bounds out", lambda: L.pqp_bounds_create(C.byref(m), None, 0, None), INVALID, None, None),
        ("bounds map", lambda: L.pqp_bounds_create(None, None, 0, C.byref(out)), INVALID, L.pqp_bounds_last_error,
         "pqp_bounds_create: map needs rows, cols >= 2, resolution > 0 and a distance layer"),
        ("dp out", lambda: L.pqp_dp_create(None, None, 8, 1, None), INVALID, None, None),
        ("dp owner", lambda: L.pqp_dp_create(None, None, 8, 1, C.byref(out)), INVALID, L.pqp_dp_last_error,
         "pqp_dp_create: a pqp_bounds_handle (the map) is required"),
        ("smoother out", lambda: L.pqp_smoother_create(C.byref(sp), 64, 1, 0, None), INVALID, None, None),
        ("smoother p_max", lambda: L.pqp_smoother_create(C.byref(sp), 3, 1, 0, C.byref(out)), INVALID,
         L.pqp_smoother_last_error, "pqp_smoother_create: 4 <= p_max <= 2000, batch_max >= 1"),
        ("smoother batch_max", lambda: L.pqp_smoother_create(C.byref(sp), 64, 0, 0, C.byref(out)), INVALID,
         L.pqp_smoother_last_error, "pqp_smoother_create: 4 <= p_max <= 2000, batch_max >= 1"),
        ("plan out", lambda: L.pqp_plan_create(C.byref(m), C.byref(pp), 64, 64, 64, 120, 1, 0, None), INVALID, None, None),
        ("plan map", lambda: L.pqp_plan_create(None, C.byref(pp), 64, 64, 64, 120, 1, 0, C.byref(out)), INVALID,
         L.pqp_plan_last_error, "pqp_plan_create: a map is required"),
        ("plan dims", lambda: L.pqp_plan_create(C.byref(m), C.byref(pp), 64, 64, 3, 120, 1, 0, C.byref(out)), INVALID,
         L.pqp_plan_last_error,
         "pqp_plan_create: r_max >= 3, p_max >= 4, layers_max >= 4, 2 <= n_max <= 511, batch_max >= 1"),
        ("plan spacing", lambda: L.pqp_plan_create(C.byref(m), C.byref(spacing), 64, 64, 64, 120, 1, 0, C.byref(out)),
         INVALID, L.pqp_plan_last_error, "pqp_plan_create: output_spacing must be positive"),
        ("plan method", lambda: L.pqp_plan_create(C.byref(m), C.byref(method), 64, 64, 64, 120, 1, 0, C.byref(out)),
         INVALID, L.pqp_plan_last_error,
         "pqp_plan_create: smoothing_method must be PQP_PLAN_SMOOTH_TENSION2 (0) or PQP_PLAN_SMOOTH_TENSION (1)"),
        ("multi out", lambda: L.pqp_multi_create(C.byref(p), 120, 8, 1, None, None), INVALID, L.pqp_multi_last_error,
         "out is null"),
        ("multi params", lambda: L.pqp_multi_create(None, 120, 8, 1, None, C.byref(out)), INVALID,
         L.pqp_multi_last_error, "invalid arguments"),
        ("multi devices", lambda: L.pqp_multi_create(C.byref(p), 120, 8, 0, None, C.byref(out)), INVALID,
         L.pqp_multi_last_error, "invalid arguments"),
    ]


def test_create_checks_before_the_device_lookup():
    L = _libs()
    dist, cases = _pre_device_cases(L)
    for name, call, code, last_error, text in cases:
        assert call() == code, name
        if last_error is not None:
            assert _err(last_error) == text, name


# --------------------------------------------------------------------------- GPU
def _free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


# The driver hands out small allocations from 2 MiB pages, so free memory moves in 2 MiB steps even when nothing
# leaks; one page is the tolerance. Round 2 is the reference: the first rounds also load modules and grow pools.
PAGE = 2 << 20
ROUNDS = 20


def _rounds(one_round):
    free = []
    for _ in range(ROUNDS):
        one_round()
        free.append(_free_bytes())
    assert abs(free[-1] - free[1]) <= PAGE, "free device memory after round %d: %d B, after round 2: %d B" % (
        ROUNDS, free[-1], free[1])


@pytest.fixture(scope="module")
def scene():
    from path_optimizer_2_b200 import sharedmap
    dmap = sharedmap.DistanceMap()
    lines = sharedmap.make_lines(16, 120, dmap=dmap)
    return dmap, lines


@pytest.mark.gpu
def test_create_checks_after_the_device_lookup(scene):
    L = _libs()
    dmap, _ = scene
    out = C.c_void_p()
    p = abi.default_params()
    assert L.pqp_create(C.byref(p), 120, 8, 99, C.byref(out)) == NO_DEVICE
    assert _err(L.pqp_last_error) == "device index out of range"
    dist, m = _tiny_map()
    assert L.pqp_bounds_create(C.byref(m), None, 99, C.byref(out)) == NO_DEVICE
    assert _err(L.pqp_bounds_last_error) == "pqp_bounds_create: no CUDA device (there is no CPU fallback)"
    sp = smoother.default_params()
    assert L.pqp_smoother_create(C.byref(sp), 64, 1, 99, C.byref(out)) == NO_DEVICE
    assert _err(L.pqp_smoother_last_error) == "pqp_smoother_create: no CUDA device (there is no CPU fallback)"
    sp.rho = 0.0
    assert L.pqp_smoother_create(C.byref(sp), 64, 1, 0, C.byref(out)) == INVALID
    assert _err(L.pqp_smoother_last_error) == "pqp_smoother_create: invalid OSQP settings"
    assert L.pqp_multi_create(C.byref(p), 120, 8, 99, None, C.byref(out)) == NO_DEVICE
    assert _err(L.pqp_multi_last_error) == "fewer CUDA devices than n_devices (there is no CPU fallback)"
    # the DP takes its device from a live bounds handle
    pbn = bounds.PathBounds(dmap.dist, dmap.res)
    dpp = dp.DpParams()
    L.pqp_dp_default_params(C.byref(dpp))
    assert L.pqp_dp_create(pbn.h, C.byref(dpp), 1, 1, C.byref(out)) == INVALID
    assert _err(L.pqp_dp_last_error) == "pqp_dp_create: layers_max >= 2, batch_max >= 1"
    dpp.lateral_spacing = 0.0
    assert L.pqp_dp_create(pbn.h, C.byref(dpp), 8, 1, C.byref(out)) == INVALID
    assert _err(L.pqp_dp_last_error) == "pqp_dp_create: spacings and range must be positive"
    dpp.lateral_spacing = 0.25
    assert L.pqp_dp_create(pbn.h, C.byref(dpp), 8, 1, C.byref(out)) == INVALID
    assert _err(L.pqp_dp_last_error) == "pqp_dp_create: more than 64 lateral samples per layer"
    pbn.close()
    # a plan reports a stage's create error under its own name
    pp = plan.default_params("TENSION")
    with pytest.raises(solver.PqpError) as e:
        plan.Planner(dmap.dist, dmap.res, r_max=64, p_max=900, layers_max=64, n_max=120, batch_max=2, params=pp)
    assert e.value.code == INVALID
    assert ("pqp_plan_create: smoothing_method TENSION: pqp_cartesian_tension_smooth: p_max = 900 too large for the "
            "Cartesian QP's shared-memory band") in str(e.value)


@pytest.mark.gpu
def test_solver_rounds_do_not_leak():
    params = abi.default_params()
    hb = synthetic.make_batch(3, 256, 120)
    infeasible = synthetic.make_batch(103, 6, 3)  # instances the FP32 kernel hands to the FP64 escalation

    def one_round():
        sv = solver.PathQpSolver(params, n_max=120, batch_max=256)
        res = sv.solve(hb, full=True)  # x_full, y_full, z_full are allocated on first use
        ref = np.zeros((hb.batch, 3, hb.n_max))
        sv.frenet_to_cartesian(hb.n, ref, res.sol)  # so is the host call's staging
        sv.close()
        small = solver.PathQpSolver(params, n_max=3, batch_max=6)
        small.solve(infeasible, full=True)
        small.close()

    _rounds(one_round)


@pytest.mark.gpu
def test_bounds_and_dp_rounds_do_not_leak(scene):
    dmap, lines = scene
    B = lines.batch
    max_s = np.array([lines.spline_rows(b)[0, lines.k[b] - 1] for b in range(B)])
    length = max_s + 3.0
    start = np.array([lines.spline_rows(b)[[4, 8], 0].tolist() + [0.0] for b in range(B)])

    def one_round():
        pbn = bounds.PathBounds(dmap.dist, dmap.res)
        pbn.compute(lines.states, lines.n, lines.spline, lines.k)  # staging grows on demand
        pbn.build_states(lines.spline, lines.k, max_s, 120)
        ds = dp.DpSearch(pbn, layers_max=64, batch_max=B)
        ds.search(lines.spline, lines.k, length, start)
        ds.close()
        pbn.close()

    _rounds(one_round)


@pytest.mark.gpu
def test_smoother_rounds_do_not_leak():
    from tests.test_smoother import corridor, raw_reference
    cases = [raw_reference(100 + b, 20 + 3 * b) for b in range(8)]
    cors = [corridor(200 + b, 10 + 4 * b) for b in range(8)]
    clear = [np.full(len(c[0]), 5.0) for c in cases]

    def one_round():
        sm = smoother.Smoother(p_max=64, batch_max=8)
        sm.tension(*[[c[i] for c in cases] for i in range(5)], full=True)
        sm.post(*[[c[i] for c in cors] for i in range(4)], full=True)
        sm.cartesian_tension(*[[c[i] for c in cases] for i in range(3)], clear, full=True)
        sm.close()

    _rounds(one_round)


@pytest.mark.gpu
def test_plan_and_multi_rounds_do_not_leak(scene):
    from path_optimizer_2_b200 import sharedmap
    dmap, _ = scene
    raw_x, raw_y, start, target = sharedmap.make_plan_inputs(4, dmap=dmap)
    hb = synthetic.make_batch(3, 64, 120)

    def one_round():
        pl = plan.Planner(dmap.dist, dmap.res, r_max=64, p_max=64, layers_max=64, n_max=255, batch_max=4,
                          params=plan.default_params("TENSION"))
        pl.plan(raw_x, raw_y, start, target, trace=True)
        pl.close()
        mg = multi.MultiGpuSolver(n_max=120, batch_max=64, n_devices=1)
        mg.solve(hb, full=True)
        mg.close()

    _rounds(one_round)


@pytest.mark.gpu
def test_failed_plan_creates_leave_nothing_behind(scene):
    """Both fail after they have allocated: TENSION at a p_max beyond the Cartesian band once the bounds, DP and
    smoother handles exist; a lattice of more than 64 lateral samples once the bounds handle has copied the map."""
    dmap, _ = scene
    tension = plan.default_params("TENSION")
    lattice = plan.default_params()
    lattice.dp.lateral_spacing = 0.25

    def one_round():
        for params, p_max in ((tension, 900), (lattice, 64)):
            with pytest.raises(solver.PqpError) as e:
                plan.Planner(dmap.dist, dmap.res, r_max=64, p_max=p_max, layers_max=64, n_max=120, batch_max=64,
                             params=params)
            assert e.value.code == INVALID

    _rounds(one_round)
