"""The path-QP kernel away from its default parameters.

Every field of pqp_params reaches the kernel through make_dev_params. Here each named set below,
applied on top of the defaults, is solved by the kernel source and compared with the oracle:
  * on the CPU, the emulated FP64 instantiation (reserved bit 2, textbook and increment form)
    against the FP64 oracle iteration for iteration (status, iteration count, rho updates, rho, x),
    cold and warm; the emulated FP32 kernel through the parity check; the infeasible batch;
  * on the GPU (-m gpu), the FP64 and FP32 handles, both launches, and the FP64 escalation.
A guard first shows that each set changes something the kernel has to follow: the solution for a
formulation set, the iteration counts or the rho schedule for a settings set.

The `caps` sets end runs off the check grid. OSQP's osqp_solve runs the loop body's rho update on
the last iteration and only then the after-loop termination check, so the returned rho, and the
rho a warm re-solve starts from, include that update whatever the check decides.
"""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import oracle
from path_optimizer_2_b200 import abi, synthetic
from tests import parity

# the problem the kernel assembles
FORMULATION = {
    # another car: the reference's gflags (planning_flags.cpp:16-22,95)
    "vehicle": dict(front_length=4.6, rear_length=-1.2, wheel_base=2.9, max_steering_angle=math.radians(30.0),
                    expected_safety_margin=0.3),
    # weight_l > 0 makes P definite in l; the others are the reference's KP_* flag values
    "weights": dict(weight_l=0.5, weight_kappa=10.0, weight_dkappa=200.0, weight_slack=3.0),
    "end_box": dict(end_l_lb=-0.3, end_l_ub=0.2),
}
# how OSQP solves it
SETTINGS = {
    "osqp": dict(rho=1.0, sigma=1e-4, alpha=1.2, eps_abs=1e-3, eps_rel=1e-4, eps_prim_inf=1e-5,
                 adaptive_rho_tolerance=3.0),
    # checks and rho updates on different iterations: updates at 35, 105, ... come without a check
    "schedule": dict(check_termination=10, adaptive_rho_interval=35, max_iter=1000),
    "no_scaling": dict(scaling=0),
    "few_passes": dict(scaling=3, adaptive_rho=0),
    # caps off the check grid; in the last two the last iteration updates rho without a scheduled check
    "caps_37": dict(max_iter=37),
    "caps_1": dict(max_iter=1),
    # (at max_iter 300 most of these runs end at rounding-level residuals, see RESIDUAL_FLOOR)
    "caps_check0": dict(check_termination=0, max_iter=150),
    "caps_off_grid": dict(check_termination=20, max_iter=50),
}
SETS = dict(FORMULATION, **SETTINGS)
LAST_ITERATION_UPDATE = ("caps_check0", "caps_off_grid")

# feasible batches of config 3 at the sizes the FP64 tests run: n -> batch
BATCHES = {3: 6, 60: 4, 120: 3, 240: 2}
# FP64 kernel against the oracle, emulated (host double arithmetic without contraction): measured worst
# |x - x_oracle| 2.4e-10 and rho 1e-7 relative over every set, size and form below
X_TOL_EMU, RHO_TOL_EMU = 1e-8, 1e-5
# on the GPU (fused multiply-adds), the bars of test_gpu_parity.py
X_TOL_GPU, RHO_TOL_GPU = 1e-5, 2e-3
# A run without termination checks iterates on long after it has converged. Where its residual norms end
# below this floor, the rho estimates of its last updates are ratios of rounding noise (measured with check 0
# and max_iter 300: residuals 1e-11 .. 1e-16, rho 1 % .. 99 % apart, 4 updates against 2), so the rho
# schedule is not compared there
RESIDUAL_FLOOR = 1e-9
INFO_RHO, INFO_RHO_UPDATES = 2, 3  # PQP_INFO_* (include/pqp.h)


def params(name, **extra):
    kw = dict(SETS[name])
    kw.update(extra)
    return abi.default_params(**kw)


def batch(n, cfg=3):
    return synthetic.make_batch(cfg, BATCHES[n], n)


def oracle_run(p, hb, b, relinearise_about=None):
    """Cold oracle solve of instance b, then (if given) the warm re-solve about `relinearise_about`."""
    n = int(hb.n[b])
    s = oracle.OracleSolver(p, hb.knots[b], hb.inst[b], n)
    s.solve()
    if relinearise_about is not None:
        s.update(*relinearise_about[:3, :n])
        s.solve()
    return s


def assert_fp64_matches_oracle(p, hb, res, res2, x_tol, rho_tol, label):
    """The FP64 kernel's cold result `res` and its warm re-solve `res2` about res.sol against the oracle:
    status and iteration count equal; above RESIDUAL_FLOOR (at least once) the number of rho updates equal and
    rho within rho_tol relative; x within x_tol."""
    compared = 0
    for b in range(hb.batch):
        for run, r, about in (("cold", res, None), ("warm", res2, res.sol[b])):
            s = oracle_run(p, hb, b, about)
            tag = "%s %s inst %d" % (label, run, b)
            got = (int(r.status[b]), int(r.iters[b]))
            assert got == (s.status, s.iters), "%s: (status, iters) %s vs oracle %s" % (tag, got, (s.status, s.iters))
            if min(s.residuals) > RESIDUAL_FLOOR:
                assert int(r.info[b, INFO_RHO_UPDATES]) == s.rho_updates, "%s: %d rho updates vs oracle %d" % (
                    tag, r.info[b, INFO_RHO_UPDATES], s.rho_updates)
                drho = abs(r.info[b, INFO_RHO] - s.rho) / s.rho
                assert drho <= rho_tol, "%s: rho %g vs oracle %g" % (tag, r.info[b, INFO_RHO], s.rho)
                compared += 1
            if s.status in parity.INFEASIBLE:
                break  # diverging iterates; the warm re-solve about them is not compared
            dx = float(np.max(np.abs(r.x_full[b, :s.nv] - s.x())))
            assert dx < x_tol, "%s: |x - x_oracle| = %g" % (tag, dx)
    assert compared >= 1, label


# --------------------------------------------------------------------------- the sets bite (CPU, oracle only)
def _solutions(p, n):
    hb = batch(n)
    return [oracle_run(p, hb, b) for b in range(hb.batch)]


def _largest_move(p, q, sizes=(60, 120)):
    """max over the test batches of |x_p - x_q|_inf; inf where the statuses differ."""
    worst = 0.0
    for n in sizes:
        for a, c in zip(_solutions(p, n), _solutions(q, n)):
            if a.status != c.status:
                return math.inf
            if a.status == abi.PQP_SOLVED:
                worst = max(worst, float(np.max(np.abs(a.x() - c.x()))))
    return worst


@pytest.mark.parametrize("name", sorted(FORMULATION))
def test_formulation_set_moves_the_solution(name):
    """A kernel that ignored any one field of the set would miss the oracle by far more than the GPU's x bar."""
    base = abi.default_params()
    assert _largest_move(params(name), base) > 100 * X_TOL_GPU, name
    for field, value in FORMULATION[name].items():
        assert _largest_move(abi.default_params(**{field: value}), base) > 100 * X_TOL_GPU, field


@pytest.mark.parametrize("name", sorted(SETTINGS))
def test_settings_set_changes_the_iteration(name):
    """The iteration counts or the rho schedule differ from the defaults' on the test batches."""
    def schedule(p):
        return [(s.status, s.iters, s.rho_updates, round(s.rho, 9)) for n in BATCHES for s in _solutions(p, n)]
    assert schedule(params(name)) != schedule(abi.default_params()), name


@pytest.mark.parametrize("name", LAST_ITERATION_UPDATE)
def test_caps_update_rho_on_a_last_iteration_the_final_check_decides(name):
    """In these sets the final, unscheduled check decides SOLVED on some instance whose rho changes on
    that same last iteration (the run up to max_iter - 1 has fewer updates), above RESIDUAL_FLOOR."""
    p = params(name)
    q = params(name, max_iter=p.max_iter - 1)
    hits = 0
    for n in BATCHES:
        hb = batch(n)
        for b in range(hb.batch):
            s, t = oracle_run(p, hb, b), oracle_run(q, hb, b)
            if (s.status == abi.PQP_SOLVED and s.iters == p.max_iter and s.rho_updates > t.rho_updates and
                    min(s.residuals) > RESIDUAL_FLOOR):
                hits += 1
    assert hits >= 1, name


def test_batches_have_active_clearance_kappa_and_end_rows():
    """The clearance rows, a kappa row and the end-l row carry multipliers in the test batches, so the
    vehicle geometry, the safety margin, the curvature limit and the end box all reach the solution."""
    def active(p, rows):
        count = 0
        for n in (60, 120):
            hb = batch(n)
            for b in range(hb.batch):
                s = oracle_run(p, hb, b)
                y = s.y()
                count += int(np.sum(np.abs(y[rows(n)]) > 1e-6))
        return count
    for p in (abi.default_params(), params("vehicle"), params("end_box")):
        assert active(p, lambda n: slice(4 * n, 6 * n)) >= 10            # front and rear clearance rows
        assert active(p, lambda n: slice(6 * n, 6 * n + 1)) >= 1          # end l in [end_l_lb, end_l_ub]
    assert active(params("vehicle"), lambda n: slice(3 * n, 4 * n)) >= 1  # |kappa| <= tan(steer) / wheel_base


# --------------------------------------------------------------------------- emulated kernel (CPU)
@pytest.mark.parametrize("n", sorted(BATCHES))
@pytest.mark.parametrize("bits", [2, 2 | 32], ids=["fp64", "fp64-incr"])
@pytest.mark.parametrize("name", sorted(SETS))
def test_emulated_fp64_kernel_matches_oracle(name, bits, n):
    """The kernel source in double: the oracle's statuses, iteration counts, rho schedule and iterates,
    cold and in the warm re-solve about the kernel's own solution."""
    from tests.emu import emu
    p = params(name)
    hb = batch(n)
    es = emu.EmuSolver(params(name, reserved=bits), n, hb.batch)
    res = es.solve(hb)
    res2 = es.resolve(hb.with_linearisation(res.sol))
    assert_fp64_matches_oracle(p, hb, res, res2, X_TOL_EMU, RHO_TOL_EMU, "%s n=%d bits=%d" % (name, n, bits))


@pytest.mark.parametrize("n", [60, 120])
@pytest.mark.parametrize("form", [32, 64], ids=["incr", "textbook"])
@pytest.mark.parametrize("name", sorted(SETS))
def test_emulated_fp32_kernel_passes_parity(name, form, n):
    """The FP32 kernel source, both step forms: the oracle's status and OSQP's termination test at the
    set's own eps, the objective and solution envelopes, cold and warm."""
    from tests.emu import emu
    p = params(name)
    hb = synthetic.make_batch(3, 3, n)
    es = emu.EmuSolver(params(name, reserved=form), n, hb.batch)
    res = es.solve(hb)
    res2 = es.resolve(hb.with_linearisation(res.sol))
    label = "%s n=%d form=%d" % (name, n, form)
    for b in range(hb.batch):
        s = parity.oracle_reference(p, hb, b)
        assert s.status not in parity.INFEASIBLE, label
        parity.check_instance(p, hb, res, b, oracle_solver=s, label=label, strict_status=True)
        if res.status[b] == abi.PQP_SOLVED:
            s = parity.oracle_reference(p, hb, b, warm_from=res.sol[b][:3, :n])
            parity.check_instance(p, hb.with_linearisation(res.sol), res2, b, oracle_solver=s, label=label + " warm",
                                  strict_status=True)


@pytest.mark.parametrize("name", ["osqp", "schedule"] + sorted(FORMULATION))
def test_emulated_kernel_certifies_infeasibility(name):
    """Config 103 at n = 3 holds primal-infeasible instances. Without the FP64 escalation the FP64 kernel
    gives the oracle's statuses and iteration counts; the FP32 increment form its statuses, at most one check
    interval apart (measured: one interval later under osqp's 10x tighter eps_prim_inf, one earlier on a
    feasible instance under schedule, none elsewhere)."""
    from tests.emu import emu
    p = params(name)
    hb = synthetic.make_batch(103, 6, 3)
    exp = [(s.status, s.iters) for s in (oracle_run(p, hb, b) for b in range(6))]
    assert any(st == abi.PQP_PRIMAL_INFEASIBLE for st, _ in exp)
    r = emu.EmuSolver(params(name, reserved=4 | 2), 3, 6).solve(hb)
    assert list(zip(r.status.tolist(), r.iters.tolist())) == exp
    r = emu.EmuSolver(params(name, reserved=4 | 32), 3, 6).solve(hb)
    assert r.status.tolist() == [st for st, _ in exp]
    assert all(abs(int(i) - it) <= p.check_termination for i, (_, it) in zip(r.iters, exp)), (r.iters, exp)


# --------------------------------------------------------------------------- pqp_create's validation (CPU)
DOUBLE_FIELDS = [f for f, t in abi.PqpParams._fields_ if t is C.c_double]
REJECTED = [
    ("adaptive_rho=2", dict(adaptive_rho=2)),
    ("adaptive_rho=-1", dict(adaptive_rho=-1)),
    ("tolerance<1", dict(adaptive_rho_tolerance=0.999)),
    ("eps_prim_inf=0", dict(eps_prim_inf=0.0)),
    ("eps_prim_inf<0", dict(eps_prim_inf=-1e-4)),
    ("eps_dual_inf=0", dict(eps_dual_inf=0.0)),
    ("eps_abs=eps_rel=0", dict(eps_abs=0.0, eps_rel=0.0)),
    ("weight_l<0", dict(weight_l=-1e-3)),
    ("weight_kappa<0", dict(weight_kappa=-1.0)),
    ("weight_dkappa<0", dict(weight_dkappa=-1.0)),
    ("weight_slack<0", dict(weight_slack=-1.0)),
    ("steering=0", dict(max_steering_angle=0.0)),
    ("steering<0", dict(max_steering_angle=-0.1)),
    ("steering=pi/2", dict(max_steering_angle=math.pi / 2)),
    ("steering>pi/2", dict(max_steering_angle=2.0)),
] + [("%s=%s" % (f, v), {f: v}) for f in DOUBLE_FIELDS for v in (math.nan, math.inf, -math.inf)]
ACCEPTED = [(name, SETS[name]) for name in sorted(SETS)] + [
    ("defaults", {}),
    ("tolerance=1", dict(adaptive_rho_tolerance=1.0)),
    ("eps_abs=0", dict(eps_abs=0.0)),
    ("eps_rel=0", dict(eps_rel=0.0)),
    ("weights=0", dict(weight_kappa=0.0, weight_dkappa=0.0, weight_slack=0.0)),
    ("adaptive_rho=0", dict(adaptive_rho=0)),
]


def _create(kw):
    """pqp_create's return code for the defaults with `kw` (a created handle is destroyed)."""
    from path_optimizer_2_b200 import solver
    solver.build_library()
    L = solver.load_library()
    h = C.c_void_p()
    rc = L.pqp_create(C.byref(abi.default_params(**kw)), 20, 1, 0, C.byref(h))
    if rc == 0:
        L.pqp_destroy(h)
    return rc


@pytest.mark.parametrize("kw", [kw for _, kw in REJECTED], ids=[i for i, _ in REJECTED])
def test_create_refuses_what_osqp_refuses(kw):
    assert _create(kw) == abi.PQP_E_INVALID


@pytest.mark.parametrize("kw", [kw for _, kw in ACCEPTED], ids=[i for i, _ in ACCEPTED])
def test_create_accepts_the_sets(kw):
    """Not refused on the parameters: a handle where a device is present, PQP_E_NO_DEVICE where none is."""
    assert _create(kw) in (0, abi.PQP_E_NO_DEVICE)


# --------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SETS))
def test_gpu_fp64_handle_matches_oracle(name):
    """The FP64 instantiation on the device; n = 400 is C = 16 with the FP64 state in global memory."""
    from path_optimizer_2_b200 import solver
    p = params(name)
    for n, nb in ((3, 6), (60, 4), (240, 2), (400, 2)):
        hb = synthetic.make_batch(3, nb, n)
        sv = solver.PathQpSolver(params(name, reserved=2), n_max=n, batch_max=nb)
        res = sv.solve(hb, full=True)
        res2 = sv.resolve(hb.with_linearisation(res.sol), full=True)
        sv.close()
        assert_fp64_matches_oracle(p, hb, res, res2, X_TOL_GPU, RHO_TOL_GPU, "gpu %s n=%d" % (name, n))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SETS))
def test_gpu_default_handle_passes_parity(name):
    """The default FP32 handle (textbook form at n = 20, increment form above, persistent launch at 240)."""
    from path_optimizer_2_b200 import solver
    p = params(name)
    for n in (20, 120, 240):
        hb = synthetic.make_batch(3, 2, n)
        sv = solver.PathQpSolver(p, n_max=n, batch_max=hb.batch)
        res = sv.solve(hb, full=True)
        res2 = sv.resolve(hb.with_linearisation(res.sol), full=True)
        sv.close()
        label = "gpu fp32 %s n=%d" % (name, n)
        for b in range(hb.batch):
            s = parity.oracle_reference(p, hb, b)
            parity.check_instance(p, hb, res, b, oracle_solver=s, label=label, strict_status=True)
            if res.status[b] == abi.PQP_SOLVED:
                s = parity.oracle_reference(p, hb, b, warm_from=res.sol[b][:3, :n])
                parity.check_instance(p, hb.with_linearisation(res.sol), res2, b, oracle_solver=s,
                                      label=label + " warm", strict_status=True)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(FORMULATION["vehicle"], **FORMULATION["weights"]), SETTINGS["schedule"]],
                         ids=["vehicle+weights", "schedule"])
def test_gpu_persistent_launch_matches_per_instance_launch(kw):
    """As test_gpu_parity.py's test of the two launches, off the default parameters."""
    from path_optimizer_2_b200 import solver
    n = 240
    hb = synthetic.make_batch(3, 9, n)
    for form in (64, 32):
        res = {}
        for bits in (16, 8):
            sv = solver.PathQpSolver(abi.default_params(reserved=bits | form, **kw), n_max=n, batch_max=hb.batch)
            r1 = sv.solve(hb, full=True)
            r2 = sv.resolve(hb.with_linearisation(r1.sol), full=True)
            res[bits] = (r1, r2)
            sv.close()
        for a, b in zip(res[16], res[8]):
            assert np.array_equal(a.status, b.status) and np.array_equal(a.iters, b.iters), form
            assert np.allclose(a.x_full, b.x_full, atol=1e-5, rtol=0)
            assert np.allclose(a.y_full, b.y_full, atol=1e-3, rtol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SETS))
def test_gpu_infeasible_batch_escalates_to_the_oracle_status(name):
    """Config 103 at n = 3 through the host call, FP64 escalation on: the oracle's statuses."""
    from path_optimizer_2_b200 import solver
    p = params(name)
    hb = synthetic.make_batch(103, 6, 3)
    exp = np.array([oracle_run(p, hb, b).status for b in range(6)])
    sv = solver.PathQpSolver(p, n_max=3, batch_max=6)
    res = sv.solve(hb)
    sv.close()
    assert np.array_equal(res.status, exp), (res.status, exp)
