"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle."""
import numpy as np
import pytest

from path_optimizer_2_b200 import abi, synthetic
from tests import parity

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def solver_mod():
    from path_optimizer_2_b200 import solver
    return solver


def _run_and_check(solver_mod, hb, params, label, warm=True, check_all=True, max_check=16, strict=True):
    sv = solver_mod.PathQpSolver(params, n_max=hb.n_max, batch_max=hb.batch)
    res = sv.solve(hb, full=True)
    idx = range(hb.batch) if check_all else range(0, hb.batch, max(1, hb.batch // max_check))
    stats = []
    for b in idx:
        s = parity.oracle_reference(params, hb, b)
        stats.append(parity.check_instance(params, hb, res, b, oracle_solver=s, label=label, strict_status=strict))
    if warm:
        hb2 = hb.with_linearisation(res.sol)
        res2 = sv.resolve(hb2, full=True)
        for b in idx:
            s0 = parity.oracle_reference(params, hb, b)
            if s0.status != abi.PQP_SOLVED or res.status[b] != abi.PQP_SOLVED:
                continue
            # the oracle is re-linearised about the GPU's first-solve result (what the caller
            # passes back, path_optimizer.cpp:153) so both sides solve the same second QP
            s = parity.oracle_reference(params, hb, b, warm_from=res.sol[b][:3, :int(hb.n[b])])
            parity.check_instance(params, hb2, res2, b, oracle_solver=s, label=label + " warm")
    assert sv.launch_count >= 1
    sv.close()
    return stats


@pytest.mark.parametrize("n", [2, 3, 20, 31, 32, 63, 64, 120, 127, 128, 240, 255, 256, 400, 511])
def test_cold_and_warm_parity(solver_mod, n):
    hb = synthetic.make_batch(100 + n, 6, n)
    _run_and_check(solver_mod, hb, abi.default_params(), "n=%d" % n)


def test_ragged_batch(solver_mod):
    hb = synthetic.make_batch(7, 24, 120, ragged=True)
    assert len(set(hb.n.tolist())) > 4
    _run_and_check(solver_mod, hb, abi.default_params(), "ragged")


def test_rough_constraints(solver_mod):
    hb = synthetic.make_batch(8, 6, 90)
    hb.p = np.array([30, 60, 0, 90, 1, 89], dtype=np.int32)
    _run_and_check(solver_mod, hb, abi.default_params(), "rough")


def test_odd_n_max_uses_plain_loads(solver_mod):
    hb = synthetic.make_batch(9, 4, 121)  # 9*121*8 bytes is not a multiple of 16 -> no TMA
    _run_and_check(solver_mod, hb, abi.default_params(), "odd")


def test_max_iter_status(solver_mod):
    params = abi.default_params(max_iter=50)
    hb = synthetic.make_batch(3, 8, 240)
    _run_and_check(solver_mod, hb, params, "cap50", warm=False)


def test_envelope_against_high_accuracy(solver_mod):
    params = abi.default_params()
    hb = synthetic.make_batch(3, 6, 120)
    sv = solver_mod.PathQpSolver(params, n_max=120, batch_max=6)
    res = sv.solve(hb, full=True)
    for b in range(hb.batch):
        s = parity.oracle_reference(params, hb, b)
        parity.check_instance(params, hb, res, b, oracle_solver=s)
    sv.close()


def test_config3_sampled(solver_mod):
    """BASELINE config[2] (B=8192, n=240) at full size: every instance must report a status,
    solved instances are spot-checked against the oracle."""
    params = abi.default_params()
    hb = synthetic.make_batch(3, 8192, 240)
    sv = solver_mod.PathQpSolver(params, n_max=240, batch_max=8192)
    res = sv.solve(hb, full=True)
    assert np.all(res.status != abi.PQP_UNSOLVED)
    assert np.mean(res.status == abi.PQP_SOLVED) > 0.95
    for b in range(0, 8192, 512):
        s = parity.oracle_reference(params, hb, b)
        parity.check_instance(params, hb, res, b, oracle_solver=s, label="cfg3")
    sv.close()


def test_full_size_batch_properties(solver_mod):
    """BASELINE configs[2] at full size (8192 x 240, ragged n) through size-independent properties:
    the result of an instance does not depend on the batch around it - repeat runs, a permuted
    batch and small sub-batches are bit-identical (each QP is one warp's private, deterministic
    computation, whichever CTA picks it up) - and every solved instance's reported residuals pass
    the termination test; the warm re-solve about the solution itself stops at its first check."""
    params = abi.default_params()
    B, n = 8192, 240
    hb = synthetic.make_batch(3, B, n, ragged=True)
    sv = solver_mod.PathQpSolver(params, n_max=n, batch_max=B)
    a = sv.solve(hb)
    # idempotence: re-linearised about its own solution, a solved instance is solved again within
    # the first two checks of the warm run
    w = sv.resolve(hb.with_linearisation(a.sol))
    ok = a.status == abi.PQP_SOLVED
    assert np.mean(w.status[ok] == abi.PQP_SOLVED) > 0.99
    assert np.median(w.iters[ok]) <= 2 * params.check_termination
    b = sv.solve(hb)
    live = np.arange(n)[None, :] < hb.n[:, None]  # sol[b][:, i >= n[b]] is not written

    def same(x, y, idx=slice(None)):
        return (np.array_equal(x.status, y.status[idx]) and np.array_equal(x.iters, y.iters[idx]) and
                np.array_equal(x.cost, y.cost[idx]) and
                np.array_equal(np.where(live[idx][:, None, :], x.sol, 0.0), np.where(live[idx][:, None, :], y.sol[idx], 0.0)))

    assert same(b, a)
    perm = np.random.default_rng(0).permutation(B)
    hp = abi.HostBatch(hb.knots[perm], hb.inst[perm], hb.n[perm])
    c = sv.solve(hp)
    assert same(c, a, perm)
    sub = np.sort(perm[:24])
    sv_small = solver_mod.PathQpSolver(params, n_max=n, batch_max=len(sub))  # plain launch instead of the streamed one
    d = sv_small.solve(abi.HostBatch(hb.knots[sub], hb.inst[sub], hb.n[sub]))
    assert same(d, a, sub)
    sv_small.close()
    assert np.all(a.status != abi.PQP_UNSOLVED) and np.mean(a.status == abi.PQP_SOLVED) > 0.95
    assert np.all(a.iters[a.status == abi.PQP_SOLVED] % params.check_termination == 0)
    sv.close()


def test_frenet_to_cartesian(solver_mod):
    from oracle import oracle
    hb, ref = synthetic.make_batch(3, 4, 120, with_ref=True)
    sv = solver_mod.PathQpSolver(abi.default_params(), n_max=120, batch_max=4)
    res = sv.solve(hb)
    out = sv.frenet_to_cartesian(hb.n, ref, res.sol)
    for b in range(4):
        n = int(hb.n[b])
        exp = oracle.frenet_to_cartesian(ref[b][:, :n], res.sol[b, 0, :n], res.sol[b, 1, :n])
        assert np.allclose(out[b][:, :n], exp, atol=1e-12, rtol=0)
    sv.close()


def test_api_errors(solver_mod):
    params = abi.default_params()
    with pytest.raises(solver_mod.PqpError):
        solver_mod.PathQpSolver(params, n_max=1, batch_max=4)
    with pytest.raises(solver_mod.PqpError):
        solver_mod.PathQpSolver(params, n_max=512, batch_max=4)
    sv = solver_mod.PathQpSolver(params, n_max=60, batch_max=2)
    hb = synthetic.make_batch(3, 2, 60)
    with pytest.raises(solver_mod.PqpError):  # resolve before solve
        sv.resolve(hb)
    bad = synthetic.make_batch(3, 2, 60)
    bad.n[0] = 1
    with pytest.raises(solver_mod.PqpError):
        sv.solve(bad)
    with pytest.raises(solver_mod.PqpError):  # batch too large
        sv.solve(synthetic.make_batch(3, 3, 60))
    sv.solve(hb)
    sv.resolve(None, batch=2)  # relinearise about the device-resident solution
    sv.close()


def test_fp64_mode_reproduces_oracle_iterates(solver_mod):
    """params.reserved bit 1: the same kernel instantiated in double. Same algorithm, same
    schedule -> the oracle's iteration counts, rho and iterates are reproduced."""
    from oracle import oracle
    p32 = abi.default_params()
    p64 = abi.default_params(reserved=2)
    for n in (3, 60, 240, 400):  # 400: C = 16, FP64 state in global memory
        hb = synthetic.make_batch(100 + n if n == 3 else 3, 6 if n < 100 else 4, n)
        sv = solver_mod.PathQpSolver(p64, n_max=n, batch_max=hb.batch)
        res = sv.solve(hb, full=True)
        for b in range(hb.batch):
            s = oracle.OracleSolver(p32, hb.knots[b], hb.inst[b], n)
            st = s.solve()
            assert res.status[b] == st and res.iters[b] == s.iters
            # rho = rho_prev * sqrt(ratio of RESIDUAL norms): iterates that agree to 1e-8 give residual norms
            # (1e-3 .. 1e-5) that agree to 1e-5 .. 1e-3 relative
            assert abs(res.info[b, 2] - s.rho) <= 2e-3 * s.rho
            if st == abi.PQP_SOLVED:
                assert np.max(np.abs(res.x_full[b, :s.nv] - s.x())) < 1e-5
        sv.close()


def test_infeasible_instance_escalates_to_fp64(solver_mod):
    """FP32 cannot resolve OSQP's infeasibility certificate (DESIGN.md); the host API re-solves
    such instances with the FP64 instantiation and reports the reference's status."""
    from oracle import oracle
    hb = synthetic.make_batch(103, 6, 3)
    ref = [oracle.OracleSolver(abi.default_params(), hb.knots[b], hb.inst[b], 3) for b in range(6)]
    exp = np.array([s.solve() for s in ref])
    assert abi.PQP_PRIMAL_INFEASIBLE in exp
    sv = solver_mod.PathQpSolver(abi.default_params(), n_max=3, batch_max=6)
    res = sv.solve(hb)
    assert np.array_equal(res.status, exp)
    sv.close()
    sv = solver_mod.PathQpSolver(abi.default_params(reserved=4), n_max=3, batch_max=6)  # escalation off
    res = sv.solve(hb)
    bad = exp == abi.PQP_PRIMAL_INFEASIBLE
    # without the FP64 run the FP32 kernel reports the cap or a certificate (possibly the "inaccurate"
    # one taken at the cap): all of them are `false` for the caller (base_solver.cpp:88)
    assert np.all(np.isin(res.status[bad], parity.INFEASIBLE + (abi.PQP_MAX_ITER_REACHED,)))
    assert np.array_equal(res.status[~bad], exp[~bad])
    sv.close()


def test_receding_horizon_ticks(solver_mod):
    from oracle import oracle
    params = abi.default_params()
    n, ticks, batch = 120, 3, 4
    ext = synthetic.make_batch(5, batch, n + ticks)
    hb = abi.HostBatch(ext.knots[:, :, :n].copy(), ext.inst, np.full(batch, n, dtype=np.int32))
    sv = solver_mod.PathQpSolver(params, n_max=n, batch_max=batch)
    res = sv.solve(hb, full=True)
    ors = [oracle.OracleSolver(params, hb.knots[b], hb.inst[b], n) for b in range(batch)]
    for o in ors:
        o.solve()
    inst, sol = hb.inst, res.sol
    for t in range(1, ticks + 1):
        knots, inst = synthetic.shift_window(ext.knots, inst, sol, t, n)
        hbt = abi.HostBatch(knots, inst, hb.n)
        res = sv.resolve(hbt, full=True)
        sol = res.sol
        for b in range(batch):
            ors[b].update_full(knots[b], inst[b])
            ors[b].solve()
            ors[b].lin = None
            parity.check_instance(params, hbt, res, b, oracle_solver=ors[b], label="tick %d" % t)
    sv.close()


def test_advance_window_on_device_matches_host_bookkeeping(solver_mod):
    """pqp_advance_window_device (one launch) against synthetic.shift_window (numpy), and a
    device-resident receding-horizon loop against the host-API loop: bit-identical."""
    import torch
    params = abi.default_params(max_iter=50, reserved=4)  # no FP64 escalation: host and device paths run the same kernel
    n, ticks, batch = 120, 4, 6
    ext = synthetic.make_batch(5, batch, n + ticks)
    hb = abi.HostBatch(ext.knots[:, :, :n].copy(), ext.inst, np.full(batch, n, dtype=np.int32))
    sv_h = solver_mod.PathQpSolver(params, n_max=n, batch_max=batch)
    sv_d = solver_mod.PathQpSolver(params, n_max=n, batch_max=batch)
    res = sv_h.solve(hb)
    dev = torch.device("cuda", 0)
    d_ext = torch.from_numpy(ext.knots).to(dev)
    d_knots, d_inst = torch.from_numpy(hb.knots).to(dev), torch.from_numpy(hb.inst).to(dev)
    d_n = torch.from_numpy(hb.n).to(dev)
    d_sol = torch.zeros((batch, 4, n), dtype=torch.float64, device=dev)
    d_cost = torch.zeros(batch, dtype=torch.float64, device=dev)
    d_status, d_iters = (torch.zeros(batch, dtype=torch.int32, device=dev) for _ in range(2))
    bi = abi.PqpBatchIn(batch, n, d_knots.data_ptr(), d_inst.data_ptr(), d_n.data_ptr(), None)
    bo = abi.PqpBatchOut(d_sol.data_ptr(), d_cost.data_ptr(), d_status.data_ptr(), d_iters.data_ptr(), None, None, None, None)
    stream = torch.cuda.current_stream().cuda_stream
    sv_d.solve_device(bi, bo, stream=stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_sol.cpu().numpy(), res.sol)
    inst, sol = hb.inst, res.sol
    for t in range(1, ticks + 1):
        knots, inst = synthetic.shift_window(ext.knots, inst, sol, t, n)
        sv_d.advance_window_device(batch, n + ticks, t, d_ext.data_ptr(), d_sol.data_ptr(), d_knots.data_ptr(),
                                   d_inst.data_ptr(), stream=stream)
        torch.cuda.synchronize()
        assert np.array_equal(d_knots.cpu().numpy(), knots) and np.array_equal(d_inst.cpu().numpy(), inst)
        sol = sv_h.resolve(abi.HostBatch(knots, inst, hb.n)).sol
        sv_d.solve_device(bi, bo, stream=stream, warm=True)
        torch.cuda.synchronize()
        assert np.array_equal(d_sol.cpu().numpy(), sol)
    with pytest.raises(solver_mod.PqpError):  # window leaves the extended reference
        sv_d.advance_window_device(batch, n + ticks, ticks + 1, d_ext.data_ptr(), d_sol.data_ptr(), d_knots.data_ptr(),
                                   d_inst.data_ptr(), stream=stream)
    sv_h.close()
    sv_d.close()


@pytest.mark.parametrize("n", [60, 120, 240])
def test_increment_form_tracks_the_oracle_iteration_counts(solver_mod, n):
    """params.reserved bit 32 (the default for n_max >= 64): ADMM step in increment form (dx solve, row
    values A x carried). Same iteration in exact arithmetic; in FP32 its rounding error scales with
    |dx|, so the kernel follows the FP64 oracle's rho schedule: identical iteration count in >= 95 %
    of instances (the textbook form reaches 85 %), never further than 4 check intervals."""
    from oracle import oracle
    hb = synthetic.make_batch(3, 256, n)
    sv = solver_mod.PathQpSolver(abi.default_params(reserved=32), n_max=n, batch_max=hb.batch)
    g = sv.solve(hb, full=True)
    sv.close()
    o, _ = oracle.solve_batch(abi.default_params(), hb, nthreads=oracle.max_threads(), full=True)
    assert np.array_equal(g.status, o.status)
    ok = o.status == abi.PQP_SOLVED
    d = g.iters[ok].astype(np.int64) - o.iters[ok]
    assert (d == 0).mean() >= 0.95 and np.abs(d).max() <= 100, ((d == 0).mean(), np.abs(d).max())
    assert abs(g.iters[ok].mean() / o.iters[ok].mean() - 1.0) < 0.01
    for b in range(0, hb.batch, 37):
        s = parity.oracle_reference(abi.default_params(), hb, b)
        parity.check_instance(abi.default_params(), hb, g, b, oracle_solver=s, label="increment form n=%d" % n)


@pytest.mark.parametrize("n", [20, 120, 240, 400])
def test_persistent_launch_matches_per_instance_launch(solver_mod, n):
    """params.reserved bit 3 / bit 4: the same solver code launched persistently (one-warp CTAs that take
    instances from a work counter) or as one CTA per instance. Same arithmetic -> same answers.
    (Default: persistent for n_max >= 128, one CTA per instance below.)"""
    hb = synthetic.make_batch(3, 9, n)
    for form in (64, 32):  # textbook / increment form of the ADMM step, the same on both sides
        res = {}
        for bits in (16, 8):
            sv = solver_mod.PathQpSolver(abi.default_params(reserved=bits | form), n_max=n, batch_max=hb.batch)
            r1 = sv.solve(hb, full=True)
            r2 = sv.resolve(hb.with_linearisation(r1.sol), full=True)
            res[bits] = (r1, r2)
            sv.close()
        for a, b in zip(res[16], res[8]):
            assert np.array_equal(a.status, b.status) and np.array_equal(a.iters, b.iters), form
            assert np.allclose(a.x_full, b.x_full, atol=1e-5, rtol=0)
            assert np.allclose(a.y_full, b.y_full, atol=1e-3, rtol=1e-4)
    params = abi.default_params(reserved=8)
    for b in range(hb.batch):
        s = parity.oracle_reference(params, hb, b)
        parity.check_instance(params, hb, res[8][0], b, oracle_solver=s, label="persistent n=%d" % n)


def test_cold_only_handle_and_device_side_size_check(solver_mod):
    """Option bit 128 (no warm state kept): same answers as the default handle, resolve is refused.
    Device-pointer calls cannot validate n[] on the host: an out-of-range n is skipped by the kernel
    with PQP_NUMERICAL_ERROR and its neighbours are untouched."""
    import torch
    params = abi.default_params()
    hb = synthetic.make_batch(3, 12, 240)
    sv = solver_mod.PathQpSolver(params, n_max=240, batch_max=12)
    a = sv.solve(hb)
    sv.close()
    sc = solver_mod.PathQpSolver(abi.default_params(reserved=128), n_max=240, batch_max=12)
    c = sc.solve(hb)
    assert np.array_equal(a.status, c.status) and np.array_equal(a.iters, c.iters) and np.array_equal(a.sol, c.sol)
    with pytest.raises(solver_mod.PqpError):
        sc.resolve(hb.with_linearisation(c.sol))
    dev = torch.device("cuda", 0)
    n_bad = hb.n.copy()
    n_bad[3], n_bad[7] = 1, 241
    d_knots, d_inst, d_n = (torch.from_numpy(v).to(dev) for v in (hb.knots, hb.inst, n_bad))
    d_sol = torch.full((12, 4, 240), -7.0, dtype=torch.float64, device=dev)
    d_cost = torch.zeros(12, dtype=torch.float64, device=dev)
    d_status, d_iters = (torch.full((12,), -1, dtype=torch.int32, device=dev) for _ in range(2))
    bi = abi.PqpBatchIn(12, 240, d_knots.data_ptr(), d_inst.data_ptr(), d_n.data_ptr(), None)
    bo = abi.PqpBatchOut(d_sol.data_ptr(), d_cost.data_ptr(), d_status.data_ptr(), d_iters.data_ptr(), None, None, None, None)
    sc.solve_device(bi, bo, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    st, sol = d_status.cpu().numpy(), d_sol.cpu().numpy()
    assert st[3] == abi.PQP_NUMERICAL_ERROR and st[7] == abi.PQP_NUMERICAL_ERROR
    assert np.all(sol[3] == -7.0) and np.all(sol[7] == -7.0)
    good = [b for b in range(12) if b not in (3, 7)]
    assert np.array_equal(st[good], a.status[good]) and np.array_equal(sol[good], a.sol[good])
    sc.close()


def test_stage_times_of_a_single_path_call(solver_mod):
    """pqp_last_stage_ms: the reference's TimeRecorder stages (base_solver.cpp:57-93) for the B = 1 call."""
    hb = synthetic.make_batch(3, 1, 120)
    sv = solver_mod.PathQpSolver(abi.default_params(), n_max=120, batch_max=1)
    sv.solve(hb)
    ms = sv.last_stage_ms
    assert ms["h2d"] >= 0 and ms["kernel"] > 0 and ms["d2h"] >= 0
    assert abs(ms["h2d"] + ms["kernel"] + ms["d2h"] - ms["total"]) < 0.05 * ms["total"] + 1e-3
    sv.close()



def test_two_handles_driven_by_two_host_threads(solver_mod):
    """A handle is single-threaded, handles are independent: two host threads that each drive their own handle
    through the synchronous host-pointer call (how bench.py keeps two batches in flight end to end) get the
    answers of a lone call, bit for bit, whatever the interleaving of their launches and copies."""
    import threading
    params = abi.default_params(reserved=128)
    hb = synthetic.make_batch(3, 1500, 240)   # > 396 resident warps: the two persistent launches really share the SMs
    ref_sv = solver_mod.PathQpSolver(params, n_max=hb.n_max, batch_max=hb.batch)
    ref = ref_sv.solve(hb)
    ref_sv.close()
    svs = [solver_mod.PathQpSolver(params, n_max=hb.n_max, batch_max=hb.batch) for _ in range(2)]
    outs, errs = [[], []], []

    def worker(k):
        try:
            for _ in range(4):
                outs[k].append(svs[k].solve(hb))
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ths = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs
    for k in range(2):
        assert len(outs[k]) == 4
        for r in outs[k]:
            assert np.array_equal(r.status, ref.status) and np.array_equal(r.iters, ref.iters)
            assert np.array_equal(r.sol, ref.sol) and np.array_equal(r.cost, ref.cost)
        svs[k].close()
