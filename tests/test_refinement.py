"""Robots beyond the conditioning limit of the sweep inversion: the opt-in refinement class (hmpc_set_refinement,
hmpc_reference_set_refinement, BatchedMPC.set_refinement, interface.reference_set_refinement).

CPU: the kernel source (tests/host_emul/kernel_source_on_host.cpp: the device-resident chain with the refinement class at its end)
against the fp64 referee — the lying robot of stress_referee.npz, a generated batch of fallen and tilted robots spanning
scaled condition numbers of up to 1.6e6 (single and double support, horizons 8 and 10), well-conditioned robots untouched
bit for bit, a non-positive pivot not handed over, and a ThreadSanitizer run.  GPU: the same through the library — the
device-resident calls, all three host-buffer modes, the reference boundary, the rollout and a captured graph."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, load_golden, rel_err
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import _p, emul_solve, host_emulation, race_driver

N = 10
KAPPA_REFINE, KAPPA_MAX, KAPPA_MAX_REFINED = 1.5e4, 1.5e5, 1e9   # hmpc_capi.cu's defaults


def _lying():
    g = np.load(os.path.join(GOLDEN, "stress_referee.npz"))
    recs = np.ascontiguousarray(g["h10_lying_records"]).view(scenarios.UPDATE_DTYPE).reshape(-1)
    return recs, g["h10_lying_referee"]


def _lying_inputs():
    """the boundary inputs behind h10_lying: record 34 of scenarios.make_stress_batch(40, 10, 8.0, 15)"""
    rng = np.random.default_rng(15)
    for _ in range(35):
        b = scenarios._stress_state(rng, N, 8.0)
    assert scenarios.to_record(b, N).tobytes() == _lying()[0][0].tobytes()
    return b


def _no_pivot_record():
    """a record whose Hessian has a zero pivot: no state weights and no input regularisation (H = 0)"""
    b = scenarios.stand_inputs(N)
    b["weights"][:] = 0.0
    b["Alpha_K"][:] = 0.0
    return scenarios.to_record(b, N)


def _referee(recs, horizon):
    """fp64 referee answers (oracle/qp_dual_active_set.py, tol 1e-12) and scaled condition numbers of the reduced QPs"""
    from oracle import oracle_py as O
    from oracle import qp_dual_active_set as G

    setup = O.make_setup(horizon)
    ref = np.zeros((len(recs), 12 * horizon))
    kap = np.zeros(len(recs))
    for k, r in enumerate(recs):
        Q = O.reduced_qp(r, setup)
        Hs = np.tril(Q["H"]) + np.tril(Q["H"], -1).T
        kap[k] = (np.diag(Hs) * np.diag(np.linalg.inv(Hs))).max()
        x, inf = G.solve(Q["H"], Q["g"], Q["A"], Q["lb"], Q["ub"], tol=1e-12, max_iter=5000)
        assert inf["status"] == 0
        ref[k, Q["var_ind"]] = x
    return ref, kap


# ---- CPU: the kernel source on the host ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul():
    return host_emulation()


def _emul_solve(L, recs, horizon, refine, ws=None, warm=0):
    """the device-resident chain on the host -> (wrench f64 [B,12N] (the kernel's double stores), status, ws, launched[4])"""
    B = len(recs)
    packed = np.ascontiguousarray(interface.pack_records(recs, horizon))
    w64 = np.zeros((B, 12 * horizon))
    ws = np.zeros((B, L.emul_ws_ints()), np.int32) if ws is None else ws
    w, st, la = emul_solve(L, horizon, packed, refine=refine, ws=ws, warm=warm, w64=w64)   # the library's default kappas
    assert np.array_equal(w64.astype(np.float32).view(np.uint32), w.view(np.uint32))
    return w64, st, ws, la


def test_refinement_source_solves_a_robot_lying_on_its_side(emul):
    """h10_lying (scaled condition number 2.9e5): code 4 without refinement, exactly as the kernel reports it today; with
    refinement the class solves it to within 2e-5 of the referee (first step) and 1e-5 (whole horizon), refined bit set."""
    recs, ref = _lying()
    w, st, ws, la = _emul_solve(emul, recs, N, False)
    assert interface.status_code(st).tolist() == [4] and interface.status_refined(st).tolist() == [0]
    assert la.tolist() == [1, 0, 0, 0]
    w, st, ws, la = _emul_solve(emul, recs, N, True)
    assert la.tolist() == [1, 0, 0, 1]
    assert interface.status_code(st).tolist() == [0] and interface.status_refined(st).tolist() == [1], hex(st[0])
    assert rel_err(w, ref, 12)[0] < 2e-5 and rel_err(w, ref)[0] < 1e-5, (rel_err(w, ref, 12), rel_err(w, ref))
    assert ws[0, 0] == 0   # the next warm call starts cold


@pytest.mark.parametrize("horizon,scale,seed,B", [(10, 24.0, 42, 24), (10, 16.0, 41, 24), (8, 16.0, 43, 24)])
def test_refinement_source_on_fallen_and_tilted_robots(emul, horizon, scale, seed, B):
    """Generated fallen / tilted robots (scenarios.make_stress_batch) under walking, standing and random contact tables:
    every handed-over instance is within 5e-5 of the referee (first step) or reports code 4, and no instance with a clean
    status is further off.  (An instance below the threshold keeps whatever the size classes return, e.g. code 3.)  Between them the batches hold 16 robots above the hand-over threshold, up to 1.6e6."""
    recs = scenarios.make_stress_batch(B, horizon, scale, seed)
    ref, kap = _referee(recs, horizon)
    w, st, _, la = _emul_solve(emul, recs, horizon, True)
    code = interface.status_code(st)
    e = rel_err(w, ref, 12)
    ok = code == 0
    assert (e[ok] < 5e-5).all(), (e[ok].max(), kap[ok][np.argmax(e[ok])])
    handed = kap > KAPPA_REFINE
    assert ((code == 0) | (code == 4) | ~handed).all(), code
    assert (interface.status_refined(st)[handed & ok] == 1).all()
    assert (interface.status_refined(st)[~handed] == 0).all()
    print("horizon %d x%g: %d records, kappa %.1e ... %.1e, %d above %.1e: %d refined, %d code 4; worst clean error %.1e" %
          (horizon, scale, B, kap.min(), kap.max(), handed.sum(), KAPPA_REFINE, int((handed & ok).sum()), int((code == 4).sum()),
           e[ok].max()))
    assert kap.max() > 1e5 and (handed & ok).sum() >= 1


def test_refinement_source_leaves_well_conditioned_robots_alone(emul):
    """A mixed batch (walking and standing robots of cfg3_h10 and the lying robot): with refinement on, every robot that is
    not handed over gets the results, status words and recorded working sets of refinement off, bit for bit."""
    g = load_golden("cfg3_h10")
    lying, _ = _lying()
    recs = np.concatenate([g["records"][:5], lying, g["records"][5:8]])
    w0, st0, ws0, la0 = _emul_solve(emul, recs, N, False)
    w1, st1, ws1, la1 = _emul_solve(emul, recs, N, True)
    keep = np.arange(len(recs)) != 5
    assert np.array_equal(w0[keep].view(np.uint64), w1[keep].view(np.uint64))
    assert np.array_equal(st0[keep], st1[keep]) and np.array_equal(ws0[keep], ws1[keep])
    assert la1[3] == 1 and interface.status_refined(st1).tolist() == [0] * 5 + [1] + [0] * 3
    # a warm call proposes the recorded sets; the handed-over robot (empty set) gets the cold refined result again
    w2, st2, ws2, _ = _emul_solve(emul, recs, N, True, ws=ws1.copy(), warm=1)
    assert np.array_equal(w2[5].view(np.uint64), w1[5].view(np.uint64)) and st2[5] == st1[5]


def test_refinement_source_does_not_hand_over_a_non_positive_pivot(emul):
    """A Hessian with a non-positive pivot is not a conditioning problem: it stays code 4 with refinement on, and the
    refinement class never sees it."""
    rec = np.array([_no_pivot_record()])
    _, st0, _, _ = _emul_solve(emul, rec, N, False)
    _, st1, _, la = _emul_solve(emul, rec, N, True)
    assert interface.status_code(st0).tolist() == [4] and np.array_equal(st0, st1) and la[3] == 0


def _rollout_robots():
    """the GPU rollout test's robots: walkers, the lying robot standing (2) and walking (6)"""
    b = _lying_inputs()
    _, inputs = scenarios.make_batch(5, 8, horizon=N, seed=3)
    inputs[2] = inputs[6] = b
    return scenarios.make_rollout(inputs, N, standing=[False, False, True, False, False, False, False, False])


def test_refinement_source_rollout_start_of_lying_robots(emul):
    """The first records the device rollout prepares for the robots started lying down: both are code 4 without
    refinement.  With it the walking one is refined; the standing one (double support, 100 active rows) is handed over but
    its refinement is rejected, so it keeps code 4 (the GPU rollout test counts the same)."""
    states, loop = _rollout_robots()
    packed = np.zeros((8, interface.record_bytes(N)), np.uint8)
    emul.emul_prepare(_p(np.ascontiguousarray(states)), 8, N, ctypes.c_double(0.04), _p(packed))
    recs = interface.unpack_records(packed, N)[[2, 6]]
    _, st0, _, _ = _emul_solve(emul, recs, N, False)
    _, st1, _, la = _emul_solve(emul, recs, N, True)
    assert interface.status_code(st0).tolist() == [4, 4] and la[3] == 2
    assert interface.status_code(st1).tolist() == [4, 0] and interface.status_refined(st1).tolist() == [0, 1], st1


def test_refinement_source_has_no_data_races(emul, tmp_path):
    """ThreadSanitizer build of the driver (every CUDA thread an OS thread, every barrier real) on h10_lying with
    refinement on: class 0 hands it over, the refinement class solves it."""
    exe = race_driver()
    recs, _ = _lying()
    f = tmp_path / "lying.bin"
    np.ascontiguousarray(interface.pack_records(recs, N)).tofile(f)
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66")
    r = subprocess.run([exe, str(f), str(N), "refine"], capture_output=True, text=True, env=env, timeout=1800)
    assert "ThreadSanitizer" not in r.stderr, r.stderr[:3000]
    assert r.returncode == 0 and "launched 1 0 0 1" in r.stdout, (r.returncode, r.stdout)
    st = int(r.stdout.split("status")[1].split()[0], 16)
    assert st & 0xff == 0 and (st >> 28) & 1 == 1


# ---- GPU: the library -----------------------------------------------------------------------------------------------------
def _mixed_batch():
    """cfg3 walkers and standing robots with the lying robot at four places, and one zero-pivot record"""
    g = load_golden("cfg3_h10")
    lying, ref = _lying()
    recs = g["records"][:60].copy()
    at = [3, 17, 40, 58]
    recs[at] = lying[0]
    recs[25] = _no_pivot_record()
    return recs, at, ref[0]


def _device_solve(mpc, recs, call="solve", shift=None):
    import torch

    B = len(recs)
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    w = torch.full((B, 12 * N), float("nan"), dtype=torch.float32, device="cuda")
    s = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    tau = torch.zeros((B, 10), dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    L = interface.lib()
    if call == "solve":
        interface._check(L.hmpc_solve_device(mpc._h, d_rec.data_ptr(), B, w.data_ptr(), s.data_ptr(), ctypes.c_void_p(st)))
    elif call == "ex":
        interface._check(L.hmpc_solve_device_ex(mpc._h, d_rec.data_ptr(), B, w.data_ptr(), s.data_ptr(), tau.data_ptr(),
                                                ctypes.c_void_p(st)))
    else:
        mpc.solve_device_warm(d_rec, B, w, s, d_tau=tau, d_shift=shift)
    torch.cuda.synchronize()
    return w.cpu().numpy(), s.cpu().numpy(), tau.cpu().numpy()


@pytest.mark.gpu
def test_device_calls_with_refinement():
    """hmpc_solve_device, _ex and _warm: the lying robots come back solved and refined, within 2e-5 of the referee; every
    other robot, the zero-pivot one included, equals refinement off bit for bit; a warm call on a handed-over robot
    reproduces the cold refined result."""
    recs, at, ref = _mixed_batch()
    B = len(recs)
    off, on = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    on.set_refinement(True)
    assert off.launches_per_solve == 3 and on.launches_per_solve == 4
    cfg = on.class_config(interface.REFINEMENT_CLASS)
    assert cfg["nb_cap"] == 2 * N and cfg["smem_bytes"] <= 227 * 1024
    others = np.setdiff1d(np.arange(B), at)
    for call in ("solve", "ex"):
        w0, s0, t0 = _device_solve(off, recs, call)
        w1, s1, t1 = _device_solve(on, recs, call)
        assert (interface.status_code(s0[at]) == 4).all()
        assert (interface.status_code(s1[at]) == 0).all() and (interface.status_refined(s1[at]) == 1).all(), s1[at]
        assert rel_err(w1[at], np.tile(ref, (len(at), 1)), 12).max() < 2e-5
        assert np.array_equal(w0[others].view(np.uint32), w1[others].view(np.uint32)) and np.array_equal(s0[others], s1[others])
        assert np.array_equal(t0[others].view(np.uint32), t1[others].view(np.uint32))
        assert interface.status_code(s1[25]) == 4 and interface.status_refined(s1[25]) == 0
    cold_w, cold_s, _ = _device_solve(on, recs, "ex")
    on.reset_warm_start()
    _device_solve(on, recs, "warm")                           # records the sets
    ww, ws_, _ = _device_solve(on, recs, "warm", shift=None)  # proposes them (shift 1 on the same records: a real proposal)
    assert (interface.status_code(ws_[at]) == 0).all()
    assert np.array_equal(ww[at].view(np.uint32), cold_w[at].view(np.uint32)) and np.array_equal(ws_[at], cold_s[at])
    off.close()
    on.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["zero_copy", "staged", "in_place", "states"])
def test_host_buffer_modes_equal_the_device_path(mode):
    """hmpc_solve_batch(_ex / _warm / _states) with refinement on: the chunk's handed-over robots are re-solved in the
    refinement class, so every host mode returns the device path's wrenches and status words."""
    recs, at, _ = _mixed_batch()
    if mode == "staged":                      # above 1536 robots the host path stages through device memory
        recs = np.concatenate([recs] * 30)
    B = len(recs)
    mpc, dev = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    mpc.set_refinement(True)
    dev.set_refinement(True)
    if mode == "states":
        b = _lying_inputs()
        _, inputs = scenarios.make_batch(3, 24, horizon=N, seed=4)
        inputs[5] = inputs[11] = b
        states = scenarios.make_states(inputs, N)
        w, s = mpc.solve_batch_states(states, strict=False)
        import torch

        d_states = torch.from_numpy(states.view(np.uint8).reshape(len(states), -1).copy()).cuda()
        d_rec = torch.zeros((len(states), interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
        dev.prepare_device(d_states, len(states), d_rec)
        torch.cuda.synchronize()
        recs = interface.unpack_records(d_rec.cpu().numpy(), N)
        at = [5, 11]
    elif mode == "in_place":
        rin = interface.page_aligned((B,), scenarios.UPDATE_DTYPE)
        rin[:] = recs
        w = interface.page_aligned((B, 12 * N), np.float64)
        s = interface.page_aligned((B,), np.int32)
        mpc.pin(rin, w, s)
        mpc.solve_batch(rin, strict=False, out=(w, s))
        w, s = w.copy(), s.copy()
    else:
        w, s = mpc.solve_batch(recs, strict=False)
    wd, sd, _ = _device_solve(dev, recs, "solve")
    assert (interface.status_refined(sd[at]) == 1).all()
    assert np.array_equal(s, sd)
    if mode == "in_place":   # the in-place mode stores the double results of the solve
        assert np.array_equal(w.astype(np.float32).view(np.uint32), wd.view(np.uint32))
    else:                    # (the zero-pivot robot's wrench is NaN: compared as bit patterns)
        assert np.array_equal(w.astype(np.float32).view(np.uint32), wd.view(np.uint32))
    # the warm host call on the same records: the refined robots again
    if mode in ("zero_copy", "staged"):
        w2, s2 = mpc.solve_batch_warm(recs, strict=False)
        assert (interface.status_refined(s2[at]) == 1).all() and np.array_equal(w2[at], wd[at].astype(np.float64))
    mpc.close()
    dev.close()


@pytest.mark.gpu
def test_reference_boundary_with_refinement():
    """update_problem_data on the lying robot: 'failed to solve!' without refinement; after
    hmpc_reference_set_refinement(1) a wrench within 2e-5 of the referee and hmpc_reference_last_rc() == HMPC_OK."""
    b = _lying_inputs()
    _, ref = _lying()

    def tick():
        interface.setup_problem(0.04, N, 0.25, 500.0)
        interface.update_problem_data(b["p"], b["v"], b["q"], b["w"], b["r"], b["joint_angles"], b["yaw"], b["weights"],
                                      b["state_trajectory"], b["Alpha_K"], b["gait"])
        return np.array([interface.get_solution(i) for i in range(12 * N)])

    interface.reference_set_refinement(False)
    tick()
    assert interface.reference_last_rc() == interface.HMPC_ERR_NOT_CONVERGED
    assert interface.status_code(interface.reference_last_status()) == 4
    interface.reference_set_refinement(True)
    try:
        w = tick()
        assert interface.reference_last_rc() == interface.HMPC_OK
        st = interface.reference_last_status()
        assert interface.status_code(st) == 0 and interface.status_refined(st) == 1
        assert rel_err(w[None], ref, 12)[0] < 2e-5
    finally:
        interface.reference_set_refinement(False)


@pytest.mark.gpu
def test_rollout_of_robots_started_lying_down():
    """hmpc_rollout_device with walkers and robots started lying down (one walking, one standing): without refinement the
    lying robots' ticks count as failures.  With it the walking one never fails, and neither does any walker.  The standing
    one is not covered: the refinement class's KKT check rejects 2 of its 4 ticks (code 4), where refinement off fails 1
    and answers the other unverified (its scaled condition number lies between the hand-over threshold and 1.5e5)."""
    import torch

    from test_rollout import _to_dev

    states, loop = _rollout_robots()
    T = 4
    fails = {}
    for on in (False, True):
        mpc = interface.BatchedMPC(8, N)
        mpc.set_refinement(on)
        d_s, d_l = _to_dev(states), _to_dev(loop)
        mpc.rollout_device(d_s, d_l, 8, T)
        torch.cuda.synchronize()
        lo = d_l.cpu().numpy().view(scenarios.ROLLOUT_DTYPE).reshape(-1)
        assert (lo["ticks"] == T).all()
        fails[on] = lo["failures"].copy()
        mpc.close()
    assert fails[False][[2, 6]].min() > 0
    assert fails[True][6] == 0 and (np.delete(fails[True], 2) == 0).all(), fails[True]
    print("failures of the standing lying robot: refinement off %d, on %d" % (fails[False][2], fails[True][2]))


@pytest.mark.gpu
def test_captured_graph_with_refinement_replays_eager_calls():
    """hmpc_solve_device_ex captured with refinement on and replayed 5 times against eager calls on a second context, bit
    for bit, with handed-over robots in the batch: the capture's memset clears the refinement list length too, so no
    replay solves a stale list."""
    import torch

    from test_graph_capture import _outputs, _same, _solve_ex

    recs, at, _ = _mixed_batch()
    B = len(recs)
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    a.set_refinement(True)
    b.set_refinement(True)
    rng = np.random.default_rng(5)
    sets = []
    for _ in range(5):
        r = recs.copy()
        r[rng.choice(B, 3, replace=False)] = _lying()[0][0]
        sets.append(torch.from_numpy(interface.pack_records(r, N)).cuda())
    rec = sets[0].clone()
    w, tau, s = _outputs(B)
    _solve_ex(a, rec, B, w, tau, s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _solve_ex(a, rec, B, w, tau, s)
    wr, taur, sr = _outputs(B)
    for k, d in enumerate(sets):
        rec.copy_(d)
        for t in (w, tau):
            t.fill_(float("nan"))
        s.fill_(-1)
        g.replay()
        _solve_ex(b, d, B, wr, taur, sr)
        torch.cuda.synchronize()
        assert _same(w, wr) and _same(tau, taur) and _same(s, sr), k
        assert interface.status_refined(s.cpu().numpy()).sum() >= 4, k
    a.close()
    b.close()
