"""Warm start in the caller's own loop: hmpc_solve_device_warm, hmpc_solve_batch_warm and the reference boundary after
hmpc_reference_set_warm_start(1).

CPU: the kernel source (tests/host_emul/warm_start_on_host.cpp) with per-robot shifts — a negative shift is a cold solve
that still records its working set, mixed shifts in one batch equal per-robot runs, an instance that overflows class 0
reaches class 1 with its proposal, and horizon 16 (no block start) is unaffected.  GPU: the calls against the device
rollout they generalise, against cold solves of the same records, against each other (device / host-buffer modes /
reference boundary), and with robots reset mid-loop."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, load_golden, rel_err
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import BUILD, DEVICE_HEADER, HERE, _host_buildable, _p


@pytest.fixture(scope="module")
def emul():
    """tests/host_emul/warm_start_on_host.cpp (the kernel-source driver plus the per-robot-shift solve), built for the host
    the way test_kernel_source_on_host.py builds its driver."""
    os.makedirs(BUILD, exist_ok=True)
    hdr = os.path.join(BUILD, "hmpc_device_host_warm.cuh")
    with open(hdr, "w") as f:
        f.write(_host_buildable(open(DEVICE_HEADER).read()))
    lib = os.path.join(BUILD, "libwarm_start_on_host.so")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-pthread",
           "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(os.path.dirname(os.path.dirname(HERE)), "include"),
           '-DHMPC_DEVICE_HEADER="%s"' % hdr, os.path.join(HERE, "warm_start_on_host.cpp"), "-o", lib, "-l:libstdc++.so.6"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return ctypes.CDLL(lib)


def _emul_solve(L, packed, N, ws=None, shift=0, shifts=None):
    """The device-resident path on the host; with `ws` the warm flag is on (scalar `shift`, or per-robot `shifts`)."""
    B = len(packed)
    w = np.zeros((B, 12 * N), np.float32)
    st = np.full(B, -1, np.int32)
    launched = np.zeros(3, np.int32)
    rc = L.emul_solve_warm(_p(packed), B, N, ctypes.c_float(0.04), ctypes.c_float(500.0), 500, _p(ws) if ws is not None else None,
                           shift, _p(shifts) if shifts is not None else None, _p(w), _p(st), _p(launched))
    assert rc == 0
    return w, st, launched


def _sets(ws):
    """the recorded working set of every robot, as a set (the proposal built from it does not depend on the order)"""
    return [sorted(ws[b, 1:1 + ws[b, 0]].tolist()) if 0 <= ws[b, 0] < ws.shape[1] else None for b in range(len(ws))]


def _bits_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


@pytest.fixture(scope="module")
def walkers_h10(emul):
    """cfg3_h10 walking and standing robots: cold results and the working sets a recording pass (empty proposals) writes."""
    g = load_golden("cfg3_h10")
    N, B = 10, 6
    packed = np.ascontiguousarray(interface.pack_records(g["records"][:B], N))
    w0, st0, _ = _emul_solve(emul, packed, N)
    assert (interface.status_code(st0) == 0).all()
    true_ws = np.zeros((B, emul.emul_ws_ints()), np.int32)
    w1, st1, _ = _emul_solve(emul, packed, N, true_ws, 0)
    assert _bits_equal(w1, w0) and np.array_equal(st1, st0) and (true_ws[:, 0] > 0).all()
    return packed, w0, st0, true_ws


def test_warm_source_negative_shift_is_a_cold_solve_that_records_its_set(emul, walkers_h10):
    """shift < 0 (no history, e.g. an environment reset): whatever the memory proposes, the robot is solved cold — results
    and status bit for bit — and its working set is recorded for the next call."""
    packed, w0, st0, true_ws = walkers_h10
    B = len(packed)
    ws = np.roll(true_ws, 1, axis=0).copy()           # every robot holds another robot's set
    w, st, _ = _emul_solve(emul, packed, 10, ws, 1, shifts=np.full(B, -1, np.int32))
    assert _bits_equal(w, w0) and np.array_equal(st, st0)
    assert _sets(ws) == _sets(true_ws)


def test_warm_source_mixed_shifts_equal_per_robot_runs(emul, walkers_h10):
    """Per-robot shifts in one batch give every robot what a whole-batch run with its shift as the scalar gives it."""
    packed, w0, _, true_ws = walkers_h10
    shifts = np.array([1, 0, -1, 2, 1, 0], np.int32)
    ws_mix = true_ws.copy()
    w_mix, st_mix, _ = _emul_solve(emul, packed, 10, ws_mix, 7, shifts=shifts)   # (the scalar is overridden)
    assert (interface.status_code(st_mix) == 0).all()
    assert np.abs(w_mix - w0).max() < 1e-5 * np.abs(w0).max()
    for s in np.unique(shifts):
        ws_s = true_ws.copy()
        w_s, st_s, _ = _emul_solve(emul, packed, 10, ws_s, int(s))
        m = shifts == s
        assert _bits_equal(w_mix[m], w_s[m]) and np.array_equal(st_mix[m], st_s[m]), s
        assert [x for x, k in zip(_sets(ws_mix), m) if k] == [x for x, k in zip(_sets(ws_s), m) if k], s
    # shift 0 proposes the optimal set itself: fewer changes than the cold solve
    assert (interface.status_iters(st_mix[shifts == 0]) < interface.status_iters(walkers_h10[2][shifts == 0])).all()


def test_warm_source_hand_over_keeps_the_proposal(emul):
    """A robot whose optimum needs more rows than class 0 holds (status ST_WS_CAP in class 0) is handed to class 1, which
    must see the same proposal: class 0 does not record a set for it.  Record 11 of the stress fixture's h10_x4 set: single
    support (10 stance blocks), 25 active rows against class 0's 24.  Warm with its own set it ends on the referee's optimum
    with fewer changes than cold."""
    g = np.load(GOLDEN + "/stress_referee.npz")
    N, idx = 10, [11]
    recs = np.ascontiguousarray(g["h10_x4_records"]).view(scenarios.UPDATE_DTYPE).reshape(-1)[idx]
    ref = g["h10_x4_referee"][idx]
    packed = np.ascontiguousarray(interface.pack_records(recs, N))
    w0, st0, la0 = _emul_solve(emul, packed, N)
    # launched[0] counts what class 0 kept: it handed the robot over, class 1 solved it
    assert la0.tolist() == [0, 1, 0] and (interface.status_code(st0) == 0).all()
    ws = np.zeros((1, emul.emul_ws_ints()), np.int32)
    _emul_solve(emul, packed, N, ws, 0)                                  # records class 1's set
    assert 24 < ws[0, 0] <= 31
    kept = ws.copy()
    w, st, la = _emul_solve(emul, packed, N, ws, 0)                      # proposes it: class 0 overflows again
    assert la.tolist() == [0, 1, 0] and (interface.status_code(st) == 0).all()
    assert interface.status_iters(st)[0] < interface.status_iters(st0)[0]
    assert _sets(ws) == _sets(kept)
    assert rel_err(w, ref, 12).max() < 5e-5 and rel_err(w, ref).max() < 1e-5
    assert np.abs(w - w0).max() < 1e-5 * np.abs(w0).max()


def test_warm_source_beyond_the_block_start_is_a_cold_solve(emul):
    """Horizon 16: working-set capacities above 31 rows, no block start.  A warm call — any shift, any proposal — is the
    cold solve bit for bit, and records an empty set."""
    g = load_golden("cfg4_h16")
    N, B = 16, 3
    packed = np.ascontiguousarray(interface.pack_records(g["records"][:B], N))
    w0, st0, la0 = _emul_solve(emul, packed, N)
    assert (la0[:2] > 0).all() and (interface.status_code(st0) == 0).all()   # both classes
    W = emul.emul_ws_ints()
    for shift, shifts in ((0, None), (1, None), (0, np.array([1, 0, -1], np.int32))):
        ws = np.zeros((B, W), np.int32)
        ws[:, 0] = 6
        ws[:, 1:7] = (np.arange(6) * 2 << 8) | 9     # Fz upper rows of leg 0 at steps 0..5
        w, st, _ = _emul_solve(emul, packed, N, ws, shift, shifts)
        assert _bits_equal(w, w0) and np.array_equal(st, st0)
        assert (ws[:, 0] == 0).all()


def test_warm_calls_reject_a_null_context():
    L = interface.lib()
    assert L.hmpc_solve_device_warm(None, None, 1, None, None, None, None, None) == interface.HMPC_ERR_ARG
    assert L.hmpc_solve_batch_warm(None, None, 1, None, None, None, None) == interface.HMPC_ERR_ARG


# ---- GPU ---------------------------------------------------------------------------------------------------------------
N, B_GPU, T_GPU = 10, 1024, 50


@pytest.fixture(scope="module")
def replay():
    """hmpc_rollout_device over B_GPU walkers for T_GPU ticks (logs of records and first-step wrenches), and the logged
    records replayed tick by tick: warm (hmpc_solve_device_warm, fresh context, shift NULL) and cold (hmpc_solve_device)."""
    import torch
    from test_rollout import _to_dev, _walkers

    B, T = B_GPU, T_GPU
    states, loop = _walkers(B, seed=11)
    mpc = interface.BatchedMPC(B, N)
    d_states, d_loop = _to_dev(states), _to_dev(loop)
    d_wlog = torch.zeros((T, B, 12), dtype=torch.float32, device="cuda")
    d_rlog = torch.zeros((T, B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    mpc.rollout_device(d_states, d_loop, B, T, d_wlog, d_rlog)
    torch.cuda.synchronize()
    lo = d_loop.cpu().numpy().view(scenarios.ROLLOUT_DTYPE).reshape(B)
    mpc.close()
    out = dict(d_rlog=d_rlog, rlog=d_rlog.cpu().numpy(), wlog=d_wlog.cpu().numpy(), loop=lo)
    out["warm"] = _replay(d_rlog, warm=True)
    out["cold"] = _replay(d_rlog, warm=False)
    return out


def _replay(d_rlog, warm=True, d_shift=None):
    import torch

    T, B = d_rlog.shape[0], d_rlog.shape[1]
    mpc = interface.BatchedMPC(B, N)
    w = torch.zeros((T, B, 12 * N), dtype=torch.float32, device="cuda")
    s = torch.zeros((T, B), dtype=torch.int32, device="cuda")
    for t in range(T):
        if warm:
            mpc.solve_device_warm(d_rlog[t], B, w[t], s[t], d_shift=None if d_shift is None else d_shift[t])
        else:
            mpc.solve_device(d_rlog[t], B, w[t], s[t])
    torch.cuda.synchronize()
    mpc.close()
    return w.cpu().numpy(), s.cpu().numpy()


@pytest.mark.gpu
def test_device_warm_replay_equals_the_rollout(replay):
    """The rollout is the shift-NULL caller of the same solve: replaying its records reproduces every tick's first-step
    wrench bit for bit, and the status words' changes add up to the loop's iters_total."""
    w, s = replay["warm"]
    assert _bits_equal(w[:, :, :12], replay["wlog"])
    assert np.array_equal(interface.status_iters(s).sum(0), replay["loop"]["iters_total"])


@pytest.mark.gpu
def test_device_warm_reaches_the_cold_optimum_with_fewer_changes(replay):
    w, s = replay["warm"]
    wc, sc = replay["cold"]
    assert (interface.status_code(s) == 0).all() and (interface.status_code(sc) == 0).all()
    e1 = rel_err(w.reshape(-1, 12 * N), wc.reshape(-1, 12 * N), 12)
    ef = rel_err(w.reshape(-1, 12 * N), wc.reshape(-1, 12 * N))
    warm_chg, cold_chg = interface.status_iters(s[1:]).mean(), interface.status_iters(sc[1:]).mean()
    print("warm vs cold replay: first-step rel err worst %.2e, whole horizon %.2e; changes per tick warm %.2f cold %.2f"
          % (e1.max(), ef.max(), warm_chg, cold_chg))
    assert e1.max() < 1e-6
    assert warm_chg < 0.5 * cold_chg


@pytest.mark.gpu
def test_host_warm_modes_equal_the_device_warm_path(replay):
    """hmpc_solve_batch_warm on the unpacked records: the chunked copy pipeline (2048 robots — the logged batch twice — in
    two chunks, so the second chunk's working sets and shifts are offset) and the in-place mode (pinned caller buffers).
    Wrenches rounded to float and statuses equal the device warm path's; no instance overflows differently."""
    w_dev, s_dev = replay["warm"]
    B, T = B_GPU, T_GPU
    staged = interface.BatchedMPC(2 * B, N)
    inplace = interface.BatchedMPC(B, N)
    rec = interface.page_aligned((B,), scenarios.UPDATE_DTYPE)
    wbuf = interface.page_aligned((B, 12 * N), np.float64)
    sbuf = interface.page_aligned((B,), np.int32)
    inplace.pin(rec, wbuf, sbuf)
    for t in range(T):
        r = interface.unpack_records(replay["rlog"][t], N)
        w2, s2 = staged.solve_batch_warm(np.concatenate([r, r]), strict=False)
        for h in (slice(0, B), slice(B, 2 * B)):
            assert _bits_equal(w2[h], w_dev[t]), t
            assert np.array_equal(s2[h], s_dev[t]), t
        rec[:] = r
        inplace.solve_batch_warm(rec, strict=False, out=(wbuf, sbuf))
        assert _bits_equal(wbuf, w_dev[t]) and np.array_equal(sbuf, s_dev[t]), t
    inplace.unpin(rec, wbuf, sbuf)
    inplace.close()
    staged.close()


@pytest.mark.gpu
def test_device_warm_resets_are_cold_solves(replay):
    """10 % of the robots get shift -1 at one random tick each: there they equal the cold solve bit for bit (results and
    status); the robots never reset are untouched by their neighbours' resets."""
    import torch

    B, T = B_GPU, T_GPU
    rng = np.random.default_rng(5)
    robots = rng.choice(B, B // 10, replace=False)
    ticks = rng.integers(1, T, len(robots))
    shifts = np.ones((T, B), np.int32)
    shifts[ticks, robots] = -1
    w, s = _replay(replay["d_rlog"], warm=True, d_shift=torch.from_numpy(shifts).cuda())
    w_dev, s_dev = replay["warm"]
    wc, sc = replay["cold"]
    assert _bits_equal(w[ticks, robots], wc[ticks, robots]) and np.array_equal(s[ticks, robots], sc[ticks, robots])
    others = np.setdiff1d(np.arange(B), robots)
    assert _bits_equal(w[:, others], w_dev[:, others]) and np.array_equal(s[:, others], s_dev[:, others])


@pytest.mark.gpu
def test_reference_boundary_warm_start(replay):
    """With hmpc_reference_set_warm_start(1), one robot's logged ticks through setup_problem + update_problem_data (the
    reference caller's sequence, every tick) give the batched warm path's solution and status for that robot.  Off (the
    default), update_problem_data is the cold solve."""
    r = 7
    w_dev, s_dev = replay["warm"]
    wc, sc = replay["cold"]
    recs = interface.unpack_records(replay["rlog"][:, r], N)

    def tick(u):
        interface.setup_problem(0.04, N, 0.25, 500.0)
        interface.update_problem_data(u["p"], u["v"], u["q"], u["w"], u["r"], u["joint_angles"], float(u["yaw"]), u["weights"],
                                      u["traj"][:12 * N], u["Alpha_K"], u["gait"][:2 * N].astype(np.int32))
        return np.array([interface.get_solution(i) for i in range(12 * N)]), interface.reference_last_status()

    interface.setup_problem(0.05, N, 0.25, 500.0)   # another dt: forgets whatever working set the context held
    interface.reference_set_warm_start(True)
    try:
        for t in range(T_GPU):
            sol, st = tick(recs[t])
            assert _bits_equal(sol, w_dev[t, r]) and st == s_dev[t, r], t
    finally:
        interface.reference_set_warm_start(False)
    for t in range(3):
        sol, st = tick(recs[t])
        assert _bits_equal(sol, wc[t, r]) and st == sc[t, r], t


@pytest.mark.gpu
def test_warm_calls_check_their_arguments():
    import torch

    L = interface.lib()
    mpc = interface.BatchedMPC(64, N)
    h = mpc._h
    stride = interface.record_bytes(N)
    d_rec = torch.zeros(65 * stride + 16, dtype=torch.uint8, device="cuda")
    d_w = torch.zeros((65, 12 * N), dtype=torch.float32, device="cuda")
    d_s = torch.zeros(65, dtype=torch.int32, device="cuda")
    p = d_rec.data_ptr()
    ERR, OK = interface.HMPC_ERR_ARG, interface.HMPC_OK
    assert L.hmpc_solve_device_warm(h, None, 4, d_w.data_ptr(), d_s.data_ptr(), None, None, None) == ERR
    assert L.hmpc_solve_device_warm(h, p, 4, None, d_s.data_ptr(), None, None, None) == ERR
    assert L.hmpc_solve_device_warm(h, p, 4, d_w.data_ptr(), None, None, None, None) == ERR
    assert L.hmpc_solve_device_warm(h, p, 65, d_w.data_ptr(), d_s.data_ptr(), None, None, None) == ERR
    assert L.hmpc_solve_device_warm(h, p + 4, 4, d_w.data_ptr(), d_s.data_ptr(), None, None, None) == ERR
    assert L.hmpc_solve_device_warm(h, p, -1, d_w.data_ptr(), d_s.data_ptr(), None, None, None) == ERR
    assert L.hmpc_solve_device_warm(h, p, 0, d_w.data_ptr(), d_s.data_ptr(), None, None, None) == OK
    recs = np.zeros(65, scenarios.UPDATE_DTYPE)
    w = np.zeros((65, 12 * N))
    s = np.zeros(65, np.int32)
    assert L.hmpc_solve_batch_warm(h, None, 4, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_warm(h, recs.ctypes.data, 4, None, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_warm(h, recs.ctypes.data, 65, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_warm(h, recs.ctypes.data, 0, w.ctypes.data, None, s.ctypes.data, None) == OK
    mpc.close()
