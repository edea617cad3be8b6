"""Candidate commands per robot, solved from its state (hmpc_solve_states_device_multi, hmpc_solve_batch_states_multi): with
the expanded state batch (row i*K + k: state i with its command replaced by cmd[i][k]), traj[i][k] must be what
hmpc_prepare_device writes for row i*K + k, wrench / status what the solve gives that prepared row, cost the certificate's
cost, best the argmin over the converged candidates, tau the _ex torques of the chosen row, and the record the prepared
chosen row, bit for bit.

CPU: the kernel source on the host (tests/host_emul/states_multi_on_host.cpp): the trajectory kernel against the single
preparation of the expanded states, the whole chain against the emulated "prepare the expanded states, solve them
with the multi-query chain, cost them", the pick against numpy, masks, ThreadSanitizer, the argument checks through the
library.  GPU (-m gpu): the library against hmpc_prepare_device + hmpc_solve_device_ex + hmpc_certify_device on the
expanded batch, masks, graph replay, the host call in both modes, K = 1 and the argument errors.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import BUILD, DEVICE_HEADER, HERE, _host_buildable, _p

CERT_DTYPE = interface.CERTIFICATE_DTYPE
CMD = scenarios.COMMAND_DTYPE
DT = 0.04
_LIB = {}


# ---- fixtures ------------------------------------------------------------------------------------------------------------
def _states(cfg, B, N, seed):
    _, inputs = scenarios.make_batch(cfg, B, horizon=N, seed=seed)
    return np.ascontiguousarray(scenarios.make_states(inputs, N))


def _stress_states(N, scale, seed, idx):
    """the states behind scenarios.make_stress_batch(., N, scale, seed)[idx]"""
    rng = np.random.default_rng(seed)
    inputs = [scenarios._stress_state(rng, N, scale) for _ in range(max(idx) + 1)]
    return np.ascontiguousarray(scenarios.make_states([inputs[i] for i in idx], N))


def _lying(N=10):
    """the robot lying on its side (stress_referee.npz h10_lying): make_stress_batch(40, 10, 8.0, 15)[34]"""
    return _stress_states(N, 8.0, 15, [34])


def expand_states(states, cmd):
    """the expanded state batch: row i*K + k is state i with its command replaced by cmd[i][k]"""
    B, K = cmd.shape
    ex = np.repeat(states, K).copy()
    ex["state_des"] = cmd["state_des"].reshape(B * K, 5)
    ex["world_position_desired"] = cmd["world_position_desired"].reshape(B * K, 2)
    return ex


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def argmin_best(st, cost):
    """numpy's pick: per robot the first minimum of the cost over the candidates with status code 0 and a finite cost"""
    ok = (interface.status_code(st) == 0) & np.isfinite(cost)
    c = np.where(ok, cost, np.inf)
    best = np.argmin(c, axis=1).astype(np.int32)
    best[~ok.any(axis=1)] = -1
    return best


# ---- the kernel source on the host ---------------------------------------------------------------------------------------
def emulation():
    """states_multi_on_host.cpp built for the host as a library, once per process (the flags of kernel_source_on_host.cpp's
    build)"""
    if "lib" not in _LIB:
        os.makedirs(BUILD, exist_ok=True)
        hdr = os.path.join(BUILD, "hmpc_device_host_states_multi.cuh")
        with open(hdr, "w") as f:
            f.write(_host_buildable(open(DEVICE_HEADER).read()))
        out = os.path.join(BUILD, "libstates_multi_on_host.so")
        cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O2", "-fPIC", "-shared",
               "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"), '-DHMPC_DEVICE_HEADER="%s"' % hdr,
               os.path.join(HERE, "states_multi_on_host.cpp"), "-l:libstdc++.so.6", "-o", out]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        _LIB["lib"] = ctypes.CDLL(out)
        _LIB["hdr"] = hdr
    return _LIB["lib"]


def emul_prepare(states, N):
    L = emulation()
    out = np.full((len(states), interface.record_bytes(N)), 0xAB, np.uint8)
    L.emul_prepare(_p(states), len(states), N, ctypes.c_double(DT), _p(out))
    return out


def emul_prepare_traj(states, cmd, N, lst=None):
    L = emulation()
    B, K = cmd.shape
    traj = np.full((B, K, 12 * N), np.nan, np.float32)
    cnt = buf = None
    if lst is not None:
        cnt = np.array([len(lst)], np.int32)
        buf = np.full(B, -7, np.int32)
        buf[:len(lst)] = lst
    L.emul_prepare_traj(_p(states), B, K, _p(np.ascontiguousarray(cmd)), N, ctypes.c_double(DT), _p(traj), _p(buf), _p(cnt))
    return traj


def emul_chain(states, cmd, N, refine=False, mask=None, out=None):
    """the multi-command states chain on the host -> dict of records, traj, wrench [B,K,12N], status, cost, best, tau, launched"""
    L = emulation()
    B, K = cmd.shape
    if out is None:
        out = dict(records=np.full((B, interface.record_bytes(N)), 0xAB, np.uint8),
                   traj=np.full((B, K, 12 * N), np.nan, np.float32), wrench=np.zeros((B, K, 12 * N), np.float32),
                   status=np.full((B, K), -1, np.int32), cost=np.zeros((B, K)), best=np.full(B, -2, np.int32),
                   tau=np.full((B, 10), np.nan, np.float32))
    o = out
    la = np.zeros(4, np.int32)
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    rc = L.emul_solve_states_multi(_p(states), _p(np.ascontiguousarray(cmd)), ctypes.c_double(DT), _p(o["records"]), _p(o["traj"]),
                                   B, K, N, int(refine), _p(m), _p(o["wrench"]), _p(o["status"]), _p(o["cost"]), _p(o["best"]),
                                   _p(o["tau"]), _p(la))
    assert rc == 0, rc
    o["launched"] = la
    return o


def emul_expanded(states, cmd, N, refine=False):
    """the reference: hmpc_prepare_device's kernel on the expanded states, hmpc_solve_device_multi's chain on robot i's record
    and the K prepared trajectories (its cost kernel included), then the cold single solve with torques (_ex) and the
    certificate's cost of the expanded prepared rows, all from the same build"""
    L = emulation()
    B, K = cmd.shape
    R = B * K
    ex = expand_states(states, cmd)
    rows = emul_prepare(ex, N)
    rs = interface.record_bytes(N)
    traj = rows[:, 54 * 4:(54 + 12 * N) * 4].copy().view(np.float32).reshape(B, K, 12 * N)
    w = np.zeros((R, 12 * N), np.float32)
    st = np.full(R, -1, np.int32)
    cost = np.zeros(R)
    rec0 = np.ascontiguousarray(rows.reshape(B, K, rs)[:, 0])
    rc = L.emul_solve_multi(_p(rec0), None, B, K, N, int(refine), None, _p(traj), _p(w), None, _p(st), _p(cost), None)
    assert rc == 0, rc
    sw = np.zeros((R, 12 * N), np.float32)
    sst = np.full(R, -1, np.int32)
    tau = np.zeros((R, 10), np.float32)
    rc = L.emul_solve(_p(rows), None, R, N, 0, int(refine), None, None, 0, 1, None, _p(sw), None, _p(sst), _p(tau), None,
                      None, None, None, None, None)
    assert rc == 0, rc
    cert = np.zeros(R, CERT_DTYPE)
    L.emul_certify(_p(rows), 0, R, N, ctypes.c_float(0.04), ctypes.c_float(500.0), None, 0, _p(sw), _p(cert), None, None)
    return dict(rows=rows.reshape(B, K, rs), traj=traj, wrench=w.reshape(B, K, -1), status=st.reshape(B, K),
                cost=cost.reshape(B, K), single=(sw.reshape(B, K, -1), sst.reshape(B, K), cert["cost"].reshape(B, K)),
                tau=tau.reshape(B, K, 10))


def check_chain(got, want, rows_on=None):
    """every output of the chain against the expanded reference, on the robots `rows_on` (all by default)"""
    on = slice(None) if rows_on is None else rows_on
    assert np.array_equal(_bits(got["traj"][on]), _bits(want["traj"][on]))
    assert np.array_equal(_bits(got["wrench"][on]), _bits(want["wrench"][on]))
    assert np.array_equal(got["status"][on], want["status"][on])
    assert np.array_equal(_bits(got["cost"][on]), _bits(want["cost"][on]))
    sw, sst, scost = want["single"]  # the multi-query chain is the single solve and the certificate, bit for bit
    assert np.array_equal(_bits(got["wrench"][on]), _bits(sw[on])) and np.array_equal(got["status"][on], sst[on])
    assert np.array_equal(_bits(got["cost"][on]), _bits(scost[on]))
    best = argmin_best(want["status"], want["cost"])[on]
    assert np.array_equal(got["best"][on], best)
    idx = np.flatnonzero(np.ones(len(want["status"]), bool)[on]) if rows_on is not None else np.arange(len(best))
    pick = np.maximum(best, 0)
    assert np.array_equal(_bits(got["records"][on]), _bits(want["rows"][idx, pick]))
    tau = np.where((best >= 0)[:, None], want["tau"][idx, pick], np.float32(0))
    assert np.array_equal(_bits(got["tau"][on]), _bits(tau))


def _walkers(N, B=3, seed=5):
    return _states(2, B, N, seed)


CASES = {  # name -> (states, N, what the case reaches)
    "walk_h10": lambda: (_walkers(10), 10),                                         # walking: class 0
    "stand_h10": lambda: (_states(1, 1, 10, 4), 10),                                # standing: class 1, robots handed over
    "mixed_h5": lambda: (_states(3, 3, 5, 6), 5),                                   # runtime horizon, both classes
    "walk_h16": lambda: (_walkers(16, 2), 16),                                      # the horizon-16 extension
    "stress_h10_x8": lambda: (_stress_states(10, 8.0, 3, [9, 21]), 10),             # ~80 active rows: escalation to class 2
}


@pytest.mark.parametrize("listed", [False, True])
@pytest.mark.parametrize("name", ["walk_h10", "stand_h10", "mixed_h5", "walk_h16"])
def test_prepare_traj_source_equals_the_expanded_preparation(name, listed):
    """The K trajectories are the traj bytes hmpc_prepare_kernel writes for the expanded states; over a list only the listed
    robots' trajectories are written."""
    states, N = CASES[name]()
    B, K = len(states), 4
    cmd = scenarios.command_candidates(states, K, seed=B + N)
    lst = np.array([i for i in range(B) if i % 2 == 0], np.int32) if listed else None
    traj = emul_prepare_traj(states, cmd, N, lst)
    want = emul_prepare(expand_states(states, cmd), N).reshape(B, K, -1)
    on = np.zeros(B, bool)
    on[np.arange(B) if lst is None else lst] = True
    wt = want[:, :, 54 * 4:(54 + 12 * N) * 4].copy().view(np.float32).reshape(B, K, 12 * N)
    assert np.array_equal(_bits(traj[on]), _bits(wt[on]))
    assert np.isnan(traj[~on]).all()
    # candidate 0 is the state's own command: the traj of hmpc_prepare_kernel on the state itself
    assert np.array_equal(wt[on, 0], emul_prepare(states, N)[on][:, 54 * 4:(54 + 12 * N) * 4].copy().view(np.float32))


@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("name", list(CASES))
def test_chain_source_equals_prepare_then_multi_solve(name, K):
    states, N = CASES[name]()
    cmd = scenarios.command_candidates(states, K, seed=K + len(name))
    got = emul_chain(states, cmd, N)
    want = emul_expanded(states, cmd, N)
    check_chain(got, want)
    assert (interface.status_code(got["status"]) == 0).mean() > 0.8
    if name == "stand_h10":
        assert got["launched"][1] == len(states)
    if name == "stress_h10_x8" and K == 8:
        assert got["launched"][2] > 0  # candidates escalated alone to class 2
    if K > 1 and name in ("walk_h10", "mixed_h5"):
        assert len(set(got["best"])) > 1 or (got["best"] != 0).any()  # the candidates move the optimum


def test_chain_source_lying_robot_with_refinement():
    """The lying robot among walkers, refinement on: each of its candidates goes to the refinement class, and the chain
    equals the expanded reference with refinement on."""
    states = np.concatenate([_walkers(10, 2), _lying()])
    K = 3
    cmd = scenarios.command_candidates(states, K, seed=9)
    got = emul_chain(states, cmd, 10, refine=True)
    assert got["launched"][3] == K
    check_chain(got, emul_expanded(states, cmd, 10, refine=True))
    assert ((got["status"][2] >> 28) & 1).all() and got["best"][2] >= 0


def test_chain_source_lying_robot_without_refinement_has_no_best():
    """Refinement off: every candidate of the lying robot ends with code 4, so best = -1, its torques are zeros and its
    record is candidate 0's."""
    states = np.concatenate([_walkers(10, 1), _lying()])
    K = 3
    cmd = scenarios.command_candidates(states, K, seed=10)
    got = emul_chain(states, cmd, 10)
    want = emul_expanded(states, cmd, 10)
    check_chain(got, want)
    assert (interface.status_code(got["status"][1]) == interface.ST_NOT_SPD).all()
    assert got["best"][1] == -1 and (_bits(got["tau"][1]) == 0).all()
    assert np.array_equal(got["records"][1], want["rows"][1, 0])


def test_chain_source_ties_pick_the_lower_candidate():
    """Two identical commands give identical costs: the lower k wins.  A candidate equal to the state's own command gives
    the cold single states solve: the record, wrench and torques of prepare + solve_ex on the state itself."""
    N = 10
    states = _walkers(N, 3, seed=8)
    cmd = scenarios.command_candidates(states, 4, seed=2)
    cmd[:, 3] = cmd[:, 1]
    cmd[:, 2] = cmd[:, 1]
    got = emul_chain(states, cmd, N)
    want = emul_expanded(states, cmd, N)
    check_chain(got, want)
    assert np.array_equal(_bits(got["cost"][:, 1]), _bits(got["cost"][:, 3]))
    assert not np.isin(got["best"], [2, 3]).any()
    # candidate 0 against the cold single states solve
    L = emulation()
    rows = emul_prepare(states, N)
    w = np.zeros((len(states), 12 * N), np.float32)
    st = np.full(len(states), -1, np.int32)
    tau = np.zeros((len(states), 10), np.float32)
    assert L.emul_solve(_p(rows), None, len(states), N, 0, 0, None, None, 0, 1, None, _p(w), None, _p(st), _p(tau), None,
                        None, None, None, None, None) == 0
    assert np.array_equal(_bits(got["wrench"][:, 0]), _bits(w)) and np.array_equal(got["status"][:, 0], st)
    own = got["best"] == 0
    assert np.array_equal(got["records"][own], rows[own]) and np.array_equal(_bits(got["tau"][own]), _bits(tau[own]))


def test_chain_source_mask_keeps_the_unlisted_rows():
    """Unlisted robots keep the sentinel bytes of all seven outputs: records, traj, wrench, status, cost, best, tau."""
    N, K = 10, 3
    states = _states(3, 6, N, 12)
    cmd = scenarios.command_candidates(states, K, seed=3)
    mask = np.array([1, 0, 0, 3, 0, 1], np.uint8)
    rng = np.random.default_rng(1)
    B = len(states)

    def sent(shape, dt):
        return rng.integers(0, 256, int(np.prod(shape)) * np.dtype(dt).itemsize, dtype=np.uint8).view(dt).reshape(shape)

    out = dict(records=sent((B, interface.record_bytes(N)), np.uint8), traj=sent((B, K, 12 * N), np.float32),
               wrench=sent((B, K, 12 * N), np.float32), status=sent((B, K), np.int32), cost=sent((B, K), np.float64),
               best=sent(B, np.int32), tau=sent((B, 10), np.float32))
    before = {k: v.copy() for k, v in out.items()}
    got = emul_chain(states, cmd, N, mask=mask, out=out)
    on = mask != 0
    check_chain({k: v[on] for k, v in got.items() if k != "launched"}, emul_expanded(states[on], cmd[on], N))
    for k, v in before.items():
        assert np.array_equal(_bits(got[k][~on]), _bits(v[~on])), k


def test_chain_source_has_no_races_under_thread_sanitizer(tmp_path):
    """The chain built with -fsanitize=thread: the preparation, the multi-query classes with escalation and refinement, the
    cost kernel and the pick kernel's warp reduction."""
    emulation()
    exe = os.path.join(BUILD, "states_multi_tsan")
    cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O1", "-g", "-fsanitize=thread", "-DHMPC_STATES_MULTI_MAIN",
           "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"),
           '-DHMPC_DEVICE_HEADER="%s"' % _LIB["hdr"], os.path.join(HERE, "states_multi_on_host.cpp"), "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("no ThreadSanitizer runtime with this toolchain: " + r.stderr[-300:])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66")
    cases = [(_walkers(10, 2), 10, 3, ()), (_states(1, 1, 10, 4), 10, 2, ()), (_states(3, 2, 5, 6), 5, 2, ()),
             (_stress_states(10, 8.0, 3, [9]), 10, 2, ()), (_lying(), 10, 2, ("refine",))]
    for states, N, K, flags in cases:
        f = tmp_path / "states.bin"
        np.ascontiguousarray(states).tofile(f)
        run = subprocess.run([exe, str(f), str(N), str(K), *flags], capture_output=True, text=True, env=env, timeout=1800)
        assert "ThreadSanitizer" not in run.stderr, run.stderr[:3000]
        assert run.returncode == 0, (run.returncode, run.stdout, run.stderr[-500:])


def test_states_multi_calls_check_their_arguments():
    """Through the library, without a GPU: a null context is rejected before anything else."""
    L = interface.lib()
    ERR = interface.HMPC_ERR_ARG
    x = np.zeros(64, np.float64)
    p = x.ctypes.data
    assert L.hmpc_solve_states_device_multi(None, p, 1, 2, p, None, DT, p, p, p, p, p, p, None, None) == ERR
    assert L.hmpc_solve_batch_states_multi(None, p, 1, 2, p, None, DT, p, p, p, p, None) == ERR
    assert L.hmpc_solve_states_device_multi(None, None, 0, 1, None, None, DT, None, None, None, None, None, None, None, None) == ERR


def test_command_dtype_is_the_states_command_bytes():
    assert CMD.itemsize == 56
    assert scenarios.STATE_DTYPE.fields["state_des"][1] == 256
    assert scenarios.STATE_DTYPE.fields["world_position_desired"][1] == 256 + CMD.fields["world_position_desired"][1]
    states = _walkers(10, 4)
    cmd = scenarios.command_candidates(states, 5, seed=1)
    assert np.array_equal(cmd[:, 0]["state_des"], states["state_des"])
    assert np.array_equal(cmd[:, 0]["world_position_desired"], states["world_position_desired"])
    assert np.array_equal(expand_states(states, cmd[:, :1]).tobytes(), states.tobytes())


# ---- GPU: the library ----------------------------------------------------------------------------------------------------
def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _alloc(B, K, N, sentinel=False):
    import torch

    o = dict(records=torch.zeros((B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda"),
             traj=torch.zeros((B, K, 12 * N), dtype=torch.float32, device="cuda"),
             wrench=torch.zeros((B, K, 12 * N), dtype=torch.float32, device="cuda"),
             status=torch.zeros((B, K), dtype=torch.int32, device="cuda"),
             cost=torch.zeros((B, K), dtype=torch.float64, device="cuda"),
             best=torch.zeros(B, dtype=torch.int32, device="cuda"),
             tau=torch.zeros((B, 10), dtype=torch.float32, device="cuda"))
    if sentinel:
        for v in o.values():
            v.view(torch.uint8).fill_(0xA7)
    return o


def _call(mpc, d_states, B, d_cmd, o, d_mask=None):
    mpc.solve_states_device_multi(d_states, B, d_cmd, o["records"], o["traj"], o["wrench"], o["status"], o["cost"], o["best"],
                                  o["tau"], d_mask=d_mask)


def _host(o):
    import torch

    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _device_multi(mpc, states, cmd, mask=None, sentinel=False):
    B, K = cmd.shape
    o = _alloc(B, K, mpc.horizon, sentinel)
    _call(mpc, _dev(states.view(np.uint8).reshape(B, -1)), B, _dev(cmd.view(np.uint8).reshape(B, K, -1)), o,
          None if mask is None else _dev(mask))
    return _host(o)


def _device_expanded(mpc, states, cmd):
    """hmpc_prepare_device + hmpc_solve_device_ex + hmpc_certify_device on the expanded states"""
    import torch

    B, K = cmd.shape
    N, R = mpc.horizon, B * K
    ex = expand_states(states, cmd)
    rows = torch.zeros((R, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    mpc.prepare_device(_dev(ex.view(np.uint8).reshape(R, -1)), R, rows)
    w = torch.zeros((R, 12 * N), dtype=torch.float32, device="cuda")
    st = torch.zeros(R, dtype=torch.int32, device="cuda")
    tau = torch.zeros((R, 10), dtype=torch.float32, device="cuda")
    cert = torch.zeros((R, CERT_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    interface._check(interface.lib().hmpc_solve_device_ex(mpc._h, rows.data_ptr(), R, w.data_ptr(), st.data_ptr(),
                                                          tau.data_ptr(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
                     allow_not_converged=True)
    mpc.certify_device(rows, R, w, cert)
    torch.cuda.synchronize()
    rows = rows.cpu().numpy()
    return dict(rows=rows.reshape(B, K, -1), traj=rows[:, 54 * 4:(54 + 12 * N) * 4].copy().view(np.float32).reshape(B, K, -1),
                wrench=w.cpu().numpy().reshape(B, K, -1), status=st.cpu().numpy().reshape(B, K),
                cost=cert.cpu().numpy().view(CERT_DTYPE).reshape(-1)["cost"].reshape(B, K).copy(),
                tau=tau.cpu().numpy().reshape(B, K, 10))


def check_device(got, want):
    assert np.array_equal(_bits(got["traj"]), _bits(want["traj"]))
    assert np.array_equal(_bits(got["wrench"]), _bits(want["wrench"]))
    assert np.array_equal(got["status"], want["status"])
    assert np.array_equal(_bits(got["cost"]), _bits(want["cost"]))
    best = argmin_best(want["status"], want["cost"])
    assert np.array_equal(got["best"], best)
    idx, pick = np.arange(len(best)), np.maximum(best, 0)
    assert np.array_equal(got["records"], want["rows"][idx, pick])
    tau = np.where((best >= 0)[:, None], want["tau"][idx, pick], np.float32(0))
    assert np.array_equal(_bits(got["tau"]), _bits(tau))


def _gpu_states(cfg, B, N=10):
    _, inputs = scenarios.make_batch(cfg, B, horizon=N, seed=scenarios.config_seed(cfg) + 78)
    return np.ascontiguousarray(scenarios.make_states(inputs, N))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,K", [(2, 8), (3, 4)])  # make_batch(2): configs[1] walkers, (3): configs[2] mixed
def test_device_states_multi_equals_the_expanded_calls(cfg, K):
    """1024 configs[1] walker states x 8 commands and 1024 configs[2] mixed states x 4, against hmpc_prepare_device +
    hmpc_solve_device_ex + hmpc_certify_device on the 8192 / 4096 expanded states; best against numpy's argmin."""
    B, N = 1024, 10
    states = _gpu_states(cfg, B)
    cmd = scenarios.command_candidates(states, K, seed=cfg)
    mpc = interface.BatchedMPC(B * K, N, device=0)
    got = _device_multi(mpc, states, cmd)
    want = _device_expanded(mpc, states, cmd)
    check_device(got, want)
    assert (interface.status_code(want["status"]) == 0).mean() > 0.95
    assert (got["best"] > 0).mean() > 0.3  # the other commands win often: the pick is not trivially candidate 0
    mpc.close()


@pytest.mark.gpu
def test_device_states_multi_mask_graph_replay_and_k1():
    """A fifth of the robots masked in leaves every other row of the seven outputs alone; a torch.cuda.graph replay with new
    states, commands and mask written into the captured buffers equals eager calls; K = 1 equals the expanded calls."""
    import torch

    B, N, K = 512, 10, 4
    states = _gpu_states(3, B)
    cmd = scenarios.command_candidates(states, K, seed=11)
    mpc = interface.BatchedMPC(B * K, N, device=0)
    mask = (np.arange(B) % 5 == 2).astype(np.uint8)
    got = _device_multi(mpc, states, cmd, mask=mask, sentinel=True)
    eager = _device_multi(mpc, states, cmd)
    on = mask != 0
    for k in got:
        assert np.array_equal(_bits(got[k][on]), _bits(eager[k][on])), k
        assert (_bits(got[k][~on]).view(np.uint8) == 0xA7).all(), k
    # graph replay: capture once, then write other inputs into the captured buffers
    d_states = _dev(states.view(np.uint8).reshape(B, -1))
    d_cmd = _dev(cmd.view(np.uint8).reshape(B, K, -1))
    d_mask = _dev(np.ones(B, np.uint8))
    o = _alloc(B, K, N)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _call(mpc, d_states, B, d_cmd, o, d_mask)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _call(mpc, d_states, B, d_cmd, o, d_mask)
    for r in range(2):
        st2 = _gpu_states(2 + r, B)
        cmd2 = scenarios.command_candidates(st2, K, seed=40 + r)
        m2 = (np.arange(B) % (2 + r) == 0).astype(np.uint8)
        d_states.copy_(_dev(st2.view(np.uint8).reshape(B, -1)))
        d_cmd.copy_(_dev(cmd2.view(np.uint8).reshape(B, K, -1)))
        d_mask.copy_(_dev(m2))
        for v in o.values():
            v.view(torch.uint8).fill_(0xA7)
        g.replay()
        rep = _host(o)
        want = _device_multi(mpc, st2, cmd2, mask=m2, sentinel=True)
        for k in rep:
            assert np.array_equal(_bits(rep[k]), _bits(want[k])), (r, k)
    # K = 1: the single states solve
    one = _device_multi(mpc, states, cmd[:, :1])
    check_device(one, _device_expanded(mpc, states, cmd[:, :1]))
    mpc.close()


@pytest.mark.gpu
def test_host_states_multi_in_place_and_staged():
    """hmpc_solve_batch_states_multi on pinned arrays (in place) and on ordinary ones (staged): equal to each other, their
    doubles rounding to the device call's floats, with the device call's status words, best and costs of those doubles'
    rows; a mask writes the listed robots only."""
    B, N, K = 256, 10, 3
    states = _gpu_states(2, B)
    cmd = scenarios.command_candidates(states, K, seed=21)
    mpc = interface.BatchedMPC(B * K, N, device=0)
    dev = _device_multi(mpc, states, cmd)
    res = {}
    for pinned in (True, False):
        alloc = interface.page_aligned if pinned else (lambda shape, dt: np.zeros(shape, dt))
        x, c = alloc((B,), scenarios.STATE_DTYPE), alloc((B, K), CMD)
        x[:], c[:] = states, cmd
        out = (alloc((B, K, 12 * N), np.float64), alloc((B, K), np.int32), alloc((B, K), np.float64), alloc((B,), np.int32),
               alloc((B, 10), np.float64))
        if pinned:
            mpc.pin(x, c, *out)
        w, st, cost, best, tau = mpc.solve_batch_states_multi(x, c, out=out, strict=False)
        assert w is out[0]
        assert interface.lib().hmpc_debug_last_states_multi_in_place() == (1 if pinned else 0)
        assert np.array_equal(_bits(w.astype(np.float32)), _bits(dev["wrench"])) and np.array_equal(st, dev["status"])
        assert np.array_equal(_bits(tau.astype(np.float32)), _bits(dev["tau"]))
        assert np.array_equal(best, argmin_best(st, cost))
        res[pinned] = (w, st, cost, best, tau)
    for a, b in zip(res[True], res[False]):
        assert np.array_equal(_bits(a), _bits(b))
    # the costs are the certificate's of the expanded prepared rows and the double wrenches
    recs = interface.unpack_records(_device_expanded(mpc, states, cmd)["rows"].reshape(B * K, -1), N)
    cert = mpc.certify_batch(recs, res[False][0].reshape(B * K, -1))
    assert np.array_equal(_bits(res[False][2].reshape(-1)), _bits(cert["cost"]))
    # a mask writes the listed robots only
    mask = (np.arange(B) % 3 == 1).astype(np.uint8)
    out = tuple(np.full_like(a, 7) for a in res[False])
    mpc.solve_batch_states_multi(states, cmd, mask=mask, out=out, strict=False)
    on = mask != 0
    for a, b in zip(out, res[False]):
        assert np.array_equal(_bits(a[on]), _bits(b[on])) and (a[~on] == 7).all()
    mpc.close()


@pytest.mark.gpu
def test_states_multi_argument_errors():
    import torch

    B, N, K = 8, 10, 2
    mpc = interface.BatchedMPC(16, N, device=0)
    states = _gpu_states(2, B)
    cmd = scenarios.command_candidates(states, K, seed=1)
    o = _alloc(B, K, N)
    d_states, d_cmd = _dev(states.view(np.uint8).reshape(B, -1)), _dev(cmd.view(np.uint8).reshape(B, K, -1))
    L, ERR = interface.lib(), interface.HMPC_ERR_ARG
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = [d_states.data_ptr(), B, K, d_cmd.data_ptr(), None, DT, o["records"].data_ptr(), o["traj"].data_ptr(),
            o["wrench"].data_ptr(), o["status"].data_ptr(), o["cost"].data_ptr(), o["best"].data_ptr(), None, st]
    assert L.hmpc_solve_states_device_multi(mpc._h, *args) == interface.HMPC_OK
    for i in (0, 3, 6, 7, 8, 9, 10, 11):  # every required pointer
        bad = list(args)
        bad[i] = None
        assert L.hmpc_solve_states_device_multi(mpc._h, *bad) == ERR, i
    for b, k in ((B, 0), (B, 3), (-1, K)):  # K < 1, B*K > capacity, B < 0
        bad = list(args)
        bad[1], bad[2] = b, k
        assert L.hmpc_solve_states_device_multi(mpc._h, *bad) == ERR, (b, k)
    bad = list(args)
    bad[1] = 0
    assert L.hmpc_solve_states_device_multi(mpc._h, *bad) == interface.HMPC_OK  # B = 0: a no-op
    w = np.zeros((B, K, 12 * N))
    i32 = np.zeros((B, K), np.int32)
    assert L.hmpc_solve_batch_states_multi(mpc._h, states.ctypes.data, B, 3, cmd.ctypes.data, None, DT, w.ctypes.data,
                                           i32.ctypes.data, w.ctypes.data, i32.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_states_multi(mpc._h, states.ctypes.data, B, K, None, None, DT, w.ctypes.data,
                                           i32.ctypes.data, w.ctypes.data, i32.ctypes.data, None) == ERR
    torch.cuda.synchronize()
    mpc.close()
