"""Warm-started, masked and state-fed sharded solves (hmpc_solve_batch_sharded_warm, hmpc_solve_batch_states_sharded_warm,
BatchedMPC.solve_batch_sharded_warm, ShardedMPC(warm=True)): each rank solves only its due robots, and the gather carries
every other robot's latest wrench.

CPU: the carry kernel's source on the host (tests/host_emul/carry_on_host.cpp) — unlisted rows get the previous buffer's
bytes, listed rows keep theirs, also under ThreadSanitizer; a two-rank gloo run of ShardedMPC's warm ticks with staggered
masks (slicing, padding and ordering; the gather's latest-row rule); the null-context checks.  GPU (one-rank NCCL group):
every sharded call against a second context running the non-sharded call over the same ticks, in place and staged."""
import ctypes
import os
import socket
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_golden
from hector_simulation_b200 import interface, scenarios, sharding
from test_kernel_source_on_host import BUILD, DEVICE_HEADER, HERE, _host_buildable, _p

N = 10
_LIB = {}
CARRY_SRC = os.path.join(HERE, "carry_on_host.cpp")


def _carry_build(name, flags):
    os.makedirs(BUILD, exist_ok=True)
    hdr = os.path.join(BUILD, "hmpc_device_host_carry.cuh")
    if "header" not in _LIB:
        with open(hdr, "w") as f:
            f.write(_host_buildable(open(DEVICE_HEADER).read()))
        _LIB["header"] = hdr
    out = os.path.join(BUILD, name)
    cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", *flags, "-I" + os.path.join(HERE, "fake_cuda"),
           "-I" + os.path.join(ROOT, "include"), '-DHMPC_DEVICE_HEADER="%s"' % hdr, CARRY_SRC, "-o", out]
    return out, subprocess.run(cmd, capture_output=True, text=True)


def carry_emulation():
    """carry_on_host.cpp built for the host as a library, once per process (the flags of kernel_source_on_host.cpp's build)"""
    if "lib" not in _LIB:
        out, r = _carry_build("libcarry_on_host.so", ["-O2", "-fPIC", "-shared", "-l:libstdc++.so.6"])
        assert r.returncode == 0, r.stderr[-3000:]
        _LIB["lib"] = ctypes.CDLL(out)
    return _LIB["lib"]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint8)


# ---- CPU: the carry kernel's source ---------------------------------------------------------------------------------------
def _carry_cases():
    rng = np.random.default_rng(3)
    out = []
    for n in (5, 10, 16):
        for B in (1, 37, 300):                  # B * 3N vectors: never a multiple of the 256-thread block here
            masks = {"empty": np.zeros(B, np.uint8), "full": np.ones(B, np.uint8),
                     "random": (rng.random(B) < 0.4).astype(np.uint8) * rng.integers(1, 256, B).astype(np.uint8),
                     "single": np.zeros(B, np.uint8)}
            masks["single"][B // 2] = 7
            out += [("N%d_B%d_%s" % (n, B, k), n, m) for k, m in masks.items()]
    return out


@pytest.mark.parametrize("name,n,mask", _carry_cases(), ids=[c[0] for c in _carry_cases()])
def test_carry_source_copies_the_unlisted_rows(name, n, mask):
    L = carry_emulation()
    B = len(mask)
    assert (B * 3 * n) % L.emul_carry_threads() != 0 and L.emul_carry_grid(B, n) * L.emul_carry_threads() >= B * 3 * n
    rng = np.random.default_rng(B * 100 + n)
    prev = rng.integers(0, 2 ** 32, (B, 12 * n), dtype=np.uint64).astype(np.uint32).view(np.float32)
    cur = rng.integers(0, 2 ** 32, (B, 12 * n), dtype=np.uint64).astype(np.uint32).view(np.float32)
    before = cur.copy()
    L.emul_carry(_p(mask), B, n, _p(prev), _p(cur))
    on = mask != 0
    assert np.array_equal(_bits(cur[on]), _bits(before[on]))       # listed rows: untouched
    assert np.array_equal(_bits(cur[~on]), _bits(prev[~on]))       # unlisted rows: the previous buffer's, byte for byte


def test_carry_source_has_no_data_races():
    """The ThreadSanitizer build of the carry (every CTA's threads at once): no two threads touch the same bytes."""
    exe, r = _carry_build("carry_tsan", ["-O1", "-g", "-fsanitize=thread", "-DHMPC_CARRY_MAIN"])
    if r.returncode != 0:
        pytest.skip("no ThreadSanitizer runtime with this toolchain: " + r.stderr[-300:])
    run = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0 and run.stdout.strip() == "ok", run.stdout + run.stderr[-3000:]
    assert "ThreadSanitizer" not in run.stderr, run.stderr[-3000:]


def test_sharded_warm_calls_reject_a_null_context():
    L = interface.lib()
    assert L.hmpc_solve_batch_sharded_warm(None, None, 1, None, None, None, None, None, None) == interface.HMPC_ERR_ARG
    assert L.hmpc_solve_batch_states_sharded_warm(None, None, 1, None, 0.04, None, None, None, None, None) == interface.HMPC_ERR_ARG


# ---- CPU: ShardedMPC's warm ticks over gloo -------------------------------------------------------------------------------
def _due(n, t, never):
    m = (np.arange(n) + t) % 5 == 0
    m[never] = False
    return m


def _tick_records(g, n, t):
    """robot i's record at tick t: golden record (i + 3t) % 64, so that every tick changes each robot's problem"""
    return (np.arange(n) + 3 * t) % len(g["records"])


def _gloo_worker(rank, world, port, n, never, ticks, q):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g = load_golden("cfg3_h10")
    keys = [bytes(r) for r in g["records"].view(np.uint8).reshape(len(g["records"]), -1)]
    seen = []

    def solve_local(recs):   # the golden fixture's oracle solutions stand in for the local solve
        rows = [keys.index(bytes(r)) for r in recs.view(np.uint8).reshape(len(recs), -1)]
        seen.append(rows)
        return g["q_soln"][rows], g["info"][rows, 1].astype(np.int32)

    sh = sharding.ShardedMPC(n, N, rank, world, lambda b: sharding.TorchBackend(b, N, world, solve_local),
                             scenarios.UPDATE_DTYPE, warm=True)
    lo, hi = sh.bounds[rank]
    latest = np.zeros((n, 12 * N), np.float32)
    ok = sh.b_local > hi - lo or rank == 0        # rank 1 holds the padded tail
    for t in range(ticks):
        idx = _tick_records(g, n, t)
        due = _due(n, t, never)
        shift = np.where(np.arange(n) % 3 == 0, -1, 1).astype(np.int32)
        seen.clear()
        w, s = sh.tick(g["records"][idx[lo:hi]], mask=due[lo:hi], shift=shift[lo:hi])
        mine = due[lo:hi]
        # the solver saw this rank's listed robots, in order, and nothing else (no padded row)
        ok &= (seen == [list(idx[lo:hi][mine])]) if mine.any() else (seen == [])
        ok &= np.array_equal(w[mine], g["q_soln"][idx[lo:hi][mine]])
        latest[due] = g["q_soln"][idx[due]].astype(np.float32)
        whole = sh.whole_batch()
        ok &= whole.shape == (n, 12 * N) and np.array_equal(whole, latest)
    ok &= not latest[never].any()                  # the never-due robot is gathered as zeros
    sh.close()
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_warm_ticks_gather_every_robots_latest_row():
    """Two ranks, 13 robots (slices of 7 and 6: rank 1 pads one row), robot i due at tick t when (i + t) % 5 == 0, robot 4
    never due, 9 ticks: after every tick whole_batch() is each robot's latest solution (zeros for robot 4) on both ranks,
    and the solver only ever sees the listed robots."""
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, 13, 4, 9, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


# ---- GPU: the library, one-rank NCCL group --------------------------------------------------------------------------------
MODES = ["in_place", "staged"]


def _walker_records(B, T, seed):
    """T ticks of a logged device rollout of B walkers, as update_data_t records"""
    import torch

    from test_rollout import _to_dev, _walkers

    states, loop = _walkers(B, seed=seed)
    roll = interface.BatchedMPC(B, N)
    d_rlog = torch.zeros((T, B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    roll.rollout_device(_to_dev(states), _to_dev(loop), B, T, None, d_rlog)
    torch.cuda.synchronize()
    roll.close()
    log = d_rlog.cpu().numpy()
    return [interface.unpack_records(log[t], N) for t in range(T)]


class _Side:
    """One context and its caller arrays: x (records or states), wrench, status; pinned in place, plain when staged."""

    def __init__(self, B, dtype, mode, sharded):
        self.mpc = interface.BatchedMPC(B, N)
        if sharded:
            self.mpc.shard_init(0, 1, interface.BatchedMPC.shard_unique_id())
        alloc = interface.page_aligned if mode == "in_place" else (lambda shape, dt: np.zeros(shape, dt))
        self.x = alloc((B,), dtype)
        self.w = alloc((B, 12 * N), np.float64)
        self.s = alloc((B,), np.int32)
        if mode == "in_place":
            self.mpc.pin(self.x, self.w, self.s)

    def close(self):
        self.mpc.close()


def _d_all(B):
    """a device buffer of NaNs, written before the library's gather stream can touch it"""
    import torch

    d = torch.full((B, 12 * N), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    return d


def _gathered(side, d_all):
    side.mpc.shard_wait()
    return d_all.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_unmasked_sharded_warm_equals_the_warm_call(mode):
    """12 ticks of 300 logged walkers: the sharded call without a mask is hmpc_solve_batch_warm — wrenches, torques and
    status words bit for bit — and d_all is the float rounding of the wrenches."""
    B, T = 300, 12
    ticks = _walker_records(B, T, seed=61)
    a = _Side(B, scenarios.UPDATE_DTYPE, mode, True)
    b = _Side(B, scenarios.UPDATE_DTYPE, mode, False)
    d_all = _d_all(B)
    for t in range(T):
        a.x[:] = ticks[t]
        b.x[:] = ticks[t]
        _, ta, _ = a.mpc.solve_batch_sharded_warm(a.x, (a.w, a.s), d_all, torques=True)
        _, tb, _ = b.mpc.solve_batch_warm(b.x, torques=True, out=(b.w, b.s))
        assert np.array_equal(_bits(a.w), _bits(b.w)) and np.array_equal(_bits(ta), _bits(tb)), t
        assert np.array_equal(a.s, b.s) and (interface.status_code(a.s) == 0).all(), t
        assert np.array_equal(_bits(_gathered(a, d_all)), _bits(a.w.astype(np.float32))), t
    a.close()
    b.close()


def _staggered(B, T, seed):
    """masks (robot i due at tick t when (i + t) % 5 == 0; robots 7, 8, 9 and every 97th never) and shifts (some -1)"""
    rng = np.random.default_rng(seed)
    never = np.zeros(B, bool)
    never[[7, 8, 9]] = True
    never[::97] = True
    masks = [(((np.arange(B) + t) % 5 == 0) & ~never).astype(np.uint8) for t in range(T)]
    shifts = [np.where(rng.random(B) < 0.1, -1, 1).astype(np.int32) for _ in range(T)]
    return masks, shifts, never


def _masked_run(a, b, xs, masks, shifts, sharded_call, plain_call):
    """the sharded call on `a` with d_all, the plain masked call on `b`, tick by tick: listed rows identical, unlisted host
    rows keep their bytes, d_all rows the latest row or zeros"""
    B = len(masks[0])
    d_all = _d_all(B)
    latest = np.zeros((B, 12 * N), np.float32)
    a.w[:] = np.nan
    a.s[:] = 0x5A5A5A5A
    b.w[:] = np.nan
    b.s[:] = 0x5A5A5A5A
    for t, (x, m, sh) in enumerate(zip(xs, masks, shifts)):
        on = m != 0
        a.x[:] = x
        b.x[:] = x
        wa0, sa0 = a.w.copy(), a.s.copy()
        _, ta, _ = sharded_call(a, d_all, m, sh)
        _, tb, _ = plain_call(b, m, sh)
        assert np.array_equal(_bits(a.w[on]), _bits(b.w[on])) and np.array_equal(_bits(ta[on]), _bits(tb[on])), t
        assert np.array_equal(a.s[on], b.s[on]) and (interface.status_code(a.s[on]) == 0).all(), t
        assert np.array_equal(_bits(a.w[~on]), _bits(wa0[~on])) and np.array_equal(a.s[~on], sa0[~on]), t
        latest[on] = a.w[on].astype(np.float32)
        assert np.array_equal(_bits(_gathered(a, d_all)), _bits(latest)), t
    return latest


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_staggered_sharded_warm_equals_the_masked_call(mode):
    """15 ticks of 1000 logged walkers with staggered masks, resets (shift -1) and a never-due group, against
    hmpc_solve_batch_masked on a second context; the never-due robots are gathered as zeros throughout."""
    B, T = 1000, 15
    ticks = _walker_records(B, T, seed=62)
    masks, shifts, never = _staggered(B, T, 63)
    a = _Side(B, scenarios.UPDATE_DTYPE, mode, True)
    b = _Side(B, scenarios.UPDATE_DTYPE, mode, False)
    latest = _masked_run(
        a, b, ticks, masks, shifts,
        lambda s, d, m, sh: s.mpc.solve_batch_sharded_warm(s.x, (s.w, s.s), d, mask=m, shift=sh, torques=True),
        lambda s, m, sh: s.mpc.solve_batch_masked(s.x, m, shift=sh, torques=True, out=(s.w, s.s)))
    assert not latest[never].any()
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_staggered_states_sharded_warm_equals_the_states_masked_call(mode):
    """The states variant: 10 ticks of 600 robot states with staggered masks and resets, against
    hmpc_solve_batch_states_masked."""
    B, T = 600, 10
    xs = []
    for t in range(T):
        _, inputs = scenarios.make_batch(2, B, horizon=N, seed=700 + t)
        xs.append(np.ascontiguousarray(scenarios.make_states(inputs, N)))
    masks, shifts, never = _staggered(B, T, 64)
    a = _Side(B, scenarios.STATE_DTYPE, mode, True)
    b = _Side(B, scenarios.STATE_DTYPE, mode, False)
    latest = _masked_run(
        a, b, xs, masks, shifts,
        lambda s, d, m, sh: s.mpc.solve_batch_sharded_warm(s.x, (s.w, s.s), d, mask=m, shift=sh, torques=True),
        lambda s, m, sh: s.mpc.solve_batch_states_masked(s.x, m, shift=sh, torques=True, out=(s.w, s.s)))
    assert not latest[never].any()
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_cold_sharded_calls_keep_the_gather_rows_current(mode):
    """A cold hmpc_solve_batch_sharded with d_all, then a masked warm call: its unlisted rows are the cold call's results.
    A cold call without d_all, then a masked warm call: its unlisted rows are that cold call's results.  An all-zero mask
    solves nothing and gathers the latest rows."""
    import torch

    B = 400
    ticks = _walker_records(B, 4, seed=65)
    a = _Side(B, scenarios.UPDATE_DTYPE, mode, True)
    d_all = _d_all(B)
    m = ((np.arange(B) % 3) == 0).astype(np.uint8)
    on = m != 0
    for t, gather_cold in ((0, True), (2, False)):
        a.x[:] = ticks[t]
        a.mpc.solve_batch_sharded(a.x, (a.w, a.s), d_all if gather_cold else None)
        cold = a.w.astype(np.float32)
        if gather_cold:
            assert np.array_equal(_bits(_gathered(a, d_all)), _bits(cold)), t
        a.x[:] = ticks[t + 1]
        a.mpc.solve_batch_sharded_warm(a.x, (a.w, a.s), d_all, mask=m)
        g = _gathered(a, d_all)
        assert np.array_equal(_bits(g[~on]), _bits(cold[~on])), t
        assert np.array_equal(_bits(g[on]), _bits(a.w[on].astype(np.float32))), t
        assert not np.array_equal(_bits(g[on]), _bits(cold[on])), t      # the ticks differ: the rows are told apart
        latest = g.copy()
        d_all.fill_(float("nan"))
        torch.cuda.synchronize()
        w0 = a.w.copy()
        a.mpc.solve_batch_sharded_warm(a.x, (a.w, a.s), d_all, mask=np.zeros(B, np.uint8))
        assert np.array_equal(_bits(_gathered(a, d_all)), _bits(latest)) and np.array_equal(_bits(a.w), _bits(w0)), t
    a.close()


@pytest.mark.gpu
def test_sharded_warm_calls_check_their_arguments():
    """Before hmpc_shard_init, B_local < 1, B_local > capacity and NULL records or states are argument errors."""
    L = interface.lib()
    ERR = interface.HMPC_ERR_ARG
    mpc = interface.BatchedMPC(64, N)
    recs = np.zeros(65, scenarios.UPDATE_DTYPE)
    states = np.zeros(65, scenarios.STATE_DTYPE)
    w = np.zeros((65, 12 * N))
    s = np.zeros(65, np.int32)
    m = np.ones(65, np.uint8)

    def rec_call(x, B):
        return L.hmpc_solve_batch_sharded_warm(mpc._h, x, B, m.ctypes.data, w.ctypes.data, None, s.ctypes.data, None, None)

    def st_call(x, B):
        return L.hmpc_solve_batch_states_sharded_warm(mpc._h, x, B, m.ctypes.data, 0.04, w.ctypes.data, None, s.ctypes.data,
                                                      None, None)

    assert rec_call(recs.ctypes.data, 4) == ERR and st_call(states.ctypes.data, 4) == ERR      # no hmpc_shard_init yet
    assert b"hmpc_shard_init" in L.hmpc_last_error()
    mpc.shard_init(0, 1, interface.BatchedMPC.shard_unique_id())
    for call, x in ((rec_call, recs.ctypes.data), (st_call, states.ctypes.data)):
        assert call(x, 0) == ERR and call(x, -1) == ERR and call(x, 65) == ERR and call(None, 4) == ERR
    assert L.hmpc_solve_batch_sharded_warm(mpc._h, recs.ctypes.data, 4, m.ctypes.data, None, None, s.ctypes.data, None,
                                           None) == ERR
    mpc.close()
