"""Solving part of the batch: hmpc_solve_device_masked, hmpc_solve_batch_masked, BatchedMPC.solve_device_masked and
BatchedMPC.solve_batch_masked solve robot i iff mask[i] != 0 and leave every other robot's results and working set alone.

CPU: the kernel source (tests/host_emul/kernel_source_on_host.cpp) — the selection kernel gives np.flatnonzero(mask) on one
emulated CTA (also under ThreadSanitizer), and a masked solve of walking and double-support robots gives the listed robots
a full solve's results, status words and working sets while the unlisted keep sentinel bytes.  GPU: the library — a full
mask against hmpc_solve_device_warm, random masks on a batch that reaches classes 1 and 2, a staggered warm loop against
one context per phase group, refinement, a captured graph replayed with other masks, the three host-buffer modes and the
argument checks."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, load_golden
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import _p, emul_solve, host_emulation, race_driver

N = 10
W_SENT, S_SENT, WS_SENT = np.uint32(0x7FA5A5A5), np.int32(0x5A5A5A5A), np.int32(0x3C3C3C3C)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint8)


# ---- CPU: the kernel source on the host ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul():
    return host_emulation()


def _select(L, mask):
    mask = np.ascontiguousarray(mask, np.uint8)
    B = len(mask)
    lst = np.full(B, -7, np.int32)
    cnt = np.full(1, -7, np.int32)
    L.emul_select(_p(mask), B, _p(lst), _p(cnt))
    return lst, int(cnt[0])


def _select_masks():
    rng = np.random.default_rng(3)
    out = [("B1_off", np.zeros(1, np.uint8)), ("B1_on", np.ones(1, np.uint8))]
    for B in (37, 512, 1300):
        out += [("empty_%d" % B, np.zeros(B, np.uint8)), ("full_%d" % B, np.ones(B, np.uint8))]
        for p in (0.2, 0.5):
            m = (rng.random(B) < p).astype(np.uint8) * rng.integers(1, 256, B).astype(np.uint8)   # any non-zero byte lists
            out.append(("random_%d_%g" % (B, p), m))
    return out


@pytest.mark.parametrize("name,mask", _select_masks(), ids=[n for n, _ in _select_masks()])
def test_select_source_gives_the_listed_robots_in_order(emul, name, mask):
    """One emulated CTA of the selection kernel: the list is np.flatnonzero(mask), ascending, and its length word is the
    count.  Covers B = 1, empty and full masks, and batches that are not a multiple of the tile."""
    lst, cnt = _select(emul, mask)
    want = np.flatnonzero(mask)
    assert cnt == len(want)
    assert np.array_equal(lst[:cnt], want)
    assert (lst[cnt:] == -7).all()          # nothing is written past the list


def test_select_source_has_no_data_races(emul, tmp_path):
    """ThreadSanitizer build of the selection kernel (every CUDA thread an OS thread, every barrier real) on masks of 1 to
    1300 robots and four densities."""
    exe = race_driver()
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66")
    r = subprocess.run([exe, "select"], capture_output=True, text=True, env=env, timeout=1800)
    assert "ThreadSanitizer" not in r.stderr, r.stderr[:3000]
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout)


def _emul_full(L, packed, ws, shifts):
    w, st, la = emul_solve(L, N, packed, ws=ws, warm=True, shifts=shifts)
    return w, st, la[:3]


def _emul_masked(L, packed, mask, ws, shifts, w, st):
    _, _, la = emul_solve(L, N, packed, mask=np.ascontiguousarray(mask, np.uint8), ws=ws, warm=True, shifts=shifts, w=w, st=st)
    return la[:3]


def test_masked_source_solves_the_listed_robots_only(emul):
    """Walking and standing robots of cfg3_h10 (the standing ones reach class 1).  Two calls: a cold one (shift -1, records
    the sets) and a warm one (shift 0, proposes them).  Listed robots get the full solve's wrench, status and working set
    bit for bit; unlisted robots' wrench rows, status words and working-set slots keep their sentinel bytes."""
    g = load_golden("cfg3_h10")
    B = 10
    packed = np.ascontiguousarray(interface.pack_records(g["records"][:B], N))
    mask = np.array([1, 0, 1, 1, 0, 1, 0, 1, 1, 0], np.uint8)
    on = mask != 0
    W = emul.emul_ws_ints()
    ws_full = np.full((B, W), WS_SENT, np.int32)   # (a recorded set overwrites the count and its entries only)
    ws_m = ws_full.copy()
    w_m = np.full((B, 12 * N), W_SENT, np.uint32).view(np.float32)
    st_m = np.full(B, S_SENT, np.int32)
    for shift in (-1, 0):
        shifts = np.full(B, shift, np.int32)
        w_f, st_f, la_f = _emul_full(emul, packed, ws_full, shifts)
        la_m = _emul_masked(emul, packed, mask, ws_m, shifts, w_m, st_m)
        assert la_f[1] > 0 and la_m[1] > 0, (la_f, la_m)                # class 1 is reached
        assert la_m[0] + la_m[1] == on.sum()
        assert np.array_equal(_bits(w_m[on]), _bits(w_f[on])) and np.array_equal(st_m[on], st_f[on]), shift
        assert np.array_equal(ws_m[on], ws_full[on]), shift
        assert (_bits(w_m[~on]) == W_SENT).all() and (st_m[~on] == S_SENT).all() and (ws_m[~on] == WS_SENT).all()
        assert (interface.status_code(st_m[on]) == 0).all()


def test_masked_calls_reject_a_null_context():
    L = interface.lib()
    assert L.hmpc_solve_device_masked(None, None, 1, None, None, None, None, None, None) == interface.HMPC_ERR_ARG
    assert L.hmpc_solve_batch_masked(None, None, 1, None, None, None, None, None) == interface.HMPC_ERR_ARG


# ---- GPU: the library -----------------------------------------------------------------------------------------------------
def _mix(B, seed, ndeg=12):
    """walking and standing robots of one cfg-3 pool and `ndeg` copies of the degenerate record (escalates to class 2)"""
    pool, _ = scenarios.make_batch(3, B + B // 2, horizon=N, seed=seed)
    deg = load_golden("degenerate_zero_force_h10")["records"][0]
    rng = np.random.default_rng(seed + 1)
    recs = pool[rng.choice(len(pool), B, replace=False)]
    at = rng.choice(B, ndeg, replace=False)
    recs[at] = deg
    return recs, at


def _sentinels(B, torch):
    w = torch.from_numpy(np.full((B, 12 * N), W_SENT, np.uint32).view(np.float32)).cuda()
    tau = torch.from_numpy(np.full((B, 10), W_SENT, np.uint32).view(np.float32)).cuda()
    s = torch.full((B,), int(S_SENT), dtype=torch.int32, device="cuda")
    return w, tau, s


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


@pytest.mark.gpu
def test_full_mask_equals_the_warm_solve():
    """A mask that lists every robot is hmpc_solve_device_warm: wrenches, torques and status words bit for bit over three
    calls with per-robot shifts (resets, same horizon, one step), so the working sets it records lead to the same next call."""
    import torch

    B = 2048
    recs, _ = _mix(B, 21)
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    rng = np.random.default_rng(22)
    for call in range(3):
        shift = torch.from_numpy(rng.integers(-1, 2, B).astype(np.int32)).cuda() if call else None
        wa, ta, sa = _sentinels(B, torch)
        wb, tb, sb = _sentinels(B, torch)
        a.solve_device_masked(d_rec, B, mask, wa, sa, d_tau=ta, d_shift=shift)
        b.solve_device_warm(d_rec, B, wb, sb, d_tau=tb, d_shift=shift)
        torch.cuda.synchronize()
        wa, ta, sa, wb, tb, sb = _np(wa, ta, sa, wb, tb, sb)
        assert np.array_equal(_bits(wa), _bits(wb)) and np.array_equal(_bits(ta), _bits(tb)) and np.array_equal(sa, sb), call
        assert (sa != S_SENT).all(), call
    a.close()
    b.close()


@pytest.mark.gpu
def test_random_masks_reach_all_classes_and_leave_the_rest():
    """4096 robots (more than two waves of class 0) with double-support robots (class 1) and degenerate ones (class 2).
    Random masks of 5 %, 20 %, 60 % and 100 %: with shift -1 (a cold solve) listed rows equal hmpc_solve_device_ex of the
    whole batch bit for bit, unlisted rows keep their sentinels.  Among the listed robots classes 1 and 2 are reached."""
    import torch

    B = 4096
    recs, at = _mix(B, 31)
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    a, ref = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    qmax1 = a.class_config(1)["qmax"]
    wf, tf, sf = _sentinels(B, torch)
    interface._check(interface.lib().hmpc_solve_device_ex(ref._h, d_rec.data_ptr(), B, wf.data_ptr(), sf.data_ptr(),
                                                          tf.data_ptr(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    cold = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(32)
    wf, tf, sf = _np(wf, tf, sf)
    blocks = (np.asarray(interface.pack_records(recs, N))[:, (54 + 12 * N) * 4:(54 + 12 * N) * 4 + 2 * N] != 0).sum(1)
    for p in (0.05, 0.2, 0.6, 1.0):
        m = rng.random(B) < p
        m[at[: 6]] = True
        w, tau, s = _sentinels(B, torch)
        a.solve_device_masked(d_rec, B, torch.from_numpy(m).cuda(), w, s, d_tau=tau, d_shift=cold)
        torch.cuda.synchronize()
        w, tau, s = _np(w, tau, s)
        assert np.array_equal(_bits(w[m]), _bits(wf[m])) and np.array_equal(_bits(tau[m]), _bits(tf[m])), p
        assert np.array_equal(s[m], sf[m]), p
        assert (_bits(w[~m]) == W_SENT).all() and (_bits(tau[~m]) == W_SENT).all() and (s[~m] == S_SENT).all(), p
        assert (blocks[m] > N).sum() > 0 and (interface.status_nactive(s[m]) > qmax1).sum() >= 6, p   # classes 1 and 2
    a.close()
    ref.close()


@pytest.mark.gpu
def test_staggered_warm_loop_equals_one_context_per_phase_group():
    """1024 walkers of a logged rollout, split into 5 phase groups (robot i in group i % 5).  Call t solves group t % 5 on
    the records of tick t, with random per-robot shifts (resets included), for 45 calls.  Every call equals, bit for bit
    with status words, one context per group warm-solving its dense sub-batch on the same records and shifts; the other
    groups' rows do not change."""
    import torch

    from test_rollout import _to_dev, _walkers

    B, T, G = 1024, 45, 5
    states, loop = _walkers(B, seed=13)
    roll = interface.BatchedMPC(B, N)
    d_rlog = torch.zeros((T, B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    roll.rollout_device(_to_dev(states), _to_dev(loop), B, T, None, d_rlog)
    torch.cuda.synchronize()
    roll.close()
    groups = [np.arange(g, B, G) for g in range(G)]
    d_groups = [torch.from_numpy(ix).cuda() for ix in groups]
    masked = interface.BatchedMPC(B, N)
    dense = [interface.BatchedMPC(len(ix), N) for ix in groups]
    w, tau, s = _sentinels(B, torch)
    rng = np.random.default_rng(14)
    for t in range(T):
        g = t % G
        ix, d_ix = groups[g], d_groups[g]
        shift = torch.from_numpy(rng.integers(-1, 3, B).astype(np.int32)).cuda()
        mask = torch.zeros(B, dtype=torch.bool, device="cuda")
        mask[d_ix] = True
        before = _np(w, tau, s)
        masked.solve_device_masked(d_rlog[t], B, mask, w, s, d_tau=tau, d_shift=shift)
        n = len(ix)
        wd, td, sd = _sentinels(n, torch)
        dense[g].solve_device_warm(d_rlog[t].index_select(0, d_ix).contiguous(), n, wd, sd, d_tau=td,
                                   d_shift=shift.index_select(0, d_ix).contiguous())
        torch.cuda.synchronize()
        wn, tn, sn = _np(w, tau, s)
        wd, td, sd = _np(wd, td, sd)
        assert np.array_equal(_bits(wn[ix]), _bits(wd)) and np.array_equal(_bits(tn[ix]), _bits(td)), t
        assert np.array_equal(sn[ix], sd), t
        rest = np.setdiff1d(np.arange(B), ix)
        assert np.array_equal(_bits(wn[rest]), _bits(before[0][rest])) and np.array_equal(sn[rest], before[2][rest]), t
        assert (sd != S_SENT).all(), t
    masked.close()
    for d in dense:
        d.close()


def _lying():
    g = np.load(os.path.join(GOLDEN, "stress_referee.npz"))
    return np.ascontiguousarray(g["h10_lying_records"]).view(scenarios.UPDATE_DTYPE).reshape(-1)[0]


@pytest.mark.gpu
def test_refinement_follows_the_mask():
    """Refinement on, h10_lying at robot 17 of 64 configs[1]-style walkers (scaled condition numbers below 400, far from
    the hand-over threshold): listed, it comes back refined and is the only refined robot.  Unlisted, its wrench and
    status keep their sentinels and no robot is refined."""
    import torch

    recs, _ = scenarios.make_batch(2, 64, horizon=N, seed=scenarios.config_seed(2) + 1)
    recs[17] = _lying()
    B = len(recs)
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    mpc = interface.BatchedMPC(B, N)
    mpc.set_refinement(True)
    inside = torch.ones(B, dtype=torch.bool, device="cuda")
    outside = inside.clone()
    outside[17] = False
    w, tau, s = _sentinels(B, torch)
    mpc.solve_device_masked(d_rec, B, inside, w, s, d_tau=tau)
    torch.cuda.synchronize()
    w1, s1 = _np(w, s)
    assert interface.status_code(s1[17]) == 0 and interface.status_refined(s1).tolist() == [0] * 17 + [1] + [0] * 46
    w, tau, s = _sentinels(B, torch)
    mpc.solve_device_masked(d_rec, B, outside, w, s, d_tau=tau)
    torch.cuda.synchronize()
    w2, s2 = _np(w, s)
    assert (_bits(w2[17]) == W_SENT).all() and s2[17] == S_SENT
    others = np.delete(s2, 17)                      # (the sentinel itself has bit 28 set)
    assert interface.status_refined(others).sum() == 0 and (others != S_SENT).all()
    mpc.close()


@pytest.mark.gpu
def test_captured_masked_solve_replays_with_other_masks():
    """One hmpc_solve_device_masked captured in a torch graph and replayed with 6 different masks written into the captured
    mask tensor (records changing too) equals eager masked calls on a second context, bit for bit, outputs carried over
    between calls so that unlisted rows are compared as well."""
    import torch

    B = 4096
    recs, _ = _mix(B, 41)
    sets = [torch.from_numpy(interface.pack_records(np.roll(recs, k * 97), N)).cuda() for k in range(3)]
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    rec = sets[0].clone()
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    w, tau, s = _sentinels(B, torch)
    we, taue, se = _sentinels(B, torch)
    a.solve_device_masked(rec, B, mask, w, s, d_tau=tau)          # loads the kernels outside the capture
    b.solve_device_masked(rec, B, mask, we, se, d_tau=taue)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        a.solve_device_masked(rec, B, mask, w, s, d_tau=tau)
    rng = np.random.default_rng(42)
    for k, p in enumerate((0.2, 0.0, 0.5, 1.0, 0.05, 0.2)):
        m = torch.from_numpy(rng.random(B) < p).cuda()
        rec.copy_(sets[k % 3])
        mask.copy_(m)
        gr.replay()
        b.solve_device_masked(sets[k % 3], B, m, we, se, d_tau=taue)
        torch.cuda.synchronize()
        for x, y in ((w, we), (tau, taue), (s, se)):
            assert np.array_equal(_bits(x.cpu().numpy()), _bits(y.cpu().numpy())), k
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["zero_copy", "copy_pipeline", "copy_pipeline_4", "in_place"])
def test_host_modes_equal_the_device_path(mode, monkeypatch):
    """hmpc_solve_batch_masked against hmpc_solve_device_masked on the same records and masks, two calls (shift NULL, then
    per-robot shifts): listed wrenches rounded to float, torques and status words are equal; unlisted rows of the caller's
    arrays keep their sentinels.  The copy pipeline runs above 1536 robots, in two chunks with helper threads and in four
    without (copy_pipeline_4: HMPC_HOST_THREADS=1); the degenerate records make the host path re-solve overflowed robots."""
    import torch

    if mode == "copy_pipeline_4":
        monkeypatch.setenv("HMPC_HOST_THREADS", "1")   # read by hmpc_create
    B = 1800 if mode.startswith("copy_pipeline") else 300
    recs, at = _mix(B, 51, ndeg=6)
    host, dev = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    if mode == "in_place":
        rin = interface.page_aligned((B,), scenarios.UPDATE_DTYPE)
        rin[:] = recs
        wh = interface.page_aligned((B, 12 * N), np.float64)
        sh = interface.page_aligned((B,), np.int32)
        host.pin(rin, wh, sh)
    else:
        rin = recs
        wh = np.zeros((B, 12 * N), np.float64)
        sh = np.zeros(B, np.int32)
    wd, td, sd = _sentinels(B, torch)
    rng = np.random.default_rng(52)
    for call in range(2):
        m = rng.random(B) < 0.4
        m[at[:3]] = True
        shift = None if call == 0 else rng.integers(-1, 2, B).astype(np.int32)
        wh[:] = np.nan
        sh[:] = S_SENT
        _, tau_h, _ = host.solve_batch_masked(rin, m, shift=shift, torques=True, strict=False, out=(wh, sh))
        dev.solve_device_masked(d_rec, B, torch.from_numpy(m).cuda(), wd, sd, d_tau=td,
                                d_shift=None if shift is None else torch.from_numpy(shift).cuda())
        torch.cuda.synchronize()
        w_, t_, s_ = _np(wd, td, sd)
        assert np.array_equal(_bits(wh[m].astype(np.float32)), _bits(w_[m])), call
        assert np.array_equal(_bits(tau_h[m].astype(np.float32)), _bits(t_[m])) and np.array_equal(sh[m], s_[m]), call
        assert np.isnan(wh[~m]).all() and (sh[~m] == S_SENT).all() and (tau_h[~m] == 0).all(), call
        assert (interface.status_nactive(sh[at[:3]]) > host.class_config(1)["qmax"]).all()
    if mode == "in_place":
        host.unpin(rin, wh, sh)
    host.close()
    dev.close()


@pytest.mark.gpu
def test_masked_calls_check_their_arguments():
    """NULL mask, B < 0 and B > capacity are argument errors, found before anything is enqueued; B = 0 is a no-op; an
    empty mask writes nothing and returns HMPC_OK, on the host too."""
    import torch

    L = interface.lib()
    mpc = interface.BatchedMPC(64, N)
    h = mpc._h
    stride = interface.record_bytes(N)
    d_rec = torch.zeros(65 * stride, dtype=torch.uint8, device="cuda")
    d_w = torch.zeros((65, 12 * N), dtype=torch.float32, device="cuda")
    d_s = torch.full((65,), 7, dtype=torch.int32, device="cuda")
    d_m = torch.zeros(65, dtype=torch.bool, device="cuda")
    p, pw, ps, pm = d_rec.data_ptr(), d_w.data_ptr(), d_s.data_ptr(), d_m.data_ptr()
    ERR, OK = interface.HMPC_ERR_ARG, interface.HMPC_OK
    assert L.hmpc_solve_device_masked(h, p, 4, None, pw, ps, None, None, None) == ERR
    assert L.hmpc_solve_device_masked(h, None, 4, pm, pw, ps, None, None, None) == ERR
    assert L.hmpc_solve_device_masked(h, p, 4, pm, None, ps, None, None, None) == ERR
    assert L.hmpc_solve_device_masked(h, p, 4, pm, pw, None, None, None, None) == ERR
    assert L.hmpc_solve_device_masked(h, p, -1, pm, pw, ps, None, None, None) == ERR
    assert L.hmpc_solve_device_masked(h, p, 65, pm, pw, ps, None, None, None) == ERR
    assert L.hmpc_solve_device_masked(h, p + 4, 4, pm, pw, ps, None, None, None) == ERR
    assert L.hmpc_solve_device_masked(h, p, 0, pm, pw, ps, None, None, None) == OK
    assert L.hmpc_solve_device_masked(h, p, 64, pm, pw, ps, None, None, None) == OK     # empty mask
    torch.cuda.synchronize()
    assert (d_s.cpu().numpy() == 7).all() and (d_w.cpu().numpy() == 0).all()
    recs = np.zeros(65, scenarios.UPDATE_DTYPE)
    w = np.full((65, 12 * N), 3.0)
    s = np.full(65, 7, np.int32)
    m = np.zeros(65, np.uint8)
    assert L.hmpc_solve_batch_masked(h, recs.ctypes.data, 4, None, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_masked(h, None, 4, m.ctypes.data, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_masked(h, recs.ctypes.data, 4, m.ctypes.data, None, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_masked(h, recs.ctypes.data, -1, m.ctypes.data, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_masked(h, recs.ctypes.data, 65, m.ctypes.data, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert L.hmpc_solve_batch_masked(h, recs.ctypes.data, 0, m.ctypes.data, w.ctypes.data, None, s.ctypes.data, None) == OK
    assert L.hmpc_solve_batch_masked(h, recs.ctypes.data, 64, m.ctypes.data, w.ctypes.data, None, s.ctypes.data, None) == OK
    assert (s == 7).all() and (w == 3.0).all()
    mpc.close()
