"""Robot states in, solved the way records are: hmpc_solve_states_device_masked, hmpc_solve_batch_states_warm,
hmpc_solve_batch_states_masked and the in-place mode of the state calls (BatchedMPC.solve_states_device_masked,
solve_batch_states_warm, solve_batch_states_masked).

CPU: the kernel source (tests/host_emul/states_chain_on_host.cpp, on top of kernel_source_on_host.cpp) — the preparation
kernel over an instance list writes the listed robots' records and nothing else, and the emulated states chain (selection ->
preparation over the list -> classes) gives what preparing every robot and then the masked record chain gives.  GPU: the
library — the fused device call against prepare_device + solve_device_masked, a staggered warm loop against the record path
on host-prepared records, a captured graph replayed with other masks and states, the three host-buffer modes and the
argument checks."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import BUILD, DEVICE_HEADER, HERE, _host_buildable, _p, emul_solve

N = 10
_LIB = {}


def states_emulation():
    """tests/host_emul/states_chain_on_host.cpp built for the host as a library, once per process: the kernel source with the
    substitutions and flags of test_kernel_source_on_host.py's build, plus the states chain's entry points."""
    if "lib" not in _LIB:
        os.makedirs(BUILD, exist_ok=True)
        hdr = os.path.join(BUILD, "hmpc_device_host_states.cuh")
        with open(hdr, "w") as f:
            f.write(_host_buildable(open(DEVICE_HEADER).read()))
        out = os.path.join(BUILD, "libstates_chain_on_host.so")
        cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O2", "-fPIC", "-shared",
               "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"), '-DHMPC_DEVICE_HEADER="%s"' % hdr,
               os.path.join(HERE, "states_chain_on_host.cpp"), "-l:libstdc++.so.6", "-o", out]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        _LIB["lib"] = ctypes.CDLL(out)
    return _LIB["lib"]
W_SENT, S_SENT, WS_SENT, R_SENT = np.uint32(0x7FA5A5A5), np.int32(0x5A5A5A5A), np.int32(0x3C3C3C3C), 0xAB


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint8)


def _states(cfg, B, seed):
    _, inputs = scenarios.make_batch(cfg, B, horizon=N, seed=seed)
    return np.ascontiguousarray(scenarios.make_states(inputs, N))


# ---- CPU: the kernel source on the host ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul():
    return states_emulation()


def _prepare(L, states, lst=None):
    B = len(states)
    out = np.full((B, interface.record_bytes(N)), R_SENT, np.uint8)
    if lst is None:
        L.emul_prepare(_p(states), B, N, ctypes.c_double(0.04), _p(out))
    else:
        lst = np.ascontiguousarray(lst, np.int32)
        cnt = np.array([len(lst)], np.int32)
        buf = np.full(max(B, 1), -7, np.int32)            # the list lives in a batch-sized region, as class 0's does
        buf[:len(lst)] = lst
        L.emul_prepare_list(_p(states), B, N, ctypes.c_double(0.04), _p(out), _p(buf), _p(cnt))
    return out


def _lists():
    rng = np.random.default_rng(5)
    out = []
    for B in (1, 37, 64, 150):
        out += [("empty_%d" % B, B, np.zeros(0, np.int32)), ("full_%d" % B, B, np.arange(B, dtype=np.int32))]
        for p in (0.2, 0.6):
            out.append(("random_%d_%g" % (B, p), B, np.flatnonzero(rng.random(B) < p).astype(np.int32)))
    return out


@pytest.mark.parametrize("name,B,lst", _lists(), ids=[n for n, _, _ in _lists()])
def test_prepare_source_over_a_list_writes_the_listed_records_only(emul, name, B, lst):
    """Preparation over an instance list: listed records are byte-identical to the preparation of every robot, unlisted
    rows keep their sentinel.  B = 1, batches that are and are not a multiple of the 64-thread block, empty and full lists."""
    states = _states(3, B, 61)
    full = _prepare(emul, states)
    got = _prepare(emul, states, lst)
    on = np.zeros(B, bool)
    on[lst] = True
    assert np.array_equal(got[on], full[on])
    assert (got[~on] == R_SENT).all()


def _emul_states(L, states, mask, ws, shifts, w, st, rec):
    la = np.zeros(4, np.int32)
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    rc = L.emul_solve_states(_p(states), ctypes.c_double(0.04), _p(rec), len(states), N, 0, _p(m), _p(ws), 1, 1, _p(shifts),
                             _p(w), None, _p(st), None, _p(la))
    assert rc == 0, rc
    return la


def test_states_chain_source_equals_prepare_then_masked_chain(emul):
    """Walking and standing robots (the standing ones reach class 1), three calls with random masks: a cold one (shift -1,
    records the sets), then warm ones (shift 0 and 1).  The emulated states chain gives the listed robots the wrench, status
    word, working set and record that preparing every robot and then the masked record chain gives, bit for bit.  Unlisted
    robots' wrench rows, status words, working-set slots and record rows keep their sentinel bytes."""
    B = 12
    states = _states(3, B, 62)
    packed = _prepare(emul, states)
    W = emul.emul_ws_ints()
    ws_r = np.full((B, W), WS_SENT, np.int32)
    ws_s = ws_r.copy()
    w_r = np.full((B, 12 * N), W_SENT, np.uint32).view(np.float32)
    st_r = np.full(B, S_SENT, np.int32)
    w_s, st_s = w_r.copy(), st_r.copy()
    rng = np.random.default_rng(63)
    reached = 0
    for call, shift in enumerate((-1, 0, 1)):
        mask = (rng.random(B) < 0.6).astype(np.uint8)
        mask[call] = 1
        on = mask != 0
        shifts = np.full(B, shift, np.int32)
        before = (w_s.copy(), st_s.copy(), ws_s.copy())
        _, _, la_r = emul_solve(emul, N, packed, mask=mask, ws=ws_r, warm=True, shifts=shifts, w=w_r, st=st_r)
        rec = np.full_like(packed, R_SENT)
        la_s = _emul_states(emul, states, mask, ws_s, shifts, w_s, st_s, rec)
        assert np.array_equal(la_s, la_r), call
        reached += la_s[1]
        assert np.array_equal(rec[on], packed[on]) and (rec[~on] == R_SENT).all(), call
        assert np.array_equal(_bits(w_s[on]), _bits(w_r[on])) and np.array_equal(st_s[on], st_r[on]), call
        assert np.array_equal(ws_s[on], ws_r[on]), call
        assert np.array_equal(_bits(w_s[~on]), _bits(before[0][~on])) and np.array_equal(st_s[~on], before[1][~on]), call
        assert np.array_equal(ws_s[~on], before[2][~on]), call
        assert (interface.status_code(st_s[on]) == 0).all(), call
    assert reached > 0                                              # class 1 was reached
    assert (_bits(w_s[st_s == S_SENT]) == W_SENT).all()


def test_unmasked_states_chain_source_equals_the_record_chain(emul):
    """Without a mask the states chain prepares every robot, then runs the device-resident chain: the in-place mode of
    hmpc_solve_batch_states.  Its results equal the record chain on the prepared records, bit for bit."""
    B = 9
    states = _states(3, B, 64)
    packed = _prepare(emul, states)
    w_r, st_r, la_r = emul_solve(emul, N, packed)
    w_s = np.zeros((B, 12 * N), np.float32)
    st_s = np.full(B, -1, np.int32)
    rec = np.full_like(packed, R_SENT)
    la_s = _emul_states(emul, states, None, None, None, w_s, st_s, rec)
    assert np.array_equal(la_s, la_r) and np.array_equal(rec, packed)
    assert np.array_equal(_bits(w_s), _bits(w_r)) and np.array_equal(st_s, st_r)


def test_state_calls_reject_a_null_context():
    L = interface.lib()
    assert L.hmpc_solve_states_device_masked(None, None, 1, None, 0.04, None, None, None, None, None, None) == interface.HMPC_ERR_ARG
    assert L.hmpc_solve_batch_states_warm(None, None, 1, 0.04, None, None, None, None) == interface.HMPC_ERR_ARG
    assert L.hmpc_solve_batch_states_masked(None, None, 1, None, 0.04, None, None, None, None) == interface.HMPC_ERR_ARG


# ---- GPU: the library -----------------------------------------------------------------------------------------------------
def _sentinels(B, torch):
    w = torch.from_numpy(np.full((B, 12 * N), W_SENT, np.uint32).view(np.float32)).cuda()
    tau = torch.from_numpy(np.full((B, 10), W_SENT, np.uint32).view(np.float32)).cuda()
    s = torch.full((B,), int(S_SENT), dtype=torch.int32, device="cuda")
    return w, tau, s


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _dev_states(states):
    import torch

    return torch.from_numpy(np.ascontiguousarray(states).view(np.uint8).reshape(len(states), 352).copy()).cuda()


@pytest.mark.gpu
def test_fused_call_equals_prepare_then_masked_solve():
    """4096 walking and standing robots, five calls with full, empty and random masks on two contexts: the fused call
    against hmpc_prepare_device of every robot + hmpc_solve_device_masked.  Listed rows of records, wrench, torques and
    status are bit-identical; unlisted rows keep their sentinels (the records' too)."""
    import torch

    B = 4096
    states = _states(3, B, 71)
    d_states = _dev_states(states)
    stride = interface.record_bytes(N)
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    rng = np.random.default_rng(72)
    d_rec_b = torch.zeros((B, stride), dtype=torch.uint8, device="cuda")
    b.prepare_device(d_states, B, d_rec_b)
    for k, p in enumerate((1.0, 0.0, 0.2, 0.6, 0.05)):
        m = rng.random(B) < p
        d_m = torch.from_numpy(m).cuda()
        d_rec_a = torch.full((B, stride), R_SENT, dtype=torch.uint8, device="cuda")
        wa, ta, sa = _sentinels(B, torch)
        wb, tb, sb = _sentinels(B, torch)
        a.solve_states_device_masked(d_states, B, d_m, d_rec_a, wa, sa, d_tau=ta)
        b.solve_device_masked(d_rec_b, B, d_m, wb, sb, d_tau=tb)
        torch.cuda.synchronize()
        ra, rb, wa, ta, sa, wb, tb, sb = _np(d_rec_a, d_rec_b, wa, ta, sa, wb, tb, sb)
        assert np.array_equal(ra[m], rb[m]) and (ra[~m] == R_SENT).all(), k
        assert np.array_equal(_bits(wa[m]), _bits(wb[m])) and np.array_equal(_bits(ta[m]), _bits(tb[m])), k
        assert np.array_equal(sa[m], sb[m]), k
        assert (_bits(wa[~m]) == W_SENT).all() and (_bits(ta[~m]) == W_SENT).all() and (sa[~m] == S_SENT).all(), k
        if p == 1.0:
            blocks = (ra[:, (54 + 12 * N) * 4:(54 + 12 * N) * 4 + 2 * N] != 0).sum(1)
            assert (blocks > N).sum() > 0 and (interface.status_code(sa) == 0).all()   # class 1 is reached
    a.close()
    b.close()


@pytest.mark.gpu
def test_staggered_warm_loop_equals_the_record_path():
    """1024 walkers over 45 ticks of a device rollout; robot i is due at tick t when (i + t) % 5 == 0, and about one robot
    in twenty is reset (shift -1) when it is due.  The fused call on the tick's states equals hmpc_solve_device_masked on
    records the host mirror of the reference's preparation built, bit for bit, with status words; rows of robots that are
    not due do not change."""
    import torch

    from test_rollout import _to_dev, _walkers
    from test_state_prepare import _host_prepared

    B, T = 1024, 45
    states0, loop = _walkers(B, seed=17)
    roll = interface.BatchedMPC(B, N)
    d_st, d_loop = _to_dev(states0), _to_dev(loop)
    ticks = []
    for t in range(T):
        ticks.append(d_st.clone())
        roll.rollout_device(d_st, d_loop, B, 1)
    torch.cuda.synchronize()
    roll.close()
    fused, rec = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    d_records = torch.zeros((B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    wf, tf, sf = _sentinels(B, torch)
    wr, tr, sr = _sentinels(B, torch)
    rng = np.random.default_rng(18)
    for t in range(T):
        due = (np.arange(B) + t) % 5 == 0
        shift = np.where(rng.random(B) < 0.05, -1, 1).astype(np.int32)
        st_np = ticks[t].cpu().numpy().view(scenarios.STATE_DTYPE).reshape(B)
        recs = np.zeros(B, scenarios.UPDATE_DTYPE)
        recs[due] = _host_prepared(st_np[due], N)
        d_m, d_sh = torch.from_numpy(due).cuda(), torch.from_numpy(shift).cuda()
        before = _np(wf, sf)
        fused.solve_states_device_masked(ticks[t], B, d_m, d_records, wf, sf, d_tau=tf, d_shift=d_sh)
        rec.solve_device_masked(torch.from_numpy(interface.pack_records(recs, N)).cuda(), B, d_m, wr, sr, d_tau=tr, d_shift=d_sh)
        torch.cuda.synchronize()
        a, b = _np(wf, tf, sf), _np(wr, tr, sr)
        for x, y in zip(a, b):
            assert np.array_equal(_bits(x), _bits(y)), t
        assert np.array_equal(_bits(a[0][~due]), _bits(before[0][~due])) and np.array_equal(a[2][~due], before[1][~due]), t
        assert (a[2][due] != S_SENT).all(), t
    fused.close()
    rec.close()


@pytest.mark.gpu
def test_captured_fused_call_replays_with_other_masks_and_states():
    """One hmpc_solve_states_device_masked captured in a torch graph and replayed with three other masks written into the
    captured mask tensor and other states written into the captured states tensor equals eager fused calls on a second
    context, bit for bit: records, wrench, torques and status, carried over between calls so that unlisted rows count."""
    import torch

    B = 2048
    sets = [_dev_states(_states(3, B, 81 + k)) for k in range(3)]
    stride = interface.record_bytes(N)
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    st = sets[0].clone()
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    ra = torch.full((B, stride), R_SENT, dtype=torch.uint8, device="cuda")
    rb = ra.clone()
    w, tau, s = _sentinels(B, torch)
    we, taue, se = _sentinels(B, torch)
    a.solve_states_device_masked(st, B, mask, ra, w, s, d_tau=tau)      # loads the kernels outside the capture
    b.solve_states_device_masked(st, B, mask, rb, we, se, d_tau=taue)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        a.solve_states_device_masked(st, B, mask, ra, w, s, d_tau=tau)
    rng = np.random.default_rng(82)
    for k, p in enumerate((0.2, 0.0, 0.6)):
        m = torch.from_numpy(rng.random(B) < p).cuda()
        st.copy_(sets[(k + 1) % 3])
        mask.copy_(m)
        gr.replay()
        b.solve_states_device_masked(sets[(k + 1) % 3], B, m, rb, we, se, d_tau=taue)
        torch.cuda.synchronize()
        for x, y in ((ra, rb), (w, we), (tau, taue), (s, se)):
            assert np.array_equal(_bits(x.cpu().numpy()), _bits(y.cpu().numpy())), k
    a.close()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("call", ["warm", "masked"])
@pytest.mark.parametrize("mode", ["zero_copy", "copy_pipeline", "in_place"])
def test_host_modes_equal_the_record_path(mode, call):
    """hmpc_solve_batch_states_warm / _masked against hmpc_solve_batch_warm / _masked on records the host mirror prepared
    from the same states, two calls (shift NULL, then per-robot shifts with resets).  Listed wrench (in place: rounded to
    float), torque and status rows are equal; unlisted rows of the caller's arrays keep their sentinels.  In place with pinned page_aligned arrays,
    zero-copy at 300 robots, the copy pipeline at 1800 robots in two chunks."""
    from test_state_prepare import _host_prepared

    B = 1800 if mode == "copy_pipeline" else 300
    states = _states(3, B, 91)
    recs = _host_prepared(states, N)
    st, rc = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    if mode == "in_place":
        sin = interface.page_aligned((B,), scenarios.STATE_DTYPE)
        sin[:] = states
        wh = interface.page_aligned((B, 12 * N), np.float64)
        sh = interface.page_aligned((B,), np.int32)
        st.pin(sin, wh, sh)
    else:
        sin = states
        wh = np.zeros((B, 12 * N), np.float64)
        sh = np.zeros(B, np.int32)
    wr = np.zeros((B, 12 * N), np.float64)
    sr = np.zeros(B, np.int32)
    rng = np.random.default_rng(92)
    for k in range(2):
        m = rng.random(B) < 0.4 if call == "masked" else np.ones(B, bool)
        shift = None if k == 0 else rng.integers(-1, 2, B).astype(np.int32)
        wh[:] = np.nan
        sh[:] = S_SENT
        wr[:] = np.nan
        sr[:] = S_SENT
        if call == "masked":
            _, tau_h, _ = st.solve_batch_states_masked(sin, m, shift=shift, torques=True, strict=False, out=(wh, sh))
            _, tau_r, _ = rc.solve_batch_masked(recs, m, shift=shift, torques=True, strict=False, out=(wr, sr))
        else:
            _, tau_h, _ = st.solve_batch_states_warm(sin, shift=shift, torques=True, strict=False, out=(wh, sh))
            _, tau_r, _ = rc.solve_batch_warm(recs, shift=shift, torques=True, strict=False, out=(wr, sr))
        if mode == "in_place":   # (the in-place mode stores the solver's doubles, the staged record path their float rounding)
            assert np.array_equal(_bits(wh[m].astype(np.float32)), _bits(wr[m].astype(np.float32))), k
        else:
            assert np.array_equal(_bits(wh[m]), _bits(wr[m])), k
        assert np.array_equal(_bits(tau_h[m]), _bits(tau_r[m])), k
        assert np.array_equal(sh[m], sr[m]) and (interface.status_code(sh[m]) == 0).all(), k
        assert np.isnan(wh[~m]).all() and (sh[~m] == S_SENT).all() and (tau_h[~m] == 0).all(), k
    if mode == "in_place":
        st.unpin(sin, wh, sh)
    st.close()
    rc.close()


@pytest.mark.gpu
def test_in_place_solve_batch_states_equals_its_staged_modes():
    """hmpc_solve_batch_states with pinned states, wrench and status runs the device-resident chain; its results are
    bit-identical to the zero-copy and copy-pipeline modes of the same call: status words and torques as they are, wrenches
    rounded to float (the staged modes return the kernels' float results, the in-place mode the doubles they round, as
    hmpc_solve_batch does)."""
    for B in (300, 1800):
        states = _states(3, B, 93)
        mpc = interface.BatchedMPC(B, N)
        w0, t0, s0 = mpc.solve_batch_states(states, torques=True)
        sin = interface.page_aligned((B,), scenarios.STATE_DTYPE)
        sin[:] = states
        wh = interface.page_aligned((B, 12 * N), np.float64)
        sh = interface.page_aligned((B,), np.int32)
        mpc.pin(sin, wh, sh)
        _, t1, _ = mpc.solve_batch_states(sin, torques=True, out=(wh, sh))
        assert np.array_equal(_bits(wh.astype(np.float32)), _bits(w0.astype(np.float32))), B
        assert np.array_equal(_bits(w0.astype(np.float32).astype(np.float64)), _bits(w0)), B
        assert np.array_equal(_bits(t1), _bits(t0)) and np.array_equal(sh, s0), B
        assert (interface.status_code(s0) == 0).all()
        mpc.unpin(sin, wh, sh)
        mpc.close()


@pytest.mark.gpu
def test_state_calls_check_their_arguments():
    """NULL mask, NULL states, NULL d_records, B < 0 and B > capacity are argument errors, found before anything is enqueued;
    B = 0 is a no-op; an empty mask writes nothing, on the host too."""
    import torch

    L = interface.lib()
    mpc = interface.BatchedMPC(64, N)
    h = mpc._h
    stride = interface.record_bytes(N)
    d_st = torch.zeros((65, 352), dtype=torch.uint8, device="cuda")
    d_rec = torch.full((65 * stride,), 9, dtype=torch.uint8, device="cuda")
    d_w = torch.zeros((65, 12 * N), dtype=torch.float32, device="cuda")
    d_s = torch.full((65,), 7, dtype=torch.int32, device="cuda")
    d_m = torch.zeros(65, dtype=torch.bool, device="cuda")
    ps, p, pw, pst, pm = d_st.data_ptr(), d_rec.data_ptr(), d_w.data_ptr(), d_s.data_ptr(), d_m.data_ptr()
    ERR, OK = interface.HMPC_ERR_ARG, interface.HMPC_OK
    f = L.hmpc_solve_states_device_masked
    assert f(h, ps, 4, None, 0.04, p, pw, pst, None, None, None) == ERR
    assert f(h, None, 4, pm, 0.04, p, pw, pst, None, None, None) == ERR
    assert f(h, ps, 4, pm, 0.04, None, pw, pst, None, None, None) == ERR
    assert f(h, ps, 4, pm, 0.04, p, None, pst, None, None, None) == ERR
    assert f(h, ps, 4, pm, 0.04, p, pw, None, None, None, None) == ERR
    assert f(h, ps, -1, pm, 0.04, p, pw, pst, None, None, None) == ERR
    assert f(h, ps, 65, pm, 0.04, p, pw, pst, None, None, None) == ERR
    assert f(h, ps, 4, pm, 0.04, p + 4, pw, pst, None, None, None) == ERR
    assert f(h, ps, 0, pm, 0.04, p, pw, pst, None, None, None) == OK
    assert f(h, ps, 64, pm, 0.04, p, pw, pst, None, None, None) == OK      # empty mask
    torch.cuda.synchronize()
    assert (d_s.cpu().numpy() == 7).all() and (d_w.cpu().numpy() == 0).all() and (d_rec.cpu().numpy() == 9).all()
    states = np.zeros(65, scenarios.STATE_DTYPE)
    w = np.full((65, 12 * N), 3.0)
    s = np.full(65, 7, np.int32)
    m = np.zeros(65, np.uint8)
    g, wm = L.hmpc_solve_batch_states_masked, L.hmpc_solve_batch_states_warm
    assert g(h, states.ctypes.data, 4, None, 0.04, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert g(h, None, 4, m.ctypes.data, 0.04, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert g(h, states.ctypes.data, 4, m.ctypes.data, 0.04, None, None, s.ctypes.data, None) == ERR
    assert g(h, states.ctypes.data, -1, m.ctypes.data, 0.04, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert g(h, states.ctypes.data, 65, m.ctypes.data, 0.04, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert g(h, states.ctypes.data, 0, m.ctypes.data, 0.04, w.ctypes.data, None, s.ctypes.data, None) == OK
    assert g(h, states.ctypes.data, 64, m.ctypes.data, 0.04, w.ctypes.data, None, s.ctypes.data, None) == OK
    assert wm(h, None, 4, 0.04, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert wm(h, states.ctypes.data, 4, 0.04, None, None, s.ctypes.data, None) == ERR
    assert wm(h, states.ctypes.data, 65, 0.04, w.ctypes.data, None, s.ctypes.data, None) == ERR
    assert wm(h, states.ctypes.data, 0, 0.04, w.ctypes.data, None, s.ctypes.data, None) == OK
    assert (s == 7).all() and (w == 3.0).all()
    mpc.close()
