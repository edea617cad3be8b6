"""CUDA-graph capture of the device-resident calls (include/hector_mpc_b200.h, "CUDA graphs").

Every replay of a captured hmpc_solve_device(_ex/_warm), hmpc_prepare_device or hmpc_rollout_device must give what an
eager call of the same function gives on the same inputs, bit for bit: wrenches, torques, status words, advanced states.
The reference for every replay is an eager call on a second context fed the same inputs.  The workloads reach all three
size classes: double-support robots go to class 1, and a falling robot whose optimal forces are all zero
(degenerate_zero_force_h10) overflows class 1 and is escalated to class 2.  Everything here runs on the GPU."""
import ctypes

import numpy as np
import pytest

from conftest import load_golden
from hector_simulation_b200 import interface, scenarios
from test_rollout import _to_dev, _walkers
from test_warm_start_calls import _bits_equal

pytestmark = pytest.mark.gpu

N = 10
B_MIX, SETS = 4096, 8
GAIT0 = (54 + 12 * N) * 4   # byte offset of the contact table in a packed record


@pytest.fixture(scope="module")
def mixed():
    """SETS packed record sets of B_MIX robots on the GPU: walking and standing robots drawn from one cfg-3 pool, and 12
    copies of the degenerate record at random places in every set.  4096 robots are more than two waves of class 0, so
    its wave barrier is engaged."""
    import torch

    pool, _ = scenarios.make_batch(3, 6144, horizon=N, seed=77)
    deg = load_golden("degenerate_zero_force_h10")["records"][0]
    rng = np.random.default_rng(78)
    sets = []
    for _ in range(SETS):
        recs = pool[rng.choice(len(pool), B_MIX, replace=False)]
        recs[rng.choice(B_MIX, 12, replace=False)] = deg
        sets.append(interface.pack_records(recs, N))
    return torch.from_numpy(np.stack(sets)).cuda()


def _outputs(B):
    """wrench f32 [B,12N], tau f32 [B,10], status i32 [B]; filled with NaN / -1 so that a result left unwritten shows"""
    import torch

    w = torch.full((B, 12 * N), float("nan"), dtype=torch.float32, device="cuda")
    tau = torch.full((B, 10), float("nan"), dtype=torch.float32, device="cuda")
    s = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    return w, tau, s


def _solve_ex(mpc, d_rec, B, w, tau, s):
    """hmpc_solve_device_ex on the current stream (the capture stream inside torch.cuda.graph)"""
    import torch

    st = torch.cuda.current_stream().cuda_stream
    interface._check(interface.lib().hmpc_solve_device_ex(mpc._h, d_rec.data_ptr(), B, w.data_ptr(), s.data_ptr(),
                                                          tau.data_ptr(), ctypes.c_void_p(st)))


def _same(a, b):
    """bit-identical tensors (floats compared as bit patterns)"""
    a, b = a.cpu().numpy(), b.cpu().numpy()
    if a.dtype == np.float32:
        return _bits_equal(a, b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_replayed_solve_equals_eager_in_all_three_classes(mixed):
    """hmpc_solve_device_ex captured once and replayed over SETS record sets copied into the captured input: every
    replay equals the eager call of a second context — and the sets really reach classes 1 and 2."""
    import torch

    B = B_MIX
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    assert a.launches_per_solve == 3
    nb_cap0, qmax1 = a.class_config(0)["nb_cap"], a.class_config(1)["qmax"]
    rec = mixed[0].clone()
    w, tau, s = _outputs(B)
    _solve_ex(a, rec, B, w, tau, s)             # eager warm-up: the kernels are loaded outside the capture
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _solve_ex(a, rec, B, w, tau, s)
    wr, taur, sr = _outputs(B)
    for k in range(SETS):
        rec.copy_(mixed[k])
        for t in (w, tau):
            t.fill_(float("nan"))
        s.fill_(-1)
        g.replay()
        _solve_ex(b, mixed[k], B, wr, taur, sr)
        torch.cuda.synchronize()
        assert _same(w, wr) and _same(tau, taur) and _same(s, sr), k
        st = s.cpu().numpy()
        blocks = (mixed[k][:, GAIT0:GAIT0 + 2 * N] != 0).sum(1).cpu().numpy()
        escalated = interface.status_nactive(st) > qmax1
        assert (blocks > nb_cap0).sum() > B // 10, k              # class 1: double support
        assert escalated.sum() >= 12 and (interface.status_code(st[escalated]) == 0).all(), k   # class 2
    a.close()
    b.close()


def test_eager_and_replayed_calls_interleave_on_one_context(mixed):
    """eager, replay, eager, eager, replay, replay, eager on one context: every call equals the second context's eager
    call on the same records, so a capture leaves the eager chain's list bookkeeping alone."""
    import torch

    B = B_MIX
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    rec = mixed[0].clone()
    w, _, s = _outputs(B)
    we, _, se = _outputs(B)
    wr, _, sr = _outputs(B)
    b.solve_device(rec, B, wr, sr)              # loads the kernels outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a.solve_device(rec, B, w, s)
    for i, kind in enumerate(("eager", "replay", "eager", "eager", "replay", "replay", "eager")):
        k = i % SETS
        if kind == "eager":
            we.fill_(float("nan"))
            se.fill_(-1)
            a.solve_device(mixed[k], B, we, se)
            out = (we, se)
        else:
            rec.copy_(mixed[k])
            w.fill_(float("nan"))
            s.fill_(-1)
            g.replay()
            out = (w, s)
        b.solve_device(mixed[k], B, wr, sr)
        torch.cuda.synchronize()
        assert _same(out[0], wr) and _same(out[1], sr), (i, kind)
    a.close()
    b.close()


def test_captured_rollout_tick_is_the_rollout():
    """hmpc_rollout_device(ticks=1) captured on context A and replayed T times equals an eager T-tick rollout on context B
    from the same initial states: every tick's first-step wrench, the final states, and the loop's counters."""
    import torch

    B, T = 1024, 50
    states, loop = _walkers(B, seed=21)
    b = interface.BatchedMPC(B, N)
    sb, lb = _to_dev(states), _to_dev(loop)
    wlog_b = torch.zeros((T, B, 12), dtype=torch.float32, device="cuda")
    b.rollout_device(sb, lb, B, T, wlog_b)
    torch.cuda.synchronize()

    a = interface.BatchedMPC(B, N)
    sa, la = _to_dev(states), _to_dev(loop)
    w1 = torch.zeros((1, B, 12), dtype=torch.float32, device="cuda")
    wlog_a = torch.full((T, B, 12), float("nan"), dtype=torch.float32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a.rollout_device(sa, la, B, 1, w1)
    for t in range(T):
        g.replay()
        wlog_a[t].copy_(w1[0])
    torch.cuda.synchronize()
    assert _same(wlog_a, wlog_b)
    assert _same(sa, sb)
    lo_a = la.cpu().numpy().view(scenarios.ROLLOUT_DTYPE).reshape(B)
    lo_b = lb.cpu().numpy().view(scenarios.ROLLOUT_DTYPE).reshape(B)
    assert np.array_equal(lo_a["iters_total"], lo_b["iters_total"]) and np.array_equal(lo_a["failures"], lo_b["failures"])
    assert _same(la, lb)
    assert (lo_a["ticks"] == T).all() and lo_a["iters_total"].sum() > 0
    a.close()
    b.close()


def test_captured_warm_solve_reads_per_robot_shifts():
    """hmpc_solve_device_warm captured with a static shift tensor and replayed over a logged walk in which 10 % of the robots
    get shift -1 at one tick each: the replays equal the eager warm replay with the same shifts, and the reset robots equal
    the cold solve there."""
    import torch

    B, T = 1024, 50
    states, loop = _walkers(B, seed=11)
    log = interface.BatchedMPC(B, N)
    d_rlog = torch.zeros((T, B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    log.rollout_device(_to_dev(states), _to_dev(loop), B, T, None, d_rlog)
    torch.cuda.synchronize()
    log.close()
    rng = np.random.default_rng(5)
    robots = rng.choice(B, B // 10, replace=False)
    ticks = rng.integers(1, T, len(robots))
    shifts = np.ones((T, B), np.int32)
    shifts[ticks, robots] = -1
    d_shifts = torch.from_numpy(shifts).cuda()

    def logs():
        return (torch.full((T, B, 12 * N), float("nan"), dtype=torch.float32, device="cuda"),
                torch.full((T, B), -1, dtype=torch.int32, device="cuda"))

    b, c = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    wb, sb = logs()
    wc, sc = logs()
    for t in range(T):
        b.solve_device_warm(d_rlog[t], B, wb[t], sb[t], d_shift=d_shifts[t])
        c.solve_device(d_rlog[t], B, wc[t], sc[t])
    torch.cuda.synchronize()

    a = interface.BatchedMPC(B, N)
    rec, shift = d_rlog[0].clone(), d_shifts[0].clone()
    w, _, s = _outputs(B)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a.solve_device_warm(rec, B, w, s, d_shift=shift)
    wa, sa = logs()
    for t in range(T):
        rec.copy_(d_rlog[t])
        shift.copy_(d_shifts[t])
        g.replay()
        wa[t].copy_(w)
        sa[t].copy_(s)
    torch.cuda.synchronize()
    assert _same(wa, wb) and _same(sa, sb)
    wa_, sa_, wc_, sc_ = wa.cpu().numpy(), sa.cpu().numpy(), wc.cpu().numpy(), sc.cpu().numpy()
    assert _bits_equal(wa_[ticks, robots], wc_[ticks, robots]) and np.array_equal(sa_[ticks, robots], sc_[ticks, robots])
    # the warm start did act: fewer changes than the cold solves over the ticks after the first
    assert interface.status_iters(sa_[1:]).mean() < 0.5 * interface.status_iters(sc_[1:]).mean()
    for m in (a, b, c):
        m.close()


def test_torch_graph_with_torch_work_around_the_mpc():
    """One torch.cuda.graph holds torch arithmetic that perturbs the device states, hmpc_prepare_device,
    hmpc_solve_device_warm and a torch reduction of the wrenches.  Every replay equals the same sequence run eagerly on a
    second context: states, wrenches, status words and the reduction."""
    import torch

    B, TICKS = 1024, 6
    states, _ = _walkers(B, seed=31)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    deltas = 0.02 * torch.randn((TICKS, B, 3), dtype=torch.float64, device="cuda", generator=gen)
    stride = interface.record_bytes(N)

    def step(mpc, d_states, delta, rec, w, s):
        d_states.view(torch.float64)[:, 3:6] += delta            # vWorld (hmpc_state_t doubles 3..5)
        mpc.prepare_device(d_states, B, rec)
        mpc.solve_device_warm(rec, B, w, s)
        first = w.view(B, N, 12)[:, 0].abs().sum(1)
        return first, first.sum()

    def buffers():
        return (_to_dev(states), torch.zeros((B, stride), dtype=torch.uint8, device="cuda")) + _outputs(B)[::2]

    warm_up = interface.BatchedMPC(B, N)    # loads the library's and torch's kernels outside the capture
    sw, rw, ww, swt = buffers()
    step(warm_up, sw, deltas[0], rw, ww, swt)
    torch.cuda.synchronize()
    warm_up.close()

    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    sa, ra, wa, st_a = buffers()
    sb, rb, wb, st_b = buffers()
    delta = torch.zeros((B, 3), dtype=torch.float64, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        first_a, total_a = step(a, sa, delta, ra, wa, st_a)
    for t in range(TICKS):
        delta.copy_(deltas[t])
        g.replay()
        first_b, total_b = step(b, sb, deltas[t], rb, wb, st_b)
        torch.cuda.synchronize()
        assert _same(sa, sb) and _same(ra, rb), t
        assert _same(wa, wb) and _same(st_a, st_b), t
        assert _same(first_a, first_b) and _same(total_a, total_b), t
    assert (interface.status_code(st_a.cpu().numpy()) == 0).all()
    a.close()
    b.close()


def test_two_captured_solves_share_the_capture_slot(mixed):
    """Two hmpc_solve_device calls of one context on two record sets, captured in sequence on one stream into one graph:
    after every replay both outputs equal the eager calls."""
    import torch

    B = B_MIX
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)
    rec1, rec2 = mixed[0].clone(), mixed[1].clone()
    w1, _, s1 = _outputs(B)
    w2, _, s2 = _outputs(B)
    wr, _, sr = _outputs(B)
    b.solve_device(rec1, B, wr, sr)             # loads the kernels outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        a.solve_device(rec1, B, w1, s1)
        a.solve_device(rec2, B, w2, s2)
    for k in range(0, SETS, 2):
        rec1.copy_(mixed[k])
        rec2.copy_(mixed[k + 1])
        for t in (w1, w2):
            t.fill_(float("nan"))
        g.replay()
        for out_w, out_s, src in ((w1, s1, mixed[k]), (w2, s2, mixed[k + 1])):
            b.solve_device(src, B, wr, sr)
            torch.cuda.synchronize()
            assert _same(out_w, wr) and _same(out_s, sr), k
    a.close()
    b.close()
