"""Several reference trajectories per robot (hmpc_solve_device_multi, hmpc_solve_batch_multi): candidate (i, k) must equal,
bit for bit, the cold solve of the expanded batch's row i*K + k (robot i's record with traj replaced by candidate k), and its
cost the certificate's cost for that row and wrench.

CPU: the kernel source on the host (tests/host_emul/multi_on_host.cpp), the multi-query chain against the emulated single
solve and certificate of the same build, in every size class, with refinement, masked, under ThreadSanitizer; the argument
checks through the library.  GPU (-m gpu): the library against hmpc_solve_device and hmpc_certify_device on the expanded
batch, masks, graph replay, the host call in both modes, K = 1.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_golden
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import BUILD, DEVICE_HEADER, HERE, _host_buildable, _p

CERT_DTYPE = interface.CERTIFICATE_DTYPE
_LIB = {}


# ---- fixtures ------------------------------------------------------------------------------------------------------------
def candidates(records, N, K, seed):
    """float32 [B, K, 12N]: candidate 0 is each record's own traj, the others that traj plus seeded perturbations (a few
    centimetres and centiradians, some velocity change) that move the optimum and often its active set"""
    rng = np.random.default_rng(seed)
    own = np.stack([np.asarray(r["traj"][: 12 * N], np.float32) for r in records])
    scale = np.tile(np.array([0.03, 0.03, 0.05, 0.02, 0.02, 0.01, 0.1, 0.1, 0.1, 0.2, 0.2, 0.05], np.float32), N)
    t = own[:, None, :] + (rng.normal(0.0, 1.0, (len(records), K, 12 * N)) * scale).astype(np.float32)
    t[:, 0] = own
    return np.ascontiguousarray(t, np.float32)


def expand(records, traj):
    """the expanded batch: row i*K + k is robot i's record with traj replaced by candidate k"""
    B, K, n = traj.shape
    ex = np.repeat(np.asarray(records), K).copy()
    for r in range(B * K):
        ex[r]["traj"][:n] = traj[r // K, r % K]
    return ex


def stress(key, idx):
    g = np.load(os.path.join(GOLDEN, "stress_referee.npz"))
    return np.ascontiguousarray(g[key + "_records"]).view(scenarios.UPDATE_DTYPE).reshape(-1)[idx]


# ---- the kernel source on the host ---------------------------------------------------------------------------------------
def multi_emulation():
    """multi_on_host.cpp built for the host as a library, once per process (the flags of kernel_source_on_host.cpp's build)"""
    if "lib" not in _LIB:
        os.makedirs(BUILD, exist_ok=True)
        hdr = os.path.join(BUILD, "hmpc_device_host_multi.cuh")
        with open(hdr, "w") as f:
            f.write(_host_buildable(open(DEVICE_HEADER).read()))
        out = os.path.join(BUILD, "libmulti_on_host.so")
        cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O2", "-fPIC", "-shared",
               "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"), '-DHMPC_DEVICE_HEADER="%s"' % hdr,
               os.path.join(HERE, "multi_on_host.cpp"), "-l:libstdc++.so.6", "-o", out]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        _LIB["lib"] = ctypes.CDLL(out)
        _LIB["hdr"] = hdr
    return _LIB["lib"]


def emul_multi(records, N, traj, raw=False, refine=False, mask=None, out=None):
    """the multi-query chain on the host -> (wrench [B*K, 12N] float32 or float64 (raw), status [B*K], cost [B*K], launched)"""
    L = multi_emulation()
    B, K = traj.shape[:2]
    rows = np.ascontiguousarray(records) if raw else interface.pack_records(records, N)
    if out is None:
        w = np.zeros((B * K, 12 * N), np.float64 if raw else np.float32)
        st = np.full(B * K, -1, np.int32)
        cost = np.zeros(B * K)
    else:
        w, st, cost = out
    launched = np.zeros(4, np.int32)
    rc = L.emul_solve_multi(None if raw else _p(rows), _p(rows) if raw else None, B, K, N, int(refine), _p(mask), _p(traj),
                            None if raw else _p(w), _p(w) if raw else None, _p(st), _p(cost), _p(launched))
    assert rc == 0, rc
    return w, st, cost, launched


def emul_single(expanded, N, raw=False, refine=False):
    """the cold single solve (emul_solve) of the expanded batch and the certificate's cost of its wrenches, same build"""
    L = multi_emulation()
    R = len(expanded)
    rows = np.ascontiguousarray(expanded) if raw else interface.pack_records(expanded, N)
    w = np.zeros((R, 12 * N), np.float64 if raw else np.float32)
    st = np.full(R, -1, np.int32)
    rc = L.emul_solve(None if raw else _p(rows), _p(rows) if raw else None, R, N, 0, int(refine), None, None, 0, 1, None,
                      None if raw else _p(w), _p(w) if raw else None, _p(st), None, None, None, None, None, None, None)
    assert rc == 0, rc
    cert = np.zeros(R, CERT_DTYPE)
    urows = rows.view(np.uint8).reshape(R, -1)
    L.emul_certify(_p(urows), int(raw), R, N, ctypes.c_float(0.04), ctypes.c_float(500.0), None, int(raw), _p(w), _p(cert),
                   None, None)
    return w, st, cert["cost"].copy()


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def assert_same(got, want):
    (w, st, cost), (ww, wst, wcost) = got, want
    assert np.array_equal(_bits(w), _bits(ww))
    assert np.array_equal(st, wst)
    assert np.array_equal(_bits(cost), _bits(wcost))


CASES = {  # name -> (records, N, what the case reaches)
    "cfg1_h10": lambda: (load_golden("cfg1_h10")["records"][:1], 10),      # standing: class 1, robots handed over whole
    "cfg2_h10": lambda: (load_golden("cfg2_h10")["records"][:3], 10),      # walking: class 0
    "cfg4_h5": lambda: (load_golden("cfg4_h5")["records"][:3], 5),         # runtime horizon, both classes
    "cfg4_h16": lambda: (load_golden("cfg4_h16")["records"][:2], 16),      # the horizon-16 extension
    "stress_h10_x8": lambda: (stress("h10_x8", [9, 21]), 10),              # ~80 active rows: escalation to class 2
}


@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("name", list(CASES))
def test_kernel_source_equals_the_expanded_single_solves(name, K):
    recs, N = CASES[name]()
    traj = candidates(recs, N, K, seed=K + len(name))
    w, st, cost, launched = emul_multi(recs, N, traj)
    assert_same((w, st, cost), emul_single(expand(recs, traj), N))
    assert (interface.status_code(st) == 0).mean() > 0.8
    if name == "cfg1_h10":
        assert launched[1] == len(recs)  # the stand goes to class 1 as one entry per robot
    if name == "stress_h10_x8" and K == 8:
        assert launched[2] > 0  # candidates escalated alone to class 2


def test_kernel_source_in_place_rows_equal_the_expanded_single_solves():
    """hmpc_solve_batch_multi's chain: update_data_t rows read in place, double wrenches, the certificate's double cost."""
    recs = np.concatenate([load_golden("cfg3_h10")["records"][:2], load_golden("cfg2_h10")["records"][3:4]])
    traj = candidates(recs, 10, 3, seed=5)
    w, st, cost, _ = emul_multi(recs, 10, traj, raw=True)
    assert_same((w, st, cost), emul_single(expand(recs, traj), 10, raw=True))


def test_kernel_source_with_refinement_equals_the_expanded_single_solves():
    """A robot lying on its side (beyond the conditioning limit) among walkers: each candidate of the lying robot is
    handed to the refinement class, and every candidate equals the expanded batch's solve with refinement on."""
    recs = np.concatenate([load_golden("cfg2_h10")["records"][:2], stress("h10_lying", [0])])
    K = 3
    traj = candidates(recs, 10, K, seed=9)
    w, st, cost, launched = emul_multi(recs, 10, traj, refine=True)
    assert launched[3] == K
    assert_same((w, st, cost), emul_single(expand(recs, traj), 10, refine=True))
    assert ((st[2 * K:] >> 28) & 1).all()  # solved by the refinement class


def test_kernel_source_mask_keeps_the_unlisted_rows():
    recs = load_golden("cfg3_h10")["records"][:5]
    K, N = 2, 10
    traj = candidates(recs, N, K, seed=3)
    mask = np.array([1, 0, 0, 3, 0], np.uint8)
    rng = np.random.default_rng(1)
    sw = rng.integers(0, 2 ** 32, (5 * K, 12 * N), dtype=np.uint64).astype(np.uint32).view(np.float32)
    ss = rng.integers(-2 ** 31, 2 ** 31, 5 * K).astype(np.int32)
    sc = rng.integers(0, 2 ** 63, 5 * K, dtype=np.uint64).view(np.float64)
    w, st, cost, _ = emul_multi(recs, N, traj, mask=mask, out=(sw.copy(), ss.copy(), sc.copy()))
    on = np.repeat(mask != 0, K)
    want = emul_single(expand(recs[mask != 0], traj[mask != 0]), N)
    assert_same((w[on], st[on], cost[on]), want)
    assert np.array_equal(_bits(w[~on]), _bits(sw[~on])) and np.array_equal(st[~on], ss[~on])
    assert np.array_equal(_bits(cost[~on]), _bits(sc[~on]))


def test_kernel_source_has_no_races_under_thread_sanitizer(tmp_path):
    """The multi-query launches built with -fsanitize=thread: the scratch round trip of a robot's later candidates, the
    skipped stages, the per-candidate stage 5, escalation (class 1 -> class 2) and the refinement class."""
    multi_emulation()
    exe = os.path.join(BUILD, "multi_tsan")
    cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O1", "-g", "-fsanitize=thread", "-DHMPC_MULTI_MAIN",
           "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"),
           '-DHMPC_DEVICE_HEADER="%s"' % _LIB["hdr"], os.path.join(HERE, "multi_on_host.cpp"), "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("no ThreadSanitizer runtime with this toolchain: " + r.stderr[-300:])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66")
    cases = [(load_golden("cfg2_h10")["records"][:2], 10, 3, ()),
             (load_golden("cfg1_h10")["records"][:1], 10, 2, ()),
             (load_golden("cfg4_h5")["records"][:2], 5, 2, ()),
             (stress("h10_x8", [9]), 10, 2, ()),
             (stress("h10_lying", [0]), 10, 2, ("refine",))]
    for recs, N, K, flags in cases:
        f = tmp_path / "rows.bin"
        np.ascontiguousarray(interface.pack_records(recs, N)).tofile(f)
        run = subprocess.run([exe, str(f), str(N), str(K), *flags], capture_output=True, text=True, env=env, timeout=1800)
        assert "ThreadSanitizer" not in run.stderr, run.stderr[:3000]
        assert run.returncode == 0, (run.returncode, run.stdout, run.stderr[-500:])


def test_multi_calls_check_their_arguments():
    """Through the library, without a GPU: a null context first, then the K and capacity checks on a context."""
    L = interface.lib()
    ERR = interface.HMPC_ERR_ARG
    x = np.zeros(64, np.float64)
    p = x.ctypes.data
    assert L.hmpc_solve_device_multi(None, p, 1, 2, p, None, p, p, None, None) == ERR
    assert L.hmpc_solve_batch_multi(None, p, 1, 2, p, None, p, p, None) == ERR
    assert L.hmpc_solve_device_multi(None, None, 0, 1, None, None, None, None, None, None) == ERR


# ---- GPU: the library ----------------------------------------------------------------------------------------------------
def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_multi(mpc, packed, traj, mask=None, sentinel=False):
    import torch

    B, K, n = traj.shape
    w = torch.zeros((B, K, n), dtype=torch.float32, device="cuda")
    st = torch.zeros((B, K), dtype=torch.int32, device="cuda")
    c = torch.zeros((B, K), dtype=torch.float64, device="cuda")
    if sentinel:
        w.view(torch.int32).fill_(0x7fc0dead)
        st.fill_(-77)
        c.view(torch.int64).fill_(0x7ff8dead)
    mpc.solve_device_multi(_dev(packed), B, _dev(traj), w, st, c, d_mask=None if mask is None else _dev(mask))
    torch.cuda.synchronize()
    return w.cpu().numpy(), st.cpu().numpy(), c.cpu().numpy()


def _device_single(mpc, expanded, N):
    import torch

    R = len(expanded)
    d = _dev(interface.pack_records(expanded, N))
    w = torch.zeros((R, 12 * N), dtype=torch.float32, device="cuda")
    st = torch.zeros(R, dtype=torch.int32, device="cuda")
    cert = torch.zeros((R, CERT_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    mpc.solve_device(d, R, w, st)
    mpc.certify_device(d, R, w, cert)
    torch.cuda.synchronize()
    return w.cpu().numpy(), st.cpu().numpy(), cert.cpu().numpy().view(CERT_DTYPE).reshape(-1)["cost"].copy()


def _batch(cfg, B, N=10):
    return scenarios.make_batch(cfg, B, horizon=N, seed=scenarios.config_seed(cfg) + 77)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,K", [(2, 8), (3, 4)])  # make_batch(2): configs[1] walkers, (3): configs[2] mixed
def test_device_multi_equals_the_expanded_single_solves(cfg, K):
    """1024 configs[1] walkers x 8 and 1024 configs[2] mixed robots x 4, against hmpc_solve_device and hmpc_certify_device
    on the 8192 / 4096 expanded records."""
    B, N = 1024, 10
    recs = _batch(cfg, B)
    traj = candidates(recs, N, K, seed=cfg)
    mpc = interface.BatchedMPC(B * K, N, device=0)
    w, st, c = _device_multi(mpc, interface.pack_records(recs, N), traj)
    ww, wst, wc = _device_single(mpc, expand(recs, traj), N)
    assert np.array_equal(_bits(w.reshape(B * K, -1)), _bits(ww))
    assert np.array_equal(st.reshape(-1), wst)
    assert np.array_equal(_bits(c.reshape(-1)), _bits(wc))
    assert (interface.status_code(wst) == 0).mean() > 0.95
    mpc.close()


@pytest.mark.gpu
def test_device_multi_mask_and_graph_replay():
    """A mask of a fifth of the robots leaves the other rows' sentinel bytes alone; a torch.cuda.graph replay equals the
    eager call; K = 1 equals hmpc_solve_device."""
    import torch

    B, N, K = 512, 10, 4
    recs = _batch(3, B)
    traj = candidates(recs, N, K, seed=11)
    packed = interface.pack_records(recs, N)
    mpc = interface.BatchedMPC(B * K, N, device=0)
    mask = (np.arange(B) % 5 == 2).astype(np.uint8)
    w, st, c = _device_multi(mpc, packed, traj, mask=mask, sentinel=True)
    ew, est, ec = _device_multi(mpc, packed, traj)
    on = mask != 0
    assert np.array_equal(_bits(w[on]), _bits(ew[on])) and np.array_equal(st[on], est[on]) and np.array_equal(_bits(c[on]), _bits(ec[on]))
    assert (w[~on].view(np.int32) == 0x7fc0dead).all() and (st[~on] == -77).all() and (c[~on].view(np.int64) == 0x7ff8dead).all()
    # graph replay
    d_rec, d_traj = _dev(packed), _dev(traj)
    gw = torch.zeros((B, K, 12 * N), dtype=torch.float32, device="cuda")
    gs = torch.zeros((B, K), dtype=torch.int32, device="cuda")
    gc = torch.zeros((B, K), dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        mpc.solve_device_multi(d_rec, B, d_traj, gw, gs, gc)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        mpc.solve_device_multi(d_rec, B, d_traj, gw, gs, gc)
    for _ in range(2):
        gw.zero_(), gs.zero_(), gc.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(_bits(gw.cpu().numpy()), _bits(ew)) and np.array_equal(gs.cpu().numpy(), est)
        assert np.array_equal(_bits(gc.cpu().numpy()), _bits(ec))
    # K = 1
    w1, st1, _ = _device_multi(mpc, packed, traj[:, :1])
    sw, sst, _ = _device_single(mpc, expand(recs, traj[:, :1]), N)
    assert np.array_equal(_bits(w1.reshape(B, -1)), _bits(sw)) and np.array_equal(st1.reshape(-1), sst)
    mpc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False])
def test_host_multi_equals_the_device_call(pinned):
    """hmpc_solve_batch_multi in place (pinned arrays) and staged: double wrenches that round to the device call's floats,
    its status words, and hmpc_certify_batch's cost of the expanded rows and those doubles."""
    B, N, K = 256, 10, 3
    recs = _batch(2, B)
    traj = candidates(recs, N, K, seed=21)
    mpc = interface.BatchedMPC(B * K, N, device=0)
    ew, est, _ = _device_multi(mpc, interface.pack_records(recs, N), traj)
    alloc = interface.page_aligned if pinned else (lambda shape, dt: np.zeros(shape, dt))
    x, t = alloc((B,), scenarios.UPDATE_DTYPE), alloc(traj.shape, np.float32)
    x[:], t[:] = recs, traj
    out = (alloc((B, K, 12 * N), np.float64), alloc((B, K), np.int32), alloc((B, K), np.float64))
    if pinned:
        mpc.pin(x, t, *out)
    w, st, c = mpc.solve_batch_multi(x, t, out=out, strict=False)
    assert w is out[0]
    assert interface.lib().hmpc_debug_last_multi_in_place() == (1 if pinned else 0)
    assert np.array_equal(_bits(w.astype(np.float32)), _bits(ew)) and np.array_equal(st, est)
    cert = mpc.certify_batch(expand(recs, traj), w.reshape(B * K, -1))
    assert np.array_equal(_bits(c.reshape(-1)), _bits(cert["cost"]))
    mpc.close()
