"""The MPC's plan: each robot's predicted state trajectory x_{k+1} = Acd x_k + Bcd u_k under the discrete model its QP was
built from (hmpc_predict_device, hmpc_predict_batch, BatchedMPC.predict_device / predict_batch).

The restatement below is the recurrence in numpy, float64, in the kernel's operation order, on the oracle's float32 x0, Acd
and Bcd.  CPU: the kernel's source on the host (tests/host_emul/predict_on_host.cpp) equals it bit for bit, with the packed
record stride and with the update_data_t stride; it agrees with the reference's own A_qp x0 + B_qp U to the float32
rounding of the reference's matrix powers; its tracking cost equals the QP objective; masks and argument checks.  GPU: the
device call on the device's own wrenches, the masked states chain, the host call in both modes, graph capture and the
objective identity against the kernel's own assembly."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_golden
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import BUILD, DEVICE_HEADER, HERE, _host_buildable, _p

FIXTURES = ["cfg1_h10", "cfg2_h10", "cfg3_h10", "cfg4_h5", "cfg4_h16"]
DT = 0.04
EPS32 = 2.0 ** -24
_LIB = {}

# the structural entries of a row of Acd (off the diagonal) and of Bcd, in the order the kernel adds them
X_TERMS = {0: (6, 7, 8), 1: (6, 7, 8), 2: (6, 7, 8), 3: (9,), 4: (10,), 5: (11,), 11: (12,)}
U_TERMS = {6: tuple(range(12)), 7: tuple(range(12)), 8: tuple(range(12)), 9: (0, 3), 10: (1, 4), 11: (2, 5)}


def restate(x0, Acd, Bcd, U, N):
    """The plan in numpy: x0 [B,13], Acd [B,13,13], Bcd [B,13,12] (float32 of the formulation), U [B,12N] -> [B,N,12] f64.
    Row r of a step: x[r], then + Acd[r,j] x[j] over the row's off-diagonal entries, then + Bcd[r,c] u[c] over its entries,
    each product and sum one rounded float64 operation."""
    A, Bm = np.asarray(Acd, np.float64), np.asarray(Bcd, np.float64)
    x = np.asarray(x0, np.float64).copy()
    U = np.asarray(U, np.float64)
    out = np.zeros((len(x), N, 12))
    for k in range(N):
        u = U[:, 12 * k:12 * k + 12]
        new = x.copy()
        for r in range(12):
            acc = x[:, r].copy()
            for j in X_TERMS.get(r, ()):
                acc = acc + A[:, r, j] * x[:, j]
            for c in U_TERMS.get(r, ()):
                acc = acc + Bm[:, r, c] * u[:, c]
            new[:, r] = acc
        x = new
        out[:, k] = x[:, :12]
    return out


def formulation(oracle, records, N):
    """the oracle's float32 x0, Acd, Bcd, A_qp of every record (the kernel's stage-1 values, bit for bit)"""
    setup = oracle.make_setup(N, dt=DT)
    F = [oracle.formulate_f32(r, setup) for r in records]
    return {k: np.array([f[k] for f in F]) for k in ("x0", "Acd", "Bcd", "A_qp", "H", "g")}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint64)


# ---- CPU: the kernel's source on the host ----------------------------------------------------------------------------------
def predict_emulation():
    """predict_on_host.cpp built for the host as a library, once per process (the flags of kernel_source_on_host.cpp's build)"""
    if "lib" not in _LIB:
        os.makedirs(BUILD, exist_ok=True)
        hdr = os.path.join(BUILD, "hmpc_device_host_predict.cuh")
        with open(hdr, "w") as f:
            f.write(_host_buildable(open(DEVICE_HEADER).read()))
        out = os.path.join(BUILD, "libpredict_on_host.so")
        cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O2", "-fPIC", "-shared",
               "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"), '-DHMPC_DEVICE_HEADER="%s"' % hdr,
               os.path.join(HERE, "predict_on_host.cpp"), "-l:libstdc++.so.6", "-o", out]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        _LIB["lib"] = ctypes.CDLL(out)
    return _LIB["lib"]


def emul_predict(L, rows, N, U, mask=None, pred=None, double=True, B=None):
    """the prediction kernel on the host over the first B (all) of `rows` (uint8 [*, stride]) -> pred [*,N,12] (f64, or f32
    with double=False)"""
    rows = np.ascontiguousarray(rows)
    B = rows.shape[0] if B is None else B
    stride = rows.shape[1]
    dt = np.float64 if double else np.float32
    U = np.ascontiguousarray(U, dt)
    if pred is None:
        pred = np.zeros((rows.shape[0], N, 12), dt)
    L.emul_predict(_p(rows), stride, B, N, ctypes.c_float(DT), _p(mask), int(double), _p(U), _p(pred))
    return pred


def _rows_raw(records):
    return np.ascontiguousarray(records).view(np.uint8).reshape(len(records), -1)


@pytest.mark.parametrize("name", FIXTURES)
def test_kernel_source_equals_the_restatement(oracle, name):
    """The fixture's records and oracle solutions: the host build of the kernel equals the restatement bit for bit, over
    packed records and over update_data_t rows, in both instantiations (float: the rounding of the restatement on the float
    wrenches)."""
    g = load_golden(name)
    N, recs, U = g["horizon"], g["records"], g["q_soln"]
    F = formulation(oracle, recs, N)
    want = restate(F["x0"], F["Acd"], F["Bcd"], U, N)
    L = predict_emulation()
    packed = interface.pack_records(recs, N)
    for rows in (packed, _rows_raw(recs)):
        got = emul_predict(L, rows, N, U)
        assert np.array_equal(_bits(got), _bits(want))
        U32 = U.astype(np.float32)
        got32 = emul_predict(L, rows, N, U32, double=False)
        want32 = restate(F["x0"], F["Acd"], F["Bcd"], U32, N).astype(np.float32)
        assert np.array_equal(_bits(got32), _bits(want32))
    assert np.isfinite(want).all()


def ref_qp_matrices(oracle):
    """tests/host_emul/ref_qp_matrices.cpp built against oracle/_ref/libref_mpc.so, once per process: the reference's
    A_qp and B_qp after its last solve, read through the shim's own matrix class"""
    if "refqp" not in _LIB:
        os.makedirs(BUILD, exist_ok=True)
        ref_dir = os.path.dirname(oracle._REF_LIB_PATH)
        out = os.path.join(BUILD, "libref_qp_matrices.so")
        cmd = ["g++", "-std=gnu++14", "-O2", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "oracle", "eigen_shim"),
               os.path.join(HERE, "ref_qp_matrices.cpp"), "-L" + ref_dir, "-l:libref_mpc.so", "-Wl,-rpath," + ref_dir,
               "-l:libstdc++.so.6", "-o", out]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        oracle.ref_lib()                      # the same libref_mpc.so object the probe's symbols resolve to
        _LIB["refqp"] = ctypes.CDLL(out)
    return _LIB["refqp"]


def _reference_plans(oracle, records, U, N):
    """A_qp x0 + B_qp U in float64 from the reference's own float32 matrices (its compiled SolverMPC.cpp), per record"""
    L, Q = oracle.ref_lib(), ref_qp_matrices(oracle)
    setup = oracle.make_setup(N, dt=DT)
    null = ctypes.c_void_p(0)
    out = np.zeros((len(records), N, 12))
    for i in range(len(records)):
        q = np.zeros(12 * N)
        x0 = np.zeros(13, np.float32)
        Aqp = np.zeros((13 * N, 13), np.float32)
        L.refshim_solve(oracle._p(records[i:i + 1]), oracle._p(setup), oracle._p(q), null, null, null, null, null,
                        oracle._p(x0), oracle._p(Aqp), null, null)
        assert (Q.refqp_rows(), Q.refqp_cols()) == (13 * N, 12 * N)
        A, B = np.zeros((13 * N, 13), np.float32), np.zeros((13 * N, 12 * N), np.float32)
        Q.refqp_copy(_p(A), _p(B))
        assert np.array_equal(A, Aqp)          # the probe reads the matrices of the solve refshim_solve just ran
        X = A.astype(np.float64) @ x0.astype(np.float64) + B.astype(np.float64) @ U[i]
        out[i] = X.reshape(N, 13)[:, :12]
    return out


def _exact_plans(F, U, N):
    """x_{k+1} = Acd x_k + Bcd u_k with numpy's float64 matrix products (no fixed order) on the same float32 matrices"""
    out = np.zeros((len(U), N, 12))
    for i in range(len(U)):
        A, B, x = (F[k][i].astype(np.float64) for k in ("Acd", "Bcd", "x0"))
        for k in range(N):
            x = A @ x + B @ U[i, 12 * k:12 * k + 12]
            out[i, k] = x[:12]
    return out


# Worst difference of the restatement from the reference's A_qp x0 + B_qp U over the three N = 10 fixtures, relative to the
# largest entry of the robot's plan (DESIGN.md §3): 5.04e-7 measured.  The restatement is the float64 product of the float32
# Acd and Bcd to 5e-16, so the whole gap is the reference's float32 rounding of the matrix powers Acd^k and of the products
# Acd^k Bcd it stores in A_qp and B_qp.  It peaks at the vertical velocity of the last step, about -0.9 m/s, the sum of ten
# gravity increments of -0.39 m/s and the ten contact-force increments that nearly cancel them.
REF_REL_MAX = 6e-7


def test_restatement_agrees_with_the_reference_matrices(oracle):
    if not oracle.has_reference_build():
        pytest.skip("oracle/_ref/libref_mpc.so (the reference's compiled formulation) is not built")
    worst = 0.0
    for name in ("cfg1_h10", "cfg2_h10", "cfg3_h10"):
        g = load_golden(name)
        N, recs, U = g["horizon"], g["records"], g["q_soln"]
        F = formulation(oracle, recs, N)
        mine = restate(F["x0"], F["Acd"], F["Bcd"], U, N)
        ref = _reference_plans(oracle, recs, U, N)
        scale = np.abs(ref).reshape(len(recs), -1).max(1)[:, None, None]
        assert (np.abs(mine - _exact_plans(F, U, N)) / scale).max() < 1e-14
        worst = max(worst, float((np.abs(mine - ref) / scale).max()))
    print("worst relative difference from A_qp x0 + B_qp U: %.3e" % worst)
    assert worst < REF_REL_MAX, worst


def objective_terms(record, U, pred, H, g, A_qp, x0, N):
    """(tracking cost of the plan, QP objective 1/2 U'HU + g'U + d'Sd, the absolute scale both are rounded against) of one
    robot; S = the record's weights (0 on gravity), alpha = its Alpha_K, X_d = its traj, d = A_qp x0 - X_d"""
    w = np.asarray(record["weights"], np.float64)
    alpha = np.tile(np.asarray(record["Alpha_K"], np.float64), N)
    traj = np.asarray(record["traj"][:12 * N], np.float64).reshape(N, 12)
    track = float((w * (pred - traj) ** 2).sum() + (alpha * U * U).sum())
    d = (A_qp.astype(np.float64) @ x0.astype(np.float64)).reshape(N, 13)[:, :12] - traj
    dSd = float((w * d * d).sum())
    H, g = H.astype(np.float64), g.astype(np.float64)
    qp = float(0.5 * U @ H @ U + g @ U + dSd)
    # (+ what one rounding of every state of the plan can move the tracking cost by: the device returns float states)
    scale = float(0.5 * np.abs(U) @ np.abs(H) @ np.abs(U) + np.abs(g) @ np.abs(U) + dSd + track
                  + 2 * (w * np.abs(pred - traj) * np.abs(pred)).sum())
    return track, qp, scale


# H and g are the reference's float32 formulation: every entry carries the rounding of float32 sums of products of float32
# matrix powers, a few units of 2^-24 relative to the sum of the magnitudes it was formed from.  The identity is held to
# OBJ_K units of 2^-24 of the absolute scale of its terms (measured worst over the fixtures: 1.0 unit).
OBJ_K = 16


@pytest.mark.parametrize("name", FIXTURES)
def test_tracking_cost_of_the_plan_is_the_qp_objective(oracle, name):
    g = load_golden(name)
    N, recs, U = g["horizon"], g["records"], g["q_soln"]
    F = formulation(oracle, recs, N)
    pred = restate(F["x0"], F["Acd"], F["Bcd"], U, N)
    worst = 0.0
    for i in range(len(recs)):
        track, qp, scale = objective_terms(recs[i], U[i], pred[i], F["H"][i], F["g"][i], F["A_qp"][i], F["x0"][i], N)
        worst = max(worst, abs(track - qp) / (EPS32 * scale))
        assert abs(track - qp) <= OBJ_K * EPS32 * scale, (i, track, qp, scale)
    print("%s: worst |tracking - objective| = %.2f units of 2^-24 of the scale" % (name, worst))


def test_kernel_source_mask_writes_the_listed_rows_only(oracle):
    g = load_golden("cfg3_h10")
    N, recs, U = g["horizon"], g["records"], g["q_soln"]
    F = formulation(oracle, recs, N)
    want = restate(F["x0"], F["Acd"], F["Bcd"], U, N)
    L = predict_emulation()
    B = len(recs)
    rng = np.random.default_rng(5)
    sentinel = rng.integers(0, 2 ** 63, (B, N, 12), dtype=np.uint64).view(np.float64)
    for m in ((rng.random(B) < 0.2) * rng.integers(1, 256, B), np.zeros(B), np.eye(1, B, B - 1)[0]):
        m = m.astype(np.uint8)
        on = m != 0
        pred = emul_predict(L, interface.pack_records(recs, N), N, U, mask=m, pred=sentinel.copy())
        assert np.array_equal(_bits(pred[on]), _bits(want[on]))
        assert np.array_equal(_bits(pred[~on]), _bits(sentinel[~on]))


def test_kernel_source_leaves_rows_beyond_the_batch_alone(oracle):
    """B = 61, 62, 63 of 64 rows (the last CTA partly empty): rows i < B are the restatement, the rows past B of the
    prediction buffer keep their bytes, whatever the records and wrenches past B hold."""
    g = load_golden("cfg3_h10")
    N, recs, U = g["horizon"], g["records"], g["q_soln"]
    F = formulation(oracle, recs, N)
    want = restate(F["x0"], F["Acd"], F["Bcd"], U, N)
    L = predict_emulation()
    assert len(recs) == 64
    sentinel = np.random.default_rng(6).integers(0, 2 ** 63, (64, N, 12), dtype=np.uint64).view(np.float64)
    for B in (61, 62, 63):
        assert L.emul_predict_grid(B) * (L.emul_predict_threads() // 32) > B
        pred = emul_predict(L, interface.pack_records(recs, N), N, U, pred=sentinel.copy(), B=B)
        assert np.array_equal(_bits(pred[:B]), _bits(want[:B]))
        assert np.array_equal(_bits(pred[B:]), _bits(sentinel[B:]))


def test_prediction_calls_reject_a_null_context():
    L = interface.lib()
    x = np.zeros(4, np.float64)
    assert L.hmpc_predict_device(None, x.ctypes.data, 1, None, x.ctypes.data, x.ctypes.data, None) == interface.HMPC_ERR_ARG
    assert L.hmpc_predict_batch(None, x.ctypes.data, 1, None, x.ctypes.data, x.ctypes.data) == interface.HMPC_ERR_ARG
    assert L.hmpc_predict_device(None, None, 0, None, None, None, None) == interface.HMPC_ERR_ARG


# ---- GPU: the library ----------------------------------------------------------------------------------------------------
def _to_dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_solve(mpc, recs, N):
    import torch

    B = len(recs)
    d_rec = _to_dev(interface.pack_records(recs, N))
    w = torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda")
    s = torch.zeros(B, dtype=torch.int32, device="cuda")
    mpc.solve_device(d_rec, B, w, s)
    return d_rec, w, s


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,B,N", [(2, 1024, 10), (3, 8192, 10), (4, 4096, 5), (4, 4096, 16)])
def test_device_prediction_equals_the_restatement(oracle, cfg, B, N):
    """hmpc_solve_device, then hmpc_predict_device on the same records and the device's own float wrenches: the float
    rounding of the restatement, bit for bit."""
    import torch

    recs, _ = scenarios.make_batch(cfg, B, horizon=N, seed=40 + cfg)
    mpc = interface.BatchedMPC(B, N)
    d_rec, w, s = _device_solve(mpc, recs, N)
    d_pred = torch.full((B, N, 12), float("nan"), dtype=torch.float32, device="cuda")
    mpc.predict_device(d_rec, B, w, d_pred)
    torch.cuda.synchronize()
    U = w.cpu().numpy()
    F = formulation(oracle, recs, N)
    want = restate(F["x0"], F["Acd"], F["Bcd"], U, N).astype(np.float32)
    assert (interface.status_code(s.cpu().numpy()) == 0).mean() > 0.99
    assert np.array_equal(_bits(d_pred.cpu().numpy()), _bits(want))
    mpc.close()


def _states(cfg, B, N, seed):
    _, inputs = scenarios.make_batch(cfg, B, horizon=N, seed=seed)
    return np.ascontiguousarray(scenarios.make_states(inputs, N))


@pytest.mark.gpu
def test_masked_states_chain_then_prediction(oracle):
    """solve_states_device_masked with about a fifth of 2048 robots due, then predict_device on its d_records with the same
    mask: listed rows are the restatement on the records the chain prepared, unlisted rows keep their bytes."""
    import torch

    B, N = 2048, 10
    mpc = interface.BatchedMPC(B, N)
    states = _states(3, B, N, 91)
    m = np.random.default_rng(92).random(B) < 0.2
    d_m = _to_dev(m)
    d_rec = torch.zeros((B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    w = torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda")
    s = torch.zeros(B, dtype=torch.int32, device="cuda")
    mpc.solve_states_device_masked(_to_dev(states.view(np.uint8).reshape(B, -1)), B, d_m, d_rec, w, s)
    sentinel = np.random.default_rng(93).integers(0, 2 ** 32, (B, N, 12), dtype=np.uint64).astype(np.uint32).view(np.float32)
    d_pred = _to_dev(sentinel)
    mpc.predict_device(d_rec, B, w, d_pred, d_mask=d_m)
    torch.cuda.synchronize()
    got = d_pred.cpu().numpy()
    recs = interface.unpack_records(d_rec.cpu().numpy()[m], N)
    F = formulation(oracle, recs, N)
    want = restate(F["x0"], F["Acd"], F["Bcd"], w.cpu().numpy()[m], N).astype(np.float32)
    assert m.sum() > 300
    assert np.array_equal(_bits(got[m]), _bits(want))
    assert np.array_equal(_bits(got[~m]), _bits(sentinel[~m]))
    mpc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["staged", "in_place"])
def test_host_prediction_equals_the_restatement(oracle, mode):
    """predict_batch on the double wrenches of solve_batch, unmasked and masked, against the restatement bit for bit; the
    library reports which mode ran (in place only with records, wrench and output all pinned)."""
    B, N = 1500, 10
    recs, _ = scenarios.make_batch(3, B, horizon=N, seed=95)
    mpc = interface.BatchedMPC(B, N)
    alloc = interface.page_aligned if mode == "in_place" else (lambda shape, dt: np.zeros(shape, dt))
    x, w, pred = alloc((B,), scenarios.UPDATE_DTYPE), alloc((B, 12 * N), np.float64), alloc((B, N, 12), np.float64)
    x[:] = recs
    if mode == "in_place":
        mpc.pin(x, w, pred)
    mpc.solve_batch(x, strict=False, out=(w, np.zeros(B, np.int32)))
    F = formulation(oracle, recs, N)
    want = restate(F["x0"], F["Acd"], F["Bcd"], w, N)
    in_place = interface.lib().hmpc_debug_last_predict_in_place
    assert mpc.predict_batch(x, w, out=pred) is pred
    assert in_place() == (mode == "in_place")
    assert np.array_equal(_bits(pred), _bits(want))
    m = np.random.default_rng(96).random(B) < 0.3
    pred[:] = np.nan
    mpc.predict_batch(x, w, mask=m, out=pred)
    assert in_place() == (mode == "in_place")
    assert np.array_equal(_bits(pred[m]), _bits(want[m])) and np.isnan(pred[~m]).all()
    if mode == "in_place":                      # an output that is not pinned: staged, the same plans
        other = mpc.predict_batch(x, w)
        assert in_place() == 0 and np.array_equal(_bits(other), _bits(want))
    mpc.close()


@pytest.mark.gpu
def test_captured_masked_states_solve_and_prediction_replay_like_eager_calls():
    """The masked states solve and the prediction captured in one torch graph, replayed with other masks and states written
    into the captured tensors, against the same two calls made eagerly on a second context: wrench, status and plan bit for
    bit after every replay."""
    import torch

    B, N = 2048, 10
    sets = [_to_dev(_states(3, B, N, 100 + k).view(np.uint8).reshape(B, -1)) for k in range(3)]
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)

    def buffers():
        return (torch.zeros((B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda"),
                torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda"),
                torch.zeros((B, N, 12), dtype=torch.float32, device="cuda"))

    def tick(mpc, st, mask, bufs):
        rec, w, s, p = bufs
        mpc.solve_states_device_masked(st, B, mask, rec, w, s)
        mpc.predict_device(rec, B, w, p, d_mask=mask)

    st = sets[0].clone()
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    ba, bb = buffers(), buffers()
    tick(a, st, mask, ba)          # loads the kernels outside the capture
    tick(b, st, mask, bb)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        tick(a, st, mask, ba)
    rng = np.random.default_rng(101)
    for k, p in enumerate((0.2, 0.0, 1.0, 0.5)):
        m = torch.from_numpy(rng.random(B) < p).cuda()
        st.copy_(sets[(k + 1) % 3])
        mask.copy_(m)
        gr.replay()
        tick(b, sets[(k + 1) % 3], m, bb)
        torch.cuda.synchronize()
        for x, y in zip(ba[1:], bb[1:]):
            x, y = x.cpu().numpy(), y.cpu().numpy()
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), k
    a.close()
    b.close()


@pytest.mark.gpu
def test_device_plan_tracking_cost_is_the_kernels_qp_objective(oracle):
    """The tracking cost of the device's plan against 1/2 U'HU + g'U + d'Sd with H and g from the kernel's own assembly
    (hmpc_assemble_device) and d'Sd from the oracle; the plan is float, one more rounding of 2^-24 per state."""
    import torch

    B, N = 256, 10
    recs, _ = scenarios.make_batch(2, B, horizon=N, seed=110)
    mpc = interface.BatchedMPC(B, N)
    d_rec, w, s = _device_solve(mpc, recs, N)
    d_pred = torch.zeros((B, N, 12), dtype=torch.float32, device="cuda")
    mpc.predict_device(d_rec, B, w, d_pred)
    qp = mpc.assemble_device(d_rec, B)
    torch.cuda.synchronize()
    H = qp["H"].cpu().numpy()
    H = np.triu(H) + np.triu(H, 1).transpose(0, 2, 1)      # upper triangle valid
    g, U, pred = qp["g"].cpu().numpy(), w.cpu().numpy().astype(np.float64), d_pred.cpu().numpy().astype(np.float64)
    F = formulation(oracle, recs, N)
    for i in range(B):
        track, q, scale = objective_terms(recs[i], U[i], pred[i], H[i], g[i], F["A_qp"][i], F["x0"][i], N)
        assert abs(track - q) <= OBJ_K * EPS32 * scale, (i, track, q, scale)
    mpc.close()


@pytest.mark.gpu
def test_prediction_calls_check_their_arguments():
    import torch

    B, N = 64, 10
    mpc = interface.BatchedMPC(B, N)
    L = interface.lib()
    ERR = interface.HMPC_ERR_ARG
    rec = torch.zeros((B + 1, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    w = torch.zeros((B + 1, 12 * N), dtype=torch.float32, device="cuda")
    p = torch.zeros((B + 1, N, 12), dtype=torch.float32, device="cuda")
    r, wp, pp = rec.data_ptr(), w.data_ptr(), p.data_ptr()
    assert L.hmpc_predict_device(mpc._h, r, B + 1, None, wp, pp, None) == ERR
    assert L.hmpc_predict_device(mpc._h, r, -1, None, wp, pp, None) == ERR
    assert L.hmpc_predict_device(mpc._h, None, 4, None, wp, pp, None) == ERR
    assert L.hmpc_predict_device(mpc._h, r, 4, None, None, pp, None) == ERR
    assert L.hmpc_predict_device(mpc._h, r, 4, None, wp, None, None) == ERR
    assert L.hmpc_predict_device(mpc._h, r, 0, None, wp, pp, None) == interface.HMPC_OK
    x = np.zeros(B + 1, scenarios.UPDATE_DTYPE)
    wh, ph = np.zeros((B + 1, 12 * N)), np.zeros((B + 1, N, 12))
    assert L.hmpc_predict_batch(mpc._h, x.ctypes.data, B + 1, None, wh.ctypes.data, ph.ctypes.data) == ERR
    assert L.hmpc_predict_batch(mpc._h, None, 4, None, wh.ctypes.data, ph.ctypes.data) == ERR
    assert L.hmpc_predict_batch(mpc._h, x.ctypes.data, 4, None, None, ph.ctypes.data) == ERR
    assert L.hmpc_predict_batch(mpc._h, x.ctypes.data, 4, None, wh.ctypes.data, None) == ERR
    assert L.hmpc_predict_batch(mpc._h, x.ctypes.data, 0, None, wh.ctypes.data, ph.ctypes.data) == interface.HMPC_OK
    ph[:] = 7.0
    assert L.hmpc_predict_batch(mpc._h, x.ctypes.data, 4, np.zeros(4, np.uint8).ctypes.data, wh.ctypes.data,
                                ph.ctypes.data) == interface.HMPC_OK
    assert (ph == 7.0).all()                                # an empty mask writes nothing
    mpc.close()
