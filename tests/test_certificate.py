"""The certificate: a first-order optimality (KKT) check of each robot's wrench for its row, made by a kernel of its own
(hmpc_certify_device, hmpc_certify_batch, BatchedMPC.certify_device / certify_batch).

The restatement below is the kernel in numpy and plain Python floats, float64, in the kernel's operation order, on the
oracle's float32 x0, Acd, Bcd, Fblk, lb and ub.  CPU: the kernel's source on the host (tests/host_emul/certify_on_host.cpp)
equals it, over both row layouts and both element types; the adjoint gradient is the oracle's HU + g; the fp64 referee's
optima pass and wrong answers fail; the kernel source's own solves pass; masks, rows past the batch, a null context and a
ThreadSanitizer run.  GPU: the device call on the device's own solves, the host call in both modes, graph capture and the
refinement class."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_golden
from hector_simulation_b200 import interface, scenarios
from test_kernel_source_on_host import BUILD, DEVICE_HEADER, HERE, _host_buildable, _p
from test_prediction import restate as restate_plan

FIXTURES = ["cfg1_h10", "cfg2_h10", "cfg3_h10", "cfg4_h5", "cfg4_h16", "degenerate_zero_force_h10"]
STRESS = ["h10_x4", "h10_x8", "h14_x4", "h10_lying"]
DT, F_MAX = 0.04, 500.0
EPS32 = 2.0 ** -24
CERT_DTYPE = np.dtype([("cost", "<f8"), ("stationarity", "<f8"), ("primal", "<f8"), ("complementarity", "<f8"),
                       ("n_active", "<i4"), ("flags", "<i4")])
_LIB = {}


# ---- the restatement ---------------------------------------------------------------------------------------------------
def constants():
    """the kernel's constants, read from its host build: act_k, act_abs, nnls_dual, nnls_pivot, tiny, and the thresholds"""
    c = np.zeros(10)
    certify_emulation().emul_certify_constants(_p(c))
    return dict(zip(("act_k", "act_abs", "dual", "pivot", "tiny", "stat_tol", "primal_tol", "compl_tol", "eps", "iters"), c))


def formulation(oracle, records, N):
    setup = oracle.make_setup(N, dt=DT, f_max=F_MAX)
    F = [oracle.formulate_f32(r, setup) for r in records]
    return {k: np.array([f[k] for f in F]) for k in ("x0", "Acd", "Bcd", "A_qp", "H", "g", "Fblk", "lb", "ub")}


def _ls(Z, P, b, pivot):
    p = [t for t in range(len(Z)) if P >> t & 1]
    L = [[0.0] * 8 for _ in range(8)]
    D, h = [0.0] * 8, [0.0] * 8
    for q in range(len(p)):
        hq = 0.0
        for c in range(6):
            hq = hq + Z[p[q]][c] * b[c]
        h[q] = hq
        for r in range(q + 1):
            g = 0.0
            for c in range(6):
                g = g + Z[p[q]][c] * Z[p[r]][c]
            for t in range(r):
                g = g - (L[q][t] * L[r][t]) * D[t]
            if r < q:
                L[q][r] = g / D[r]
            else:
                gqq = 0.0
                for c in range(6):
                    gqq = gqq + Z[p[q]][c] * Z[p[q]][c]
                if not g > pivot * gqq:
                    return None
                D[q] = g
    for q in range(len(p)):
        v = h[q]
        for t in range(q):
            v = v - L[q][t] * h[t]
        h[q] = v
    for q in range(len(p)):
        h[q] = h[q] / D[q]
    for q in range(len(p) - 1, -1, -1):
        v = h[q]
        for t in range(q + 1, len(p)):
            v = v - L[t][q] * h[t]
        h[q] = v
    z = [0.0] * len(Z)
    for q in range(len(p)):
        z[p[q]] = h[q]
    return z


def nnls_restated(Z, b, C):
    """Lawson-Hanson as cert_nnls runs it: y >= 0 minimising ||Z'y - b||"""
    k = len(Z)
    P = out = 0
    bmax = max(abs(v) for v in b)
    tol = C["dual"] * bmax
    y = [0.0] * k
    for _ in range(int(C["iters"])):
        r = []
        for c in range(6):
            v = b[c]
            for t in range(k):
                if P >> t & 1:
                    v = v - Z[t][c] * y[t]
            r.append(v)
        best, wb = -1, tol
        for t in range(k):
            if (P | out) >> t & 1:
                continue
            w = 0.0
            for c in range(6):
                w = w + Z[t][c] * r[c]
            if w > wb:
                wb, best = w, t
        if best < 0:
            break
        P |= 1 << best
        for inner in range(8):
            z = _ls(Z, P, b, C["pivot"])
            if z is None or (inner == 0 and not z[best] > 0.0):
                P &= ~(1 << best)
                out |= 1 << best
                break
            out = 0
            if all(z[t] > 0.0 for t in range(k) if P >> t & 1):
                y = [z[t] if P >> t & 1 else 0.0 for t in range(k)]
                break
            a, tmin = 2.0, -1
            for t in range(k):
                if P >> t & 1 and not z[t] > 0.0:
                    at = y[t] / (y[t] - z[t])
                    if at < a:
                        a, tmin = at, t
            if tmin < 0:
                break
            for t in range(k):
                if P >> t & 1:
                    y[t] = y[t] + a * (z[t] - y[t])
            y[tmin] = 0.0
            for t in range(k):
                if P >> t & 1 and not y[t] > 0.0:
                    P &= ~(1 << t)
                    y[t] = 0.0
    return y


def _col12(leg, c):
    return 3 * leg + c if c < 3 else 6 + 3 * leg + (c - 3)


def restate(F, records, U, N):
    """The certificate in numpy: F the oracle's float32 formulation of the records, U [B,12N] (the values the kernel reads,
    as float64) -> (cert [B] CERT_DTYPE, lambda [B,N,2,8] f64, gradient [B,12N], [B,2] the
    gradient and row scales)"""
    C = constants()
    B = len(records)
    U = np.asarray(U, np.float64)
    X = restate_plan(F["x0"], F["Acd"], F["Bcd"], U, N)
    XA = restate_plan(np.abs(F["x0"]), np.abs(F["Acd"]), np.abs(F["Bcd"]), np.abs(U), N)
    S = np.array([r["weights"] for r in records], np.float32).astype(np.float64)
    Al = np.array([r["Alpha_K"] for r in records], np.float32).astype(np.float64)
    traj = np.array([r["traj"][:12 * N] for r in records], np.float32).astype(np.float64).reshape(B, N, 12)
    gait = np.array([r["gait"][:2 * N] for r in records]).reshape(B, N, 2)
    Acd, Bcd = F["Acd"].astype(np.float64), F["Bcd"].astype(np.float64)
    # cost: lane r's terms step by step, then the lanes in order
    c = np.zeros((B, 12))
    for k in range(N):
        e = X[:, k] - traj[:, k]
        u = U[:, 12 * k:12 * k + 12]
        c = c + (S * e) * e
        c = c + (Al * u) * u
    J = np.zeros(B)
    for r in range(12):
        J = J + c[:, r]
    # adjoint and gradient
    S2, A2 = 2.0 * S, 2.0 * Al
    p, q = np.zeros((B, 12)), np.zeros((B, 12))
    G, GA = np.zeros((B, 12 * N)), np.zeros((B, 12 * N))
    for k in range(N, 0, -1):
        acc, acca = p.copy(), q.copy()
        for j in range(12):
            for r in ((0, 1, 2) if 6 <= j < 9 else ((j - 6,) if j >= 9 else ())):
                acc[:, j] = acc[:, j] + Acd[:, r, j] * p[:, r]
                acca[:, j] = acca[:, j] + np.abs(Acd[:, r, j]) * q[:, r]
        xd = traj[:, k - 1]
        p = acc + S2 * (X[:, k - 1] - xd)
        q = acca + np.abs(S2) * (XA[:, k - 1] + np.abs(xd))
        u = U[:, 12 * (k - 1):12 * k]
        g, ga = np.zeros((B, 12)), np.zeros((B, 12))
        for j in range(12):
            for r in ((6, 7, 8, 9 + j % 3) if j < 6 else (6, 7, 8)):
                g[:, j] = g[:, j] + Bcd[:, r, j] * p[:, r]
                ga[:, j] = ga[:, j] + np.abs(Bcd[:, r, j]) * q[:, r]
        G[:, 12 * (k - 1):12 * k] = g + A2 * u
        GA[:, 12 * (k - 1):12 * k] = ga + np.abs(A2) * np.abs(u)
    cert = np.zeros(B, CERT_DTYPE)
    lam = np.zeros((B, N, 2, 8))
    scales = np.zeros((B, 2))
    for i in range(B):
        Fb, lb, ub = F["Fblk"][i].astype(np.float64), F["lb"][i].astype(np.float64), F["ub"][i].astype(np.float64)
        stat = prim = comp = ps = gs = 0.0
        nact, swing = 0, False
        blocks = []
        for s in range(N):
            for leg in range(2):
                fz = float(np.float32(F_MAX) * np.float32(gait[i, s, leg]))
                cols = [12 * s + _col12(leg, c) for c in range(6)]
                u = [float(U[i, col]) for col in cols]
                A = [[float(Fb[8 * leg + t, _col12(leg, c)]) for c in range(6)] for t in range(8)]
                stance = not abs(fz) < 1e-4
                if stance:
                    gs = max(gs, max(GA[i, col] for col in cols))
                    v = []
                    for t in range(8):
                        vt = rs = 0.0
                        for cc in range(6):
                            vt = vt + A[t][cc] * u[cc]
                            rs = rs + abs(A[t][cc]) * abs(u[cc])
                        ps = max(ps, rs)
                        v.append(vt)
                    blocks.append((s, leg, cols, u, A, v))
                else:
                    for x in u:
                        if x != 0.0:
                            swing = True
                            prim = max(prim, abs(x))
        tol = (C["act_k"] * C["eps"]) * ps + C["act_abs"]
        for s, leg, cols, u, A, v in blocks:
            gb = [float(G[i, col]) for col in cols]
            Z, sl, up, rowof = [], [], [], []
            for t in range(8):
                lo, hi = lb[16 * s + 8 * leg + t], ub[16 * s + 8 * leg + t]
                haslo, hashi = lo > -1e10, hi < 1e10
                slo = v[t] - lo if haslo else 1e300
                shi = hi - v[t] if hashi else 1e300
                prim = max(prim, -slo, -shi)
                atlo, athi = slo <= tol, shi <= tol
                if atlo or athi:
                    upper = athi and (not atlo or shi < slo)
                    Z.append([-x for x in A[t]] if upper else A[t])
                    sl.append(abs(shi if upper else slo))
                    up.append(upper)
                    rowof.append(t)
            y = nnls_restated(Z, gb, C)
            nact += len(Z)
            res = list(gb)
            for t in range(len(Z)):
                for cc in range(6):
                    res[cc] = res[cc] - y[t] * Z[t][cc]
            stat = max(stat, max(abs(x) for x in res))
            for t in range(len(Z)):
                comp = max(comp, y[t] * sl[t])
                lam[i, s, leg, rowof[t]] = -y[t] if up[t] else y[t]
        gsc, psc = max(gs, C["tiny"]), max(ps, C["tiny"])
        scales[i] = gsc, psc
        cert[i] = (J[i], stat / gsc, prim / psc, comp / (gsc * psc), nact, 0)
        f = (4 if swing else 0) | (8 if not cert[i]["stationarity"] <= C["stat_tol"] else 0)
        f |= (16 if not cert[i]["primal"] <= C["primal_tol"] else 0) | (32 if not cert[i]["complementarity"] <= C["compl_tol"] else 0)
        cert[i]["flags"] = f or 1
    return cert, lam, G, scales


# ---- the kernel's source on the host -----------------------------------------------------------------------------------
def certify_emulation():
    """certify_on_host.cpp built for the host as a library, once per process (the flags of kernel_source_on_host.cpp's build)"""
    if "lib" not in _LIB:
        os.makedirs(BUILD, exist_ok=True)
        hdr = os.path.join(BUILD, "hmpc_device_host_certify.cuh")
        with open(hdr, "w") as f:
            f.write(_host_buildable(open(DEVICE_HEADER).read()))
        out = os.path.join(BUILD, "libcertify_on_host.so")
        cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O2", "-fPIC", "-shared",
               "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"), '-DHMPC_DEVICE_HEADER="%s"' % hdr,
               os.path.join(HERE, "certify_on_host.cpp"), "-l:libstdc++.so.6", "-o", out]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        L = ctypes.CDLL(out)
        assert L.emul_certify_bytes() == CERT_DTYPE.itemsize
        _LIB["lib"] = L
    return _LIB["lib"]


def emul_certify(rows, N, U, update_rows, double=True, mask=None, cert=None, lam=None, B=None, grad=False):
    """the certificate kernel on the host over the first B (all) of `rows` (uint8 [*, stride]) -> (cert, lambda, gradient)"""
    L = certify_emulation()
    rows = np.ascontiguousarray(rows)
    B = rows.shape[0] if B is None else B
    dt = np.float64 if double else np.float32
    U = np.ascontiguousarray(U, dt)
    cert = np.zeros(rows.shape[0], CERT_DTYPE) if cert is None else cert
    lam = np.zeros((rows.shape[0], N, 2, 8), dt) if lam is None else lam
    g = np.zeros((rows.shape[0], 12 * N)) if grad else None
    L.emul_certify(_p(rows), int(update_rows), B, N, ctypes.c_float(DT), ctypes.c_float(F_MAX), _p(mask), int(double), _p(U),
                   _p(cert), _p(lam), _p(g))
    return cert, lam, g


def _rows(records, N, update_rows):
    if update_rows:
        return np.ascontiguousarray(records).view(np.uint8).reshape(len(records), -1)
    return interface.pack_records(records, N)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a.view(np.uint64)


def _close(got, want, rel=1e-12):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want).max(initial=0.0) <= rel * max(np.abs(want).max(initial=0.0), 1e-300)


def assert_equals_restatement(got, want, float_out=False):
    (c, lam, g), (wc, wlam, wg, _) = got, want
    assert np.array_equal(_bits(c["cost"]), _bits(wc["cost"]))
    if g is not None:
        assert np.array_equal(_bits(g), _bits(wg))
    assert np.array_equal(c["n_active"], wc["n_active"]) and np.array_equal(c["flags"], wc["flags"])
    for k in ("stationarity", "primal", "complementarity"):
        assert np.allclose(c[k], wc[k], rtol=1e-12, atol=1e-300), k
    wlam = wlam.astype(np.float32) if float_out else wlam
    assert _close(lam, wlam)


def fixture(name):
    """(records, N, wrenches) of a fixture: the oracle's solutions, and the referee's for the degenerate robot"""
    if name in STRESS:
        g = np.load(os.path.join(GOLDEN, "stress_referee.npz"))
        recs = np.ascontiguousarray(g[name + "_records"]).view(scenarios.UPDATE_DTYPE).reshape(-1)
        return recs, g[name + "_referee"].shape[1] // 12, g[name + "_referee"]
    g = load_golden(name)
    return g["records"], g["horizon"], g.get("q_referee", g["q_soln"])


@pytest.mark.parametrize("name", FIXTURES + ["stress_referee"])
def test_kernel_source_equals_the_restatement(oracle, name):
    """Both row layouts, both element types: cost and gradient bit for bit, the measures and multipliers within 1e-12."""
    sets = [fixture(s) for s in STRESS] if name == "stress_referee" else [fixture(name)]
    for recs, N, U in sets:
        F = formulation(oracle, recs, N)
        want64 = restate(F, recs, U, N)
        U32 = U.astype(np.float32)
        want32 = restate(F, recs, U32, N)
        for upd in (False, True):
            rows = _rows(recs, N, upd)
            assert_equals_restatement(emul_certify(rows, N, U, upd, grad=True), want64)
            assert_equals_restatement(emul_certify(rows, N, U32, upd, double=False, grad=True), want32, float_out=True)


# H and g are the reference's float32 formulation: each entry carries the rounding of float32 sums of products, a few units
# of 2^-24 of the magnitude of its terms.  The adjoint gradient equals HU + g to GRAD_K units of 2^-24 of the robot's
# gradient scale (the largest absolute-value gradient entry of its stance legs); measured worst over the fixtures: 1.91
# units (cfg2_h10), asserted at 8.
GRAD_K = 8


@pytest.mark.parametrize("name", FIXTURES[:5])
def test_adjoint_gradient_is_HU_plus_g(oracle, name):
    recs, N, U = fixture(name)
    F = formulation(oracle, recs, N)
    _, _, G = emul_certify(_rows(recs, N, False), N, U, False, grad=True)
    scales = restate(F, recs, U, N)[3]
    worst = 0.0
    for i in range(len(F["H"])):        # (the fixtures keep H and g of their first records)
        H = F["H"][i].astype(np.float64)
        H = np.triu(H) + np.triu(H, 1).T
        hug = H @ U[i] + F["g"][i].astype(np.float64)
        d = np.abs(G[i] - hug)[_stance_cols(recs[i], N)].max(initial=0.0) / (EPS32 * scales[i, 0])
        worst = max(worst, d)
    print("%s: worst |adjoint - (HU + g)| = %.2f units of 2^-24 of the gradient scale" % (name, worst))
    assert worst <= GRAD_K


def _stance_cols(record, N):
    gait = np.asarray(record["gait"][:2 * N]).reshape(N, 2)
    return np.array([gait[k // 12, (k % 12 // 3) & 1] != 0 for k in range(12 * N)])


def _tols():
    C = constants()
    return {"stationarity": C["stat_tol"], "primal": C["primal_tol"], "complementarity": C["compl_tol"]}


def _all_referee_optima(oracle):
    """(name, records, N, U) of the fp64 referee's optima: the stress fixture's, the degenerate robot's, and
    qp_dual_active_set.solve run on the reduced QPs of the oracle fixtures"""
    from oracle import qp_dual_active_set as QP

    out = [(s,) + fixture(s) for s in STRESS + ["degenerate_zero_force_h10"]]
    for name in FIXTURES[:5]:
        recs, N, _ = fixture(name)
        setup = oracle.make_setup(N)
        Us = []
        for r in recs:
            R = oracle.reduced_qp(r, setup)
            x, info = QP.solve(R["H"], R["g"], R["A"], R["lb"], R["ub"])
            assert info["status"] == 0
            u = np.zeros(12 * N)
            u[R["var_ind"]] = x
            Us.append(u)
        out.append((name + "_referee", recs, N, np.array(Us)))
    return out


# The measured floors over the referee's optima and the oracle's solutions, both instantiations (DESIGN.md §7):
# stationarity 1.13e-7 (cfg2_h10), primal 1.19e-8 (float wrenches of h10_x4), complementarity 5.3e-11.  The thresholds
# HMPC_CERT_*_TOL are 2e-6, 2e-7 and 1e-9: margins of 17x, 16x and 19x.
FLOORS = {"stationarity": 1.2e-7, "primal": 1.2e-8, "complementarity": 6e-11}


def test_referee_optima_pass_at_the_rounding_floor(oracle):
    """Every referee optimum passes with its measures at the floor; each block's residual is no worse than scipy's NNLS on
    the same candidate rows."""
    from scipy.optimize import nnls

    for name, recs, N, U in _all_referee_optima(oracle):
        for double in (True, False):
            W = U if double else U.astype(np.float32)
            c, lam, _ = emul_certify(_rows(recs, N, True), N, W, True, double=double)
            assert (c["flags"] == 1).all(), (name, c)
            for k, f in FLOORS.items():
                assert c[k].max() <= f, (name, k, c[k].max())
        F = formulation(oracle, recs, N)
        _, _, G, scales = restate(F, recs, U, N)
        gait = np.array([r["gait"][:2 * N] for r in recs]).reshape(len(recs), N, 2)
        for i in range(len(recs)):
            for s in range(N):
                for leg in range(2):
                    if not gait[i, s, leg]:
                        assert (lam[i, s, leg] == 0).all()
                        continue
                    cols = [12 * s + _col12(leg, cc) for cc in range(6)]
                    A = np.array([[F["Fblk"][i][8 * leg + t, _col12(leg, cc)] for cc in range(6)] for t in range(8)], np.float64)
                    on = lam[i, s, leg] != 0
                    mine = np.abs(G[i, cols] - A.T @ lam[i, s, leg]).max()
                    # scipy on the rows the kernel found active, signed as the kernel signed them
                    sg = np.where(lam[i, s, leg] < 0, -1.0, 1.0)
                    y, _ = nnls((A * sg[:, None])[on].T, G[i, cols]) if on.any() else (None, 0)
                    ref = np.abs(G[i, cols] - ((A * sg[:, None])[on].T @ y if on.any() else 0)).max()
                    assert mine - ref <= FLOORS["stationarity"] * scales[i, 0], (name, i, s, leg)


def _largest_stance_foot(record, U, N):
    gait = np.asarray(record["gait"][:2 * N]).reshape(N, 2)
    best = max(((abs(U[12 * s + 3 * leg + 2]), s, leg) for s in range(N) for leg in range(2) if gait[s, leg]))
    return best[1], best[2]


# What the perturbations of the referee optima measured (DESIGN.md §7), over their 243 robots:
#   scale      the largest stance force x (1 + 1e-3): 238 fail, the median at 16x the stationarity threshold; a 1e-3 change
#              of one force is not always 100x the rounding floor of the whole gradient, and 5 robots move along
#              directions their QP barely sees.
#   friction   fx of that foot moved so that -mu fx + fz < 0 by 1e-3 of fz: all but one fail, the median at 2500x.
#   zero_step  that step's twelve entries zeroed: every robot fails, the smallest at 28x (a foot at zero force sits on
#              every row's bound, so part of the gradient is absorbed by its multipliers).
#   swing      a swing entry set to 1e-3 of that force: every robot with a swing leg fails by HMPC_CERT_SWING.
@pytest.mark.parametrize("kind", ["scale", "zero_step", "friction", "swing"])
def test_wrong_answers_fail(oracle, kind):
    tol = _tols()
    measures, passed = [], 0
    for name, recs, N, U in _all_referee_optima(oracle):
        W = U.copy()
        keep = np.ones(len(recs), bool)
        for i in range(len(recs)):
            s, leg = _largest_stance_foot(recs[i], U[i], N)
            fz = 12 * s + 3 * leg + 2
            if kind == "scale":
                W[i, fz] *= 1 + 1e-3
            elif kind == "zero_step":
                W[i, 12 * s:12 * s + 12] = 0.0
            elif kind == "friction":
                W[i, fz - 2] = (W[i, fz] * (1 + 1e-3)) / 2.0
            else:
                gait = np.asarray(recs[i]["gait"][:2 * N]).reshape(N, 2)
                sw = [(a, b) for a in range(N) for b in range(2) if not gait[a, b]]
                if not sw:
                    keep[i] = False
                    continue
                W[i, 12 * sw[0][0] + 3 * sw[0][1] + 2] = 1e-3 * abs(U[i, fz])
        c, _, _ = emul_certify(_rows(recs, N, True), N, W, True)
        c = c[keep]
        passed += int((c["flags"] & 1).sum())
        if kind == "swing":
            assert (c["flags"] & 4).all()
        key = "primal" if kind == "friction" else "stationarity"
        measures += list(c[key] / tol[key])
    m = np.array(measures)
    print("%s: %d of %d pass; measure / threshold: smallest %.3g, median %.3g" % (kind, passed, len(m), m.min(), np.median(m)))
    if kind in ("zero_step", "swing"):
        assert passed == 0
    if kind == "zero_step":
        assert m.min() >= 20
    if kind == "scale":
        assert passed <= 5 and np.median(m) >= 10
    if kind == "friction":
        assert passed <= 1 and np.median(m) >= 100


def test_qpoases_answers_on_the_stress_fixtures(oracle):
    """qpOASES' answers: those more than 1e-3 off the referee fail; where the smaller errors land is printed."""
    g = np.load(os.path.join(GOLDEN, "stress_referee.npz"))
    for name in STRESS:
        recs, N, ref = fixture(name)
        q = g[name + "_qpoases"]
        err = np.abs(q - ref).max(1) / np.maximum(np.abs(ref).max(1), 1e-9)
        c, _, _ = emul_certify(_rows(recs, N, True), N, q, True)
        assert (c["flags"][err > 1e-3] & 1 == 0).all()
        print("%s: qpOASES error %.1e..%.1e, stationarity %.1e..%.1e, %d of %d pass" % (
            name, err.min(), err.max(), c["stationarity"].min(), c["stationarity"].max(), (c["flags"] == 1).sum(), len(c)))


def test_kernel_source_solves_pass(oracle):
    """emul_solve (the solve kernel's source on the host) on the fixture records: every status-0 robot's float wrench passes."""
    from test_kernel_source_on_host import emul_solve, host_emulation

    L = host_emulation()
    for name in ["cfg2_h10", "cfg3_h10", "cfg4_h5", "cfg4_h16"]:
        recs, N, _ = fixture(name)
        packed = interface.pack_records(recs, N)
        w, st, _ = emul_solve(L, N, packed=packed)
        ok = interface.status_code(st) == 0
        assert ok.mean() > 0.9
        c, _, _ = emul_certify(packed, N, w, False, double=False)
        assert (c["flags"][ok] == 1).all(), (name, c[ok][c["flags"][ok] != 1])


def test_mask_and_rows_beyond_the_batch_keep_their_bytes(oracle):
    recs, N, U = fixture("cfg3_h10")
    B = len(recs)
    rows = _rows(recs, N, False)
    want, wlam, _ = emul_certify(rows, N, U, False)
    rng = np.random.default_rng(7)
    sc = rng.integers(0, 256, B * CERT_DTYPE.itemsize, dtype=np.uint8).view(CERT_DTYPE)
    sl = rng.integers(0, 2 ** 63, (B, N, 2, 8), dtype=np.uint64).view(np.float64)
    for m in ((rng.random(B) < 0.3).astype(np.uint8) * 7, np.zeros(B, np.uint8), np.eye(1, B, B - 1)[0].astype(np.uint8)):
        on = m != 0
        c, lam, _ = emul_certify(rows, N, U, False, mask=m, cert=sc.copy(), lam=sl.copy())
        assert c[on].tobytes() == want[on].tobytes() and c[~on].tobytes() == sc[~on].tobytes()
        assert np.array_equal(_bits(lam[on]), _bits(wlam[on])) and np.array_equal(_bits(lam[~on]), _bits(sl[~on]))
    for b in (61, 62, 63):
        assert certify_emulation().emul_certify_grid(b) * 4 > b
        c, lam, _ = emul_certify(rows, N, U, False, cert=sc.copy(), lam=sl.copy(), B=b)
        assert c[:b].tobytes() == want[:b].tobytes() and c[b:].tobytes() == sc[b:].tobytes()
        assert np.array_equal(_bits(lam[b:]), _bits(sl[b:]))


def test_non_finite_inputs_never_pass(oracle):
    recs, N, U = fixture("cfg3_h10")
    W = U[:4].copy()
    W[0, 5] = np.nan
    W[1, 0] = np.inf
    r = recs[:4].copy()
    r[2]["traj"][3] = np.nan
    r[3]["q"][0] = np.nan
    c, _, _ = emul_certify(_rows(r, N, True), N, W, True)
    assert (c["flags"] & 2).all() and not (c["flags"] & 1).any()


def test_certify_calls_reject_a_null_context():
    L = interface.lib()
    x = np.zeros(64, np.float64)
    ERR = interface.HMPC_ERR_ARG
    assert L.hmpc_certify_device(None, x.ctypes.data, 1, None, x.ctypes.data, x.ctypes.data, None, None) == ERR
    assert L.hmpc_certify_batch(None, x.ctypes.data, 1, None, x.ctypes.data, x.ctypes.data, None) == ERR
    assert L.hmpc_certify_device(None, None, 0, None, None, None, None, None) == ERR


def test_kernel_source_has_no_races_under_thread_sanitizer(tmp_path):
    """The kernel over the stress fixture's h10_x8 robots, built with -fsanitize=thread: every shared-memory access of a
    warp is ordered by its __syncwarp / shuffles."""
    hdr = os.path.join(BUILD, "hmpc_device_host_certify.cuh")
    certify_emulation()
    exe = os.path.join(BUILD, "certify_tsan")
    cmd = ["g++", "-std=c++17", "-ffp-contract=off", "-w", "-pthread", "-O1", "-g", "-fsanitize=thread", "-DHMPC_CERTIFY_MAIN",
           "-I" + os.path.join(HERE, "fake_cuda"), "-I" + os.path.join(ROOT, "include"), '-DHMPC_DEVICE_HEADER="%s"' % hdr,
           os.path.join(HERE, "certify_on_host.cpp"), "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("no ThreadSanitizer runtime with this toolchain: " + r.stderr[-300:])
    recs, N, U = fixture("h10_x8")
    recs, U = recs[:8], U[:8]
    f = tmp_path / "rows.bin"
    f.write_bytes(np.array([len(recs), N], np.int32).tobytes() + np.ascontiguousarray(recs).tobytes()
                  + np.ascontiguousarray(U, np.float64).tobytes())
    run = subprocess.run([exe, str(f)], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0 and "WARNING: ThreadSanitizer" not in run.stderr, run.stderr[-3000:]
    assert run.stdout.strip() == "ok %d" % len(recs)


# ---- GPU: the library ----------------------------------------------------------------------------------------------------
def _to_dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _dev_cert(B):
    import torch

    return torch.zeros((B, CERT_DTYPE.itemsize), dtype=torch.uint8, device="cuda")


def _host_cert(d):
    return np.ascontiguousarray(d.cpu().numpy()).view(interface.CERTIFICATE_DTYPE).reshape(-1)


def _assert_sample_equals_restatement(oracle, recs, N, U, cert, lam, idx):
    """the rows `idx`: cost bit for bit, measures within 1e-12, multipliers (in their element type) equal"""
    F = formulation(oracle, recs[idx], N)
    want, wlam, _, _ = restate(F, recs[idx], np.asarray(U[idx], np.float64), N)
    assert np.array_equal(_bits(cert["cost"][idx]), _bits(want["cost"]))
    assert np.array_equal(cert["flags"][idx], want["flags"]) and np.array_equal(cert["n_active"][idx], want["n_active"])
    for k in ("stationarity", "primal", "complementarity"):
        assert np.allclose(cert[k][idx], want[k], rtol=1e-12, atol=1e-300), k
    assert _close(lam[idx], wlam.astype(lam.dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,B,N", [(2, 1024, 10), (3, 8192, 10), (4, 4096, 5), (4, 4096, 16)])
def test_device_certificate_of_the_device_solves(oracle, cfg, B, N):
    """hmpc_solve_device, then hmpc_certify_device on the same records and float wrenches: every status-0 robot passes, and a
    strided sample equals the float restatement."""
    import torch

    recs, _ = scenarios.make_batch(cfg, B, horizon=N, seed=40 + cfg)
    mpc = interface.BatchedMPC(B, N)
    d_rec = _to_dev(interface.pack_records(recs, N))
    w = torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda")
    s = torch.zeros(B, dtype=torch.int32, device="cuda")
    mpc.solve_device(d_rec, B, w, s)
    d_cert = _dev_cert(B)
    d_lam = torch.full((B, N, 2, 8), float("nan"), dtype=torch.float32, device="cuda")
    mpc.certify_device(d_rec, B, w, d_cert, d_lam)
    torch.cuda.synchronize()
    cert, lam, U = _host_cert(d_cert), d_lam.cpu().numpy(), w.cpu().numpy()
    ok = interface.status_code(s.cpu().numpy()) == 0
    assert ok.mean() > 0.99
    bad = cert[ok][cert["flags"][ok] != 1]
    print("cfg %d B %d N %d: %d of %d status-0 robots pass; worst stationarity %.2e primal %.2e complementarity %.2e" % (
        cfg, B, N, ok.sum() - len(bad), ok.sum(), cert["stationarity"][ok].max(), cert["primal"][ok].max(),
        cert["complementarity"][ok].max()))
    assert len(bad) == 0, bad[:8]
    _assert_sample_equals_restatement(oracle, recs, N, U, cert, lam, np.arange(0, B, max(1, B // 128)))
    mpc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["staged", "in_place"])
def test_host_certificate_equals_the_restatement(oracle, mode):
    """certify_batch on the double wrenches of solve_batch, unmasked and masked; the library reports which mode ran."""
    B, N = 1500, 10
    recs, _ = scenarios.make_batch(3, B, horizon=N, seed=95)
    mpc = interface.BatchedMPC(B, N)
    alloc = interface.page_aligned if mode == "in_place" else (lambda shape, dt: np.zeros(shape, dt))
    x, w = alloc((B,), scenarios.UPDATE_DTYPE), alloc((B, 12 * N), np.float64)
    cert, lam = alloc((B,), interface.CERTIFICATE_DTYPE), alloc((B, N, 2, 8), np.float64)
    x[:] = recs
    if mode == "in_place":
        mpc.pin(x, w, cert, lam)
    mpc.solve_batch(x, strict=False, out=(w, np.zeros(B, np.int32)))
    in_place = interface.lib().hmpc_debug_last_certify_in_place
    got, _ = mpc.certify_batch(x, w, out=cert, lam=lam)
    assert got is cert and in_place() == (mode == "in_place")
    assert (cert["flags"] == 1).mean() > 0.99
    _assert_sample_equals_restatement(oracle, recs, N, w, cert, lam, np.arange(0, B, 12))
    full, full_lam = cert.copy(), lam.copy()
    m = np.random.default_rng(96).random(B) < 0.3
    cert[:] = np.frombuffer(b"\xab" * cert.nbytes, interface.CERTIFICATE_DTYPE)
    lam[:] = np.nan
    mpc.certify_batch(x, w, mask=m, out=cert, lam=lam)
    assert in_place() == (mode == "in_place")
    assert cert[m].tobytes() == full[m].tobytes() and np.array_equal(_bits(lam[m]), _bits(full_lam[m]))
    assert (cert[~m].view(np.uint8) == 0xAB).all() and np.isnan(lam[~m]).all()
    other = mpc.certify_batch(x, w)                     # no multipliers, a new array: staged, the same certificates
    assert in_place() == 0 and other.tobytes() == full.tobytes()
    mpc.close()


@pytest.mark.gpu
def test_captured_states_solve_prediction_and_certificate_replay_like_eager_calls():
    """masked states solve -> predict -> certify in one torch graph, replayed with other masks and states, against the same
    calls made eagerly on a second context: every output bit for bit; unlisted robots keep their certificate bytes."""
    import torch

    B, N = 2048, 10

    def states(seed):
        _, inputs = scenarios.make_batch(3, B, horizon=N, seed=seed)
        return _to_dev(np.ascontiguousarray(scenarios.make_states(inputs, N)).view(np.uint8).reshape(B, -1))

    sets = [states(100 + k) for k in range(3)]
    a, b = interface.BatchedMPC(B, N), interface.BatchedMPC(B, N)

    def buffers():
        return (torch.zeros((B, interface.record_bytes(N)), dtype=torch.uint8, device="cuda"),
                torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda"),
                torch.zeros((B, N, 12), dtype=torch.float32, device="cuda"), _dev_cert(B),
                torch.zeros((B, N, 2, 8), dtype=torch.float32, device="cuda"))

    def tick(mpc, st, mask, bufs):
        rec, w, s, p, c, lam = bufs
        mpc.solve_states_device_masked(st, B, mask, rec, w, s)
        mpc.predict_device(rec, B, w, p, d_mask=mask)
        mpc.certify_device(rec, B, w, c, lam, d_mask=mask)

    st = sets[0].clone()
    mask = torch.ones(B, dtype=torch.bool, device="cuda")
    ba, bb = buffers(), buffers()
    tick(a, st, mask, ba)
    tick(b, st, mask, bb)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        tick(a, st, mask, ba)
    rng = np.random.default_rng(101)
    for k, p in enumerate((0.2, 0.0, 1.0, 0.5)):
        m = torch.from_numpy(rng.random(B) < p).cuda()
        before = ba[4].clone()
        st.copy_(sets[(k + 1) % 3])
        mask.copy_(m)
        gr.replay()
        tick(b, sets[(k + 1) % 3], m, bb)
        torch.cuda.synchronize()
        for x, y in zip(ba[1:], bb[1:]):
            assert np.array_equal(x.cpu().numpy().view(np.uint8), y.cpu().numpy().view(np.uint8)), k
        mm = m.cpu().numpy()
        assert np.array_equal(ba[4].cpu().numpy()[~mm], before.cpu().numpy()[~mm])
        s = bb[2].cpu().numpy()
        c = _host_cert(ba[4])
        listed_ok = mm & (interface.status_code(s) == 0)
        assert (c["flags"][listed_ok] == 1).all(), k
    a.close()
    b.close()


@pytest.mark.gpu
def test_refined_lying_robot_passes_and_what_the_certificate_says_without_refinement():
    """h10_lying among 63 walkers: with refinement on it comes back with bit 28 and passes; without it (code 4) the
    certificate of its wrench is printed."""
    import torch

    g = np.load(os.path.join(GOLDEN, "stress_referee.npz"))
    lying = np.ascontiguousarray(g["h10_lying_records"]).view(scenarios.UPDATE_DTYPE).reshape(-1)
    walk, _ = scenarios.make_batch(2, 63, horizon=10, seed=7)
    recs = np.concatenate([walk[:31], lying, walk[31:]])
    B, N = len(recs), 10
    for refine in (True, False):
        mpc = interface.BatchedMPC(B, N)
        mpc.set_refinement(refine)
        d_rec = _to_dev(interface.pack_records(recs, N))
        w = torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda")
        s = torch.zeros(B, dtype=torch.int32, device="cuda")
        mpc.solve_device(d_rec, B, w, s)
        d_cert = _dev_cert(B)
        mpc.certify_device(d_rec, B, w, d_cert)
        torch.cuda.synchronize()
        st, cert = s.cpu().numpy(), _host_cert(d_cert)
        print("refinement %s: lying robot status 0x%08x, certificate %s" % (refine, st[31], cert[31]))
        walkers = np.arange(B) != 31
        assert (cert["flags"][walkers] == 1).all()
        if refine:
            assert interface.status_code(st[31:32])[0] == 0 and st[31] & (1 << 28)
            assert cert["flags"][31] == 1
        else:
            assert interface.status_code(st[31:32])[0] == 4
        mpc.close()


@pytest.mark.gpu
def test_certify_calls_check_their_arguments():
    import torch

    B, N = 64, 10
    mpc = interface.BatchedMPC(B, N)
    L = interface.lib()
    ERR = interface.HMPC_ERR_ARG
    rec = torch.zeros((B + 1, interface.record_bytes(N)), dtype=torch.uint8, device="cuda")
    w = torch.zeros((B + 1, 12 * N), dtype=torch.float32, device="cuda")
    c = _dev_cert(B + 1)
    r, wp, cp = rec.data_ptr(), w.data_ptr(), c.data_ptr()
    assert L.hmpc_certify_device(mpc._h, r, B + 1, None, wp, cp, None, None) == ERR
    assert L.hmpc_certify_device(mpc._h, r, -1, None, wp, cp, None, None) == ERR
    assert L.hmpc_certify_device(mpc._h, None, 4, None, wp, cp, None, None) == ERR
    assert L.hmpc_certify_device(mpc._h, r, 4, None, None, cp, None, None) == ERR
    assert L.hmpc_certify_device(mpc._h, r, 4, None, wp, None, None, None) == ERR
    assert L.hmpc_certify_device(mpc._h, r, 0, None, wp, cp, None, None) == interface.HMPC_OK
    x = np.zeros(B + 1, scenarios.UPDATE_DTYPE)
    wh, ch = np.zeros((B + 1, 12 * N)), np.zeros(B + 1, interface.CERTIFICATE_DTYPE)
    assert L.hmpc_certify_batch(mpc._h, x.ctypes.data, B + 1, None, wh.ctypes.data, ch.ctypes.data, None) == ERR
    assert L.hmpc_certify_batch(mpc._h, None, 4, None, wh.ctypes.data, ch.ctypes.data, None) == ERR
    assert L.hmpc_certify_batch(mpc._h, x.ctypes.data, 4, None, None, ch.ctypes.data, None) == ERR
    assert L.hmpc_certify_batch(mpc._h, x.ctypes.data, 4, None, wh.ctypes.data, None, None) == ERR
    assert L.hmpc_certify_batch(mpc._h, x.ctypes.data, 0, None, wh.ctypes.data, ch.ctypes.data, None) == interface.HMPC_OK
    ch["cost"] = 7.0
    assert L.hmpc_certify_batch(mpc._h, x.ctypes.data, 4, np.zeros(4, np.uint8).ctypes.data, wh.ctypes.data, ch.ctypes.data,
                                None) == interface.HMPC_OK
    assert (ch["cost"] == 7.0).all()
    mpc.close()
