#!/usr/bin/env python
"""Device time of the multi-command states call (hmpc_solve_states_device_multi) against preparing and solving the expanded
state batch.

    python tools/states_multi_ab.py [--reps 60] [--warmup 10] [--out FILE]

Workloads: B in {128, 1024} walking robots (configs[1]-style states) at horizon 10, K in {1, 4, 8, 16} candidate commands each
(the state's own and seeded perturbations: scenarios.command_candidates), resident on the GPU.  Three arms alternate
repetition by repetition (the order rotates) on one context, so that clock and thermal drift hit them alike:
  fused     hmpc_solve_states_device_multi: preparation, solve, cost, pick, torques of the chosen candidates
  expanded  hmpc_prepare_device of the B*K expanded states (row i*K + k = state i with command k) + hmpc_solve_device_ex
  gather    expanded, then a torch argmin over the certificate's costs of the status-0 candidates (hmpc_certify_device) and
            a gather of the chosen wrench rows and torques: what a caller without the fused call writes
Each is timed with CUDA events around its own work on the stream, with the host kept out of the window: a spin kernel
(torch.cuda._sleep, about SLEEP_US) is enqueued first, then the start event, the arm's calls and the end event.  The host
enqueue time of each arm (perf_counter around its calls) is reported too.  A repetition whose enqueue took more than half
the spin is not counted.  After the timed repetitions the fused call's wrenches, status words and torques of the chosen
candidates are compared bit for bit with the expanded arm's.
Prints one line per workload (medians, p10-p90, fused / expanded, fused / gather) and a JSON summary with the card's name and
power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hector_simulation_b200 import interface, scenarios  # noqa: E402

SLEEP_US = 3000.0
ARMS = ("fused", "expanded", "gather")


def power_limit():
    try:
        import subprocess

        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def _pct(v):
    return dict(us_median=float(np.median(v)), us_p10=float(np.percentile(v, 10)), us_p90=float(np.percentile(v, 90)))


def run(B, K, N, reps, warmup):
    import torch

    _, inputs = scenarios.make_batch(2, B, horizon=N, seed=scenarios.config_seed(2) + 7)  # configs[1]: walkers
    states = np.ascontiguousarray(scenarios.make_states(inputs, N))
    cmd = scenarios.command_candidates(states, K, seed=B + K)
    ex = np.repeat(states, K).copy()
    ex["state_des"] = cmd["state_des"].reshape(B * K, 5)
    ex["world_position_desired"] = cmd["world_position_desired"].reshape(B * K, 2)
    R, rs = B * K, interface.record_bytes(N)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d_states, d_cmd, d_ex = dev(states.view(np.uint8).reshape(B, -1)), dev(cmd.view(np.uint8).reshape(B, K, -1)), dev(ex.view(np.uint8).reshape(R, -1))
    mpc = interface.BatchedMPC(R, N)
    f32, i32, f64 = torch.float32, torch.int32, torch.float64
    rec = torch.zeros((B, rs), dtype=torch.uint8, device="cuda")
    traj = torch.zeros((B, K, 12 * N), dtype=f32, device="cuda")
    wm = torch.zeros((B, K, 12 * N), dtype=f32, device="cuda")
    sm = torch.zeros((B, K), dtype=i32, device="cuda")
    cm = torch.zeros((B, K), dtype=f64, device="cuda")
    bm = torch.zeros(B, dtype=i32, device="cuda")
    tm = torch.zeros((B, 10), dtype=f32, device="cuda")
    rex = torch.zeros((R, rs), dtype=torch.uint8, device="cuda")
    we = torch.zeros((R, 12 * N), dtype=f32, device="cuda")
    se = torch.zeros(R, dtype=i32, device="cuda")
    te = torch.zeros((R, 10), dtype=f32, device="cuda")
    cert = torch.zeros((R, interface.CERTIFICATE_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream()
    L = interface.lib()

    def expanded():
        mpc.prepare_device(d_ex, R, rex)
        L.hmpc_solve_device_ex(mpc._h, rex.data_ptr(), R, we.data_ptr(), se.data_ptr(), te.data_ptr(), ctypes.c_void_p(stream.cuda_stream))

    def gather():
        expanded()
        mpc.certify_device(rex, R, we, cert)
        cost = cert.view(f64)[:, 0].view(B, K)
        ok = ((se & 0xFF) == 0).view(B, K) & torch.isfinite(cost)
        best = torch.where(ok, cost, torch.full_like(cost, float("inf"))).argmin(dim=1)
        rows = torch.arange(B, device="cuda") * K + best
        return we.index_select(0, rows), te.index_select(0, rows)

    arms = {"fused": lambda: mpc.solve_states_device_multi(d_states, B, d_cmd, rec, traj, wm, sm, cm, bm, tm),
            "expanded": expanded, "gather": gather}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    torch.cuda._sleep(1_000_000)
    e1.record(stream)
    torch.cuda.synchronize()
    cycles = int(1_000_000 * SLEEP_US / (e0.elapsed_time(e1) * 1e3))
    t = {a: [] for a in arms}
    h = {a: [] for a in arms}
    dropped = 0
    for r in range(warmup + reps):
        order = ARMS[r % 3:] + ARMS[:r % 3]
        for a in order:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(cycles)
            h0 = time.perf_counter()
            e0.record(stream)
            arms[a]()
            e1.record(stream)
            h1 = time.perf_counter()
            torch.cuda.synchronize()
            if r >= warmup:
                if (h1 - h0) * 1e6 > 0.5 * SLEEP_US:
                    dropped += 1
                    continue
                t[a].append(e0.elapsed_time(e1) * 1e3)
                h[a].append((h1 - h0) * 1e6)
    same_w = bool(np.array_equal(wm.reshape(R, -1).cpu().numpy().view(np.uint32), we.cpu().numpy().view(np.uint32)))
    same_s = bool(np.array_equal(sm.reshape(-1).cpu().numpy(), se.cpu().numpy()))
    best = bm.cpu().numpy()
    pick = np.arange(B) * K + np.maximum(best, 0)
    tau_want = np.where((best >= 0)[:, None], te.cpu().numpy()[pick], np.float32(0))
    same_t = bool(np.array_equal(tm.cpu().numpy().view(np.uint32), tau_want.view(np.uint32)))
    codes = interface.status_code(se.cpu().numpy())
    mpc.close()
    row = dict(B=B, K=K, N=N, reps=reps, dropped=dropped, bit_identical=same_w and same_s and same_t,
               nonzero_status=int((codes != 0).sum()), best_not_0=int((best > 0).sum()))
    for a in arms:
        row[a] = _pct(t[a])
        row[a]["enqueue_us_median"] = float(np.median(h[a]))
    row["fused_over_expanded"] = row["fused"]["us_median"] / row["expanded"]["us_median"]
    row["fused_over_gather"] = row["fused"]["us_median"] / row["gather"]["us_median"]
    return row


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), rows=[])
    print("device: %s, %s" % (res["device"], res["power_limit"]), flush=True)
    for B in (128, 1024):
        for K in (1, 4, 8, 16):
            row = run(B, K, 10, a.reps, a.warmup)
            res["rows"].append(row)
            print("B=%4d K=%2d: us median (p10-p90) fused %8.1f (%.1f-%.1f)  expanded %8.1f (%.1f-%.1f)  gather %8.1f "
                  "(%.1f-%.1f)  fused/expanded %.3f  fused/gather %.3f | enqueue us fused %.1f expanded %.1f gather %.1f | "
                  "bit-identical %s | nonzero status %d | best>0 %d | dropped %d" %
                  (B, K, row["fused"]["us_median"], row["fused"]["us_p10"], row["fused"]["us_p90"], row["expanded"]["us_median"],
                   row["expanded"]["us_p10"], row["expanded"]["us_p90"], row["gather"]["us_median"], row["gather"]["us_p10"],
                   row["gather"]["us_p90"], row["fused_over_expanded"], row["fused_over_gather"],
                   row["fused"]["enqueue_us_median"], row["expanded"]["enqueue_us_median"], row["gather"]["enqueue_us_median"],
                   row["bit_identical"], row["nonzero_status"], row["best_not_0"], row["dropped"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
