#!/usr/bin/env python
"""Device time of the multi-query solve (hmpc_solve_device_multi) against the single solve of the expanded batch.

    python tools/multi_ab.py [--reps 60] [--warmup 10] [--out FILE]

Workloads: B in {128, 1024} walking robots (configs[1]-style records) at horizon 10, K in {1, 4, 8, 16} candidate reference
trajectories each (the record's own and seeded perturbations of it), packed and resident on the GPU.  Two arms alternate
repetition by repetition on one context, so that clock and thermal drift hit them alike:
  multi     hmpc_solve_device_multi of the B robots x K candidates, no cost
  expanded  hmpc_solve_device (cold) of the B*K expanded records (row i*K + k = robot i's record with traj k)
Each is timed with CUDA events around its own work on the stream, with the host kept out of the window: a spin kernel
(torch.cuda._sleep, about SLEEP_US) is enqueued first, then the start event, the arm's call and the end event.  A repetition
whose enqueue took more than half the spin is not counted.  After the timed repetitions the outputs of both arms are compared
bit for bit (wrenches and status words).
Prints one line per workload (medians, p10-p90, multi / expanded) and a JSON summary with the card's name and power limit,
read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hector_simulation_b200 import interface, scenarios  # noqa: E402

SLEEP_US = 3000.0


def power_limit():
    try:
        import subprocess

        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def candidates(recs, N, K, seed):
    rng = np.random.default_rng(seed)
    own = np.stack([np.asarray(r["traj"][: 12 * N], np.float32) for r in recs])
    scale = np.tile(np.array([0.03, 0.03, 0.05, 0.02, 0.02, 0.01, 0.1, 0.1, 0.1, 0.2, 0.2, 0.05], np.float32), N)
    t = own[:, None, :] + (rng.normal(0.0, 1.0, (len(recs), K, 12 * N)) * scale).astype(np.float32)
    t[:, 0] = own
    return np.ascontiguousarray(t, np.float32)


def run(B, K, N, reps, warmup):
    import torch

    recs, _ = scenarios.make_batch(2, B, horizon=N, seed=scenarios.config_seed(2) + 7)  # configs[1]: walkers
    traj = candidates(recs, N, K, seed=B + K)
    ex = np.repeat(recs, K).copy()
    for r in range(B * K):
        ex[r]["traj"][: 12 * N] = traj[r // K, r % K]
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    d_ex = torch.from_numpy(interface.pack_records(ex, N)).cuda()
    d_traj = torch.from_numpy(traj).cuda()
    mpc = interface.BatchedMPC(B * K, N)
    wm = torch.zeros((B, K, 12 * N), dtype=torch.float32, device="cuda")
    sm = torch.zeros((B, K), dtype=torch.int32, device="cuda")
    we = torch.zeros((B * K, 12 * N), dtype=torch.float32, device="cuda")
    se = torch.zeros(B * K, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream()
    arms = {"multi": lambda: mpc.solve_device_multi(d_rec, B, d_traj, wm, sm),
            "expanded": lambda: mpc.solve_device(d_ex, B * K, we, se)}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    torch.cuda._sleep(1_000_000)
    e1.record(stream)
    torch.cuda.synchronize()
    cycles = int(1_000_000 * SLEEP_US / (e0.elapsed_time(e1) * 1e3))
    t = {a: [] for a in arms}
    dropped = 0
    for r in range(warmup + reps):
        order = ("multi", "expanded") if r % 2 == 0 else ("expanded", "multi")
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
    same_w = bool(np.array_equal(wm.reshape(B * K, -1).cpu().numpy().view(np.uint32), we.cpu().numpy().view(np.uint32)))
    same_s = bool(np.array_equal(sm.reshape(-1).cpu().numpy(), se.cpu().numpy()))
    codes = interface.status_code(se.cpu().numpy())
    mpc.close()
    row = dict(B=B, K=K, N=N, reps=reps, dropped=dropped, bit_identical=same_w and same_s, nonzero_status=int((codes != 0).sum()))
    for a in arms:
        row[a] = dict(us_median=float(np.median(t[a])), us_p10=float(np.percentile(t[a], 10)), us_p90=float(np.percentile(t[a], 90)))
    row["multi_over_expanded"] = row["multi"]["us_median"] / row["expanded"]["us_median"]
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
            print("B=%4d K=%2d: us median (p10-p90) multi %8.1f (%.1f-%.1f)  expanded %8.1f (%.1f-%.1f)  ratio %.3f | "
                  "bit-identical %s | nonzero status %d | dropped %d" %
                  (B, K, row["multi"]["us_median"], row["multi"]["us_p10"], row["multi"]["us_p90"], row["expanded"]["us_median"],
                   row["expanded"]["us_p10"], row["expanded"]["us_p90"], row["multi_over_expanded"], row["bit_identical"],
                   row["nonzero_status"], row["dropped"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
