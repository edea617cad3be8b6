#!/usr/bin/env python
"""Device time of the certificate (hmpc_certify_device) against the solve it follows.

    python tools/certify_ab.py [--reps 200] [--warmup 20] [--out FILE]

Workloads: B = 1024 and 4096 walking robots at horizon 10, and 1024 at horizon 16 (configs[1]-style records), packed and
resident on the GPU.  Two arms alternate repetition by repetition on one context, so that clock and thermal drift hit them
alike:
  solve    hmpc_solve_device (cold) of all B robots
  certify  hmpc_certify_device of all B robots on the records and wrenches of that solve, with the multipliers
Each is timed with CUDA events around its own work on the stream, with the host kept out of the window: a spin kernel
(torch.cuda._sleep, about SLEEP_US) is enqueued first, then the start event, the arm's call and the end event, so the GPU
reaches the start event only after the host has finished enqueueing the arm.  The host time from the start event's record
to the end event's record is reported too (`enqueue_us`); a repetition whose enqueue took more than half the spin is
not counted.
Prints one line per workload and a JSON summary with the card's name and power limit, measured in the same run.
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

SLEEP_US = 2000.0


def power_limit():
    try:
        import subprocess

        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run(B, N, reps, warmup):
    import torch

    recs, _ = scenarios.make_batch(2, B, horizon=N, seed=scenarios.config_seed(2) + 7)
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    mpc = interface.BatchedMPC(B, N)
    w = torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda")
    s = torch.zeros(B, dtype=torch.int32, device="cuda")
    cert = torch.zeros((B, interface.CERTIFICATE_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    lam = torch.zeros((B, N, 2, 8), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream()
    arms = {"solve": lambda: mpc.solve_device(d_rec, B, w, s), "certify": lambda: mpc.certify_device(d_rec, B, w, cert, lam)}
    # cycles of the spin: calibrated against the events, so that it lasts about SLEEP_US at the clock the card runs
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    torch.cuda._sleep(1_000_000)
    e1.record(stream)
    torch.cuda.synchronize()
    cycles = int(1_000_000 * SLEEP_US / (e0.elapsed_time(e1) * 1e3))
    t = {a: [] for a in arms}
    enq = {a: [] for a in arms}
    dropped = 0
    for r in range(warmup + reps):
        order = ("solve", "certify") if r % 2 == 0 else ("certify", "solve")
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
                enq[a].append((h1 - h0) * 1e6)
    codes = interface.status_code(s.cpu().numpy())
    flags = cert.cpu().numpy().view(interface.CERTIFICATE_DTYPE).reshape(-1)["flags"]
    mpc.close()
    row = dict(B=B, N=N, reps=reps, nonzero_status=int((codes != 0).sum()),
               status0_not_passing=int(((codes == 0) & (flags != interface.CERT_PASS)).sum()), dropped=dropped)
    for a in arms:
        row[a] = dict(device_us_median=float(np.median(t[a])), device_us_p10=float(np.percentile(t[a], 10)),
                      device_us_p90=float(np.percentile(t[a], 90)), enqueue_us_median=float(np.median(enq[a])))
    row["certify_over_solve"] = row["certify"]["device_us_median"] / row["solve"]["device_us_median"]
    return row


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), rows=[])
    print("device: %s, %s" % (res["device"], res["power_limit"]), flush=True)
    for B, N in ((1024, 10), (4096, 10), (1024, 16)):
        row = run(B, N, a.reps, a.warmup)
        res["rows"].append(row)
        print("B=%4d N=%2d: device us median (p10-p90) solve %7.1f (%.1f-%.1f)  certify %6.2f (%.2f-%.2f)  ratio %.4f | "
              "host enqueue us solve %.1f certify %.1f | status-0 not passing %d | dropped %d" %
              (B, N, row["solve"]["device_us_median"], row["solve"]["device_us_p10"], row["solve"]["device_us_p90"],
               row["certify"]["device_us_median"], row["certify"]["device_us_p10"], row["certify"]["device_us_p90"],
               row["certify_over_solve"], row["solve"]["enqueue_us_median"], row["certify"]["enqueue_us_median"],
               row["status0_not_passing"], row["dropped"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
