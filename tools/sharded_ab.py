#!/usr/bin/env python
"""A/B of the warm masked sharded tick (hmpc_solve_batch_sharded_warm) on one GPU, a one-rank NCCL group.

    python tools/sharded_ab.py [--ticks 200] [--warmup 10] [--out FILE]

Workloads: B = 1024 and 4096 walking robots (configs[1]-style records, horizon 10) in registered host arrays (the in-place
mode), the float wrenches gathered into a device buffer every tick.  A fifth of the robots is due per tick (robot i in ticks
t with (i + t) % 5 == 0).  Three arms, each on its own context, alternate tick by tick so that clock and thermal drift hit
them alike:
  sharded_masked  hmpc_solve_batch_sharded_warm with the tick's mask (shift NULL), gather
  sharded_cold    hmpc_solve_batch_sharded of every robot, gather
  masked          hmpc_solve_batch_masked with the tick's mask (no gather: the single-GPU call)
Wall time per tick is the host clock around the call, which ends in a synchronisation of the solve; for the sharded arms
also around the call plus hmpc_shard_wait (the gather landed).  A separate short run under torch.profiler gives the carry
kernel's device time.  Outputs are checked: the sharded masked arm's listed rows equal the masked arm's bit for bit (same
warm-start history), its gathered rows equal each robot's latest row, and the cold arm's gathered rows are its wrenches'
float rounding.  Prints one line per workload and a JSON summary with the card's name, power limit and max SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hector_simulation_b200 import interface, scenarios  # noqa: E402

N = 10
ARMS = ("sharded_masked", "sharded_cold", "masked")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return r.stdout.strip().splitlines()[0]


def run(B, ticks, warmup):
    import torch

    recs, _ = scenarios.make_batch(2, B, horizon=N, seed=scenarios.config_seed(2) + 7)
    masks = [((np.arange(B) + t) % 5 == 0).astype(np.uint8) for t in range(5)]
    side = {}
    for a in ARMS:
        mpc = interface.BatchedMPC(B, N)
        if a.startswith("sharded"):
            mpc.shard_init(0, 1, interface.BatchedMPC.shard_unique_id())
        x = interface.page_aligned((B,), scenarios.UPDATE_DTYPE)
        x[:] = recs
        w = interface.page_aligned((B, 12 * N), np.float64)
        s = interface.page_aligned((B,), np.int32)
        mpc.pin(x, w, s)
        d_all = torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda")
        side[a] = (mpc, x, w, s, d_all)
    torch.cuda.synchronize()

    def call(a, m):
        mpc, x, w, s, d_all = side[a]
        if a == "sharded_masked":
            mpc.solve_batch_sharded_warm(x, (w, s), d_all, mask=m)
        elif a == "sharded_cold":
            mpc.solve_batch_sharded(x, (w, s), d_all)
        else:
            mpc.solve_batch_masked(x, m, out=(w, s))

    t_call = {a: [] for a in ARMS}
    t_wait = {a: [] for a in ARMS if a.startswith("sharded")}
    latest = np.zeros((B, 12 * N), np.float32)
    same_listed = gather_ok = cold_gather_ok = True
    for t in range(warmup + ticks):
        m = masks[t % 5]
        for a in ARMS[t % 3:] + ARMS[:t % 3]:
            h0 = time.perf_counter()
            call(a, m)
            h1 = time.perf_counter()
            if a.startswith("sharded"):
                side[a][0].shard_wait()
            h2 = time.perf_counter()
            if t >= warmup:
                t_call[a].append((h1 - h0) * 1e6)
                if a in t_wait:
                    t_wait[a].append((h2 - h0) * 1e6)
        on = m != 0
        ws, wm = side["sharded_masked"][2], side["masked"][2]
        same_listed &= np.array_equal(ws[on].view(np.uint8), wm[on].view(np.uint8))
        latest[on] = ws[on].astype(np.float32)
        if t % 10 == 0 or t == warmup + ticks - 1:   # (the device-to-host copies stay out of most ticks)
            gather_ok &= np.array_equal(side["sharded_masked"][4].cpu().numpy().view(np.uint32), latest.view(np.uint32))
            wc, dc = side["sharded_cold"][2], side["sharded_cold"][4]
            cold_gather_ok &= np.array_equal(dc.cpu().numpy().view(np.uint32), wc.astype(np.float32).view(np.uint32))
    cold_vs_masked = float(np.max(np.abs(side["sharded_cold"][2] - side["masked"][2]) /
                                  np.maximum(np.abs(side["masked"][2]).max(1, keepdims=True), 1e-9)))
    codes = [int((interface.status_code(side[a][3]) != 0).sum()) for a in ARMS]

    # the carry kernel's device time, in a run of its own under the profiler
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(20):
            call("sharded_masked", masks[t % 5])
        side["sharded_masked"][0].shard_wait()
        torch.cuda.synchronize()
    carry = [e.device_time_total for e in prof.events() if "carry" in e.name and e.device_time_total > 0]
    for a in ARMS:
        side[a][0].close()
    row = dict(B=B, due=0.2, ticks=ticks, listed_rows_bit_identical=bool(same_listed), gather_latest_rows=bool(gather_ok),
               cold_gather_is_float_rounding=bool(cold_gather_ok), cold_vs_masked_max_rel=cold_vs_masked,
               nonzero_codes=dict(zip(ARMS, codes)),
               carry_kernel_us=dict(n=len(carry), median=float(np.median(carry)) if carry else None,
                                    max=float(np.max(carry)) if carry else None))
    for a in ARMS:
        row[a] = dict(call_us_p50=float(np.percentile(t_call[a], 50)), call_us_p99=float(np.percentile(t_call[a], 99)))
        if a in t_wait:
            row[a].update(call_and_wait_us_p50=float(np.percentile(t_wait[a], 50)),
                          call_and_wait_us_p99=float(np.percentile(t_wait[a], 99)))
    return row


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(device=torch.cuda.get_device_name(0), card=card(), ticks=a.ticks, rows=[])
    print("card (name, power limit, max SM clock): %s" % res["card"], flush=True)
    for B in (1024, 4096):
        row = run(B, a.ticks, a.warmup)
        res["rows"].append(row)
        print("B=%4d due 0.2: call us p50/p99  sharded_masked %7.1f/%7.1f  sharded_cold %7.1f/%7.1f  masked %7.1f/%7.1f | "
              "+shard_wait p50/p99 sharded_masked %7.1f/%7.1f sharded_cold %7.1f/%7.1f | carry us %s | listed identical %s, "
              "gather latest %s, cold gather %s" %
              (B, row["sharded_masked"]["call_us_p50"], row["sharded_masked"]["call_us_p99"], row["sharded_cold"]["call_us_p50"],
               row["sharded_cold"]["call_us_p99"], row["masked"]["call_us_p50"], row["masked"]["call_us_p99"],
               row["sharded_masked"]["call_and_wait_us_p50"], row["sharded_masked"]["call_and_wait_us_p99"],
               row["sharded_cold"]["call_and_wait_us_p50"], row["sharded_cold"]["call_and_wait_us_p99"],
               row["carry_kernel_us"]["median"], row["listed_rows_bit_identical"], row["gather_latest_rows"],
               row["cold_gather_is_float_rounding"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
