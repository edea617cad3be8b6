#!/usr/bin/env python
"""A/B of the masked solve (hmpc_solve_device_masked) against the two ways a caller solves a changing subset without it.

    python tools/masked_ab.py [--ticks 60] [--out FILE]

Workloads: B = 1024 and 4096 walking robots (configs[1]-style records, horizon 10), packed and resident on the GPU.  The due
fraction is 1/5 (robot i is due in ticks t with (i + t) % 5 == 0: a different fifth every tick, as with a reference-style
controller whose robots were reset at different times) or 1 (every robot every tick).  Three arms alternate tick by tick,
each on its own context, so that clock and thermal drift hit them alike:
  masked   hmpc_solve_device_masked with the tick's bool mask (warm, shift NULL)
  full     hmpc_solve_device_warm of all B robots
  compact  torch compaction: nonzero -> index_select of the records -> hmpc_solve_device_ex of the dense batch -> index_copy_
           of wrench, torques and status back into the batch's rows
Every tick is timed with CUDA events around the arm's work on the stream (device time), and with the host clock from the
first enqueue to the end of a synchronize (wall time); the host time to enqueue is reported too, since the compaction waits
for the count of due robots there.  Outputs are checked: listed rows of the masked arm agree with the full arm's (both warm,
from different working-set histories: relative error), and a masked call with shift -1 (a cold solve) equals the compaction
arm's cold solve bit for bit.  Prints one line per workload and writes a JSON summary with the card's name and power limit.
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

N = 10
ARMS = ("masked", "full", "compact")


def power_limit():
    try:
        import subprocess

        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run(B, due, ticks, warmup):
    import torch

    recs, _ = scenarios.make_batch(2, B, horizon=N, seed=scenarios.config_seed(2) + 7)
    d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
    period = int(round(1 / due))
    masks = [torch.from_numpy((np.arange(B) + t) % period == 0).cuda() for t in range(period)]
    ctx = {a: interface.BatchedMPC(B, N) for a in ARMS}
    out = {a: (torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda"), torch.zeros((B, 10), dtype=torch.float32, device="cuda"),
               torch.zeros(B, dtype=torch.int32, device="cuda")) for a in ARMS}
    dense = (torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda"), torch.zeros((B, 10), dtype=torch.float32, device="cuda"),
             torch.zeros(B, dtype=torch.int32, device="cuda"))
    stream = torch.cuda.current_stream()
    L = interface.lib()

    def compact(mask):
        w, tau, s = out["compact"]
        idx = torch.nonzero(mask).squeeze(1)          # waits for the count
        n = idx.numel()
        if n:
            sub = d_rec.index_select(0, idx)
            interface._check(L.hmpc_solve_device_ex(ctx["compact"]._h, sub.data_ptr(), n, dense[0].data_ptr(), dense[2].data_ptr(),
                                                    dense[1].data_ptr(), ctypes.c_void_p(stream.cuda_stream)))
            w.index_copy_(0, idx, dense[0][:n])
            tau.index_copy_(0, idx, dense[1][:n])
            s.index_copy_(0, idx, dense[2][:n])

    def arm(a, mask):
        w, tau, s = out[a]
        if a == "masked":
            ctx[a].solve_device_masked(d_rec, B, mask, w, s, d_tau=tau)
        elif a == "full":
            ctx[a].solve_device_warm(d_rec, B, w, s, d_tau=tau)
        else:
            compact(mask)

    t_dev = {a: [] for a in ARMS}
    t_wall = {a: [] for a in ARMS}
    t_enq = {a: [] for a in ARMS}
    max_rel = 0.0
    for t in range(warmup + ticks):
        mask = masks[t % period]
        order = ARMS[t % 3:] + ARMS[:t % 3]
        for a in order:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            h0 = time.perf_counter()
            e0.record(stream)
            arm(a, mask)
            e1.record(stream)
            h1 = time.perf_counter()
            torch.cuda.synchronize()
            h2 = time.perf_counter()
            if t >= warmup:
                t_dev[a].append(e0.elapsed_time(e1) * 1e3)
                t_enq[a].append((h1 - h0) * 1e6)
                t_wall[a].append((h2 - h0) * 1e6)
        m = mask.cpu().numpy()
        wm, wf = out["masked"][0].cpu().numpy()[m], out["full"][0].cpu().numpy()[m]
        den = np.maximum(np.abs(wf).max(1, keepdims=True), 1e-9)
        max_rel = max(max_rel, float((np.abs(wm - wf) / den).max()))
    # cold parity: a masked call with shift -1 against the compaction arm's cold solve of the same robots
    cold = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    mask = masks[1 % period]
    wc, tc, sc = (x.clone() for x in out["compact"])
    ctx["masked"].solve_device_masked(d_rec, B, mask, wc, sc, d_tau=tc, d_shift=cold)
    compact(mask)
    torch.cuda.synchronize()
    m = mask.cpu().numpy()
    same = all(np.array_equal(x.cpu().numpy()[m].view(np.uint8), y.cpu().numpy()[m].view(np.uint8))
               for x, y in zip((wc, tc, sc), out["compact"]))
    codes = interface.status_code(out["masked"][2].cpu().numpy())
    for c in ctx.values():
        c.close()
    row = dict(B=B, due=due, ticks=ticks, cold_bit_identical=bool(same), warm_vs_full_max_rel=max_rel,
               masked_codes_nonzero=int((codes != 0).sum()))
    for a in ARMS:
        row[a] = dict(device_us_median=float(np.median(t_dev[a])), device_us_p90=float(np.percentile(t_dev[a], 90)),
                      wall_us_median=float(np.median(t_wall[a])), wall_us_p90=float(np.percentile(t_wall[a], 90)),
                      enqueue_us_median=float(np.median(t_enq[a])))
    return row


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), ticks=a.ticks, rows=[])
    print("device: %s, %s" % (res["device"], res["power_limit"]), flush=True)
    for B in (1024, 4096):
        for due in (0.2, 1.0):
            row = run(B, due, a.ticks, a.warmup)
            res["rows"].append(row)
            print("B=%4d due %.1f: device us (median) masked %7.1f full %7.1f compact %7.1f | wall us masked %7.1f full %7.1f "
                  "compact %7.1f | enqueue us masked %5.1f compact %5.1f | cold bit-identical %s, warm rel %.1e" %
                  (B, due, row["masked"]["device_us_median"], row["full"]["device_us_median"], row["compact"]["device_us_median"],
                   row["masked"]["wall_us_median"], row["full"]["wall_us_median"], row["compact"]["wall_us_median"],
                   row["masked"]["enqueue_us_median"], row["compact"]["enqueue_us_median"], row["cold_bit_identical"],
                   row["warm_vs_full_max_rel"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
