#!/usr/bin/env python
"""A/B of the state-path calls: where the time of hmpc_solve_batch_states goes, what its in-place mode and the masked call
save on the host, and what the fused device call saves against preparing every robot.

    python tools/states_ab.py [--ticks 200] [--out FILE]

Workloads: B = 1024 and 4096 walkers (configs[5]-style states, horizon 10).  The due fraction is 1/5 (robot i is due in
ticks t with (i + t) % 5 == 0) or 1.

  trace     HMPC_TRACE=1 on the staged hmpc_solve_batch_states (a child process): medians of the microseconds from entry to
            each trace point — per chunk: states copied into the pinned staging, chunk enqueued; then per chunk: synchronized;
            then the end of the result conversion.
  host      three arms alternate tick by tick, each on its own context; wall time of the call (ticks per second = 1 / median):
              staged         hmpc_solve_batch_states on unpinned arrays (what bench.py's e2e_states runs)
              in_place       the same call on pinned page_aligned arrays (the device-resident chain)
              masked_place   hmpc_solve_batch_states_masked in place with a fifth of the robots due
            Checks: staged and in_place results are bit-identical every tick (wrenches rounded to float: the in-place mode
            returns the solver's doubles); a final masked call with shift -1 (a cold solve) equals the staged results on
            its listed rows the same way.
  device    two arms alternate, each on its own context, states resident on the GPU; device time (CUDA events) and host
            enqueue time:
              fused          hmpc_solve_states_device_masked
              prepare_all    hmpc_prepare_device of all B robots + hmpc_solve_device_masked
            Check: listed rows of wrench, torques and status are bit-identical between the arms every tick.
Prints one line per row and a JSON summary with the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hector_simulation_b200 import interface, scenarios  # noqa: E402

N = 10


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def walkers(B, seed):
    _, inputs = scenarios.make_batch(5, B, horizon=N, seed=seed)
    states, _ = scenarios.make_rollout(inputs, N)
    return np.ascontiguousarray(states)


def med(x):
    return float(np.median(x))


def f32(w):
    """the bits of a double wrench rounded to float: the staged modes return float results, the in-place mode doubles"""
    return np.ascontiguousarray(w.astype(np.float32)).view(np.uint32)


def trace_child(B, ticks):
    """(runs with HMPC_TRACE=1) staged solve_batch_states calls; the library prints one trace line per call on stderr"""
    states = walkers(B, 5)
    mpc = interface.BatchedMPC(B, N)
    w, s = np.zeros((B, 12 * N)), np.zeros(B, np.int32)
    for _ in range(ticks):
        mpc.solve_batch_states(states, strict=False, out=(w, s))
    mpc.close()


def trace(B, ticks):
    env = dict(os.environ, HMPC_TRACE="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--trace-child", str(B), "--ticks", str(ticks)],
                       capture_output=True, text=True, env=env, timeout=1200)
    rows = [[float(v) for v in m.group(1).split()] for m in re.finditer(r"us since entry: ([0-9. ]+?)\s+\(", r.stderr)]
    rows = rows[min(10, len(rows) // 4):]                       # the first calls load kernels and warm the pool
    if not rows:
        return dict(error=r.stderr[-500:])
    pts = np.median(np.array(rows), axis=0)
    return dict(B=B, calls=len(rows), points_us=[round(float(v), 1) for v in pts])


def host(B, ticks, warmup):
    states = walkers(B, 6)
    arms = ("staged", "in_place", "masked_place")
    ctx = {a: interface.BatchedMPC(B, N) for a in arms}
    nw = 12 * N
    out = {"staged": (np.zeros((B, nw)), np.zeros(B, np.int32))}
    pin_st = {}
    for a in ("in_place", "masked_place"):   # (one pinned copy per context: a context unregisters what it pinned)
        pin_st[a] = interface.page_aligned((B,), scenarios.STATE_DTYPE)
        pin_st[a][:] = states
        out[a] = (interface.page_aligned((B, nw), np.float64), interface.page_aligned((B,), np.int32))
        ctx[a].pin(pin_st[a], *out[a])
    masks = [((np.arange(B) + t) % 5 == 0) for t in range(5)]
    wall = {a: [] for a in arms}
    same = True
    for t in range(warmup + ticks):
        order = arms[t % 3:] + arms[:t % 3]
        for a in order:
            h0 = time.perf_counter()
            if a == "staged":
                ctx[a].solve_batch_states(states, strict=False, out=out[a])
            elif a == "in_place":
                ctx[a].solve_batch_states(pin_st[a], strict=False, out=out[a])
            else:
                ctx[a].solve_batch_states_masked(pin_st[a], masks[t % 5], strict=False, out=out[a])
            if t >= warmup:
                wall[a].append((time.perf_counter() - h0) * 1e6)
        same &= np.array_equal(f32(out["staged"][0]), f32(out["in_place"][0]))
        same &= np.array_equal(out["staged"][1], out["in_place"][1])
    m = masks[0]
    w, s = out["masked_place"]
    ctx["masked_place"].solve_batch_states_masked(pin_st["masked_place"], m, shift=np.full(B, -1, np.int32), strict=False, out=(w, s))
    cold_same = np.array_equal(f32(w[m]), f32(out["staged"][0][m])) and np.array_equal(s[m], out["staged"][1][m])
    codes = int((interface.status_code(out["staged"][1]) != 0).sum())
    for a in ("in_place", "masked_place"):
        ctx[a].unpin(pin_st[a], *out[a])
    for c in ctx.values():
        c.close()
    row = dict(B=B, ticks=ticks, staged_vs_in_place_bit_identical=bool(same), masked_cold_bit_identical=bool(cold_same),
               staged_codes_nonzero=codes)
    for a in arms:
        row[a] = dict(wall_us_median=med(wall[a]), wall_us_p90=float(np.percentile(wall[a], 90)), ticks_per_s=1e6 / med(wall[a]))
    return row


def device(B, due, ticks, warmup):
    import torch

    states = walkers(B, 7)
    d_st = torch.from_numpy(states.view(np.uint8).reshape(B, 352).copy()).cuda()
    stride = interface.record_bytes(N)
    arms = ("fused", "prepare_all")
    ctx = {a: interface.BatchedMPC(B, N) for a in arms}
    rec = {a: torch.zeros((B, stride), dtype=torch.uint8, device="cuda") for a in arms}
    out = {a: (torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda"), torch.zeros((B, 10), dtype=torch.float32, device="cuda"),
               torch.zeros(B, dtype=torch.int32, device="cuda")) for a in arms}
    period = int(round(1 / due))
    masks = [torch.from_numpy((np.arange(B) + t) % period == 0).cuda() for t in range(period)]
    stream = torch.cuda.current_stream()
    t_dev = {a: [] for a in arms}
    t_enq = {a: [] for a in arms}
    same = True
    for t in range(warmup + ticks):
        mask = masks[t % period]
        for a in (arms if t % 2 == 0 else arms[::-1]):
            w, tau, s = out[a]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            h0 = time.perf_counter()
            e0.record(stream)
            if a == "fused":
                ctx[a].solve_states_device_masked(d_st, B, mask, rec[a], w, s, d_tau=tau)
            else:
                ctx[a].prepare_device(d_st, B, rec[a])
                ctx[a].solve_device_masked(rec[a], B, mask, w, s, d_tau=tau)
            e1.record(stream)
            h1 = time.perf_counter()
            torch.cuda.synchronize()
            if t >= warmup:
                t_dev[a].append(e0.elapsed_time(e1) * 1e3)
                t_enq[a].append((h1 - h0) * 1e6)
        m = mask.cpu().numpy()
        for x, y in zip(out["fused"], out["prepare_all"]):
            same &= np.array_equal(x.cpu().numpy()[m].view(np.uint8), y.cpu().numpy()[m].view(np.uint8))
    for c in ctx.values():
        c.close()
    row = dict(B=B, due=due, ticks=ticks, listed_bit_identical=bool(same))
    for a in arms:
        row[a] = dict(device_us_median=med(t_dev[a]), device_us_p90=float(np.percentile(t_dev[a], 90)),
                      enqueue_us_median=med(t_enq[a]))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-child", type=int, default=0, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.trace_child:
        trace_child(a.trace_child, a.ticks)
        return
    import torch

    res = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), ticks=a.ticks, trace=[], host=[], device_rows=[])
    print("device: %s, %s" % (res["device"], res["power_limit"]), flush=True)
    for B in (1024, 4096):
        row = trace(B, min(a.ticks, 100))
        res["trace"].append(row)
        print("trace B=%4d: us since entry (medians) %s" % (B, row.get("points_us", row)), flush=True)
    for B in (1024, 4096):
        row = host(B, a.ticks, a.warmup)
        res["host"].append(row)
        print("host  B=%4d: wall us (median) staged %7.1f in_place %7.1f masked_place %7.1f | ticks/s %7.0f %7.0f %7.0f | "
              "staged==in_place %s, masked cold==staged %s" %
              (B, row["staged"]["wall_us_median"], row["in_place"]["wall_us_median"], row["masked_place"]["wall_us_median"],
               row["staged"]["ticks_per_s"], row["in_place"]["ticks_per_s"], row["masked_place"]["ticks_per_s"],
               row["staged_vs_in_place_bit_identical"], row["masked_cold_bit_identical"]), flush=True)
    for B in (1024, 4096):
        for due in (0.2, 1.0):
            row = device(B, due, a.ticks, a.warmup)
            res["device_rows"].append(row)
            print("device B=%4d due %.1f: device us (median) fused %7.1f prepare_all %7.1f | enqueue us fused %5.1f prepare_all %5.1f | "
                  "listed bit-identical %s" %
                  (B, due, row["fused"]["device_us_median"], row["prepare_all"]["device_us_median"],
                   row["fused"]["enqueue_us_median"], row["prepare_all"]["enqueue_us_median"], row["listed_bit_identical"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
