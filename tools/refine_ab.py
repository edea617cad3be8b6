#!/usr/bin/env python
"""A/B of the refinement class (hmpc_set_refinement): device time of hmpc_solve_device with refinement on against off.

    python tools/refine_ab.py [--reps 30] [--out FILE]

Workloads: configs[1]-style batches (1024 walking robots, horizon 10) in which 0 %, 1 % and 10 % of the robots are replaced
by a robot lying on its side (tests/golden/stress_referee.npz, h10_lying: scaled condition number 2.9e5, code 4 without
refinement), plus one lying robot alone (the cost of a handed-over instance).  The packed records are resident on the GPU;
every sample is one eager call timed with CUDA events on its stream, and the two arms alternate sample by sample on two
contexts so that clock and thermal drift hit both alike.  Prints one line per workload and writes a JSON summary.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hector_simulation_b200 import interface, scenarios  # noqa: E402

N = 10


def lying_record():
    g = np.load(os.path.join(ROOT, "tests", "golden", "stress_referee.npz"))
    return np.ascontiguousarray(g["h10_lying_records"]).view(scenarios.UPDATE_DTYPE).reshape(-1)[0]


def workload(B, frac, seed=1):
    recs, _ = scenarios.make_batch(2, B, horizon=N, seed=scenarios.config_seed(2) + seed) if B > 1 else (None, None)
    if B == 1:
        return np.array([lying_record()])
    nf = int(round(frac * B))
    if nf:
        recs[np.random.default_rng(seed).choice(B, nf, replace=False)] = lying_record()
    return recs


def power_limit():
    try:
        import subprocess

        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = []
    for B, frac in ((1, 1.0), (1024, 0.0), (1024, 0.01), (1024, 0.10)):
        recs = workload(B, frac)
        d_rec = torch.from_numpy(interface.pack_records(recs, N)).cuda()
        ctx = {on: interface.BatchedMPC(B, N) for on in (False, True)}
        ctx[True].set_refinement(True)
        out = {on: (torch.zeros((B, 12 * N), dtype=torch.float32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda"))
               for on in (False, True)}
        times = {False: [], True: []}
        stream = torch.cuda.current_stream()
        for rep in range(a.reps + 3):
            for on in ((False, True) if rep % 2 == 0 else (True, False)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                ctx[on].solve_device(d_rec, B, out[on][0], out[on][1])
                e1.record(stream)
                torch.cuda.synchronize()
                if rep >= 3:
                    times[on].append(e0.elapsed_time(e1) * 1e3)
        s_off, s_on = out[False][1].cpu().numpy(), out[True][1].cpu().numpy()
        row = dict(B=B, fallen=frac, n_fallen=int((interface.status_code(s_off) == 4).sum()),
                   refined=int(interface.status_refined(s_on).sum()), not_solved_on=int((interface.status_code(s_on) != 0).sum()),
                   off_us_median=float(np.median(times[False])), on_us_median=float(np.median(times[True])),
                   off_us_min=float(np.min(times[False])), on_us_min=float(np.min(times[True])))
        row["on_over_off"] = row["on_us_median"] / row["off_us_median"]
        rows.append(row)
        print("B=%4d fallen %4.1f%% (%3d code 4 off, %3d refined on): off %8.1f us, on %8.1f us (median of %d), on/off %.3f" %
              (B, 100 * frac, row["n_fallen"], row["refined"], row["off_us_median"], row["on_us_median"], a.reps, row["on_over_off"]),
              flush=True)
        for c in ctx.values():
            c.close()
    res = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), reps=a.reps, rows=rows)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
