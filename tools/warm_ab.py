"""Warm versus cold start on the same ticks (DESIGN.md §6).

One device rollout (hmpc_rollout_device) of configs[1]'s size — 1024 walkers, horizon 10 — logs the packed records of
every tick.  The log is then replayed tick by tick through hmpc_solve_device (cold) and hmpc_solve_device_warm (warm,
shift NULL: every robot moved one step, as in the loop), the two arms alternating in one process after a warm-up pass of
each.  Each tick is timed with CUDA events.  The warm arm starts every pass from hmpc_reset_warm_start, so its tick 0 is a
cold start, as a loop's first tick is.

Prints one JSON line: QP/s of each arm over all timed passes, per-tick p50 / p99 (us), mean working-set changes per robot
and tick (ticks >= 1), the outputs' agreement, and the GPU's name and power limit read in the same run.  --stamps adds
the median clock cycles per stage of one mid-loop tick of each arm (hmpc_debug_set_clock_buffer), for class-0 robots.

    python tools/warm_ab.py [--batch 1024] [--ticks 200] [--passes 5] [--stamps] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from hector_simulation_b200 import interface, scenarios  # noqa: E402

N = 10


def gpu_card(device):
    """name and power limit of the card the numbers are measured on"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [x.strip() for x in r.stdout.strip().split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clk)
    except Exception as e:  # the measurement stands, the label says what is missing
        return dict(name=torch.cuda.get_device_name(device), power_limit="unknown (%s)" % e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--passes", type=int, default=5, help="timed passes per arm, alternating")
    ap.add_argument("--stamps", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("warm_ab: no CUDA device")
    B, T = a.batch, a.ticks
    dev = torch.device("cuda", 0)

    # the ticks: one closed loop on the device, its records logged
    states, loop = scenarios.make_rollout(scenarios.make_batch(5, B, horizon=N, seed=2024)[1], N)
    ctx = interface.BatchedMPC(B, N)
    d_states = torch.from_numpy(states.view(np.uint8).reshape(B, -1).copy()).to(dev)
    d_loop = torch.from_numpy(loop.view(np.uint8).reshape(B, -1).copy()).to(dev)
    d_rlog = torch.zeros((T, B, interface.record_bytes(N)), dtype=torch.uint8, device=dev)
    ctx.rollout_device(d_states, d_loop, B, T, None, d_rlog)
    torch.cuda.synchronize()
    ctx.close()

    mpc = interface.BatchedMPC(B, N)
    d_w = {k: torch.zeros((T, B, 12 * N), dtype=torch.float32, device=dev) for k in ("cold", "warm")}
    d_s = {k: torch.zeros((T, B), dtype=torch.int32, device=dev) for k in ("cold", "warm")}
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(T)]

    def run_pass(arm, timed):
        if arm == "warm":
            mpc.reset_warm_start()
        for t in range(T):
            if timed:
                ev[t][0].record()
            if arm == "warm":
                mpc.solve_device_warm(d_rlog[t], B, d_w[arm][t], d_s[arm][t])
            else:
                mpc.solve_device(d_rlog[t], B, d_w[arm][t], d_s[arm][t])
            if timed:
                ev[t][1].record()
        torch.cuda.synchronize()
        return [ev[t][0].elapsed_time(ev[t][1]) * 1e3 for t in range(T)] if timed else None

    for arm in ("cold", "warm"):
        run_pass(arm, False)
    per_tick = {"cold": [], "warm": []}
    for _ in range(a.passes):
        for arm in ("cold", "warm"):
            per_tick[arm] += run_pass(arm, True)

    res = dict(workload="device rollout log replayed, B=%d N=%d, %d ticks x %d passes per arm" % (B, N, T, a.passes),
               card=gpu_card(0))
    for arm in ("cold", "warm"):
        us = np.array(per_tick[arm])
        st = d_s[arm].cpu().numpy()
        res[arm] = dict(qp_per_s=round(B * len(us) / (us.sum() * 1e-6)), tick_p50_us=round(float(np.percentile(us, 50)), 1),
                        tick_p99_us=round(float(np.percentile(us, 99)), 1),
                        changes_per_tick=round(float(interface.status_iters(st[1:]).mean()), 2),
                        not_optimal=int((interface.status_code(st) != 0).sum()))
    w = {k: d_w[k].cpu().numpy().reshape(-1, 12 * N) for k in d_w}
    d1 = np.linalg.norm(w["warm"][:, :12] - w["cold"][:, :12], axis=1) / np.maximum(np.linalg.norm(w["cold"][:, :12], axis=1), 1e-9)
    res["warm_vs_cold_first_step_rel_err_max"] = float(d1.max())
    res["warm_speedup"] = round(res["warm"]["qp_per_s"] / res["cold"]["qp_per_s"], 3)

    if a.stamps:
        # one mid-loop tick of each arm with the stage clock stamps on (a separate, untimed run of the same ticks)
        names = {"assembly": (0, 3), "sweep inversion": (3, 4), "active set": (4, 5), "polish + scatter": (5, 6)}
        mid = T // 2
        clk = torch.zeros((B, 32), dtype=torch.int64, device=dev)
        res["stage_cycles_median_class0"] = {}
        for arm in ("cold", "warm"):
            if arm == "warm":
                mpc.reset_warm_start()
            for t in range(mid + 1):
                if t == mid:
                    clk.zero_()
                    interface.lib().hmpc_debug_set_clock_buffer(ctypes.c_void_p(clk.data_ptr()))
                f = mpc.solve_device_warm if arm == "warm" else mpc.solve_device
                f(d_rlog[t], B, d_w[arm][t], d_s[arm][t])
                if t == mid:
                    interface.lib().hmpc_debug_set_clock_buffer(None)
            torch.cuda.synchronize()
            c = clk.cpu().numpy()
            nb = (d_rlog[mid].cpu().numpy()[:, (54 + 12 * N) * 4:(54 + 12 * N) * 4 + 2 * N] != 0).sum(1)
            sel = (nb <= N) & (interface.status_code(d_s[arm][mid].cpu().numpy()) == 0)
            res["stage_cycles_median_class0"][arm] = {k: float(np.median(c[sel, j] - c[sel, i])) for k, (i, j) in names.items()}
    mpc.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "warm_ab.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
