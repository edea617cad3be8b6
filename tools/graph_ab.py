"""Eager calls against CUDA-graph replays of the same ticks (DESIGN.md §6).

The ticks are tools/warm_ab.py's: walkers of make_batch(5, seed=2024) at horizon 10 in a device closed loop.  The loop
runs one tick per hmpc_rollout_device call, and the robot states in front of every tick are logged.  A batch of B robots
replays the first B robots' logged states (robots are independent, so B = 1024 is warm_ab.py's workload).  One tick is
what a caller's MPC step does: hmpc_prepare_device on the tick's states, then hmpc_solve_device_warm (shift NULL).
Two arms, each on its own context, alternating passes after a warm-up pass of each:

  eager  the two calls through interface.BatchedMPC, every tick;
  graph  the same two calls captured once with torch.cuda.graph, CUDAGraph.replay() every tick.

Both arms read a tick's states from a static device buffer, written by a device copy in front of the tick and outside
the timed span, and start every pass from hmpc_reset_warm_start.  Per tick: the CUDA-event time of the tick's work on the
stream, and the host wall time to enqueue it (the Python calls with their ctypes marshalling, or CUDAGraph.replay).
An untimed pass of each arm logs the first-step wrenches and status words of every tick; the two arms must agree bit
for bit.

The JSON line also lists the nodes and edges of one captured prepare + warm solve, read through the driver API, to show
whether stream capture turned the chain's programmatic dependent launches into programmatic edges.  It carries the GPU's
name, power limit and max SM clock, read in the same run.

    python tools/graph_ab.py [--batches 1,64,1024,4096] [--ticks 200] [--passes 5] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

from hector_simulation_b200 import interface, scenarios  # noqa: E402
from warm_ab import gpu_card  # noqa: E402

N = 10
NODE_TYPES = {0: "kernel", 1: "memcpy", 2: "memset", 3: "host", 4: "graph", 5: "empty"}
EDGE_TYPES = {0: "default", 1: "programmatic"}


def graph_edges(g):
    """nodes and edges of a captured graph (CUDAGraph(keep_graph=True)), through the driver API"""
    cu = ctypes.CDLL("libcuda.so.1")
    graph = ctypes.c_void_p(g.raw_cuda_graph())
    n = ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(graph, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(graph, nodes, ctypes.byref(n)) == 0

    def label(node):
        t = ctypes.c_int(-1)
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(t)) == 0
        name = NODE_TYPES.get(t.value, str(t.value))
        if t.value == 0:  # CUDA_KERNEL_NODE_PARAMS_v2: func, gridDim[3], blockDim[3], ...
            buf = (ctypes.c_uint32 * 64)()
            if cu.cuGraphKernelNodeGetParams_v2(ctypes.c_void_p(node), buf) == 0:
                name += " grid %d x %d threads" % (buf[2], buf[5])
        return name

    labels = {nd: label(nd) for nd in nodes}
    m = ctypes.c_size_t(0)
    if cu.cuGraphGetEdges_v2(graph, None, None, None, ctypes.byref(m)) != 0:
        return dict(nodes=list(labels.values()), edges="cuGraphGetEdges_v2 unavailable")
    src, dst = (ctypes.c_void_p * m.value)(), (ctypes.c_void_p * m.value)()
    data = (ctypes.c_uint8 * (8 * m.value))()   # CUgraphEdgeData: from_port, to_port, type, reserved[5]
    assert cu.cuGraphGetEdges_v2(graph, src, dst, data, ctypes.byref(m)) == 0
    edges = [dict(src=labels[src[i]], dst=labels[dst[i]], type=EDGE_TYPES.get(data[8 * i + 2], str(data[8 * i + 2])),
                  from_port=int(data[8 * i])) for i in range(m.value)]
    return dict(nodes=[labels[nd] for nd in nodes], edges=edges)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,64,1024,4096")
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--passes", type=int, default=5, help="timed passes per arm, alternating")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("graph_ab: no CUDA device")
    batches = [int(x) for x in a.batches.split(",")]
    BMAX, T = max(batches), a.ticks
    dev = torch.device("cuda", 0)
    stride = interface.record_bytes(N)

    # the ticks: one closed loop on the device, the states in front of every tick logged
    states, loop = scenarios.make_rollout(scenarios.make_batch(5, BMAX, horizon=N, seed=2024)[1], N)
    ctx = interface.BatchedMPC(BMAX, N)
    d_states = torch.from_numpy(states.view(np.uint8).reshape(BMAX, -1).copy()).to(dev)
    d_loop = torch.from_numpy(loop.view(np.uint8).reshape(BMAX, -1).copy()).to(dev)
    slog = torch.zeros((T, BMAX, d_states.shape[1]), dtype=torch.uint8, device=dev)
    for t in range(T):
        slog[t].copy_(d_states)
        ctx.rollout_device(d_states, d_loop, BMAX, 1)
    torch.cuda.synchronize()
    ctx.close()

    res = dict(workload="prepare + warm solve per tick, walkers at N=%d, %d logged ticks x %d timed passes per arm" % (N, T, a.passes),
               card=gpu_card(0), batches={})

    for B in batches:
        arms = {}
        for arm in ("eager", "graph"):
            mpc = interface.BatchedMPC(B, N)
            buf = dict(states=torch.zeros((B, slog.shape[2]), dtype=torch.uint8, device=dev),
                       rec=torch.zeros((B, stride), dtype=torch.uint8, device=dev),
                       w=torch.zeros((B, 12 * N), dtype=torch.float32, device=dev),
                       s=torch.zeros(B, dtype=torch.int32, device=dev))
            arms[arm] = dict(mpc=mpc, buf=buf)

        def tick_calls(arm):
            m, b = arms[arm]["mpc"], arms[arm]["buf"]
            m.prepare_device(b["states"], B, b["rec"])
            m.solve_device_warm(b["rec"], B, b["w"], b["s"])

        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(T)]

        def run_pass(arm, timed, log=None):
            b = arms[arm]["buf"]
            arms[arm]["mpc"].reset_warm_start()
            host = []
            for t in range(T):
                b["states"].copy_(slog[t, :B])
                if timed:
                    ev[t][0].record()
                t0 = time.perf_counter()
                if arm == "graph":
                    arms[arm]["g"].replay()
                else:
                    tick_calls(arm)
                host.append((time.perf_counter() - t0) * 1e6)
                if timed:
                    ev[t][1].record()
                if log is not None:
                    log[0][t].copy_(b["w"][:, :12])
                    log[1][t].copy_(b["s"])
            torch.cuda.synchronize()
            return ([ev[t][0].elapsed_time(ev[t][1]) * 1e3 for t in range(T)], host) if timed else None

        run_pass("eager", False)            # loads every kernel before the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            tick_calls("graph")
        arms["graph"]["g"] = g
        run_pass("graph", False)
        dev_us = {"eager": [], "graph": []}
        host_us = {"eager": [], "graph": []}
        for _ in range(a.passes):
            for arm in ("eager", "graph"):
                d, h = run_pass(arm, True)
                dev_us[arm] += d
                host_us[arm] += h
        logs = {}
        for arm in ("eager", "graph"):
            logs[arm] = (torch.zeros((T, B, 12), dtype=torch.float32, device=dev), torch.zeros((T, B), dtype=torch.int32, device=dev))
            run_pass(arm, False, logs[arm])
        same = bool(torch.equal(logs["eager"][0].view(torch.int32), logs["graph"][0].view(torch.int32)) and
                    torch.equal(logs["eager"][1], logs["graph"][1]))
        out = dict(identical_outputs=same)
        for arm in ("eager", "graph"):
            d, h = np.array(dev_us[arm]), np.array(host_us[arm])
            out[arm] = dict(tick_p50_us=round(float(np.percentile(d, 50)), 1), tick_p99_us=round(float(np.percentile(d, 99)), 1),
                            qp_per_s=round(B * len(d) / (d.sum() * 1e-6)),
                            enqueue_p50_us=round(float(np.percentile(h, 50)), 1), enqueue_p99_us=round(float(np.percentile(h, 99)), 1))
        out["graph_speedup"] = round(out["graph"]["qp_per_s"] / out["eager"]["qp_per_s"], 3)
        if B == max(batches):
            # the shape of one captured tick (a separate capture that is never launched)
            pg = torch.cuda.CUDAGraph(keep_graph=True)
            with torch.cuda.graph(pg):
                tick_calls("graph")
            res["captured_tick"] = graph_edges(pg)
            del pg
        res["batches"][str(B)] = out
        del g
        for arm in arms.values():
            arm["mpc"].close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "graph_ab.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
