"""Batch sharding across GPUs (SURVEY.md §8e) — the host-side driver of the library's hmpc_shard_* entry points.

Robots are independent, so a batch that exceeds one device is cut into contiguous, equally sized slices, one process
per GPU; every rank runs the identical kernels on its slice (hmpc_solve_batch_sharded: the slice's results come back to
the rank's own host arrays, in place) and the path's only exchange is ONE all-gather of the float wrenches — issued by the
library (ncclAllGather on a side stream, overlapped with the next tick) when a consumer wants the whole batch on every
device.  `ShardedMPC.tick` is the one function both bench.py (NCCL, GPUs) and tests/test_sharding_gloo.py (gloo, CPU, the
oracle standing in for the local solve) drive; what differs is the `backend` that solves a slice and moves the gather.

With warm=True a tick is hmpc_solve_batch_sharded_warm: warm-started, and with a mask only the due robots are solved; the
gather still delivers every robot's latest wrench (zeros before its first solve).
"""
from __future__ import annotations

import numpy as np


def shard_bounds(batch: int, world: int) -> list[tuple[int, int]]:
    """Contiguous [lo, hi) per rank over slices of ceil(batch / world) robots; the tail ranks may hold fewer (or none)."""
    per = -(-batch // world)
    return [(min(r * per, batch), min((r + 1) * per, batch)) for r in range(world)]


class GpuBackend:
    """The product path: libhector_mpc_b200 on this rank's GPU, NCCL for the gather (inside the library)."""

    def __init__(self, b_local: int, horizon: int, rank: int, world: int, device: int, broadcast_bytes):
        import torch

        from . import interface

        self.torch = torch
        self.mpc = interface.BatchedMPC(b_local, horizon, device=device)
        uid = interface.BatchedMPC.shard_unique_id() if rank == 0 else None
        uid = broadcast_bytes(uid)            # rank 0's 128 bytes to everybody (any torch.distributed backend)
        self.mpc.shard_init(rank, world, uid)
        self.d_all = torch.zeros((world * b_local, 12 * horizon), dtype=torch.float32, device=f"cuda:{device}")
        self.h_all = torch.zeros((world * b_local, 12 * horizon), dtype=torch.float32).pin_memory()

    def register(self, recs, out_w, out_s):
        self.mpc.pin(recs, out_w, out_s)      # the control loop's arrays: solved in place from now on

    def solve(self, recs, out_w, out_s, gather: bool, warm: bool = False, mask=None, shift=None):
        d_all = self.d_all if gather else None
        if warm:
            self.mpc.solve_batch_sharded_warm(recs, (out_w, out_s), d_all, mask=mask, shift=shift)
        else:
            self.mpc.solve_batch_sharded(recs, (out_w, out_s), d_all)

    def wait(self):
        self.mpc.shard_wait()

    def gathered(self) -> np.ndarray:
        self.mpc.shard_wait()
        with self.torch.cuda.device(self.d_all.device):
            self.h_all.copy_(self.d_all)
            self.torch.cuda.synchronize()
        return self.h_all.numpy()

    def close(self):
        self.mpc.close()


class TorchBackend:
    """Any local solver + torch.distributed for the gather (the CPU test: oracle + gloo).  The library's gather semantics:
    solve_local sees the listed records only, and the gather sends every robot's latest row (zeros before its first
    solve).  The solver stands in for a cold one, so `warm` and `shift` change nothing here."""

    def __init__(self, b_local: int, horizon: int, world: int, solve_local, group=None):
        import torch
        import torch.distributed as dist

        self.torch, self.dist, self.group = torch, dist, group
        self.solve_local = solve_local
        self.all = torch.zeros((world * b_local, 12 * horizon), dtype=torch.float32)
        self.latest = np.zeros((b_local, 12 * horizon), dtype=np.float32)

    def register(self, recs, out_w, out_s):
        pass

    def solve(self, recs, out_w, out_s, gather: bool, warm: bool = False, mask=None, shift=None):
        rows = np.arange(len(recs)) if mask is None else np.flatnonzero(mask)
        if len(rows):
            w, s = self.solve_local(recs[rows])
            out_w[rows] = w
            out_s[rows] = s
            self.latest[rows] = out_w[rows]
        if gather:
            self.dist.all_gather_into_tensor(self.all, self.torch.from_numpy(self.latest), group=self.group)

    def wait(self):
        pass

    def gathered(self) -> np.ndarray:
        return self.all.numpy()

    def close(self):
        pass


class ShardedMPC:
    """One tick of a batch of `batch` robots spread over `world` ranks.

    tick(records_local) solves this rank's slice (padded to the common slice size with copies of its last record, so that
    every rank moves the same number of elements in the gather) and returns views of the slice's results;
    whole_batch() assembles the gathered wrenches of the last tick in global robot order.  `record_dtype` is
    scenarios.UPDATE_DTYPE (records) or scenarios.STATE_DTYPE (robot states, warm ticks only).

    warm=True: every tick is warm-started, and tick(mask=..., shift=...) solves only the robots its mask lists; the padded
    tail is never listed, so it is never solved."""

    def __init__(self, batch: int, horizon: int, rank: int, world: int, backend_factory, record_dtype, warm: bool = False):
        self.batch, self.horizon, self.rank, self.world, self.warm = batch, horizon, rank, world, warm
        self.bounds = shard_bounds(batch, world)
        self.lo, self.hi = self.bounds[rank]
        self.b_local = max(h - l for l, h in self.bounds)
        self.backend = backend_factory(self.b_local)
        from .interface import page_aligned   # registered (pinned) arrays own their pages

        self.recs = page_aligned(self.b_local, record_dtype)
        self.out_w = page_aligned((self.b_local, 12 * horizon), np.float64)
        self.out_s = page_aligned(self.b_local, np.int32)
        self.backend.register(self.recs, self.out_w, self.out_s)
        self.mask = np.zeros(self.b_local, np.uint8)
        self.shift = np.zeros(self.b_local, np.int32)

    def local_slice(self, records_global: np.ndarray) -> np.ndarray:
        return records_global[self.lo:self.hi]

    @property
    def records(self) -> np.ndarray:
        """This rank's registered record array (first hi - lo entries are its robots): a control loop fills it in place and
        calls tick() without arguments — no copy, like hmpc_solve_batch on pinned arrays."""
        return self.recs

    def tick(self, records_local: np.ndarray | None = None, gather: bool = True, mask=None, shift=None):
        """mask / shift (warm ticks only): this rank's slices, [hi - lo] each; None lists every robot / moves each one step."""
        n = self.hi - self.lo
        if records_local is not None:
            assert len(records_local) == n
            self.recs[:n] = records_local
        if 0 < n < self.b_local:
            self.recs[n:] = self.recs[n - 1]      # padding: a valid problem, its results are dropped
        elif n == 0:
            self.recs[:] = 0
        if not self.warm:
            assert mask is None and shift is None, "mask and shift need ShardedMPC(warm=True)"
            self.backend.solve(self.recs, self.out_w, self.out_s, gather and self.world > 1)
            return self.out_w[:n], self.out_s[:n]
        m = None
        if mask is not None or n < self.b_local:  # the padded tail is never listed
            self.mask[:n] = 1 if mask is None else (np.asarray(mask) != 0)
            self.mask[n:] = 0
            m = self.mask
        s = None
        if shift is not None:
            self.shift[:n] = shift
            self.shift[n:] = 0
            s = self.shift
        self.backend.solve(self.recs, self.out_w, self.out_s, gather and self.world > 1, True, m, s)
        return self.out_w[:n], self.out_s[:n]

    def whole_batch(self) -> np.ndarray:
        """[batch, 12N] float32 wrenches of the last tick(gather=True), global robot order: each robot's latest result (zeros
        before its first solve)."""
        if self.world == 1:
            return self.out_w[: self.hi - self.lo].astype(np.float32)
        g = self.backend.gathered().reshape(self.world, self.b_local, 12 * self.horizon)
        return np.concatenate([g[r, : h - l] for r, (l, h) in enumerate(self.bounds)], axis=0)

    def close(self):
        self.backend.close()
