"""Developer check of the multi-GPU path's warm masked ticks on a box with >= 2 GPUs:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29534 tests/tools/shard_check_masked.py
every rank ticks its slice through sharding.ShardedMPC(warm=True) (hmpc_solve_batch_sharded_warm, library NCCL gather) with
staggered masks (robot i due at tick t when (i + t) % 5 == 0), and rank 0 checks the gathered batch after every tick against
a single-GPU hmpc_solve_batch_masked of all robots with the same masks."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from hector_simulation_b200 import interface, scenarios, sharding  # noqa: E402


def main():
    world, rank, lr = int(os.environ["WORLD_SIZE"]), int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    N, B = 10, 1000  # not a multiple of the world size: the tail slice is padded, and its padding is never listed

    def bcast(b):
        box = [b]
        dist.broadcast_object_list(box, src=0)
        return box[0]

    recs, _ = scenarios.make_batch(3, B, horizon=N, seed=4321)
    sh = sharding.ShardedMPC(B, N, rank, world, lambda bl: sharding.GpuBackend(bl, N, rank, world, lr, bcast), scenarios.UPDATE_DTYPE,
                             warm=True)
    print(f"rank {rank}: slice {sh.lo}:{sh.hi} of {B}, b_local {sh.b_local}", flush=True)
    mine = sh.local_slice(recs)
    one = interface.BatchedMPC(B, N, device=lr) if rank == 0 else None
    w1, s1 = np.zeros((B, 12 * N)), np.zeros(B, np.int32)
    ok = True
    for t in range(12):
        m = ((np.arange(B) + t) % 5 == 0).astype(np.uint8)
        sh.tick(mine, mask=m[sh.lo:sh.hi])
        whole = sh.whole_batch()
        torch.cuda.synchronize()
        if rank == 0:
            one.solve_batch_masked(recs, m, out=(w1, s1))
            # unlisted rows: each robot's latest result, or zeros before its first solve, in both
            same = np.array_equal(whole, w1.astype(np.float32))
            print(f"rank 0 tick {t}: gathered batch equals the single-GPU masked solve: {same}", flush=True)
            ok &= same
    if rank == 0:
        one.close()
    assert ok
    sh.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
