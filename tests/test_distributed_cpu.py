"""Host-side logic of the data-parallel path, world_size 2 over gloo on CPU (no GPU, no kernels):
replica broadcast and the averaged gradient exchange used by scsfm.trainer / bench.py."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import free_port


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from scsfm.exchange import GradExchange
    torch.manual_seed(100 + rank)
    params = [torch.randn(1000), torch.randn(37)]        # two "arenas" (disp, pose), different per rank
    grads = [torch.randn(1000), torch.randn(37)]
    ex = GradExchange(world)
    ex.broadcast_params(params)
    local = [g.clone() for g in grads]
    for g in grads:
        ex.allreduce_async(g)
    ex.wait()
    gathered = [[torch.zeros_like(g) for _ in range(world)] for g in local]
    for lst, g in zip(gathered, local):
        dist.all_gather(lst, g)
    ok = all(torch.allclose(g, sum(lst) / world, atol=1e-6) for g, lst in zip(grads, gathered))
    ref = [p.clone() for p in params]
    for p in ref:
        dist.broadcast(p, 0)
    ok = ok and all(torch.equal(p, r) for p, r in zip(params, ref))
    # sharding helper: contiguous, equal shards of the global batch
    from scsfm.exchange import shard_batch
    full = torch.arange(8 * 3).view(8, 3)
    mine = shard_batch(full, rank, world)
    ok = ok and mine.shape[0] == 4 and int(mine[0, 0]) == rank * 12
    out[rank] = bool(ok)
    dist.destroy_process_group()


def test_gradient_exchange_world2_gloo():
    world = 2
    with mp.Manager() as m:
        out = m.dict()
        mp.spawn(_worker, args=(world, free_port(), out), nprocs=world, join=True)
        assert dict(out) == {0: True, 1: True}
