"""world_size-2 gloo test (CPU) of the data-parallel host logic: the sharded gradient exchange (slice bounds, reduce-scatter, all-gather)."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _worker_sharded(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from xrnerf_b200.train import ShardedExchange, shard_range
    n = 1003                                                       # not a multiple of world * 8: the last slice is short
    ex = ShardedExchange(n)
    ok = ex.world == world and ex.per % 8 == 0 and ex.padded == ex.per * world and ex.padded >= n
    ok = ok and (ex.begin, ex.end) == (min(rank * ex.per, n), min((rank + 1) * ex.per, n))
    # gradient exchange: every rank contributes rank+1 times a ramp; the owner of a slice receives the sum of that slice
    g = torch.zeros(ex.padded); g[:n] = torch.arange(n, dtype=torch.float32) * (rank + 1)
    mine = torch.zeros(ex.per)
    ex.reduce_scatter_sum(g, mine)
    want = torch.zeros(ex.padded); want[:n] = torch.arange(n, dtype=torch.float32) * sum(range(1, world + 1))
    ok = ok and torch.equal(mine, want[rank * ex.per:(rank + 1) * ex.per])
    # parameter exchange: each rank updates its slice; the all-gather rebuilds the whole (padded) vector on every rank
    full = torch.zeros(ex.padded)
    ex.all_gather(full, mine * 0.5)
    ok = ok and torch.equal(full, want * 0.5)
    # the slices tile [0, n) exactly
    cover = torch.zeros(n)
    for r in range(world):
        b, e, _, _ = shard_range(n, world, r)
        cover[b:e] += 1
    ok = ok and bool((cover == 1).all())
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_sharded_gradient_exchange_gloo_world2():
    """host logic of the sharded data-parallel step (xrnerf_b200/train.py: reduce-scatter of the gradient -> Adam on the rank's slice -> all-gather of the updated copy)
    on the gloo backend (no reduce_scatter there: the all_reduce + slice fallback gives the same result)"""
    import socket
    s = socket.socket(); s.bind(('127.0.0.1', 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    ps = [ctx.Process(target=_worker_sharded, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = [q.get(timeout=120) for _ in ps]
    for p in ps:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]
