"""The worker-id-sharded pick through both exchanges — a gloo all-gather between two host-synchronised calls and the peer-memory
exchange (CUDA IPC mappings, stores + flags, no collective) — on indexes where the shards' searches depart from the whole fleet's.

The sharded pick is the reference search run on each shard's index alone, merged in rank order (tests/sharded_oracle.py).  On the
synth indexes of tests/test_gpu_sharded.py that is also the whole-fleet pick; on the crafted indexes of sharded_oracle.departure_case
it is not (DESIGN.md §4d).  Here both exchanges must give the per-shard pick on every rank, and it must differ from the whole fleet's.
The two ranks share cuda:0 when the box has one GPU."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _departure_worker(rank, world, port, kind, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from smg_b200 import CacheAwareConfig
    from smg_b200.sharding import ShardedEventRouter
    from tests.sharded_oracle import departure_case, seq_blocks
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ndev = torch.cuda.device_count()
    bs = 16
    case = departure_case(kind, bs)
    urls = [f"http://{nm}:8000" for nm in case["names"]]
    cfg = CacheAwareConfig(eviction_interval_secs=0, cache_threshold=0.3, balance_abs_threshold=64, balance_rel_threshold=1.5, block_size=bs)
    router = ShardedEventRouter(urls, rank, world, cfg, jump_size=8, device_id=rank % max(ndev, 1), max_tokens_per_request=16 * bs)
    for k, (g, hs) in enumerate(sorted(case["stores"].items())):
        if router.owns(g):
            router.indexer.apply_stored(router.local_id(g), seq_blocks(hs, 1 + 100 * k))
    router.set_fleet_state(case["loads"], np.ones(len(urls), np.uint8))

    def all_gather(arr):
        t = torch.from_numpy(arr.copy())
        outs = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(outs, t)
        return np.concatenate([o.numpy() for o in outs])
    router.connect_peers(all_gather)
    reqs = [case["tokens"]] * 4 + [np.zeros(0, np.uint32)]
    flat = np.concatenate(reqs).astype(np.uint32)
    offs = np.zeros(len(reqs) + 1, np.uint32)
    np.cumsum([len(r) for r in reqs], out=offs[1:])
    got = router.select(flat, offs, 16 * bs, all_gather)
    fused = router.select_fused(flat, offs, 16 * bs)
    ret[rank] = (got.tolist(), fused.tolist(), case["sharded"], case["whole"])
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("kind", ["count_test", "retain_guard"])
def test_sharded_pick_departs_from_whole_fleet(kind):
    """Crafted indexes on which the shards' searches disagree with the whole fleet's: the gloo and peer-memory exchanges both give the
    per-shard pick, on every rank."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = 29650 + len(kind)
    procs = [ctx.Process(target=_departure_worker, args=(r, 2, port, kind, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
    assert all(p.exitcode == 0 for p in procs)
    for r in range(2):
        got, fused, sharded, whole = ret[r]
        assert sharded != whole
        assert got == fused and got[:4] == [sharded] * 4, (r, got, fused)
