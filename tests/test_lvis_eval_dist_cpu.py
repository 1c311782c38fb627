"""CPU, world_size 2, gloo: ``parallel.all_gather_rows``, the collective the LVIS evaluator gathers its per-rank pools with (a
different row count per rank, rank order, the per-rank heads)."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from util import ROOT


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    from mqdet_b200 import parallel
    dist.init_process_group("gloo", rank=rank, world_size=world)
    n = [5, 0][rank] if port % 2 else [3, 7][rank]
    rows = torch.arange(n * 9, dtype=torch.int32).view(n, 9) + 1000 * rank
    head = torch.tensor([n, 100 + rank, rank], dtype=torch.int64)
    parts, heads = parallel.all_gather_rows(rows, head)
    want_n = [5, 0] if port % 2 else [3, 7]
    ok = [int(h[0]) for h in heads] == want_n and [int(h[1]) for h in heads] == [100, 101]
    for r, p in enumerate(parts):
        ok = ok and torch.equal(p, torch.arange(want_n[r] * 9, dtype=torch.int32).view(want_n[r], 9) + 1000 * r)
    ret[rank] = bool(ok)
    dist.barrier()
    dist.destroy_process_group()


def test_all_gather_rows_world2():
    mgr = mp.Manager()
    for off in (0, 1):   # odd port: one rank holds no rows
        ret = mgr.dict()
        port = 31000 + 2 * (os.getpid() % 1000) + off
        mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
        assert dict(ret) == {0: True, 1: True}


def test_all_gather_rows_single_process_is_identity():
    from mqdet_b200 import parallel
    rows, head = torch.ones(4, 9, dtype=torch.int32), torch.tensor([4, 4, 0])
    parts, heads = parallel.all_gather_rows(rows, head)
    assert len(parts) == 1 and parts[0] is rows and heads[0] is head
