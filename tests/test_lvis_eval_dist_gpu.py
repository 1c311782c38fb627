"""GPU, world_size 2, gloo (both ranks on cuda:0): the LVIS evaluator's ``synchronize_between_processes``.  Rank r scores its
own updates; after the gather the result equals ONE evaluator fed rank 0's updates and then rank 1's (the reference's
rank-order concatenation, lvis_eval.py:800-806), with score ties across ranks going to the lower rank."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

import lvis_eval_oracle as lo
from util import ROOT

pytestmark = pytest.mark.gpu


def _packed(upd):
    from test_lvis_eval_gpu import _packed as p
    import torch
    return p(upd, torch.device("cuda:0"))


def _worker(rank, world, port, name, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    gt, updates, topk, fixed_ap = lo.pin_cases()[name]
    half = (len(updates) + 1) // 2
    mine = updates[:half] if rank == 0 else updates[half:]
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, "cuda:0"), topk=topk, fixed_ap=fixed_ap, pool_rows=1 << 16)
    for u in mine:
        ev.update_packed(*_packed(u))
    ev.synchronize_between_processes()
    lines = ev.summarize()
    if rank == 0:
        ret["precision"], ret["recall"] = ev.eval["precision"].tobytes(), ev.eval["recall"].tobytes()
        ret["results"] = [float(v) for v in ev.results.values()]
        ret["lines"] = lines
    else:
        ret["rank1_summary"] = lines
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("name", ["fixed_cut", "standard"])
def test_two_ranks_equal_one_rank_in_rank_order(name, dev):
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    gt, updates, topk, fixed_ap = lo.pin_cases()[name]
    one = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev), topk=topk, fixed_ap=fixed_ap, pool_rows=1 << 16)
    for u in updates:
        one.update_packed(*_packed(u))
    lines = one.summarize()
    ret = mp.Manager().dict()
    port = 32000 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, name, ret), nprocs=2, join=True)
    assert ret["precision"] == one.eval["precision"].tobytes()
    assert ret["recall"] == one.eval["recall"].tobytes()
    assert ret["results"] == [float(v) for v in one.results.values()]
    assert ret["lines"] == lines and ret["rank1_summary"] is None
    o = lo.run_oracle(gt, updates, topk, fixed_ap)
    assert np.array_equal(one.eval["precision"], o.precision)
