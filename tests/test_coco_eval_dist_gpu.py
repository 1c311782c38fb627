"""GPU, world_size 2, gloo (both ranks on cuda:0): the COCO evaluator's ``synchronize_between_processes``.  Rank r scores its
own updates; after the gather (each rank's pool cut to its top 100 per (image, category) first) the result equals ONE evaluator
fed rank 0's updates and then rank 1's, with score ties across ranks going to the lower rank.  A detection on an image outside
the GT file seen by rank 1 only still raises on rank 0 (its count travels with the gather)."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

import coco_eval_oracle as co
from util import ROOT

pytestmark = pytest.mark.gpu


def _packed(upd, gt):
    from test_coco_eval_gpu import _packed as p
    import torch
    return p(upd, torch.device("cuda:0"), gt)


def _worker(rank, world, port, name, foreign, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.engine.coco_eval import CocoEvaluator, CocoGroundTruth
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    gt, updates = co.pin_cases()[name]
    half = (len(updates) + 1) // 2
    mine = updates[:half] if rank == 0 else updates[half:]
    ev = CocoEvaluator(CocoGroundTruth(gt, "cuda:0"), pool_rows=1 << 16)
    for u in mine:
        ev.update_packed(*_packed(u, gt))
    if foreign and rank == 1:
        pk, ids, s, o = _packed(mine[0][:1], gt)
        ev.update_packed(pk, [424242], s, o)
    ev.synchronize_between_processes()
    if rank == 0:
        try:
            ev.accumulate()
        except MqdetError as e:
            ret["error"] = str(e)
        else:
            stats = ev.summarize()
            ret["precision"], ret["recall"] = ev.eval["precision"].tobytes(), ev.eval["recall"].tobytes()
            ret["stats"] = [float(v) for v in stats]
    else:
        ret["rank1_summary"] = ev.summarize() if not foreign else None
    dist.barrier()
    dist.destroy_process_group()


def _spawn(name, foreign):
    ret = mp.Manager().dict()
    port = 32000 + (os.getpid() % 2000) + (7 if foreign else 0)
    mp.spawn(_worker, args=(2, port, name, foreign, ret), nprocs=2, join=True)
    return ret


@pytest.mark.parametrize("name", ["dense", "crowd_id0"])
def test_two_ranks_equal_one_rank_in_rank_order(name, dev):
    from mqdet_b200.engine.coco_eval import CocoEvaluator, CocoGroundTruth
    gt, updates = co.pin_cases()[name]
    one = CocoEvaluator(CocoGroundTruth(gt, dev), pool_rows=1 << 16)
    for u in updates:
        one.update_packed(*_packed(u, gt))
    stats = one.summarize()
    ret = _spawn(name, False)
    assert ret["precision"] == one.eval["precision"].tobytes()
    assert ret["recall"] == one.eval["recall"].tobytes()
    assert ret["stats"] == [float(v) for v in stats] and ret["rank1_summary"] is None
    o, _ = co.run_oracle(gt, updates)
    assert np.array_equal(one.eval["precision"], o.eval["precision"])


def test_foreign_image_on_one_rank_raises_after_the_gather(dev):
    ret = _spawn("basic", True)
    assert "do not correspond" in ret["error"]
