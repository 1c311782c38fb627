"""GPU: the vision-query bank extraction over a dataset.  The ground-truth ROI, capped-append and merge kernels bit for bit against
the restatement (tests/query_extract_oracle.py, pinned to the reference by tests/test_query_extract_cpu.py), and
``engine.query_extract.extract_query_bank`` on synthetic MQ-GLIP-T and MQ-GroundingDINO-T against a host loop of the model's own
``extract_query`` over the same mixed-size batches: bit for bit, reruns identical, a warm call reads nothing on the host before its
final copy, the saved file detects as the in-memory bank does, and two ranks over gloo give the one-rank bank."""
import functools
import os
import sys
from collections import defaultdict

import pytest
import torch
import torch.multiprocessing as mp

import query_extract_oracle as qo
from util import ROOT

pytestmark = pytest.mark.gpu


def _gts(g, sizes, max_boxes=9, labels=12):
    """Per image (boxes [n, 4], labels [n], (w, h)): random boxes, some on the image borders, some whose expansion leaves the image
    entirely (clipped to empty), every fifth image without boxes."""
    out = []
    for i, (h, w) in enumerate(sizes):
        n = 0 if i % 5 == 4 else int(torch.randint(1, max_boxes + 1, (1,), generator=g))
        x1 = torch.rand(n, generator=g) * w * 0.9
        y1 = torch.rand(n, generator=g) * h * 0.9
        b = torch.stack([x1, y1, x1 + 2 + torch.rand(n, generator=g) * w * 0.4, y1 + 2 + torch.rand(n, generator=g) * h * 0.4], 1)
        if n >= 3:
            b[0] = torch.tensor([0.0, 0.0, float(w), float(h)])                        # the whole image, both borders
            b[1] = torch.tensor([float(w) + 4, 1.0, float(w) + 20, 9.0])               # outside: clipped to empty
            b[2, 2] = float(w - 1)                                                       # on the right border
        out.append((b, torch.randint(1, labels + 1, (n,), generator=g), (w, h)))
    return out


def test_gt_rois_vs_restatement(dev):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(11)
    sizes = [(480, 640), (427, 640), (640, 480), (375, 500), (333, 500), (612, 612), (640, 427), (500, 375)]
    gts = _gts(g, sizes, max_boxes=40)
    gts.append((torch.tensor([[3.0, 5.0, 3.0, 9.0], [10.0, 10.0, 10.5, 10.25]]), torch.tensor([2, 3]), (64, 48)))   # zero width
    sizes.append((48, 64))
    rwh = [(1066, 800) if w > h else (800, 1066) for h, w in sizes]
    rwh[3], rwh[-1] = (1000, 750), (1066, 800)
    idx = list(range(len(sizes)))
    first = {i: 1000 + 17 * i for i in idx}
    rois, labels, arrival, count = ops.query_gt_rois([(gts[i][0], gts[i][1], gts[i][2], rwh[i], first[i]) for i in idx], 1.5, dev)
    want_r, want_l, want_a = qo.batch_rois(gts, idx, rwh, 1.5, first)
    n = int(count)
    assert n == want_r.shape[0] and n < sum(b.shape[0] for b, _, _ in gts)
    assert torch.equal(rois[:n].cpu(), want_r)
    assert torch.equal(labels[:n].cpu().long(), want_l) and torch.equal(arrival[:n].cpu().long(), want_a)
    assert (want_r[:, 3] == torch.tensor([float(w - 1) for w, _ in rwh])[want_r[:, 0].long()]).any()   # a box clipped at a border


def test_gt_rois_no_boxes(dev):
    from mqdet_b200 import ops
    z = (torch.zeros(0, 4), torch.zeros(0, dtype=torch.long), (64, 48), (800, 600), 0)
    rois, labels, arrival, count = ops.query_gt_rois([z, z], 1.5, dev)
    assert int(count) == 0 and rois.shape == (0, 5)


def _pure_cap(feats_list, labels_list, counts, max_query):
    bank = defaultdict(list)
    for f, l, n in zip(feats_list, labels_list, counts):
        qo.cap_append(bank, l[:n], f[:n], max_query)
    return bank


@pytest.mark.parametrize("max_query", [5, 5000])
def test_append_and_infinite_similarity_are_a_pure_cap(dev, max_query):
    """``query_bank_append`` and ``query_bank_update`` with sim_thr = +inf (s > +inf is false for every s, NaN included) both give
    the pure per-label cap, also for calls with zero rows; the arrival numbers sit beside their rows."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(max_query)
    C, L = 256, 9
    feats_list, labels_list, counts = [], [], []
    for step in range(12):
        R = 64
        n = 0 if step in (3, 7) else R - 3 * step
        f = torch.randn(R, C, generator=g)
        f[5] = f[4]                                                     # exact duplicates: cosine 1
        feats_list.append(f)
        labels_list.append(torch.randint(0, L, (R,), generator=g))
        counts.append(n)
    want = _pure_cap(feats_list, labels_list, counts, max_query)
    cap = max_query
    a, u = ops.QueryBank(L, cap, C, dev), ops.QueryBank(L, cap, C, dev)
    arr = torch.zeros((L, cap), dtype=torch.int32, device=dev)
    base = 0
    for f, l, n in zip(feats_list, labels_list, counts):
        fd, ld = f.to(dev), l.to(torch.int32).to(dev)
        cnt = torch.tensor([n], dtype=torch.int32, device=dev)
        ad = torch.arange(base, base + f.shape[0], dtype=torch.int32, device=dev)
        ops.query_bank_append(a, fd, ld, ad, cnt, max_query, arr)
        ops.query_bank_update(u, fd, ld, cnt, max_query, float("inf"))
        base += f.shape[0]
    for qb in (a, u):
        got = qb.as_dict(qb.count.cpu())
        assert qo.same_bank(got, want)
    if max_query == 5:
        assert max(len(v) for v in want.values()) == 5
    # the arrival of row j of label k: the global index of the j-th kept feature of label k
    seen, base = defaultdict(list), 0
    for f, l, n in zip(feats_list, labels_list, counts):
        for i in range(n):
            if len(seen[int(l[i])]) < max_query:
                seen[int(l[i])].append(base + i)
        base += f.shape[0]
    arr_h, cnt_h = arr.cpu(), a.count.cpu()
    for k in range(L):
        assert arr_h[k, :int(cnt_h[k])].tolist() == seen[k]
    assert torch.equal(a.norm, u.norm)


@pytest.mark.parametrize("G", [2, 3])
def test_merge_vs_restatement(dev, G):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(40 + G)
    C, L, K = 64, 7, 6
    # rows of the one-GPU sequence: arrival a -> (label, rank); each rank keeps its first K per label
    N = 200
    lab = torch.randint(0, L, (N,), generator=g)
    rank = torch.randint(0, G, (N,), generator=g)
    feats = torch.randn(N, C, generator=g)
    parts, counts, banks = [], torch.zeros((G, L), dtype=torch.int64), []
    for r in range(G):
        bank, arr = defaultdict(list), defaultdict(list)
        sel = torch.nonzero(rank == r).flatten()
        qo.cap_append(bank, lab[sel], feats[sel], K, sel, arr)
        banks.append((bank, arr))
        rows = []
        for k in range(L):
            for j, a in enumerate(arr[k]):
                rows.append(torch.cat([torch.tensor([k, a], dtype=torch.int32).view(torch.float32), bank[k][j, 0]]))
            counts[r, k] = len(arr[k])
        parts.append(torch.stack(rows).to(dev) if rows else torch.zeros(0, 2 + C, device=dev))
    out, cnt = ops.query_bank_merge(parts, counts, K, C)
    want = qo.merge(banks, K)
    got = {k: out[k, :int(cnt[k]), None].cpu() for k in range(L) if cnt[k] > 0}
    assert qo.same_bank(got, want)
    # the merge equals the one-rank cap
    assert qo.same_bank(got, qo.cap_append(defaultdict(list), lab, feats, K))


# ---------------------------------------------------------------------------------------------------------------------
# end to end: synthetic MQ-GLIP-T and MQ-GroundingDINO-T
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [(150, 203), (203, 150), (128, 160), (160, 128), (150, 203), (96, 160), (203, 150), (150, 203), (128, 160), (140, 140),
         (150, 203), (96, 160), (203, 150), (128, 160), (150, 203), (160, 128), (150, 203), (96, 160), (140, 140), (128, 160)]


@functools.lru_cache(maxsize=2)
def _model(kind):
    from oracle import synth
    dev = torch.device("cuda:0")
    if kind == "glip":
        from test_gcp_many_queries_gpu import _glip
        model = _glip(synth.detector_sd(synth.Gen(2024), bias0=-1.5), dev, 5)
    else:
        from test_gdino_asm_gpu import _build_model, _gdino_case
        sd = _gdino_case(3033, 1, 160, 224, 13, 2, 2, 100)[0]
        model = _build_model(sd, 2, 2, 100, dev)
    cfg = model.cfg
    cfg.INPUT.MIN_SIZE_TEST, cfg.INPUT.MAX_SIZE_TEST = 160, 256
    cfg.TEST.IMS_PER_BATCH = 4
    return model


def _data(seed=5):
    g = torch.Generator().manual_seed(seed)
    imgs = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy() for h, w in SIZES]
    return imgs, _gts(g, SIZES, max_boxes=8, labels=6)


def _targets(gts):
    from mqdet_b200.structures.bounding_box import BoxList
    out = []
    for b, l, wh in gts:
        t = BoxList(b.clone(), wh, mode="xyxy")
        t.add_field("labels", l.clone())
        out.append(t)
    return out


def _host_loop(model, imgs, targets, batches, max_query):
    """tools/train_net.py's loop: per batch the test transform, the loader's BoxList.resize, model.extract_query."""
    from mqdet_b200.engine.transforms import TestTransform
    bank = defaultdict(list)
    tt = TestTransform(model.cfg)
    for idx in batches:
        il, _ = tt([imgs[i] for i in idx], torch.device("cuda:0"), mixed_sizes=True)
        tg = [targets[i].resize((w, h)) for i, (h, w) in zip(idx, il.image_sizes)]
        bank = model.extract_query(il, tg, bank, max_query_number=max_query)
    return bank


@pytest.mark.parametrize("kind", ["glip", "gdino"])
@pytest.mark.parametrize("max_query", [5, 5000])
def test_engine_equals_host_extract_query(dev, kind, max_query):
    from mqdet_b200.engine.batches import reference_test_batches
    from mqdet_b200.engine.query_extract import extract_query_bank
    model = _model(kind)
    model.cfg.VISION_QUERY.MAX_QUERY_NUMBER = max_query
    imgs, gts = _data()
    targets = _targets(gts)
    batches = reference_test_batches([im.shape[:2] for im in imgs], 4, True)
    assert batches != [list(range(i, min(i + 4, len(imgs)))) for i in range(0, len(imgs), 4)]     # aspect grouping reorders
    want = _host_loop(model, imgs, targets, batches, max_query)
    got = extract_query_bank(model, imgs, targets, model.cfg)
    assert qo.same_bank(got, want)
    rows = sum(len(v) for v in want.values())
    if max_query == 5:
        assert max(len(v) for v in want.values()) == 5 and rows < sum(len(b) for b, _, _ in gts)
    else:
        assert rows > 60
    again = extract_query_bank(model, imgs, targets, model.cfg)
    assert qo.same_bank(again, got)                                    # reruns are bit-identical
    # the explicit batch list of the reference's loader without aspect grouping
    flat = reference_test_batches([im.shape[:2] for im in imgs], 4, False)
    assert qo.same_bank(extract_query_bank(model, imgs, targets, model.cfg, batches=flat),
                        _host_loop(model, imgs, targets, flat, max_query))


def test_warm_call_reads_nothing_on_the_host_before_the_copy(dev):
    """Under sync debug mode 'error' up to the one device->host copy (the row counts), which lifts the mode as it starts."""
    from mqdet_b200.engine.query_extract import extract_query_bank
    model = _model("glip")
    model.cfg.VISION_QUERY.MAX_QUERY_NUMBER = 5
    imgs, gts = _data(9)
    targets = _targets(gts)
    dev_imgs = [torch.from_numpy(im).to(dev) for im in imgs]
    want = extract_query_bank(model, dev_imgs, targets, model.cfg)
    torch.cuda.synchronize()
    orig_cpu, copies = torch.Tensor.cpu, []

    def cpu(self, *a, **k):
        if self.is_cuda:
            copies.append(tuple(self.shape))
            torch.cuda.set_sync_debug_mode(0)
        return orig_cpu(self, *a, **k)

    torch.Tensor.cpu = cpu
    torch.cuda.set_sync_debug_mode("error")
    try:
        bank = extract_query_bank(model, dev_imgs, targets, model.cfg)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        torch.Tensor.cpu = orig_cpu
    L = max(int(l.max()) for _, l, _ in gts if len(l)) + 1
    assert copies == [(L,)]
    assert qo.same_bank(bank, want)


@pytest.mark.parametrize("kind", ["glip", "gdino"])
def test_saved_bank_detects_as_the_memory_bank(dev, kind, tmp_path):
    from mqdet_b200.engine.query_extract import extract_query_bank
    from mqdet_b200.structures.image_list import to_image_list
    from oracle import synth
    model = _model(kind)
    model.cfg.VISION_QUERY.MAX_QUERY_NUMBER = 5
    imgs, gts = _data(3)
    bank = extract_query_bank(model, imgs, _targets(gts), model.cfg)
    path = str(tmp_path / "bank.pth")
    model.save_query_bank(bank, path)
    on_disk = torch.load(path, weights_only=True)
    assert qo.same_bank(on_disk, bank) and all(v.device.type == "cpu" for v in on_disk.values())
    ids, am, pmap = synth.prompt(6, 2, 256, synth.Gen(1))
    assert sorted(k for k, v in bank.items() if len(v)) == sorted(pmap)
    caps = {"input_ids": ids, "attention_mask": am}
    il = to_image_list([torch.from_numpy(imgs[0]).permute(2, 0, 1).float().to(dev)], 32)
    outs = []
    for load in (lambda: model.set_query_bank(bank), lambda: model.load_query_bank(path)):
        load()
        outs.append(model.forward_device(il, caps, pmap)["det_packed"].cpu())
    assert torch.equal(outs[0], outs[1])


def _worker(rank, world, port, kind, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    from mqdet_b200.engine.query_extract import extract_query_bank
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    model = _model(kind)
    for K in (5, 5000):
        model.cfg.VISION_QUERY.MAX_QUERY_NUMBER = K
        imgs, gts = _data()
        bank = extract_query_bank(model, imgs, _targets(gts), model.cfg)
        ret[(rank, K)] = {int(k): v.cpu() for k, v in bank.items()}
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_over_gloo_give_the_one_rank_bank(dev):
    from mqdet_b200.engine.query_extract import extract_query_bank
    model = _model("glip")
    want = {}
    for K in (5, 5000):
        model.cfg.VISION_QUERY.MAX_QUERY_NUMBER = K
        imgs, gts = _data()
        want[K] = extract_query_bank(model, imgs, _targets(gts), model.cfg)
    ret = mp.Manager().dict()
    port = 34000 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, "glip", ret), nprocs=2, join=True)
    for K in (5, 5000):
        for r in range(2):
            assert qo.same_bank(ret[(r, K)], want[K]), (r, K)
