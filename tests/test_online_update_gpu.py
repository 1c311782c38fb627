"""GPU: the test-time vision-query update.  The candidate and bank-update kernels bit for bit against the restatement
(tests/online_update_oracle.py, pinned to the reference by tests/test_online_update_cpu.py), and ``engine.online_update`` on synthetic
MQ-GLIP-T and MQ-GroundingDINO-T (5-shot starting bank, 3 turns) against a host loop of one-image forwards + ``extract_query
(exclude_similar=True)``: B = 4 batches equal B = 1, reruns are bit-identical, a warm turn reads nothing on the host."""
import functools
from collections import defaultdict

import pytest
import torch

import online_update_oracle as ou

pytestmark = pytest.mark.gpu


def _rows(g, B, M, counts, wh):
    w, h = wh
    pk = torch.zeros(B, M + 1, 6)
    for b, n in enumerate(counts):
        x1 = torch.rand(M, generator=g) * w * 1.1 - 0.05 * w
        y1 = torch.rand(M, generator=g) * h * 1.1 - 0.05 * h
        pk[b, :M, 0], pk[b, :M, 1] = x1, y1
        pk[b, :M, 2] = x1 + torch.rand(M, generator=g) * w * 0.5
        pk[b, :M, 3] = y1 + torch.rand(M, generator=g) * h * 0.5
        pk[b, :M, 4] = torch.rand(M, generator=g)
        pk[b, :M, 5] = torch.randint(1, 9, (M,), generator=g).float()
        pk[b, 3, 4] = 0.6                                              # exactly the threshold: dropped
        pk[b, 4, :4] = torch.tensor([w + 3.0, 2.0, w + 40.0, 9.0])      # outside the image: clipped to empty
        pk[b, 4, 4] = 0.95
        pk[b, M, 0] = float(n)
    return pk


@pytest.mark.parametrize("M,counts", [(100, [100, 0, 37, 100]), (900, [900, 5]), (7, [7])])
def test_candidates_vs_restatement(dev, M, counts):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(M)
    wh = (203, 150)
    pk = _rows(g, len(counts), M, counts, wh)
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    rois, labels, count = ops.query_candidates(pk.to(dev), wh, 0.6, 1.5, bad)
    n = int(count)
    want_b, want_l, want_i = [], [], []
    for b in range(len(counts)):
        boxes, lab = ou.candidates(pk[b], wh, 0.6, 1.5)
        want_b.append(boxes), want_l.append(lab), want_i.append(torch.full((boxes.shape[0],), float(b)))
    assert n == sum(x.shape[0] for x in want_b) and int(bad) == 0
    assert torch.equal(rois[:n, 1:].cpu(), torch.cat(want_b)) and torch.equal(rois[:n, 0].cpu(), torch.cat(want_i))
    assert torch.equal(labels[:n].cpu().long(), torch.cat(want_l))


def test_candidates_bad_count_rows(dev):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(1)
    pk = _rows(g, 3, 20, [20, 20, 4], (64, 48))
    pk[0, 20, 0] = 20.5
    pk[1, 20, 0] = 21.0
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    rois, labels, count = ops.query_candidates(pk.to(dev), (64, 48), 0.6, 1.5, bad)
    boxes, _ = ou.candidates(pk[2], (64, 48), 0.6, 1.5)
    assert int(bad) == 2 and int(count) == boxes.shape[0] and torch.equal(rois[:int(count), 1:].cpu(), boxes)
    ops.query_candidates(pk.to(dev), (64, 48), 0.6, 1.5, bad)
    assert int(bad) == 4                                               # the counter accumulates over calls


def _features(g, R, C, dirs, noise):
    cl = torch.randint(0, dirs.shape[0], (R,), generator=g)
    return dirs[cl] + noise * torch.randn(R, C, generator=g)


@pytest.mark.parametrize("max_query", [100, 6])
def test_bank_update_vs_restatement(dev, max_query):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(7 + max_query)
    C, L = 256, 9
    dirs = torch.randn(40, C, generator=g)
    start = defaultdict(list)
    for k in (1, 4):
        start[k] = _features(g, 5, C, dirs, 0.3)[:, None, :]
    qb = ops.QueryBank.from_dict(start, L, max_query, C, dev)
    bank = ou.copy_bank(start)
    margin = float("inf")
    for step in range(4):
        R = 60
        n = R - 7 * step                                               # the rows past the device count are never read
        feats = _features(g, R, C, dirs, 0.25)
        labels = torch.randint(1, L, (R,), generator=g)
        margin = min(margin, ou.bank_update(bank, labels[:n], feats[:n], max_query, 0.85))
        feats[n:] = float("nan")
        ops.query_bank_update(qb, feats.to(dev), labels.to(torch.int32).to(dev), torch.tensor([n], dtype=torch.int32, device=dev),
                              max_query, 0.85)
    assert margin > 1e-3
    got = qb.as_dict(qb.count.cpu())
    assert sorted(k for k, v in bank.items() if len(v)) == sorted(got)
    for k in got:
        assert torch.equal(got[k].cpu(), bank[k]), k
    if max_query == 6:
        assert max(len(v) for v in bank.values()) == 6


# ---------------------------------------------------------------------------------------------------------------------
# end to end: synthetic MQ-GLIP-T and MQ-GroundingDINO-T, 5-shot starting bank, 3 turns
# ---------------------------------------------------------------------------------------------------------------------
SIZES = [(150, 203)] * 5 + [(128, 160)] * 3


@functools.lru_cache(maxsize=2)
def _case(kind):
    from oracle import synth
    dev = torch.device("cuda:0")
    if kind == "glip":
        from test_gcp_many_queries_gpu import _glip
        gen = synth.Gen(2024)
        sd = synth.detector_sd(gen, bias0=-1.5)
        ids, am, pmap = synth.prompt(10, 2, 256, gen)
        model = _glip(sd, dev, 100)
        imgs = [synth.images(gen, 1, h, w)[0].to(dev) for h, w in SIZES]
    else:
        from test_gdino_asm_gpu import _build_model, _gdino_case
        sd, ids, am, pmap, _, _ = _gdino_case(3033, 1, 160, 224, 13, 2, 2, 100)
        gen = synth.Gen(77)
        model = _build_model(sd, 2, 2, 100, dev)
        model.cfg.VISION_QUERY.NUM_QUERY_PER_CLASS = model.query_selector.num_query_per_class = 100
        imgs = [synth.rgb_images(gen, 1, h, w)[0].to(dev) for h, w in SIZES]
    start = synth.query_bank(pmap, 5, synth.Gen(5))
    caps = {"input_ids": ids, "attention_mask": am}
    # the synthetic detectors score lower than trained ones: a threshold that keeps the first image's 30 (MQ-GLIP) or 10 best boxes
    from mqdet_b200.structures.image_list import to_image_list
    model.set_query_bank({k: v.clone() for k, v in start.items()})
    il = to_image_list([imgs[0]], 32)
    pk = (model.forward_device(il, caps, pmap)["det_packed"][0] if kind == "glip" else
          model.forward_chunked_device(il, [caps], [pmap])["det_packed"][0, 0]).cpu()
    scores = pk[:int(pk[-1, 0]), 4].sort(descending=True)[0]
    thr = float(scores[min((30 if kind == "glip" else 10) - 1, len(scores) - 1)]) - 1e-4
    return model, caps, pmap, start, imgs, thr


def _prepare(kind, turns=3):
    model, caps, pmap, start, imgs, thr = _case(kind)
    model.set_query_bank({k: v.clone() for k, v in start.items()})
    vq = model.cfg.VISION_QUERY
    vq.NUM_TURNS, vq.MAX_TEST_QUERY_NUMBER, vq.SCORE_THRESHOLD = turns, 100, thr
    # the synthetic MQ-GLIP's boxes move little from turn to turn: a higher similarity threshold lets every turn add rows, so the
    # banks after turns 1, 2 and 3 differ and the evaluation bank check below can tell them apart
    vq.SIMILARITY_THRESHOLD = 0.95 if kind == "glip" else 0.85
    return model, caps, pmap, start, imgs


def _host_loop(kind, model, caps, pmap, start, imgs):
    """The reference's loop: one image at a time, forward, scores > SCORE_THRESHOLD, extract_query(exclude_similar=True); the bank
    installed at the start of every turn after the first."""
    from mqdet_b200.structures.bounding_box import BoxList
    from mqdet_b200.structures.image_list import to_image_list
    vq = model.cfg.VISION_QUERY
    bank = ou.copy_bank(start)
    banks, kept_total = [], 0
    for turn in range(vq.NUM_TURNS):
        if turn > 0:
            model.set_query_bank({k: v.clone() for k, v in banks[-1].items()})
        for im in imgs:
            il = to_image_list([im], 32)
            if kind == "glip":
                out = model.forward_device(il, caps, pmap)
                pk, pyr = out["det_packed"][0].cpu(), out["pyramid16"]
            else:
                out = model.forward_chunked_device(il, [caps], [pmap])
                pk, pyr = out["det_packed"][0, 0].cpu(), out["pyramid16"]
            off, maps = 0, []
            for h, w in out["levels"].sizes:
                maps.append(pyr[:, off:off + h * w].float().transpose(1, 2).reshape(1, -1, h, w).contiguous())
                off += h * w
            h, w = il.image_sizes[0]
            n = int(pk[-1, 0])
            bl = BoxList(pk[:n, :4].clone(), (w, h), mode="xyxy")
            bl.add_field("scores", pk[:n, 4].clone())
            bl.add_field("labels", pk[:n, 5].long())
            kept = bl[bl.get_field("scores") > vq.SCORE_THRESHOLD]
            kept_total += len(kept)
            bank = model.extract_query(targets=[kept], query_images=bank, visual_features=maps, exclude_similar=True,
                                       max_query_number=vq.MAX_TEST_QUERY_NUMBER)
        banks.append(ou.copy_bank(bank))
    return banks, kept_total


def _assert_banks_equal(got, want, what):
    kg = sorted(int(k) for k, v in got.items() if len(v))
    kw = sorted(int(k) for k, v in want.items() if len(v))
    assert kg == kw, (what, kg, kw)
    for k in kg:
        assert torch.equal(got[k].cpu(), want[k].cpu()), (what, k, got[k].shape, want[k].shape)


@pytest.mark.parametrize("kind", ["glip", "gdino"])
def test_online_update_end_to_end(dev, kind):
    from mqdet_b200.engine.online_update import make_batches, online_update
    model, caps, pmap, start, imgs = _prepare(kind)
    want, kept = _host_loop(kind, model, caps, pmap, start, imgs)
    assert kept > 3 * len(imgs)
    res = {}
    for B in (1, 4):
        model, caps, pmap, start, imgs = _prepare(kind)
        res[B] = online_update(model, make_batches(imgs, B), caps, pmap, model.cfg, bank=start)
        assert len(res[B]["banks"]) == 3
        for t in range(3):
            _assert_banks_equal(res[B]["banks"][t], want[t], f"{kind} B={B} turn {t}")
        _assert_banks_equal(res[B]["eval_bank"], want[1], f"{kind} B={B} eval bank")     # the bank after turn 2
        _assert_banks_equal(model.query_selector.query_bank, want[1], f"{kind} B={B} model bank")
    rows = [sum(len(v) for v in b.values()) for b in [start] + want]
    assert rows[0] < rows[1] < rows[2] < rows[3], rows             # every turn grew the bank: the eval bank is turn 2's, no other
    model, caps, pmap, start, imgs = _prepare(kind)
    again = online_update(model, make_batches(imgs, 4), caps, pmap, model.cfg, bank=start)
    for t in range(3):                                                  # reruns are bit-identical
        _assert_banks_equal(again["banks"][t], res[4]["banks"][t], f"{kind} rerun turn {t}")


def test_one_turn_leaves_the_evaluation_bank(dev):
    from mqdet_b200.engine.online_update import make_batches, online_update
    model, caps, pmap, start, imgs = _prepare("glip", turns=1)
    res = online_update(model, make_batches(imgs, 4), caps, pmap, model.cfg, bank=start)
    _assert_banks_equal(res["eval_bank"], start, "one turn: the model keeps its bank")
    assert sum(len(v) for v in res["banks"][0].values()) > sum(len(v) for v in start.values())


def test_warm_turn_reads_nothing_on_the_host(dev):
    from mqdet_b200 import ops
    from mqdet_b200.engine.online_update import make_batches, online_update, update_turn
    for kind in ("glip", "gdino"):
        model, caps, pmap, start, imgs = _prepare(kind, turns=1)
        imgs = imgs[:4] + imgs[5:] + imgs[5:6]   # the prompt caches hold one batch size: batches of 4 + 4 images of two sizes
        batches = make_batches(imgs, 4)
        online_update(model, batches, caps, pmap, model.cfg, bank=start)      # warms the prompt and geometry caches
        qb = ops.QueryBank.from_dict(start, 14, 100, 256, dev)
        bad = torch.zeros(1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            update_turn(model, batches, caps, pmap, qb, model.cfg, bad)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        assert int(bad) == 0 and int(qb.count.sum()) > sum(len(v) for v in start.values())
