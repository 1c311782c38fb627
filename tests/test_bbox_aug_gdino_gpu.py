"""GPU: test-time augmentation for MQ-GroundingDINO — ``ops.bbox_aug_collect_packed`` (csrc/bbox_aug.cu) against the restatement
tests/bbox_aug_gdino_oracle.py (pinned to the reference's box_aug.py by tests/test_bbox_aug_gdino_cpu.py), and
``engine/bbox_aug`` with a ``GroundingDINO`` model against box_aug.py restated over ``GroundingDINO.forward`` run on each image
alone, as the reference runs it."""
import functools

import pytest
import torch

import bbox_aug_gdino_oracle as go
import bbox_aug_oracle as bo
from test_bbox_aug_gpu import _check

pytestmark = pytest.mark.gpu


def _packed(g, B, M, counts, size):
    """[B, M + 1, 6]: M GroundingDINO-shaped rows per image (rows past the count must not be read), rows 0..2 with areas lo^2
    and hi^2 of the range (32, 100) exactly and one just above lo^2; row M = (counts[b], 0, ...)."""
    pk = torch.zeros(B, M + 1, 6)
    for b, c in enumerate(counts):
        bx, s, lab = go.gdino_rows(g, M, size, 13)
        bx[:3] = torch.tensor([[10., 10., 41., 41.], [0., 0., 99., 99.], [10., 10., 42., 41.]])
        pk[b, :M, :4], pk[b, :M, 4], pk[b, :M, 5] = bx, s, lab.float()
        pk[b, M, 0] = c
    return pk


def _assert_merged_equal(m, want, what):
    for b, w in enumerate(want):
        n = int(m.count[b])
        assert n == w["boxes"].shape[0] and int(m.overflow[b]) == w["overflow"], (what, b, n, int(m.overflow[b]), w["overflow"])
        assert torch.equal(m.boxes[b, :n].cpu(), w["boxes"]), (what, b)
        assert torch.equal(m.scores[b, :n].cpu(), w["scores"]), (what, b)
        assert torch.equal(m.labels[b, :n].cpu().long(), w["labels"]), (what, b)


@pytest.mark.parametrize("cap", [4000, 700])
def test_collect_packed_vs_restatement(dev, cap):
    """Counts 0, 1, M, M - 1 and bad count rows (M + 1, 2.5, -1, NaN); three passes (two flipped, two with a range whose bounds
    the first rows hit exactly), appended behind each other; cap = 700 makes the last pass overflow."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(77)
    M, orig = 900, (640, 480)
    counts = [0.0, 1.0, float(M), float(M - 1), float(M + 1), 2.5, -1.0, float("nan")]
    B = len(counts)
    passes = [(_packed(g, B, M, counts, (533, 400)), (533, 400), False, (32, 100)),
              (_packed(g, B, M, counts, (533, 400)), (533, 400), True, (32, 100)),
              (_packed(g, B, M, counts, (800, 600)), (800, 600), True, None)]
    m, want = ops.MergedBoxes(B, cap, dev), go.empty_merged(B, cap)
    for pk, size, flip, rng in passes:
        ops.bbox_aug_collect_packed(m, pk.to(dev), size, orig, flip=flip, keep_range=rng)
        go.collect_packed(want, pk, size, orig, flip, rng)
    _assert_merged_equal(m, want, f"cap {cap}")
    assert all(w["overflow"] & go.BAD_COUNT for w in want[4:]) and not any(w["overflow"] & go.BAD_COUNT for w in want[:4])
    assert (cap < 2 * M) == any(0 < w["overflow"] < go.BAD_COUNT for w in want)
    # exactly on lo^2 / hi^2: dropped; just above lo^2: kept (image 2, first pass, count M)
    k = bo.range_keep(passes[0][0][2, :3, :4], 32, 100)
    assert k.tolist() == [False, False, True]
    # a bad count row raises at unpack, with the merge in between
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.engine import bbox_aug
    cls = torch.arange(1, 14, dtype=torch.int32, device=dev)
    packed = ops.nms_by_class(m.boxes, m.scores, m.labels, m.count, cls, 0.6, top_n=1000, max_out=1056, overflow=m.overflow)
    with pytest.raises(MqdetError, match="count row"):
        bbox_aug.unpack(packed[4:5], [orig])
    bbox_aug.unpack(packed[:1], [orig])
    with pytest.raises(MqdetError, match="did not fit" if cap < 2 * M else "count row"):
        bbox_aug.unpack(packed, [orig] * B)


def test_collect_packed_equals_cand_collect(dev):
    """The packed rows of a pass and the same rows as cand_* arrays (cand_totals = the counts) fill the merged buffers
    identically, bit for bit, across a flipped and a ranged pass and an overflow."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(78)
    M, B, orig = 300, 3, (500, 375)
    m1, m2 = ops.MergedBoxes(B, 400, dev), ops.MergedBoxes(B, 400, dev)
    for size, flip, rng, counts in (((667, 500), True, (16, 400), [300, 0, 123]), ((333, 250), False, None, [1, 300, 299]),
                                    ((667, 500), False, (0, 256), [300, 300, 300])):
        pk = _packed(g, B, M, counts, size)
        ops.bbox_aug_collect_packed(m1, pk.to(dev), size, orig, flip=flip, keep_range=rng)
        ops.bbox_aug_collect(m2, pk[:, :M, :4].contiguous().to(dev), pk[:, :M, 4].contiguous().to(dev),
                             pk[:, :M, 5].contiguous().to(dev), torch.tensor(counts, dtype=torch.int32, device=dev), size, orig,
                             flip=flip, keep_range=rng)
    for a, b in ((m1.boxes, m2.boxes), (m1.scores, m2.scores), (m1.labels, m2.labels), (m1.count, m2.count), (m1.overflow, m2.overflow)):
        assert torch.equal(a, b)
    assert int(m1.overflow.sum()) > 0 and int(m1.count.min()) > 0


# ---------------------------------------------------------------------------------------------------------------------
# the engine with a synthetic MQ-GroundingDINO-T (2 + 2 layers, 100 queries, 13-class prompt, K = 5)
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def _model_case():
    from test_gdino_asm_gpu import _build_model, _gdino_case
    sd, ids, am, pmap, bank, _ = _gdino_case(3033, 1, 160, 224, 13, 2, 2, 100)
    model = _build_model(sd, 2, 2, 100, torch.device("cuda:0"))
    model.query_selector.set_query_bank(bank)
    return model, {"input_ids": ids, "attention_mask": am}, pmap


def _model(**test):
    model, caps, pmap = _model_case()
    t = model.cfg.TEST
    base = dict(SCALES=(128, 176), RANGES=((0, 10000), (16, 150)), MAX_SIZE=1000, FLIP=True, SPECIAL_NMS="none", TH=0.6,
                PRE_NMS_TOP_N=1000, NUM_CLASSES=14, SELECT_CLASSES=())
    base.update(test)
    for k, v in base.items():
        setattr(t, k, v)
    return model, caps, pmap


def _u8(seed, h, w):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)


def _alone(model, img, caps, pmap, dev):
    """box_aug.py over GroundingDINO.forward on one image: per scale (and flip) the reference's transform, one forward (B = 1),
    the BoxList in pass coordinates; then the restatement of the merge."""
    from mqdet_b200.engine.transforms import TestTransform
    from mqdet_b200.structures.image_list import ImageList
    t = model.cfg.TEST
    per_pass = []
    for i, rng, flip in bo.passes(t):
        il, orig = TestTransform(model.cfg, t.SCALES[i], t.MAX_SIZE)([img], dev, pad=False)
        x = il.tensors
        h, w = x.shape[-2:]
        x = torch.flip(x, dims=[-1]) if flip else x
        bl = model(ImageList(bo.pad_to(x, 32), [(h, w)]), captions=caps, positive_map=pmap)[0]
        per_pass.append(((w, h), flip, rng, [(bl.bbox.cpu(), bl.get_field("scores").cpu(), bl.get_field("labels").cpu())]))
    want, _ = bo.merge_candidates(per_pass, orig, t)
    return want[0], sum(c[0][0].shape[0] for *_, c in per_pass)


@pytest.mark.parametrize("special", ["none", "vote"])
def test_im_detect_bbox_aug_images_equals_box_aug_over_forward(dev, special):
    from mqdet_b200.engine import bbox_aug
    model, caps, pmap = _model(SPECIAL_NMS=special)
    vote = special == "vote"
    pair = [_u8(1, 150, 203), _u8(2, 150, 203)]
    single = [_u8(3, 181, 131)]
    for imgs in (pair, single):
        got = bbox_aug.im_detect_bbox_aug_images(model, imgs, caps, pmap)
        assert len(got) == len(imgs)
        for b, (r, img) in enumerate(zip(got, imgs)):
            want, n_cand = _alone(model, img, caps, pmap, dev)
            assert r.size == (img.shape[1], img.shape[0]) and n_cand > 0 and len(r) > 0
            _check((r.bbox, r.get_field("scores"), r.get_field("labels")), want, vote, f"{special} image {b} of {len(imgs)}")


def test_batch_equals_one_image_calls_and_reruns(dev):
    from mqdet_b200.engine import bbox_aug
    from mqdet_b200.engine.transforms import TestTransform, upload
    model, caps, pmap = _model(SPECIAL_NMS="vote")
    t = model.cfg.TEST
    imgs = upload([_u8(4, 150, 203), _u8(5, 150, 203)], dev)

    def run(ims):
        batches, orig = [], None
        for s in t.SCALES:
            il, orig = TestTransform(model.cfg, s, t.MAX_SIZE)(ims, dev, pad=False)
            batches.append(il.tensors)
        return bbox_aug.im_detect_bbox_aug_device(model, batches, orig, caps, pmap), batches

    (packed, merged), batches = run(imgs)
    assert merged.cap == 4 * 100 and int(merged.count.min()) > 0
    for b in range(2):
        (one, _), _ = run(imgs[b:b + 1])
        assert torch.equal(packed[b], one[0]), f"image {b}: the batch differs from the image alone"
    (again, _), _ = run(imgs)
    assert torch.equal(again, packed), "reruns must be bit-identical"
    with pytest.raises(NotImplementedError):
        bbox_aug.im_detect_bbox_aug_device(model, batches, [(203, 150), (204, 150)], caps, pmap)


def test_one_pass_holds_the_rows_of_forward(dev):
    """One scale at the image's own size, no flip, no range, TH <= 0 and no per-image cut: the merged result holds exactly the
    rows of ``forward`` on each image alone (per class: the merge lists classes in ascending order)."""
    from mqdet_b200.engine import bbox_aug
    from mqdet_b200.structures.image_list import ImageList
    from mqdet_b200.engine.transforms import TestTransform
    model, caps, pmap = _model(SCALES=(150,), RANGES=(), FLIP=False, TH=0.0, PRE_NMS_TOP_N=0)
    imgs = [_u8(6, 150, 203), _u8(7, 150, 203)]
    res = bbox_aug.im_detect_bbox_aug_images(model, imgs, caps, pmap)
    for img, r in zip(imgs, res):
        il, _ = TestTransform(model.cfg, 150, 1000)([img], dev)
        assert tuple(il.image_sizes[0]) == (150, 203)
        q = model(ImageList(il.tensors, il.image_sizes), captions=caps, positive_map=pmap)[0]
        assert len(r) == len(q) > 0
        for c in range(1, 14):
            a, b = r.get_field("labels") == c, q.get_field("labels").cpu() == c
            assert torch.equal(r.bbox[a], q.bbox.cpu()[b]) and torch.equal(r.get_field("scores")[a], q.get_field("scores").cpu()[b]), c


@pytest.mark.parametrize("which", ["mq_groundingdino_t", "mq_glip_t"])
def test_warm_call_never_waits_for_the_device(dev, which):
    """Between the first forward and the one device->host copy a warm call launches without synchronising with the device
    (torch raises on any synchronising call under sync debug mode 'error'), for both detectors; its result equals the cold
    call's.  GroundingDINO: every scale is a new geometry of the chunked path's pass state."""
    from mqdet_b200.engine import bbox_aug
    from mqdet_b200.engine.transforms import TestTransform, upload
    if which == "mq_groundingdino_t":
        model, caps, pmap = _model(SPECIAL_NMS="vote")
    else:
        from test_bbox_aug_gpu import _detector
        over = {"TEST.SCALES": (150, 180), "TEST.RANGES": ((0, 10000), (16, 150)), "TEST.MAX_SIZE": 1000, "TEST.FLIP": True,
                "TEST.SPECIAL_NMS": "vote", "TEST.TH": 0.6, "TEST.PRE_NMS_TOP_N": 1000, "TEST.NUM_CLASSES": 11}
        model, _, _, ids, am, pmap, _ = _detector(dev, **over)
        caps = {"input_ids": ids, "attention_mask": am}
    t = model.cfg.TEST
    imgs = upload([_u8(8, 150, 203), _u8(9, 150, 203)], dev)
    batches = [TestTransform(model.cfg, s, t.MAX_SIZE)(imgs, dev, pad=False)[0].tensors for s in t.SCALES]
    orig = [(203, 150)] * 2
    cold, _ = bbox_aug.im_detect_bbox_aug_device(model, batches, orig, caps, pmap)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        warm, _ = bbox_aug.im_detect_bbox_aug_device(model, batches, orig, caps, pmap)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(warm, cold)
    assert sum(len(r) for r in bbox_aug.unpack(warm, orig)) > 0
