"""GPU: the multi-scale / flip test-time augmentation kernels (csrc/bbox_aug.cu) and ``engine/bbox_aug.py`` against the CPU
restatement tests/bbox_aug_oracle.py (itself pinned to the reference's box_aug.py by tests/test_bbox_aug_cpu.py)."""
import glob
import importlib.util
import os
from types import SimpleNamespace as NS

import pytest
import torch

import bbox_aug_oracle as bo
from util import ROOT, assert_close, load_sd

pytestmark = pytest.mark.gpu

CASES = sorted(bo.pin_cases())


def _merged(per_image, dev, cap=None):
    """[(boxes, scores, labels)] per image -> ops.MergedBoxes holding them"""
    from mqdet_b200 import ops
    cap = max([b.shape[0] for b, _, _ in per_image] + [1]) if cap is None else cap
    m = ops.MergedBoxes(len(per_image), cap, dev)
    for i, (b, s, l) in enumerate(per_image):
        n = b.shape[0]
        m.boxes[i, :n], m.scores[i, :n], m.labels[i, :n] = b.to(dev), s.to(dev), l.to(dev).int()
    m.count.copy_(torch.tensor([b.shape[0] for b, _, _ in per_image], dtype=torch.int32))
    return m


def _rows(packed, b):
    pk = packed.cpu()
    n = int(pk[b, -1, 0])
    assert n <= pk.shape[1] - 1
    return pk[b, :n, :4], pk[b, :n, 4], pk[b, :n, 5].long()


def _nms(m, test, dev, max_out=None):
    from mqdet_b200 import ops
    cls = torch.tensor(sorted(bo.class_list(test)), dtype=torch.int32, device=dev)
    mode = "vote" if test.SPECIAL_NMS == "vote" else "nms"
    return ops.nms_by_class(m.boxes, m.scores, m.labels, m.count, cls, test.TH, mode=mode, top_n=test.PRE_NMS_TOP_N,
                            max_out=m.cap if max_out is None else max_out)


def _check(got, want, vote, what):
    (gb, gs, gl), (wb, ws, wl) = got, want
    assert torch.equal(gl, wl) and torch.equal(gs, ws), what
    if vote:
        if wb.numel():
            assert_close(gb, wb, 1e-4, what + ": voted boxes")
            assert ((gb - wb).abs() <= 1e-4 * wb.abs() + 1e-4).all(), what
    else:
        assert torch.equal(gb, wb), what


@pytest.mark.parametrize("shape", [(2, 3, 5, 7, 8, 7), (2, 3, 37, 51, 64, 64), (1, 3, 150, 203, 160, 224)])
def test_hflip_pad_equals_flip_and_zero_pad(dev, shape):
    from mqdet_b200 import ops
    B, C, h, w, H, W = shape
    x = torch.randn(B, C, h, w, generator=torch.Generator().manual_seed(w))
    want = torch.zeros(B, C, H, W)
    want[..., :h, :w] = torch.flip(x, dims=[-1])
    assert torch.equal(ops.hflip_pad(x.to(dev), (H, W)).cpu(), want)


def _collect_case(c, dev, cap, B=1):
    from mqdet_b200 import ops
    m = ops.MergedBoxes(B, cap, dev)
    for size, flip, rng, b, s, l in c["passes"]:
        n = b.shape[0]
        S = n + 3                                   # rows beyond the pass's count are ignored
        cb, cs, cl = torch.full((B, S, 4), 7.0), torch.full((B, S), 0.5), torch.full((B, S), 1.0)
        cb[0, :n], cs[0, :n], cl[0, :n] = b, s, l.float()
        tot = torch.zeros(B, dtype=torch.int32)
        tot[0] = n
        ops.bbox_aug_collect(m, cb.to(dev), cs.to(dev), cl.to(dev), tot.to(dev), size, c["orig_size"], flip=flip, keep_range=rng)
    return m


@pytest.mark.parametrize("name", CASES)
def test_collect_then_merge_equals_restatement_on_the_pinned_cases(dev, name):
    c = bo.pin_cases()[name]
    want = bo.run_case(c)
    ub, us, ul = want["union"]
    m = _collect_case(c, dev, cap=max(ub.shape[0], 1) + 5, B=2)      # image 1 stays empty
    n = int(m.count[0])
    assert n == ub.shape[0] and int(m.count[1]) == 0 and int(m.overflow.sum()) == 0
    assert torch.equal(m.boxes[0, :n].cpu(), ub) and torch.equal(m.scores[0, :n].cpu(), us)
    assert torch.equal(m.labels[0, :n].cpu().long(), ul)
    vote = c["test"].SPECIAL_NMS == "vote" and c["test"].TH > 0
    packed = _nms(m, c["test"], dev)
    _check(_rows(packed, 0), want["result"], vote, name)
    assert int(packed[1, -1, 0]) == 0
    assert torch.equal(packed, _nms(m, c["test"], dev)), "reruns must be bit-identical"


def test_collect_overflow_is_counted_and_raises(dev):
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.engine import bbox_aug
    c = bo.pin_cases()["equal_nms"]
    full = bo.run_case(c)["union"][0].shape[0]
    m = _collect_case(c, dev, cap=full - 7)
    assert int(m.count[0]) == full - 7 and int(m.overflow[0]) == 7
    from mqdet_b200 import ops
    cls = torch.arange(1, 6, dtype=torch.int32, device=dev)
    packed = ops.nms_by_class(m.boxes, m.scores, m.labels, m.count, cls, 0.5, top_n=1000, max_out=m.cap, overflow=m.overflow)
    with pytest.raises(MqdetError, match="did not fit"):
        bbox_aug.unpack(packed, [c["orig_size"]])
    small = ops.nms_by_class(m.boxes, m.scores, m.labels, m.count, cls, 0.0, top_n=0, max_out=8)
    with pytest.raises(MqdetError, match="exceed"):
        bbox_aug.unpack(small, [c["orig_size"]])


def _random_set(n, seed, n_labels=80):
    """jittered copies of n / 20 objects over 80 classes, one class holding half of the boxes"""
    g = torch.Generator().manual_seed(seed)
    b, s, l = bo._objects(g, max(n // 20, 1), 20, (1333, 800), n_labels, jitter=10.0)
    half = torch.randperm(b.shape[0], generator=g)[: b.shape[0] // 2]
    l[half] = 7
    return b, s, l


@pytest.mark.parametrize("n,mode", [(200, "none"), (200, "vote"), (5000, "none"), (5000, "vote"), (120000, "none"), (120000, "vote")])
def test_nms_by_class_random_sets(dev, n, mode):
    b, s, l = _random_set(n, n)
    test = NS(SPECIAL_NMS=mode, TH=0.6, PRE_NMS_TOP_N=1000, NUM_CLASSES=81, SELECT_CLASSES=())
    per_image = [(b, s, l), (torch.zeros(0, 4), torch.zeros(0), torch.zeros(0, dtype=torch.long))]
    if n == 200:   # a second, different image and an empty one
        per_image.append(_random_set(150, 9))
    m = _merged(per_image, dev)
    packed = _nms(m, test, dev, max_out=1056)
    for i, u in enumerate(per_image):
        want = bo.merge(*u, bo.class_list(test), test.TH, "vote" if mode == "vote" else "nms", test.PRE_NMS_TOP_N)
        _check(_rows(packed, i), want, mode == "vote", f"random {n} {mode} image {i}")
    if n == 120000:
        assert int(packed[0, -1, 0]) >= 1000
    assert torch.equal(packed, _nms(m, test, dev, max_out=1056))
    # without the per-image cut (every survivor returned)
    if n <= 5000:
        test.PRE_NMS_TOP_N = 0
        packed = _nms(m, test, dev)
        want = bo.merge(b, s, l, bo.class_list(test), test.TH, "vote" if mode == "vote" else "nms", 0)
        _check(_rows(packed, 0), want, mode == "vote", f"random {n} {mode} uncut")


def test_nms_by_class_equals_reference_nms_kernel(dev):
    so = glob.glob(os.path.join(ROOT, "oracle", "_ref", "mqdet_ref_C*.so"))
    if not so:
        pytest.skip("the reference's compiled extension is not built (oracle/build_ref.py)")
    spec = importlib.util.spec_from_file_location("mqdet_ref_C", so[0])
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    b, s, l = _random_set(200, 77, n_labels=1)
    l[:] = 1
    s = torch.linspace(0.95, 0.05, b.shape[0])[torch.randperm(b.shape[0], generator=torch.Generator().manual_seed(1))]  # tie-free
    keep = ref.nms(b.to(dev), s.to(dev), 0.6).cpu()
    test = NS(SPECIAL_NMS="none", TH=0.6, PRE_NMS_TOP_N=0, NUM_CLASSES=2, SELECT_CLASSES=())
    gb, gs, _ = _rows(_nms(_merged([(b, s, l)], dev), test, dev), 0)
    assert torch.equal(gb, b[keep]) and torch.equal(gs, s[keep])


def test_drop_in_remove_boxes_and_merge(dev):
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.engine import bbox_aug
    from mqdet_b200.structures.bounding_box import BoxList
    c = bo.pin_cases()["equal_vote"]
    size, _, rng, b, s, l = c["passes"][0]
    bl = BoxList(b.to(dev), size)
    bl.add_field("scores", s.to(dev))
    bl.add_field("labels", l.to(dev))
    kept = bbox_aug.remove_boxes([bl], *rng)[0]
    k = bo.range_keep(b, *rng)
    assert torch.equal(kept.bbox.cpu(), b[k]) and torch.equal(kept.get_field("scores").cpu(), s[k])
    cfg = mq_glip_t_cfg(**{"TEST.SPECIAL_NMS": "vote", "TEST.NUM_CLASSES": 6})
    ub, us, ul = bo.run_case(c)["union"]
    u = BoxList(ub.to(dev), c["orig_size"])
    u.add_field("scores", us.to(dev))
    u.add_field("labels", ul.to(dev))
    r = bbox_aug.merge_result_from_multi_scales([u], cfg)[0]
    assert r.bbox.is_cuda and r.size == c["orig_size"]
    _check((r.bbox.cpu(), r.get_field("scores").cpu(), r.get_field("labels").cpu()), bo.run_case(c)["result"], True, "drop-in merge")


def _detector(dev, **over):
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
    from oracle import synth
    gen = synth.Gen(2024)
    sd = synth.detector_sd(gen, bias0=-1.5)
    ids, am, pmap = synth.prompt(10, 2, 256, gen)
    bank = synth.query_bank(pmap, 5, gen)
    model = GeneralizedVLRCNN_New(mq_glip_t_cfg(**over))
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    model = load_sd(model, full).to(dev).eval()
    model.query_selector.set_query_bank(bank)
    return model, gen, sd, ids, am, pmap, bank


def _iou(a, b):
    x1, y1 = torch.max(a[:, None, 0], b[None, :, 0]), torch.max(a[:, None, 1], b[None, :, 1])
    x2, y2 = torch.min(a[:, None, 2], b[None, :, 2]), torch.min(a[:, None, 3], b[None, :, 3])
    inter = (x2 - x1 + 1).clamp(min=0) * (y2 - y1 + 1).clamp(min=0)
    aa = (a[:, 2] - a[:, 0] + 1) * (a[:, 3] - a[:, 1] + 1)
    ab = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
    return inter / (aa[:, None] + ab[None] - inter)


@pytest.mark.parametrize("special", ["none", "vote"])
def test_im_detect_bbox_aug_end_to_end(dev, special):
    from mqdet_b200.engine import bbox_aug
    from oracle import synth
    over = {"TEST.SCALES": (135, 150, 180), "TEST.RANGES": ((24, 10000), (0, 10000), (0, 120)), "TEST.FLIP": True,
            "TEST.SPECIAL_NMS": special, "TEST.TH": 0.6, "TEST.PRE_NMS_TOP_N": 1000, "TEST.NUM_CLASSES": 11}
    model, gen, sd, ids, am, pmap, bank = _detector(dev, **over)
    B = 2
    imgs = [synth.images(gen, B, h, w)[..., :h, :w].contiguous() for h, w in ((135, 182), (150, 203), (180, 244))]   # padded: at least 2 x 2 at stride 128
    orig = [(203, 150)] * B
    caps = {"input_ids": ids, "attention_mask": am}
    packed, merged = bbox_aug.im_detect_bbox_aug_device(model, [x.to(dev) for x in imgs], orig, caps, pmap)
    res = bbox_aug.unpack(packed, orig)
    t = model.cfg.TEST
    # the merge alone, fed the device's own candidates: identical to the restatement's merge of those candidates
    for b in range(B):
        n = int(merged.count[b])
        assert n > 0
        want = bo.merge(merged.boxes[b, :n].cpu(), merged.scores[b, :n].cpu(), merged.labels[b, :n].cpu().long(), bo.class_list(t),
                        t.TH, "vote" if special == "vote" else "nms", t.PRE_NMS_TOP_N)
        _check((res[b].bbox, res[b].get_field("scores"), res[b].get_field("labels")), want, special == "vote", f"e2e merge image {b}")
    # the whole augmented detection against the restatement over the oracle's detector
    ref, _ = bo.im_detect_bbox_aug(imgs, orig, ids, am, pmap, bank, sd, t)
    for b, r in enumerate(res):
        rb, rs, rl = ref[b]
        assert r.size == (203, 150) and abs(len(r) - rb.shape[0]) <= max(10, rb.shape[0] // 10), (len(r), rb.shape[0])
        iou = _iou(rb, r.bbox)
        same = rl[:, None] == r.get_field("labels")[None]
        matched = ((iou > 0.9) & same & ((rs[:, None] - r.get_field("scores")[None]).abs() < 2e-2)).any(1)
        # voting is discontinuous in the candidates: a score changed by the detector's fp16 noise moves a box to another cluster
        # and with it the cluster's mean box, so fewer voted boxes match one to one (the merge itself is exact, above)
        need = 0.75 if special == "vote" else 0.85
        assert matched.float().mean().item() >= need, f"image {b}: only {matched.float().mean().item():.2f} matched"


def test_single_pass_equals_the_detector_before_its_cut(dev):
    """One pass at the original size, no flip, no ranges, TH = MODEL.ATSS.NMS_TH and no per-image cut: the detections of
    ``model.forward`` with DETECTIONS_PER_IMG out of the way — the candidates are what the reference hands to box_aug."""
    from mqdet_b200.engine import bbox_aug
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    over = {"TEST.SCALES": (150,), "TEST.RANGES": (), "TEST.FLIP": False, "TEST.TH": 0.6, "TEST.PRE_NMS_TOP_N": 0,
            "TEST.NUM_CLASSES": 11, "MODEL.ATSS.DETECTIONS_PER_IMG": 4000}
    model, gen, sd, ids, am, pmap, bank = _detector(dev, **over)
    B, h, w = 2, 150, 203
    img = synth.images(gen, B, h, w)[..., :h, :w].contiguous().to(dev)   # synth pads; the engine pads again
    caps = {"input_ids": ids, "attention_mask": am}
    res = bbox_aug.im_detect_bbox_aug(model, [img], [(w, h)] * B, caps, pmap)
    pad = img.new_zeros((B, 3, 160, 224))
    pad[..., :h, :w] = img
    base = model(ImageList(pad, [(h, w)] * B), captions=caps, positive_map=pmap)
    for r, q in zip(res, base):
        assert len(r) == len(q) > 0
        key = lambda bl: sorted(zip(bl.get_field("labels").tolist(), bl.get_field("scores").tolist(), bl.bbox.tolist()))  # noqa: E731
        assert key(r) == key(q)
