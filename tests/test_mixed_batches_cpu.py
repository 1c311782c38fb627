"""CPU: padded batches of differently sized images.  ``engine.batches.reference_test_batches`` against the reference's own
``GroupedBatchSampler`` (compiled as it is from maskrcnn_benchmark/data/samplers/grouped_batch_sampler.py) over a
``SequentialSampler`` and against torch's ``BatchSampler``, with the group ids of data/build.py (bisect_right([1], h / w)); and
tests/transform_oracle.py on images of different target sizes against the reference's Resize -> ToTensor -> Normalize ->
to_image_list; the reference's ATSSPostProcessor on a two-size padded batch against the restatement with per-image clip sizes
(recorded for tests/test_mixed_batches_gpu.py); and a host-logic dry run of ``online_update`` over mixed batches
(tests/hostlogic/mixed_batches_case.py).  The reference's results are recorded under tests/golden/mixed_batches_pins.pt, so the comparisons also run where
the reference is absent."""
import bisect
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import refpin
import transform_oracle as to
from oracle import ref_loader, restate, synth
from test_transform_cpu import GDINO, GLIP, _images, _run_reference
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "mixed_batches_pins.pt")
_store = None


def pinned(name, fn):
    global _store
    if _store is None:
        _store = torch.load(PIN_FILE, weights_only=True) if os.path.exists(PIN_FILE) else {}
    if ref_loader.available():
        val = fn()
        if os.environ.get("MQDET_RECORD_PINS") == "1":
            _store[name] = refpin._shrink(val, True)
            torch.save(_store, PIN_FILE)
        return val
    assert name in _store, f"{name}: no recorded result in {PIN_FILE}"
    return refpin._expand(_store[name])


def _reference_batches(image_hw, ims_per_batch, aspect_grouping):
    """make_batch_data_sampler(dataset, SequentialSampler, aspect_grouping, ims_per_batch, drop_last=False) of data/build.py."""
    sampler = torch.utils.data.sampler.SequentialSampler(range(len(image_hw)))
    if not aspect_grouping:
        return {"batches": [torch.tensor(b) for b in torch.utils.data.sampler.BatchSampler(sampler, ims_per_batch, drop_last=False)]}
    path = os.path.join(ref_loader.REF, "maskrcnn_benchmark", "data", "samplers", "grouped_batch_sampler.py")
    spec = importlib.util.spec_from_file_location("ref_grouped_batch_sampler", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    group_ids = [bisect.bisect_right([1], float(h) / float(w)) for h, w in image_hw]   # _quantize(_compute_aspect_ratios, [1])
    return {"batches": [torch.tensor(b) for b in mod.GroupedBatchSampler(sampler, group_ids, ims_per_batch, drop_uneven=False)]}


def _sizes(seed, n):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        r = rng.random()
        h, w = int(rng.integers(200, 900)), int(rng.integers(200, 900))
        out.append((w, w) if r < 0.15 else (h, w))            # some squares: h / w = 1 goes to group 1
    return out


SAMPLER_CASES = [
    ("landscape_then_portrait_runs", [(480, 640)] * 11 + [(640, 480)] * 5 + [(480, 640)] * 3, 8),
    ("uneven_tails", [(480, 640), (640, 480)] * 9 + [(500, 500)], 8),
    ("squares_join_portrait", [(500, 500), (480, 640), (333, 333), (640, 427), (480, 640)], 2),
    ("one_group_only", [(427, 640)] * 13, 4),
    ("random_sizes", _sizes(3, 157), 8),
    ("random_sizes_b1", _sizes(4, 23), 1),
]


@pytest.mark.parametrize("grouping", [True, False], ids=["grouped", "sequential"])
@pytest.mark.parametrize("case", SAMPLER_CASES, ids=[c[0] for c in SAMPLER_CASES])
def test_reference_test_batches_vs_reference_sampler(case, grouping):
    from mqdet_b200.engine.batches import reference_test_batches
    name, hw, bs = case
    want = pinned(f"sampler_{name}_{grouping}", lambda: _reference_batches(hw, bs, grouping))["batches"]
    got = reference_test_batches(hw, bs, grouping)
    assert got == [b.tolist() for b in want]
    assert sorted(i for b in got for i in b) == list(range(len(hw)))


def test_reference_test_batches_config_and_errors():
    from mqdet_b200.config import mq_glip_l_cfg, mq_glip_t_cfg, mq_groundingdino_t_cfg
    from mqdet_b200.engine.batches import reference_test_batches
    for cfg in (mq_glip_t_cfg(), mq_glip_l_cfg(), mq_groundingdino_t_cfg()):
        assert cfg.TEST.IMS_PER_BATCH == 8 and cfg.DATALOADER.ASPECT_RATIO_GROUPING is True
    assert reference_test_batches([], 8) == []
    assert reference_test_batches([(2, 3), (3, 2), (2, 3)], 8) == [[0, 2], [1]]
    with pytest.raises(ValueError, match="ims_per_batch"):
        reference_test_batches([(2, 3)], 0)


def test_make_batches_reference_order():
    from mqdet_b200.engine.online_update import make_batches
    hw = [(20, 30), (30, 20), (26, 30), (20, 30), (30, 26)]
    imgs = [torch.zeros(3, h, w) for h, w in hw]
    default = make_batches(imgs, 8)
    assert [il.image_sizes for il in default] == [[s] for s in hw]          # the default still splits at every size change
    ref = make_batches(imgs, 8, 32, orig_hw=hw)
    assert [il.image_sizes for il in ref] == [[hw[0], hw[2], hw[3]], [hw[1], hw[4]]]
    assert [tuple(il.tensors.shape) for il in ref] == [(3, 3, 32, 32), (2, 3, 32, 32)]
    with pytest.raises(ValueError, match="orig_hw"):
        make_batches(imgs, 8, orig_hw=hw[:2])


# (name, image sizes (h, w) resizing to different targets, size, max_size, normalisation, SIZE_DIVISIBILITY)
MIXED_CASES = [
    ("mixed_landscape_portrait_bgr255", [(17, 23), (23, 17), (40, 60)], 30, 60, GLIP, 32),
    ("mixed_clamp_and_keep_rgb", [(13, 90), (24, 31), (61, 47)], 24, 50, GDINO, 8),
    ("mixed_no_pad_rgb", [(75, 11), (11, 75)], 9, 80, GDINO, 0),
]


@pytest.mark.parametrize("case", MIXED_CASES, ids=[c[0] for c in MIXED_CASES])
def test_restatement_vs_reference_transform_mixed_targets(case):
    name, sizes, size, max_size, norm, div = case
    assert len({to.get_size((w, h), size, max_size) for h, w in sizes}) == len(sizes)
    want = pinned(name, lambda: _run_reference(sizes, size, max_size, norm, div, seed=len(name)))
    batch, resized = to.transform(_images(sizes, len(name)), size, max_size, norm["mean"], norm["std"], norm["fmt"], div)
    assert torch.equal(batch, want["batch"])
    assert [tuple(r.shape[:2]) for r in resized] == [tuple(s) for s in want["sizes"].tolist()]


# ---------------------------------------------------------------------------------------------------------------------
# the reference's ATSSPostProcessor on a padded batch of two image sizes
# ---------------------------------------------------------------------------------------------------------------------
ATSS_LEVELS, ATSS_STRIDES = [(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)], [8, 16, 32, 64, 128]
ATSS_IMAGE_HW = [(160, 224), (123, 150)]          # padded to 160 x 224 (the level grids above); image 1 clips to 150 x 123
ATSS_C = 20


def atss_two_size_inputs():
    """Head outputs of a two-image padded batch (seeded): box regressions [B, 4, h, w] (after the level Scale), centerness logits
    [B, 1, h, w] and dot-product logits [B, h * w, T] per level, the positive map and the anchors of each level."""
    gen = synth.Gen(43)
    B, T = len(ATSS_IMAGE_HW), 256
    _, _, pmap = synth.prompt(ATSS_C, 2, T, gen)
    regs = [gen.randn(B, 4, h, w, scale=1.5) for h, w in ATSS_LEVELS]
    ctrs = [gen.randn(B, 1, h, w) for h, w in ATSS_LEVELS]
    dots = [gen.randn(B, h * w, T, scale=1.5) - 2.5 for h, w in ATSS_LEVELS]
    anc = [restate.anchors_level(h, w, s, 8.0 * s) for (h, w), s in zip(ATSS_LEVELS, ATSS_STRIDES)]
    return pmap, regs, ctrs, dots, anc


def atss_two_size_reference():
    """ATSSPostProcessor.forward from the reference's own file (ml_nms substituted by the pinned restatement); each image's anchors
    carry that image's own size, as the reference's AnchorGenerator builds them from ImageList.image_sizes, and clip_to_image clips
    to it.  -> per image [n, 6] = box, score, label."""
    pmap, regs, ctrs, dots, anc = atss_two_size_inputs()
    B = len(ATSS_IMAGE_HW)
    inf = ref_loader.rpn_inference(lambda b, s, l, t: restate.ml_nms(b, s, l, t))
    BoxList = sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList
    coder = sys.modules["maskrcnn_benchmark.modeling.box_coder"].BoxCoder(weights=(10.0, 10.0, 5.0, 5.0))
    post = inf.ATSSPostProcessor(pre_nms_thresh=0.05, pre_nms_top_n=1000, nms_thresh=0.6, fpn_post_nms_top_n=100, min_size=0,
                                 num_classes=ATSS_C + 1, box_coder=coder, score_agg="MEAN")
    anchors = [[BoxList(a.clone(), (w, h), mode="xyxy") for a in anc] for h, w in ATSS_IMAGE_HW]
    cls = [torch.zeros(B, ATSS_C, h, w) for h, w in ATSS_LEVELS]
    with torch.no_grad():
        out = post(regs, ctrs, anchors, cls, None, dots, pmap)
    return {f"det{b}": torch.cat([r.bbox, r.get_field("scores")[:, None], r.get_field("labels")[:, None].float()], 1)
            for b, r in enumerate(out)}


def canon(x):
    """Detections [n, 6] in a canonical order (the reference's topk(sorted=False) order is implementation-defined)."""
    key = x[:, 4].double() * 1e6 + x[:, 5].double() * 1e-3 + x[:, 0].double() * 1e-9
    return x[torch.argsort(key)]


def test_atss_two_size_batch_reference_vs_restatement():
    """The reference's post-processor on a two-size padded batch, recorded for tests/test_mixed_batches_gpu.py, equals the
    restatement run per image with that image's own clip size; image 1 really is clipped to its own, smaller size."""
    ref = pinned("atss_two_sizes", atss_two_size_reference)
    pmap, regs, ctrs, dots, anc = atss_two_size_inputs()
    for b, (h, w) in enumerate(ATSS_IMAGE_HW):
        parts = [restate.atss_level_candidates(dots[l][b], regs[l][b].permute(1, 2, 0).reshape(-1, 4), ctrs[l][b].reshape(-1), anc[l],
                                               pmap, ATSS_C, w, h) for l in range(len(ATSS_LEVELS))]
        boxes, scores, labels = (torch.cat([p[k] for p in parts]) for k in ("boxes", "scores", "labels"))
        keep = restate.select_over_all_levels(boxes, scores, labels, 0.6, 100)
        got = torch.cat([boxes[keep], scores[keep, None], labels[keep, None].float()], 1)
        want = ref[f"det{b}"]
        assert got.shape == want.shape and want.shape[0] > 20, (b, got.shape, want.shape)
        assert torch.allclose(canon(got), canon(want), rtol=1e-6, atol=1e-5)
        assert float(want[:, 0:4:2].max()) <= w - 1 and float(want[:, 1:4:2].max()) <= h - 1
    assert float(ref["det1"][:, 2].max()) == ATSS_IMAGE_HW[1][1] - 1          # boxes reach the smaller image's own border


def test_online_update_host_logic_mixed_batches():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostlogic", "mixed_batches_case.py")], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PASS mixed online_update" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
