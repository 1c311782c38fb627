"""GPU: the test transform kernels (csrc/transform.cu) and engine/transforms.py against the reference pipeline — PIL's bilinear
resize, torchvision's to_tensor / normalize with the reference's format handling, zero padding as to_image_list — and
``predict`` / ``im_detect_bbox_aug_images`` against the detectors fed the host-transformed batches.  Every comparison is exact."""
import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image

import transform_oracle as to

pytestmark = pytest.mark.gpu

GLIP = dict(mean=[103.530, 116.280, 123.675], std=[57.375, 57.120, 58.395], fmt="bgr255")
GDINO = dict(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225], fmt="rgb")


def _images(sizes, seed):
    rng = np.random.default_rng(seed)
    out = []
    for h, w in sizes:
        # smooth structure plus noise: resampling of both flat areas and edges is exercised
        yy, xx = np.mgrid[0:h, 0:w]
        base = (np.stack([xx * 255.0 / max(w - 1, 1), yy * 255.0 / max(h - 1, 1), (xx + yy) % 256], -1)).astype(np.int64)
        out.append(np.clip(base + rng.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8))
    return out


def _host_pipeline(images, size, max_size, norm, div):
    """The reference's Resize -> ToTensor -> Normalize, with PIL and torchvision, then to_image_list: (padded batch, resized
    uint8 images)."""
    chw, resized = [], []
    for im in images:
        h, w = im.shape[:2]
        pil = F.resize(Image.fromarray(im), list(to.get_size((w, h), size, max_size)))
        resized.append(np.asarray(pil))
        t = F.to_tensor(pil)
        if "bgr" in norm["fmt"]:
            t = t[[2, 1, 0]]
        if "255" in norm["fmt"]:
            t = t * 255
        chw.append(F.normalize(t, mean=norm["mean"], std=norm["std"]))
    return to.pad_batch(chw, div), resized


def _cfg(norm, size=800, max_size=1333, div=32):
    from types import SimpleNamespace as NS
    fmt = "" if norm["fmt"] == "bgr255" else norm["fmt"]
    return NS(INPUT=NS(PIXEL_MEAN=norm["mean"], PIXEL_STD=norm["std"], MIN_SIZE_TEST=size, MAX_SIZE_TEST=max_size, FORMAT=fmt,
                       TO_BGR255=True), DATALOADER=NS(SIZE_DIVISIBILITY=div))


@pytest.mark.parametrize("pair", [(4000, 1333), (3000, 1000), (640, 1066), (480, 800), (1, 7), (7, 1), (2, 1), (800, 800),
                                  (10000, 10), (1333, 4000), (997, 333)])
def test_resize_coeffs_equal_restatement(dev, pair):
    from mqdet_b200 import ops
    n_in, n_out = pair
    t = ops.resize_coeffs(n_in, n_out, dev).cpu().long()
    lo, n, k = to.coeffs(n_in, n_out)
    assert t.shape == (n_out, 2 + k.shape[1])
    assert torch.equal(t[:, 0], torch.from_numpy(lo)) and torch.equal(t[:, 1], torch.from_numpy(n))
    assert torch.equal(t[:, 2:], torch.from_numpy(k))


CASES = {
    # name: (source sizes (h, w), MIN_SIZE_TEST, MAX_SIZE_TEST, SIZE_DIVISIBILITY)
    "lvis_like": ([(480, 640)], 800, 1333, 32),
    "portrait": ([(640, 427)], 800, 1333, 32),
    "downscale_4000x3000": ([(3000, 4000)], 1000, 1333, 32),
    "downscale_clamped": ([(1500, 6000)], 800, 1333, 32),
    "three_sources_one_target": ([(480, 640), (600, 800), (3000, 4000)], 800, 1333, 32),
    "same_size": ([(800, 1201)], 800, 1333, 32),
    "tiny": ([(1, 2), (2, 4)], 3, 100, 32),
    "no_padding": ([(37, 53)], 45, 1000, 0),
}


@pytest.mark.parametrize("fmt", ["bgr255", "rgb"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_transform_equals_reference_pipeline(dev, name, fmt):
    from mqdet_b200.engine import transforms as tr
    sizes, size, max_size, div = CASES[name]
    norm = GLIP if fmt == "bgr255" else GDINO
    images = _images(sizes, seed=len(name))
    want, want_u8 = _host_pipeline(images, size, max_size, norm, div)
    il, orig, resized = tr.TestTransform(_cfg(norm, size, max_size, div))(images, dev, want_resized=True)
    oh, ow = il.image_sizes[0]
    assert orig == [(w, h) for h, w in sizes]
    assert all(tuple(r.shape[:2]) == (oh, ow) for r in want_u8)
    for b, r in enumerate(want_u8):
        assert np.array_equal(resized[b].cpu().numpy(), r), f"image {b}: uint8 resize differs from PIL"
    got = il.tensors.cpu()
    assert got.shape == want.shape and torch.equal(got, want)
    assert (got[..., oh:, :] == 0).all() and (got[..., :, ow:] == 0).all()


def test_inputs_as_tensors_and_device_tensors(dev):
    from mqdet_b200.engine import transforms as tr
    images = _images([(120, 160), (150, 200)], 3)
    cfg = _cfg(GLIP, 240, 400)
    ref, _ = tr.TestTransform(cfg)(images, dev)
    for form in (lambda a: torch.from_numpy(a), lambda a: torch.from_numpy(a).to(dev)):
        il, _ = tr.TestTransform(cfg)([form(a) for a in images], "cuda")
        assert torch.equal(il.tensors, ref.tensors)
    assert ref.tensors.is_cuda and ref.image_sizes == [(240, 320)] * 2


def test_more_images_than_one_launch_takes(dev):
    from mqdet_b200.engine import transforms as tr
    sizes = [(7 + i % 3, 9 + i % 3) for i in range(70)]
    sizes = [(h, w) for h, w in sizes if to.get_size((w, h), 12, 100) == to.get_size((9, 7), 12, 100)]
    images = _images(sizes, 8) * 2
    assert len(images) > 64
    want, _ = _host_pipeline(images, 12, 100, GLIP, 32)
    il, _ = tr.TestTransform(_cfg(GLIP, 12, 100))(images, dev)
    assert torch.equal(il.tensors.cpu(), want)


def test_mixed_target_sizes_raise(dev):
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.engine import transforms as tr
    with pytest.raises(MqdetError, match="different sizes"):
        tr.TestTransform(_cfg(GLIP))(_images([(480, 640), (640, 480)], 1), dev)


@pytest.mark.parametrize("out_hw", [(37, 91), (91, 53), (37, 53), (5, 200)])
def test_one_dimension_unchanged_equals_pil(dev, out_hw):
    """ops.test_transform at sizes get_size does not produce: one pass skipped by PIL, an identity pass here."""
    from mqdet_b200 import ops
    im = _images([(37, 53)], 4)[0]
    oh, ow = out_hw
    x = torch.from_numpy(im).to(dev)
    out, resized = ops.test_transform([x], [ops.resize_coeffs(53, ow, dev)], [ops.resize_coeffs(37, oh, dev)], out_hw, (oh + 3, ow + 5),
                                      GDINO["mean"], GDINO["std"], want_resized=True)
    ref = np.asarray(Image.fromarray(im).resize((ow, oh), Image.BILINEAR))
    assert np.array_equal(resized[0].cpu().numpy(), ref)
    want = torch.nn.functional.pad(to.normalize(ref, GDINO["mean"], GDINO["std"], "rgb"), (0, 5, 0, 3))[None]
    assert torch.equal(out.cpu(), want)


@pytest.mark.parametrize("which", ["mq_glip_t", "mq_groundingdino_t"])
def test_predict_equals_forward_on_host_transformed_batch(dev, which):
    from mqdet_b200.engine import transforms as tr
    from mqdet_b200.structures.image_list import ImageList
    from test_coco_eval_models_gpu import _gdino, _glip
    build = _glip if which == "mq_glip_t" else _gdino
    model, caps, pmap, _, _ = build(dev)
    model.cfg.INPUT.MIN_SIZE_TEST, model.cfg.INPUT.MAX_SIZE_TEST = 160, 224
    norm = GLIP if which == "mq_glip_t" else GDINO
    assert tr.TestTransform(model.cfg).bgr == (which == "mq_glip_t")
    images = _images([(120, 168), (150, 210)], 21)       # two source sizes, one target: 160 x 224
    host, _ = _host_pipeline(images, 160, 224, norm, 32)
    il = ImageList(host.to(dev), [(160, 224)] * 2)
    out = model.forward_device(il, caps, pmap)
    det_host, num_host = out["det"].clone(), out["num"].clone()
    base = model(il, captions=caps, positive_map=pmap)
    res = tr.predict(model, images, caps, pmap)
    dil, _ = tr.TestTransform(model.cfg)(images, dev)
    assert torch.equal(dil.tensors, il.tensors) and dil.image_sizes == il.image_sizes
    out = model.forward_device(dil, caps, pmap)
    assert torch.equal(out["det"], det_host) and torch.equal(out["num"], num_host)
    assert sum(len(r) for r in res) > 0
    for r, q, (h, w) in zip(res, base, [(120, 168), (150, 210)]):
        q = q.resize((w, h))
        assert r.size == (w, h) and r.mode == "xyxy"
        assert torch.equal(r.bbox, q.bbox)
        assert torch.equal(r.get_field("scores"), q.get_field("scores")) and torch.equal(r.get_field("labels"), q.get_field("labels"))


def test_im_detect_bbox_aug_images_equals_host_transformed_batches(dev):
    from mqdet_b200.engine import bbox_aug
    from test_bbox_aug_gpu import _detector
    over = {"TEST.SCALES": (135, 150, 180), "TEST.RANGES": ((24, 10000), (0, 10000), (0, 120)), "TEST.FLIP": True,
            "TEST.MAX_SIZE": 1000, "TEST.SPECIAL_NMS": "vote", "TEST.TH": 0.6, "TEST.PRE_NMS_TOP_N": 1000, "TEST.NUM_CLASSES": 11}
    model, _, _, ids, am, pmap, _ = _detector(dev, **over)
    caps = {"input_ids": ids, "attention_mask": am}
    images = _images([(120, 162)] * 2, 33)
    batches = []
    for s in model.cfg.TEST.SCALES:
        x, _ = _host_pipeline(images, s, 1000, GLIP, 0)
        batches.append(x.to(dev))
    want = bbox_aug.im_detect_bbox_aug(model, batches, [(162, 120)] * 2, caps, pmap)
    got = bbox_aug.im_detect_bbox_aug_images(model, images, caps, pmap)
    assert sum(len(r) for r in got) > 0
    for g, w in zip(got, want):
        assert g.size == w.size == (162, 120)
        assert torch.equal(g.bbox, w.bbox)
        assert torch.equal(g.get_field("scores"), w.get_field("scores")) and torch.equal(g.get_field("labels"), w.get_field("labels"))
