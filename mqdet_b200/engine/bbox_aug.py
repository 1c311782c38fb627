"""Multi-scale + horizontal-flip test-time augmentation for MQ-GLIP and MQ-GroundingDINO, drop-in for
maskrcnn_benchmark/data/datasets/evaluation/box_aug.py (``TEST.USE_MULTISCALE``).

The detector runs on every image at each of ``TEST.SCALES`` and again on the flipped image when ``TEST.FLIP``; boxes outside
the scale's ``TEST.RANGES`` are dropped, every pass is mapped back to the original image, and the union is merged per class
(``TEST.SPECIAL_NMS``: plain NMS or box voting at ``TEST.TH``) and cut to ``TEST.PRE_NMS_TOP_N`` per image.

The reference merges on the host (a Python loop over the classes of every image, a ``.cpu()`` + ``kthvalue`` + ``.item()``
per image, numpy ``np.delete`` per voting cluster).  Here the candidates of a pass never leave the device: each pass appends
to a per-image device buffer (``ops.bbox_aug_collect``), one ``ops.nms_by_class`` merges the whole batch, and the packed result
is the one device->host copy.  Nothing synchronises with the host between the first forward and that copy.

What a pass hands to the merge is what the reference's box_aug.py receives from the model: for MQ-GLIP the pre-NMS candidates
of ATSSPostProcessor (``cand_*``, bbox_aug_enabled), for MQ-GroundingDINO its final output (convert_groundingdino_to_glip_output:
every query above box_threshold, in query order, clipped, no NMS), i.e. the packed rows of ``gdino_detections``
(``ops.bbox_aug_collect_packed``).  A GroundingDINO pass runs through ``forward_chunked_device`` with the prompt as its only
chunk: that path takes the fusion layers' stable-softmax maximum per image, so every image of the batch gets what the
reference's one-image forward gives it (``forward_device`` takes one maximum over the whole batch).
"""
import torch

from .. import ops
from .._lib import MqdetError
from ..structures.bounding_box import BoxList
from ..structures.image_list import ImageList
from .transforms import TestTransform, model_device, upload

_MODES = {"none": "nms", "nms": "nms", "vote": "vote"}


def _mode(test_cfg):
    key = test_cfg.SPECIAL_NMS
    if key in ("soft-nms", "soft-vote"):
        raise NotImplementedError(f"TEST.SPECIAL_NMS = {key!r} is not implemented (plain NMS and 'vote' are)")
    if key not in _MODES:
        raise ValueError(f"TEST.SPECIAL_NMS = {key!r}")
    return _MODES[key]


def _classes(test_cfg, device):
    sel = [int(c) for c in test_cfg.SELECT_CLASSES]
    if sel != sorted(set(sel)):   # the result lists the classes in table order; the reference walks SELECT_CLASSES as given
        raise ValueError(f"TEST.SELECT_CLASSES must be ascending without repeats (got {tuple(sel)})")
    cls = sel if len(sel) else list(range(1, int(test_cfg.NUM_CLASSES)))
    return ops.upload_async(torch.tensor(cls, dtype=torch.int32), device)


def result_rows(test_cfg, cap):
    """Rows of the packed result: PRE_NMS_TOP_N plus head-room for the scores tied at the cut (as
    ``GeneralizedVLRCNN_New.max_out``); without a cut every merged box can remain."""
    n = int(test_cfg.PRE_NMS_TOP_N)
    return (n + 28 + 31) // 32 * 32 if n > 0 else int(cap)


def unpack(packed, sizes):
    """Packed [B, rows + 1, 6] (host or device) -> list[BoxList] (mode xyxy, fields labels / scores); sizes: (w, h) per image.
    Raises when the merged buffer or the result rows were too small: nothing is clipped silently."""
    pk = packed.cpu()
    rows = pk.shape[1] - 1
    res = []
    for b, size in enumerate(sizes):
        n, lost = int(round(float(pk[b, rows, 0]))), int(round(float(pk[b, rows, 1])))
        if lost >= ops.BBOX_AUG_BAD_COUNT:
            raise MqdetError(f"image {b}: a detector pass gave a count row that is not an integer in [0, rows]")
        if lost:
            raise MqdetError(f"image {b}: {lost} candidates did not fit in the merged buffer; raise `cap`")
        if n > rows:
            raise MqdetError(f"image {b}: {n} merged detections (score ties at the PRE_NMS_TOP_N cut) exceed the {rows}-row result buffer")
        d = pk[b, :n]
        bl = BoxList(d[:, :4].clone(), tuple(size), mode="xyxy")
        bl.add_field("scores", d[:, 4].clone())
        bl.add_field("labels", d[:, 5].long())
        res.append(bl)
    return res


def remove_boxes(boxlist_ts, min_scale, max_scale):
    """box_aug.py:150-163 for CUDA BoxLists: keeps boxes with min_scale^2 < w * h < max_scale^2 (both strict), order kept."""
    out = []
    for bl in boxlist_ts:
        mode = bl.mode
        bl = bl.convert("xyxy")
        n = len(bl)
        if n == 0:
            out.append(bl.convert(mode))
            continue
        dev = bl.bbox.device
        m = ops.MergedBoxes(1, n, dev)
        idx = torch.arange(n, dtype=torch.float32, device=dev)[None].contiguous()   # carried as the score: survivors' indices
        ops.bbox_aug_collect(m, bl.bbox[None].contiguous(), idx, torch.zeros_like(idx),
                             torch.full((1,), n, dtype=torch.int32, device=dev), (1, 1), (1, 1),
                             keep_range=(min_scale, max_scale))
        keep = m.scores[0, :int(m.count.item())].long()
        out.append(bl[keep].convert(mode))
    return out


def merge_result_from_multi_scales(boxlists, cfg, cap=None):
    """box_aug.py:166-206 for CUDA BoxLists (fields ``scores``, ``labels``): per-class NMS / voting and the per-image cut of
    ``cfg.TEST``, one kernel sequence for all images."""
    t = cfg.TEST
    mode = _mode(t)
    dev = boxlists[0].bbox.device
    B = len(boxlists)
    cap = max([len(bl) for bl in boxlists] + [1]) if cap is None else int(cap)
    m = ops.MergedBoxes(B, cap, dev)
    for b, bl in enumerate(boxlists):
        n = len(bl)
        m.boxes[b, :n] = bl.convert("xyxy").bbox
        m.scores[b, :n] = bl.get_field("scores")
        m.labels[b, :n] = bl.get_field("labels").to(torch.int32)
    m.count.copy_(torch.tensor([len(bl) for bl in boxlists], dtype=torch.int32))
    packed = ops.nms_by_class(m.boxes, m.scores, m.labels, m.count, _classes(t, dev), float(t.TH), mode=mode,
                              top_n=int(t.PRE_NMS_TOP_N), max_out=result_rows(t, cap))
    return [r.to(dev) for r in unpack(packed, [bl.size for bl in boxlists])]


@torch.no_grad()
def im_detect_bbox_aug_device(model, images_by_scale, orig_sizes, captions, positive_map, cap=None):
    """Device-resident form of ``im_detect_bbox_aug``: returns (packed fp32 [B, rows + 1, 6], merged ``ops.MergedBoxes``);
    packed rows are (x1, y1, x2, y2, score, label) in original-image coordinates, row ``rows`` = (count, candidates lost to a
    full merged buffer, 0...).  ``cap``: merged candidates kept per image (default: every candidate of every pass, for
    MQ-GroundingDINO passes x num_queries)."""
    from ..modeling.groundingdino.groundingdino import GroundingDINO
    gdino = isinstance(model, GroundingDINO)
    cfg = model.cfg
    t = cfg.TEST
    mode = _mode(t)
    scales = list(t.SCALES)
    if len(images_by_scale) != len(scales):
        raise ValueError(f"{len(images_by_scale)} image batches for {len(scales)} TEST.SCALES")
    ranges = list(t.RANGES) if len(t.RANGES) == len(scales) else [None] * len(scales)
    B = images_by_scale[0].shape[0]
    if any(tuple(s) != tuple(orig_sizes[0]) for s in orig_sizes):
        raise NotImplementedError("im_detect_bbox_aug batches images of one original size; call it per size group")
    classes = _classes(t, images_by_scale[0].device)
    div = int(cfg.DATALOADER.SIZE_DIVISIBILITY)
    merged = None
    for x, rng in zip(images_by_scale, ranges):
        if not x.is_cuda:
            raise MqdetError("im_detect_bbox_aug: CUDA images required (no CPU fallback)")
        x = x.float().contiguous()
        h, w = x.shape[-2:]
        H, W = (-(-h // div) * div, -(-w // div) * div) if div > 0 else (h, w)
        for flip in ((False, True) if t.FLIP else (False,)):
            if flip:
                batch = ops.hflip_pad(x, (H, W))
            else:
                batch = x.new_zeros((B, x.shape[1], H, W))
                batch[..., :h, :w] = x
            images = ImageList(batch, [(h, w)] * B)
            if gdino:
                out = model.forward_chunked_device(images, [captions], [positive_map], chunks_per_pass=1)
                S = out["det_packed"].shape[2] - 1
            else:
                out = model.forward_device(images, captions, positive_map)
                S = out["cand_scores"].shape[1]
            if merged is None:
                passes = len(scales) * (2 if t.FLIP else 1)
                merged = ops.MergedBoxes(B, min(S * passes, ops.BBOX_AUG_MAX_CAP) if cap is None else cap, x.device)
            if gdino:
                ops.bbox_aug_collect_packed(merged, out["det_packed"][0], (w, h), orig_sizes[0], flip=flip, keep_range=rng)
            else:
                ops.bbox_aug_collect(merged, out["cand_boxes"], out["cand_scores"], out["cand_labels"], out["cand_totals"], (w, h),
                                     orig_sizes[0], flip=flip, keep_range=rng)
    packed = ops.nms_by_class(merged.boxes, merged.scores, merged.labels, merged.count, classes, float(t.TH), mode=mode,
                              top_n=int(t.PRE_NMS_TOP_N), max_out=result_rows(t, merged.cap), overflow=merged.overflow)
    return packed, merged


def im_detect_bbox_aug(model, images_by_scale, orig_sizes, captions, positive_map, cap=None):
    """box_aug.py:12-62 -> list[BoxList] in original-image coordinates.

    images_by_scale: one fp32 CUDA batch [B, 3, h_i, w_i] per entry of ``TEST.SCALES``, already resized
    (``T.Resize(scale, TEST.MAX_SIZE)``) and normalised, not padded — resizing is work of the data pipeline, as in the
    reference; the flipped passes are made here on the device.  orig_sizes: (width, height) per image.  The images of a batch
    share their size in every pass (the restriction of ``forward_device``) and their original size.  ``model``: MQ-GLIP
    (``GeneralizedVLRCNN_New``) or MQ-GroundingDINO (``GroundingDINO``; each image's result is the one it gets alone)."""
    packed, _ = im_detect_bbox_aug_device(model, images_by_scale, orig_sizes, captions, positive_map, cap)
    return unpack(packed, orig_sizes)


def im_detect_bbox_aug_images(model, images_u8, captions, positive_map, cap=None):
    """box_aug.py:12-62 from decoded images, as the reference runs it (im_detect_bbox_scale on the original PIL images):
    images_u8 = uint8 HWC RGB numpy arrays or tensors of one original size -> list[BoxList] in original-image coordinates.
    Each image crosses to the device once; every ``TEST.SCALES`` batch is made from it there by
    ``TestTransform(cfg, scale, TEST.MAX_SIZE)`` (bit-identical to the reference's transform), then merged as
    ``im_detect_bbox_aug``."""
    cfg = model.cfg
    dev = model_device(model)
    images = upload(images_u8, dev)
    batches, orig = [], None
    for scale in cfg.TEST.SCALES:
        il, orig = TestTransform(cfg, scale, cfg.TEST.MAX_SIZE)(images, dev, pad=False)
        batches.append(il.tensors)
    packed, _ = im_detect_bbox_aug_device(model, batches, orig, captions, positive_map, cap)
    return unpack(packed, orig)
