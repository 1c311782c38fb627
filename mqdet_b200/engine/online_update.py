"""MQ-Det's test-time vision-query update (``VISION_QUERY.NUM_TURNS``), drop-in for ``online_update``
(maskrcnn_benchmark/engine/inference.py:383-497), which tools/test_grounding_net.py:184-187 runs before the evaluation when
``VISION_QUERY.OFFLINE_WITH_ONLINE`` is set (the finetuning-free ODinW protocol, configs/vision_query_5shot/odinw.yaml).

Per turn the detector runs over the test set with the bank it loaded at the start of the turn; every detection scoring above
``SCORE_THRESHOLD`` is grown by ``EXPAND_RATIO``, clipped, pooled from the detector's own pyramid and appended to the bank unless its
label already has ``MAX_TEST_QUERY_NUMBER`` rows or a row of that label is more similar than ``SIMILARITY_THRESHOLD``.  The bank grows
across turns; it is installed in the model at the start of every turn after the first.

Here a batch of images goes through three launches after its forward (``ops.query_candidates``, ``ops.roi_align_levels_counted``,
``ops.query_bank_update``) on a device-resident ``ops.QueryBank``; nothing is read on the host inside a turn, and one device->host
copy (the row counts) ends it.  The exception is the detector's prompt state (selected vision queries, token tables), which depends on
the bank: the first batch after a bank is installed rebuilds it on the host, and so does a batch whose size differs from the one
before (the prompt state and the GCP index table are cached for one batch size).  The bank only depends on the order of the images, so batches of consecutive images of one size give
what the reference's one-image loop gives.

Quirk kept from the reference: ``online_update`` installs the bank of turn t - 1 at the start of turn t and the evaluation that follows
does not reload it, so the evaluation uses the bank as it was after turn NUM_TURNS - 1 (with one turn, the bank the model had before).
``online_update`` leaves the model in that state and returns that bank as ``eval_bank``, next to the bank after every turn.
"""
import os

import torch

from .. import ops
from .._lib import MqdetError
from ..structures.image_list import to_image_list


def check_config(cfg):
    """The paths the reference cannot run raise ``NotImplementedError`` naming the key."""
    if getattr(cfg.TEST, "USE_MULTISCALE", False):
        raise NotImplementedError("VISION_QUERY.NUM_TURNS with TEST.USE_MULTISCALE: the reference's online_update raises "
                                  "NotImplementedError for multi-scale test-time augmentation")
    task = getattr(cfg.TEST, "EVAL_TASK", "detection")
    if task != "detection":
        raise NotImplementedError(f"VISION_QUERY.NUM_TURNS with TEST.EVAL_TASK={task!r}: the reference's online_update implements "
                                  "the detection task only")
    if not getattr(cfg.VISION_QUERY, "SELECT_FPN_LEVEL", True):
        raise NotImplementedError("VISION_QUERY.NUM_TURNS with VISION_QUERY.SELECT_FPN_LEVEL=False: the reference's "
                                  "extract_query(exclude_similar=True) asserts one pooled scale per query")
    tests = getattr(getattr(cfg, "DATASETS", None), "TEST", ()) or ()
    if any("lvis" in str(t) for t in tests):
        raise NotImplementedError("VISION_QUERY.NUM_TURNS on an LVIS DATASETS.TEST: the reference's LVIS branch of online_update "
                                  "reads no detections (IndexError)")


def make_batches(images, max_batch, size_divisible=32):
    """Consecutive images (fp32 [3, h, w] device tensors, normalised) -> ImageLists of at most ``max_batch`` images of one size, in
    order; a new batch starts when the size changes."""
    if max_batch < 1:
        raise ValueError(f"max_batch must be >= 1, got {max_batch}")
    out, cur = [], []
    for im in images:
        if cur and (len(cur) == max_batch or tuple(cur[0].shape[-2:]) != tuple(im.shape[-2:])):
            out.append(to_image_list(cur, size_divisible))
            cur = []
        cur.append(im)
    if cur:
        out.append(to_image_list(cur, size_divisible))
    return out


def _is_gdino(model):
    from ..modeling.groundingdino.groundingdino import GroundingDINO
    return isinstance(model, GroundingDINO)


def _detect(model, images, captions, positive_map):
    """One forward -> (packed rows [B, M + 1, 6], fp16 pyramid [B, N, C], levels, (w, h)).  MQ-GroundingDINO runs the chunked path
    with the prompt as its only chunk: it takes the fusion softmax maximum per image, as the reference's one-image forward does."""
    if _is_gdino(model):
        out = model.forward_chunked_device(images, [captions], [positive_map])
        packed = out["det_packed"][0]
    else:
        out = model.forward_device(images, captions, positive_map)
        packed = out["det_packed"]
    sizes = out["image_sizes"]
    h, w = sizes[0]
    if any(tuple(s) != (h, w) for s in sizes):
        raise MqdetError("online_update: every batch holds images of one size (see make_batches)")
    return packed, out["pyramid16"], out["levels"], (int(w), int(h))


def update_turn(model, batches, captions, positive_map, bank, cfg, bad):
    """One turn over ``batches`` with the model's current bank: forward, candidates, pooling and bank update per batch, all on the
    device.  ``bad`` (int32 [1], device) counts the images whose count row was malformed.  Reads nothing on the host."""
    vq, pooler = cfg.VISION_QUERY, model.pooler
    for images in batches:
        images = to_image_list(images, cfg.DATALOADER.SIZE_DIVISIBILITY)
        packed, pyr16, levels, wh = _detect(model, images, captions, positive_map)
        if levels.n != len(pooler.scales):
            raise MqdetError(f"pooler has {len(pooler.scales)} scales but the pyramid has {levels.n} levels")
        rois, labels, count = ops.query_candidates(packed, wh, vq.SCORE_THRESHOLD, vq.EXPAND_RATIO, bad)
        feats = ops.roi_align_levels_counted(pyr16, levels, pooler.scales, rois, count, pooler.output_size[0], pooler.sampling_ratio)
        ops.query_bank_update(bank, feats, labels, count, vq.MAX_TEST_QUERY_NUMBER, vq.SIMILARITY_THRESHOLD)
    return bank


@torch.no_grad()
def online_update(model, batches, captions, positive_map, cfg, bank=None):
    """Run ``VISION_QUERY.NUM_TURNS`` turns of the test-time update over ``batches`` (ImageLists of consecutive images of one size, in
    dataset order; see ``make_batches``) with one prompt (``captions``, ``positive_map``: the detection prompt of the dataset).

    ``bank``: the starting bank {label: [n, 1, C]}; by default ``torch.load(VISION_QUERY.QUERY_BANK_PATH)`` when that file exists,
    else empty.  Returns {"banks": the bank after every turn, "eval_bank": the bank the evaluation that follows uses (the model's
    bank on return)}, each in the reference's format (a ``defaultdict(list)`` of device tensors [n, 1, C]; ``save_query_bank``
    writes it to disk)."""
    check_config(cfg)
    vq = cfg.VISION_QUERY
    if model.query_selector is None:
        raise MqdetError("online_update needs VISION_QUERY.ENABLED (a query selector)")
    if model.pooler is None:
        raise MqdetError("online_update needs cfg.MODEL.ROI_BOX_HEAD (POOLER_RESOLUTION / POOLER_SCALES / POOLER_SAMPLING_RATIO)")
    batches = list(batches)
    if not batches:
        raise ValueError("online_update: no images")
    dev = to_image_list(batches[0]).tensors.device
    if bank is None and vq.QUERY_BANK_PATH and os.path.exists(vq.QUERY_BANK_PATH):
        # the reference pickles its banks as defaultdict(list), which the weights-only unpickler refuses; the file is the user's
        # own query bank, read as the reference reads it
        bank = torch.load(vq.QUERY_BANK_PATH, map_location=dev, weights_only=False)
    labels = [int(k) for k in positive_map] + [int(k) for k in (bank or {})]
    C = cfg.MODEL.BACKBONE.OUT_CHANNELS if not _is_gdino(model) else model.hidden_dim
    qb = ops.QueryBank.from_dict(bank, max(labels) + 1, vq.MAX_TEST_QUERY_NUMBER, C, dev)
    bad = torch.zeros((1,), dtype=torch.int32, device=dev)
    banks = []
    for turn in range(int(vq.NUM_TURNS)):
        if turn > 0:
            model.set_query_bank(banks[-1])    # fixed for the whole turn; only the device bank grows
        update_turn(model, batches, captions, positive_map, qb, cfg, bad)
        host = torch.cat([qb.count, bad]).cpu()    # the one device->host copy of the turn
        if int(host[-1]):
            raise MqdetError(f"online_update: {int(host[-1])} detector result(s) had a count row that is not an integer in [0, rows]")
        banks.append(qb.as_dict(host[:-1]))
    return {"banks": banks, "eval_bank": model.query_selector.query_bank}
