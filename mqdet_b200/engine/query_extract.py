"""Vision-query bank extraction over a dataset on the GPU, for MQ-GLIP and MQ-GroundingDINO: drop-in for the loop of
``tools/train_net.py --extract_query`` (tools/train_net.py:256-336), which tools/extract_vision_query.py runs over a training split
to build the bank every MQ-Det workflow starts from.

The reference's loop calls ``model.extract_query(images, targets, query_images)`` once per test-loader batch (exclude_similar=False,
cap VISION_QUERY.MAX_QUERY_NUMBER): the ground-truth boxes, already resized to the test size by the loader, are grown by EXPAND_RATIO
and clipped (``expand_bbox``), pooled from the detector's own pyramid (7x7 ROIAlignV2 at the FPN level of each box, mean over the
bins) and appended to their label in order until the label holds MAX_QUERY_NUMBER rows.

Here a batch is the device test transform, the backbone-only forward and three launches (``ops.query_gt_rois``,
``ops.roi_align_levels_counted``, ``ops.query_bank_append``) on a device-resident ``ops.QueryBank``; the batch loop reads nothing on
the host, and the row counts cross to the host once at the end.  The bank is dense fp32 [L, MAX_QUERY_NUMBER, C] on the device:
0.4 GB for COCO (81 x 5000 x 256), 1.9 GB for Objects365 (366 x 5000 x 256).

Several ranks (``group``): batch b of the one-GPU batch list goes to rank b mod G.  Every kept box carries its arrival number (its
position in the one-GPU sequence of boxes), each rank caps per label in its own order, which keeps every row the one-GPU cap takes
from that rank, and one ``parallel.all_gather_rows`` of (label, arrival, feature) feeds ``ops.query_bank_merge``: per label the rows
of all ranks in arrival order, the first MAX_QUERY_NUMBER kept.  Every rank returns the one-GPU bank, bit for bit; the reference's
per-rank ``_rank{r}`` files (each capped on its own shard) are deliberately not reproduced.
"""
from collections import defaultdict

import torch
import torch.distributed as dist

from .. import ops, parallel
from .._lib import MqdetError
from .batches import reference_test_batches
from .transforms import TestTransform, model_device


def _is_gdino(model):
    from ..modeling.groundingdino.groundingdino import GroundingDINO
    return isinstance(model, GroundingDINO)


def check_config(cfg):
    """DATASETS.FEW_SHOT, when set, must equal VISION_QUERY.MAX_QUERY_NUMBER (train_net.py:257-258); SELECT_FPN_LEVEL=False
    (the all-level CustomPooler) is off in every MQ config and refused, as the detectors' own ``extract_query`` refuses it."""
    vq = cfg.VISION_QUERY
    few = getattr(getattr(cfg, "DATASETS", None), "FEW_SHOT", 0)
    if few and few != vq.MAX_QUERY_NUMBER:
        raise ValueError(f"DATASETS.FEW_SHOT = {few} but VISION_QUERY.MAX_QUERY_NUMBER = {vq.MAX_QUERY_NUMBER}: to extract the "
                         "right query instances, set VISION_QUERY.MAX_QUERY_NUMBER = DATASETS.FEW_SHOT")
    if not getattr(vq, "SELECT_FPN_LEVEL", True):
        raise NotImplementedError("VISION_QUERY.SELECT_FPN_LEVEL=False (CustomPooler over all levels) is off in every MQ config")
    if int(vq.MAX_QUERY_NUMBER) < 1:
        raise ValueError(f"VISION_QUERY.MAX_QUERY_NUMBER must be >= 1, got {vq.MAX_QUERY_NUMBER}")


def _gt(target, i):
    """A target BoxList (xyxy, a 'labels' field, size = the original (w, h)) -> (boxes fp32 [n, 4], labels int64 [n], (w, h))."""
    if target.mode != "xyxy":
        raise MqdetError(f"target {i}: xyxy boxes required (got {target.mode!r})")
    return target.bbox.detach().cpu().float(), target.get_field("labels").detach().cpu().long(), tuple(int(v) for v in target.size)


def _pyramid(model, tensors):
    """The backbone-only forward of the detector's own ``extract_query`` -> (fp16 pyramid [B, N, C], levels)."""
    if _is_gdino(model):
        _, pyr16, sizes = model.visual_features(tensors)
        return pyr16, ops.get_levels(sizes, tensors.device)
    feats = model.backbone.body.forward_flat(tensors)
    return model.backbone.fpn.forward_flat([feats[i] for i in (1, 2, 3)])


def _bank_dict(rows, count_host):
    """Views of the dense device rows [L, cap, C] in the reference's format: a ``defaultdict(list)`` {label: [n, 1, C]} over the
    labels that have rows, in label order."""
    out = defaultdict(list)
    for k, n in enumerate(count_host.tolist()):
        if n > 0:
            out[k] = rows[k, :n, None, :]
    return out


@torch.no_grad()
def extract_query_bank(model, images_u8, targets, cfg, batches=None, group=None):
    """The vision-query bank of a dataset: ``images_u8`` = decoded uint8 RGB images [h, w, 3] (numpy arrays or tensors), ``targets``
    = their ground truth as BoxLists (xyxy, a 'labels' field, in original-image coordinates: what the dataset yields before the test
    transform), in dataset order.  ``batches``: lists of dataset indices, by default the reference's test loader's
    (``reference_test_batches(sizes, TEST.IMS_PER_BATCH, DATALOADER.ASPECT_RATIO_GROUPING)``); each batch goes through
    ``TestTransform(mixed_sizes=True)``.  ``group``: a process group of several ranks, each passing the whole dataset; rank r runs
    the batches b with b mod G = r, and every rank returns the one-GPU bank.

    Returns the bank the reference's loop of ``model.extract_query`` builds over the same batches, bit for bit, in its format: a
    ``defaultdict(list)`` {label: fp32 [n, 1, C]} of views of one dense device tensor.  ``model.save_query_bank(bank, path)``
    writes it as tools/extract_vision_query.py does; ``model.load_query_bank`` / ``set_query_bank`` read it back."""
    check_config(cfg)
    vq = cfg.VISION_QUERY
    if model.pooler is None:
        raise MqdetError("extract_query_bank needs cfg.MODEL.ROI_BOX_HEAD (POOLER_RESOLUTION / POOLER_SCALES / POOLER_SAMPLING_RATIO)")
    dev = model_device(model)
    if dev.type != "cuda":
        raise MqdetError("extract_query_bank: a CUDA model required (no CPU fallback)")
    images_u8 = list(images_u8)
    if len(targets) != len(images_u8):
        raise ValueError(f"{len(targets)} targets for {len(images_u8)} images")
    gts = [_gt(t, i) for i, t in enumerate(targets)]
    for i, (im, (_, _, (w, h))) in enumerate(zip(images_u8, gts)):
        if (int(im.shape[1]), int(im.shape[0])) != (w, h):
            raise MqdetError(f"target {i} is for a {w}x{h} image but image {i} is {im.shape[1]}x{im.shape[0]}")
    if batches is None:
        batches = reference_test_batches([(h, w) for _, _, (w, h) in gts], cfg.TEST.IMS_PER_BATCH,
                                         cfg.DATALOADER.ASPECT_RATIO_GROUPING)
    batches = [list(b) for b in batches]
    seq = [i for b in batches for i in b]
    if sorted(seq) != list(range(len(seq))) or any(not 0 <= i < len(images_u8) for i in seq):
        raise ValueError("batches must hold every index of a subset of the images once")
    # arrival number of an image's first box: the boxes of the images before it in the one-GPU sequence
    first_box, n = {}, 0
    for i in seq:
        first_box[i] = n
        n += gts[i][0].shape[0]
    if n >= 1 << 31:
        raise MqdetError(f"extract_query_bank: {n} boxes; arrival numbers are int32")
    labels_all = [int(v) for _, lab, _ in gts for v in lab.tolist()]
    if any(v < 0 for v in labels_all):
        raise MqdetError("extract_query_bank: negative labels")
    L = max(labels_all, default=0) + 1
    C = model.hidden_dim if _is_gdino(model) else cfg.MODEL.BACKBONE.OUT_CHANNELS
    K = int(vq.MAX_QUERY_NUMBER)
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank(group) if world > 1 else 0

    qb = ops.QueryBank(L, K, C, dev)
    arrival = torch.zeros((L, K), dtype=torch.int32, device=dev)
    transform, pooler = TestTransform(cfg), model.pooler
    for b in range(rank, len(batches), world):
        idx = batches[b]
        if not idx or sum(gts[i][0].shape[0] for i in idx) == 0:
            continue                                       # no box to pool: the bank cannot change
        il, _ = transform([images_u8[i] for i in idx], dev, mixed_sizes=True)
        pyr16, levels = _pyramid(model, il.tensors)
        if levels.n != len(pooler.scales):
            raise MqdetError(f"pooler has {len(pooler.scales)} scales but the pyramid has {levels.n} levels")
        rois, labels, arr, count = ops.query_gt_rois(
            [(gts[i][0], gts[i][1], gts[i][2], (rw, rh), first_box[i]) for i, (rh, rw) in zip(idx, il.image_sizes)], vq.EXPAND_RATIO, dev)
        feats = ops.roi_align_levels_counted(pyr16, levels, pooler.scales, rois, count, pooler.output_size[0], pooler.sampling_ratio)
        ops.query_bank_append(qb, feats, labels, arr, count, K, arrival)

    count_host = qb.count.cpu()                            # the one device->host copy of a single rank
    if world == 1:
        return _bank_dict(qb.rows, count_host)
    # several ranks: this rank's rows, label-major and in arrival order within a label, as (label bits, arrival bits, feature)
    keep = torch.tensor([l * K + j for l, c in enumerate(count_host.tolist()) for j in range(c)], dtype=torch.int64)
    lab = torch.tensor([l for l, c in enumerate(count_host.tolist()) for _ in range(c)], dtype=torch.int32)
    keep_d, lab_d = ops.upload_async(keep, dev), ops.upload_async(lab, dev)
    rows = torch.cat([lab_d[:, None].view(torch.float32), arrival.view(-1).index_select(0, keep_d)[:, None].view(torch.float32),
                      qb.rows.view(L * K, C).index_select(0, keep_d)], 1)
    head = torch.cat([torch.tensor([rows.shape[0]], dtype=torch.int64), count_host.to(torch.int64)]).to(dev)
    parts, heads = parallel.all_gather_rows(rows, head, group)
    counts = torch.stack(heads).cpu()[:, 1:]
    merged, count_all = ops.query_bank_merge([p.contiguous() for p in parts], counts, K, C)
    return _bank_dict(merged, count_all)
