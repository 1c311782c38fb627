"""Restatement of MQ-Det's test-time vision-query update (maskrcnn_benchmark/engine/inference.py:383-497 with extract_query
(exclude_similar=True), generalized_vl_rcnn_new.py:32-49 and :231-288) on the CPU, one image at a time, in the reference's own tensor
operations.  tests/test_online_update_cpu.py pins it to the reference; the GPU tests compare the kernels and the engine against it.

The detector and the pooler are parameters: ``detect(image, bank) -> packed rows [M + 1, 6]`` (the bank the model holds during the
turn) and ``pool(image, boxes [R, 4]) -> features [R, C]``.
"""
from collections import defaultdict

import torch
import torch.nn.functional as F

BAD_COUNT = -1


def candidates(packed, wh, score_thr, expand_ratio):
    """One image's packed rows [M + 1, 6] -> (boxes [R, 4], labels [R] int64), or BAD_COUNT for a count row that is not an integer in
    [0, M]: score filter (strict), expand_bbox, clip_to_image(remove_empty=True)."""
    M = packed.shape[0] - 1
    c = float(packed[M, 0])
    if not (0 <= c <= M and c == int(c)):
        return BAD_COUNT
    rows = packed[:int(c)]
    rows = rows[rows[:, 4] > score_thr]
    bbox = rows[:, :4]
    box_w, box_h = bbox[:, 2] - bbox[:, 0], bbox[:, 3] - bbox[:, 1]
    diff_w = (box_w * expand_ratio - box_w) / 2
    diff_h = (box_h * expand_ratio - box_h) / 2
    b = bbox + torch.stack([-diff_w, -diff_h, diff_w, diff_h], dim=1)
    w, h = wh
    b = torch.stack((b[:, 0].clamp(min=0, max=w - 1), b[:, 1].clamp(min=0, max=h - 1), b[:, 2].clamp(min=0, max=w - 1),
                     b[:, 3].clamp(min=0, max=h - 1)), dim=-1)
    keep = (b[:, 3] > b[:, 1]) & (b[:, 2] > b[:, 0])
    return b[keep], rows[keep, 5].long()


def bank_update(bank, labels, feats, max_query, sim_thr):
    """extract_query's loop (:268-288) with exclude_similar: ``bank`` {label: [n, 1, C]} (a defaultdict(list)), features [R, C] in
    order.  Returns the smallest |similarity - sim_thr| met (inf when no test ran)."""
    margin = float("inf")
    for label, feat in zip(labels.tolist(), feats[:, None, :]):
        n = len(bank[label])
        if n >= max_query:
            continue
        if n > 0:
            sim = torch.einsum("b n d, n d -> b n", F.normalize(bank[label], p=2, dim=-1), F.normalize(feat, p=2, dim=-1))
            margin = min(margin, float((sim - sim_thr).abs().min()))
            if (sim > sim_thr).sum() > 0:
                continue
        bank[label] = feat[None] if n == 0 else torch.cat([bank[label], feat[None]])
    return margin


def copy_bank(bank):
    out = defaultdict(list)
    for k, v in (bank or {}).items():
        out[int(k)] = v.clone() if torch.is_tensor(v) else list(v)
    return out


def online_update(detect, pool, images, sizes, start_bank, model_bank, num_turns, score_thr=0.6, expand_ratio=1.5, max_query=100,
                  sim_thr=0.85):
    """``images``: image keys in dataset order, ``sizes`` their (w, h); ``start_bank``: torch.load(QUERY_BANK_PATH) or None;
    ``model_bank``: the bank the model holds before the update.  -> (bank after every turn, the bank the evaluation uses, the smallest
    similarity margin met)."""
    bank = copy_bank(start_bank)
    held = model_bank
    banks, margin = [], float("inf")
    for turn in range(num_turns):
        if turn > 0:
            held = copy_bank(banks[-1])
        for im, wh in zip(images, sizes):
            c = candidates(detect(im, held), wh, score_thr, expand_ratio)
            if c is BAD_COUNT:
                raise ValueError(f"image {im}: bad count row")
            boxes, labels = c
            if boxes.shape[0]:
                margin = min(margin, bank_update(bank, labels, pool(im, boxes), max_query, sim_thr))
        banks.append(copy_bank(bank))
    return banks, held, margin
