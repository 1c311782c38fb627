"""Restatement of vision-only evaluation (VISION_QUERY.MASK_DURING_INFERENCE, generalized_vl_rcnn_new.py:397-407) that the GPU
tests compare against: per element (one reference forward of one image), one ``random.random()`` per category row of the
positive map in prompt order, drawn for every category; the tokens of a category whose draw is below TEXT_DROPOUT and that
has vision queries become the mask token.  Pinned to the reference's own code by tests/test_vision_only_cpu.py."""
import random

import torch

MASK_TOKEN_ID = 103


def token_rows(positive_map, T):
    """Labels with at least one token, in the positive map's order, and their token positions as bool rows [C, T]."""
    labels = [k for k, v in positive_map.items() if len(v) != 0]
    rows = torch.zeros((len(labels), T), dtype=torch.bool)
    for j, label in enumerate(labels):
        rows[j, positive_map[label]] = True
    return labels, rows


def has_query(labels, bank, k):
    """QuerySelector's per-category flag at inference: 1 when the category gets at least one of its bank rows."""
    return [int(not isinstance(bank[l], list) and min(len(bank[l]), k) > 0) for l in labels]


def draw(has, rate):
    """One forward's draws: a flag per category, 1 = mask its tokens."""
    return [int(random.random() < rate and h == 1) for h in has]


def apply(ids, rows, flags, mask_id=MASK_TOKEN_ID):
    """ids [T] with the rows of the flagged categories set to mask_id (a new tensor)."""
    out = ids.clone()
    for j, f in enumerate(flags):
        if f:
            out[rows[j]] = mask_id
    return out


def forward_ids(ids, positive_map, has, rate, n_images, mask_id=MASK_TOKEN_ID):
    """The ids of ``n_images`` consecutive one-image forwards over one prompt (ids [T]) -> [n_images, T]."""
    _, rows = token_rows(positive_map, ids.shape[-1])
    return torch.stack([apply(ids, rows, draw(has, rate), mask_id) for _ in range(n_images)])


def chunked_ids(chunks, has, rate, n_images, mask_id=MASK_TOKEN_ID):
    """chunks: [(ids [T], positive_map)], has: per chunk -> [n_chunks, n_images, T], drawn in the reference's loop order
    (engine/inference.py:600-625: images outer, chunks inner)."""
    T = chunks[0][0].shape[-1]
    rows = [token_rows(pm, T)[1] for _, pm in chunks]
    out = torch.empty((len(chunks), n_images, T), dtype=torch.long)
    for b in range(n_images):
        for c, (ids, _) in enumerate(chunks):
            out[c, b] = apply(ids, rows[c], draw(has[c], rate), mask_id)
    return out


def kernel(ids, tok_cat, flags, mask_id):
    """mqdet_mask_prompt_tokens as include/mqdet_b200.h specifies it: ids i64 [E, T], tok_cat i32 [E, T], flags u8 [E, C]."""
    C = flags.shape[1]
    c = tok_cat.long()
    ok = (c >= 0) & (c < C)
    hit = torch.zeros_like(ok)
    if C:
        hit[ok] = flags.gather(1, c.clamp(0, C - 1))[ok] != 0
    return torch.where(hit, torch.full_like(ids, mask_id), ids)
