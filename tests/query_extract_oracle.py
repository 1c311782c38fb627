"""Restatement of the vision-query bank extraction loop (tools/train_net.py:256-336 over GeneralizedVLRCNN_New.extract_query,
generalized_vl_rcnn_new.py:231-288, exclude_similar=False) on the host, in fp32 torch ops, and of its several-rank form.

* ``resize_boxes``: the test loader's BoxList.resize to the Resize(MIN_SIZE_TEST, MAX_SIZE_TEST) size;
* ``expand_clip``: expand_bbox (generalized_vl_rcnn_new.py:32-49) with clip_to_image(remove_empty=True);
* ``extract``: batches in order, images in batch order, kept boxes in target order, appended to their label until it holds
  ``max_query`` rows (no similarity test);
* ``extract_ranks``: batch b on rank b mod G, each rank capped per label in its own order, then per label all ranks' rows in
  arrival order (the box's position in the one-GPU sequence of boxes), the first ``max_query`` kept.

tests/test_query_extract_cpu.py pins it to the reference's own code; the GPU tests compare the kernels and the engine with it.
"""
from collections import defaultdict

import torch


def resize_boxes(boxes, orig_wh, new_wh):
    """BoxList.resize: ratios new / orig in double, rounded to fp32, one fp32 multiply per coordinate."""
    rx, ry = float(new_wh[0]) / float(orig_wh[0]), float(new_wh[1]) / float(orig_wh[1])
    r = torch.tensor([rx, ry, rx, ry], dtype=torch.float64).float()
    return boxes.float() * r


def expand_clip(boxes, wh, ratio):
    """expand_bbox + clip_to_image(remove_empty=True) -> (boxes [k, 4], keep mask [n])."""
    b = boxes.float()
    bw, bh = b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]
    dw, dh = (bw * ratio - bw) / 2, (bh * ratio - bh) / 2
    nb = b + torch.stack([-dw, -dh, dw, dh], dim=1)
    w, h = wh
    nb[:, 0].clamp_(min=0, max=w - 1)
    nb[:, 1].clamp_(min=0, max=h - 1)
    nb[:, 2].clamp_(min=0, max=w - 1)
    nb[:, 3].clamp_(min=0, max=h - 1)
    keep = (nb[:, 3] > nb[:, 1]) & (nb[:, 2] > nb[:, 0])
    return nb[keep], keep


def batch_rois(gts, idx, resized_wh, ratio, first_box):
    """The kept rows of one batch in image-then-box order: (rois [k, 5] = (image index in the batch, box), labels [k], arrival [k])."""
    rois, labels, arrival = [], [], []
    for j, (i, wh) in enumerate(zip(idx, resized_wh)):
        boxes, lab, owh = gts[i]
        nb, keep = expand_clip(resize_boxes(boxes, owh, wh), wh, ratio)
        rois.append(torch.cat([torch.full((nb.shape[0], 1), float(j)), nb], 1))
        labels.append(lab[keep].long())
        arrival.append(first_box[i] + torch.nonzero(keep).flatten())
    return torch.cat(rois), torch.cat(labels), torch.cat(arrival)


def first_boxes(gts, batches):
    """Image -> arrival number of its first box: the boxes of the images before it in the one-GPU sequence."""
    out, n = {}, 0
    for b in batches:
        for i in b:
            out[i] = n
            n += gts[i][0].shape[0]
    return out


def cap_append(bank, labels, feats, max_query, arrivals=None, bank_arrival=None):
    """extract_query's append with exclude_similar=False: each feature to its label unless the label holds ``max_query`` rows."""
    for j, (label, feat) in enumerate(zip(labels.tolist(), feats)):
        n = len(bank[label])
        if n >= max_query:
            continue
        bank[label] = feat[None, None] if n == 0 else torch.cat([bank[label], feat[None, None]])
        if bank_arrival is not None:
            bank_arrival[label].append(int(arrivals[j]))
    return bank


def extract(gts, batches, resized_wh, pool, max_query, ratio=1.5, ranks=None):
    """The bank of the loop: ``gts`` = per image (boxes [n, 4] original coordinates, labels [n], (w, h)); ``resized_wh`` = per image
    its test size (w, h); ``pool(i, boxes)`` -> features [k, C] of image i's expanded boxes.  With ``ranks`` = (r, G) only the
    batches b with b mod G = r, and the arrival numbers of the rows as well."""
    first = first_boxes(gts, batches)
    bank, arr = defaultdict(list), defaultdict(list)
    for b, idx in enumerate(batches):
        if ranks is not None and b % ranks[1] != ranks[0]:
            continue
        rois, labels, arrival = batch_rois(gts, idx, [resized_wh[i] for i in idx], ratio, first)
        feats = torch.cat([pool(i, rois[rois[:, 0] == j, 1:]) for j, i in enumerate(idx)]) if rois.shape[0] else torch.zeros(0, 1)
        cap_append(bank, labels, feats, max_query, arrival, arr)
    return (bank, arr) if ranks is not None else bank


def merge(rank_banks, max_query):
    """[(bank, arrivals)] of every rank -> per label the rows of all ranks in arrival order, the first ``max_query``."""
    out = defaultdict(list)
    labels = sorted({k for bank, _ in rank_banks for k, v in bank.items() if len(v)})
    for k in labels:
        rows = [(a, bank[k][j]) for bank, arr in rank_banks if len(bank[k]) for j, a in enumerate(arr[k])]
        rows.sort(key=lambda t: t[0])
        out[k] = torch.stack([r for _, r in rows[:max_query]])
    return out


def extract_ranks(gts, batches, resized_wh, pool, max_query, G, ratio=1.5):
    return merge([extract(gts, batches, resized_wh, pool, max_query, ratio, ranks=(r, G)) for r in range(G)], max_query)


def same_bank(a, b):
    ka = sorted(int(k) for k, v in a.items() if len(v))
    kb = sorted(int(k) for k, v in b.items() if len(v))
    return ka == kb and all(torch.equal(a[k].cpu(), b[k].cpu()) for k in ka)
