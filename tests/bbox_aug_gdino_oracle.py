"""Plain torch restatement of what box_aug.py does with one MQ-GroundingDINO pass, from the packed detector rows
(x1, y1, x2, y2, score, label; row M = (count, ...)) that ``gdino_detections`` writes: BoxList.transpose for a flipped pass,
remove_boxes, BoxList.resize to the original image, appended behind the earlier passes.  Pinned to the reference's own
box_aug.py and BoxList by tests/test_bbox_aug_gdino_cpu.py and used as the expected result by tests/test_bbox_aug_gdino_gpu.py.
The per-box arithmetic is tests/bbox_aug_oracle.py's (``collect_pass``); what is restated here is how the packed rows feed it.
"""
import torch

import bbox_aug_oracle as bo

BAD_COUNT = 1 << 30    # ops.BBOX_AUG_BAD_COUNT


def rows_of(packed_b):
    """One image's packed rows [M + 1, 6] -> (boxes, scores, labels) of its first `count` rows, or None for a count that is not
    an integer in [0, M]."""
    M = packed_b.shape[0] - 1
    c = float(packed_b[M, 0])
    if not (0 <= c <= M and c == int(c)):
        return None
    n = int(c)
    return packed_b[:n, :4].clone(), packed_b[:n, 4].clone(), packed_b[:n, 5].long()


def collect_packed(merged, packed, pass_size, orig_size, flip=False, keep_range=None):
    """Append one pass (packed [B, M + 1, 6]) to ``merged`` = per image dict(boxes, scores, labels, overflow) with room for
    ``merged[b]["cap"]`` rows: the restatement of ops.bbox_aug_collect_packed."""
    for b, m in enumerate(merged):
        r = rows_of(packed[b])
        if r is None:
            m["overflow"] |= BAD_COUNT
            continue
        bx, sc, lb = bo.collect_pass(*r, pass_size, orig_size, flip, keep_range)
        k = min(bx.shape[0], m["cap"] - m["boxes"].shape[0])
        m["boxes"] = torch.cat([m["boxes"], bx[:k]])
        m["scores"] = torch.cat([m["scores"], sc[:k]])
        m["labels"] = torch.cat([m["labels"], lb[:k]])
        m["overflow"] += bx.shape[0] - k
    return merged


def empty_merged(B, cap):
    return [dict(boxes=torch.zeros(0, 4), scores=torch.zeros(0), labels=torch.zeros(0, dtype=torch.long), overflow=0, cap=cap)
            for _ in range(B)]


def pack(boxes, scores, labels, M):
    """(boxes, scores, labels) of one image -> packed [M + 1, 6] with the count row (rows past the count hold noise)."""
    n = boxes.shape[0]
    out = torch.full((M + 1, 6), 3.0)
    out[:n, :4], out[:n, 4], out[:n, 5] = boxes, scores, labels.float()
    out[M] = 0.0
    out[M, 0] = n
    return out


def gdino_rows(g, n, size, n_labels, box_threshold=0.05):
    """GroundingDINO-shaped output of one pass: n rows in query order (no NMS: overlapping copies of a few objects), scores above
    box_threshold, boxes from cxcywh in [0, 1] to pixels, clipped to [0, W - 1] x [0, H - 1] (many touch the border)."""
    W, H = size
    cxcy = torch.rand(n, 2, generator=g) * 1.2 - 0.1
    wh = torch.rand(n, 2, generator=g) * 0.5 + 0.01
    b = torch.cat([cxcy - wh / 2, cxcy + wh / 2], 1) * torch.tensor([W, H, W, H], dtype=torch.float32)
    b[:, 0::2] = b[:, 0::2].clamp(0, W - 1)
    b[:, 1::2] = b[:, 1::2].clamp(0, H - 1)
    s = box_threshold + (1 - box_threshold) * torch.rand(n, generator=g) ** 3
    lab = torch.randint(1, n_labels + 1, (n,), generator=g)
    return b.float(), s.float(), lab


def pin_cases():
    """name -> dict(orig_size, M, passes = [(pass_size, flip, keep_range, boxes, scores, labels)], test = TEST namespace)"""
    from types import SimpleNamespace as NS
    g = torch.Generator().manual_seed(4321)

    def test(**kw):
        d = dict(SPECIAL_NMS="none", TH=0.6, PRE_NMS_TOP_N=1000, NUM_CLASSES=14, SELECT_CLASSES=(), FLIP=True, SCALES=(), RANGES=())
        d.update(kw)
        return NS(**d)

    cases = {}
    # two scales + flip of a 640 x 480 image, 900 queries in every pass; the 900-row pass fills its buffer exactly
    sizes = [(533, 400), (533, 400), (800, 600), (800, 600)]
    counts = [900, 640, 0, 357]
    p = []
    for (w, h), flip, n, rng in zip(sizes, (False, True, False, True), counts, ((32, 400), (32, 400), None, None)):
        b, s, lab = gdino_rows(g, n, (w, h), 13)
        if n:  # a box of area exactly lo^2 = 32 x 32 (dropped) and one just above (kept)
            b[0] = torch.tensor([10., 10., 41., 41.])
            b[1] = torch.tensor([10., 10., 42., 41.])
        p.append(((w, h), flip, rng, b, s, lab))
    cases["two_scales_flip_nms"] = dict(orig_size=(640, 480), M=900, passes=p, test=test())
    cases["two_scales_flip_vote"] = dict(orig_size=(640, 480), M=900, passes=p, test=test(SPECIAL_NMS="vote"))
    cases["two_scales_flip_th0"] = dict(orig_size=(640, 480), M=900, passes=p, test=test(TH=0.0, PRE_NMS_TOP_N=0))
    # unequal width / height ratios, a pass with a single row, an empty flipped pass
    q = []
    for (w, h), flip, n in (((500, 374), False, 1), ((500, 374), True, 0), ((1000, 749), False, 300), ((1000, 749), True, 299)):
        b, s, lab = gdino_rows(g, n, (w, h), 13)
        q.append(((w, h), flip, (0, 10000) if w == 500 else (0, 256), b, s, lab))
    cases["unequal_ratios_nms"] = dict(orig_size=(667, 500), M=300, passes=q, test=test(PRE_NMS_TOP_N=100))
    cases["unequal_ratios_vote"] = dict(orig_size=(667, 500), M=300, passes=q, test=test(SPECIAL_NMS="vote", PRE_NMS_TOP_N=100))
    e = torch.zeros(0, 4), torch.zeros(0), torch.zeros(0, dtype=torch.long)
    cases["all_empty"] = dict(orig_size=(640, 480), M=900, passes=[((800, 600), False, None, *e), ((800, 600), True, None, *e)],
                              test=test())
    return cases


def run_case(c):
    """-> dict(union = merged candidates (boxes, scores, labels), result = (boxes, scores, labels)), the passes going through
    their packed form."""
    M = c["M"]
    merged = empty_merged(1, M * len(c["passes"]))
    for size, flip, rng, b, s, lab in c["passes"]:
        collect_packed(merged, pack(b, s, lab, M)[None], size, c["orig_size"], flip, rng)
    m = merged[0]
    assert m["overflow"] == 0
    mode = "vote" if c["test"].SPECIAL_NMS == "vote" else "nms"
    res = bo.merge(m["boxes"], m["scores"], m["labels"], bo.class_list(c["test"]), c["test"].TH, mode, c["test"].PRE_NMS_TOP_N)
    return {"union": (m["boxes"], m["scores"], m["labels"]), "result": res}
