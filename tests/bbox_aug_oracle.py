"""Plain torch / numpy restatement of the multi-scale + flip test-time augmentation of
maskrcnn_benchmark/data/datasets/evaluation/box_aug.py, pinned to the reference's own code by tests/test_bbox_aug_cpu.py and
used as the expected result by tests/test_bbox_aug_gpu.py.

All box arithmetic is fp32 with every operation rounded (numpy / torch on the CPU never contract a multiply-add).
Rules the reference leaves open, fixed here and in DESIGN.md section 4:
  * equal scores inside a class are ordered by ascending index in the merged list (a stable descending sort);
  * suppression uses IoU > TH (csrc/cuda/nms.cu:62), voting uses IoU >= TH (bbox_vote's numpy code).
"""
import numpy as np
import torch

ONE = np.float32(1.0)


def flip_boxes(boxes, pass_w):
    """BoxList.transpose(FLIP_LEFT_RIGHT): x1' = W - x2 - 1, x2' = W - x1 - 1 (TO_REMOVE = 1)."""
    out = boxes.clone()
    out[:, 0] = pass_w - boxes[:, 2] - 1
    out[:, 2] = pass_w - boxes[:, 0] - 1
    return out


def range_keep(boxes, lo, hi):
    """remove_boxes (box_aug.py:150-163): lo^2 < w * h < hi^2, both strict, on fp32 w = x2 - x1 + 1, h = y2 - y1 + 1."""
    w = boxes[:, 2] - boxes[:, 0] + 1
    h = boxes[:, 3] - boxes[:, 1] + 1
    a = w * h
    return (a > torch.tensor(lo * lo, dtype=torch.float32)) & (a < torch.tensor(hi * hi, dtype=torch.float32))


def resize_boxes(boxes, pass_size, orig_size):
    """BoxList.resize: ratios in double, the product an fp32 multiply by the ratio rounded to fp32."""
    rx, ry = float(orig_size[0]) / float(pass_size[0]), float(orig_size[1]) / float(pass_size[1])
    r = torch.tensor([rx, ry, rx, ry], dtype=torch.float64).float()
    return boxes * r


def collect_pass(boxes, scores, labels, pass_size, orig_size, flip=False, keep_range=None):
    """One pass's candidates (pass coordinates) -> what im_detect_bbox_aug appends for it: un-flip, range filter, resize."""
    boxes = boxes.float()
    if flip:
        boxes = flip_boxes(boxes, pass_size[0])
    if keep_range is not None:
        k = range_keep(boxes, *keep_range)
        boxes, scores, labels = boxes[k], scores[k], labels[k]
    return resize_boxes(boxes, pass_size, orig_size), scores, labels


def _iou_one(b, i, js):
    """IoU of box i with boxes js, the +1 convention of nms.cu:15-23 (bbox_vote's numpy lines compute the same expression)."""
    area = (b[:, 2] - b[:, 0] + ONE) * (b[:, 3] - b[:, 1] + ONE)
    left = np.maximum(b[i, 0], b[js, 0]); right = np.minimum(b[i, 2], b[js, 2])
    top = np.maximum(b[i, 1], b[js, 1]); bottom = np.minimum(b[i, 3], b[js, 3])
    w = np.maximum(right - left + ONE, np.float32(0)); h = np.maximum(bottom - top + ONE, np.float32(0))
    inter = w * h
    return inter / (area[i] + area[js] - inter)


def score_order(scores):
    """descending, equal scores by ascending index"""
    return np.argsort(-scores.astype(np.float64), kind="stable")


def nms_class(boxes, scores, th):
    """nms_cuda on one class: kept indices, ascending (nms.cu:139-142)."""
    n = boxes.shape[0]
    order = score_order(scores)
    b = boxes[order]
    removed = np.zeros(n, dtype=bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        if i + 1 < n:
            js = np.arange(i + 1, n)
            removed[js[_iou_one(b, i, js) > np.float32(th)]] = True
    return np.sort(order[np.asarray(keep, dtype=np.int64)])


def vote_class(boxes, scores, th):
    """bbox_vote (box_aug.py:241-287) on one class with more than one box -> (boxes [k,4], scores [k], members): clusters in
    creation order; `members[c]` = the cluster's indices into the class in score order (head first).  Sums run in that order
    in fp32."""
    n = boxes.shape[0]
    order = score_order(scores)
    b, s = boxes[order], scores[order]
    taken = np.zeros(n, dtype=bool)
    ob, os_, members = [], [], []
    for i in range(n):
        if taken[i]:
            continue
        js = np.arange(i, n)
        m = js[(~taken[js]) & (_iou_one(b, i, js) >= np.float32(th))]
        taken[m] = True
        members.append(order[m])
        if m.size <= 1:
            ob.append(b[i]); os_.append(s[i])
            continue
        prod = (b[m] * s[m, None]).astype(np.float32)
        num = np.cumsum(prod, axis=0, dtype=np.float32)[-1]
        den = np.cumsum(s[m], dtype=np.float32)[-1]
        ob.append((num / den).astype(np.float32)); os_.append(s[m].max())
    return np.stack(ob).astype(np.float32), np.asarray(os_, dtype=np.float32), members


def merge(boxes, scores, labels, classes, th, mode="nms", top_n=1000, want_members=False):
    """merge_result_from_multi_scales for one image: tensors in, (boxes, scores, labels) tensors out."""
    b = boxes.detach().cpu().numpy().astype(np.float32).reshape(-1, 4)
    s = scores.detach().cpu().numpy().astype(np.float32)
    lab = labels.detach().cpu().numpy().astype(np.int64)
    ob, os_, ol, om = [], [], [], []
    for c in classes:
        idx = np.nonzero(lab == c)[0]
        if idx.size == 0:
            continue
        if th <= 0 or (mode == "vote" and idx.size <= 1):
            cb, cs, mem = b[idx], s[idx], [idx[i:i + 1] for i in range(idx.size)]
        elif mode == "vote":
            cb, cs, mem = vote_class(b[idx], s[idx], th)
            mem = [idx[m] for m in mem]
        else:
            k = idx[nms_class(b[idx], s[idx], th)]
            cb, cs, mem = b[k], s[k], [k[i:i + 1] for i in range(k.size)]
        ob.append(cb); os_.append(cs); ol.append(np.full(cs.shape[0], c, dtype=np.int64)); om.extend(mem)
    if not ob:
        out = (torch.zeros(0, 4), torch.zeros(0), torch.zeros(0, dtype=torch.long))
        return out + ([],) if want_members else out
    ob, os_, ol = np.concatenate(ob), np.concatenate(os_), np.concatenate(ol)
    n = os_.shape[0]
    if n > top_n > 0:
        thr = np.sort(os_)[n - top_n]          # kthvalue(n - top_n + 1): the top_n-th largest
        k = os_ >= thr
        ob, os_, ol = ob[k], os_[k], ol[k]
        om = [m for m, f in zip(om, k) if f]
    out = (torch.from_numpy(ob), torch.from_numpy(os_), torch.from_numpy(ol))
    return out + (om,) if want_members else out


def class_list(test_cfg):
    sel = list(getattr(test_cfg, "SELECT_CLASSES", ()))
    return sel if len(sel) else list(range(1, test_cfg.NUM_CLASSES))


def passes(test_cfg):
    """[(scale index, keep_range or None, flipped)] in the order im_detect_bbox_aug runs them."""
    rng = list(test_cfg.RANGES) if len(test_cfg.RANGES) == len(test_cfg.SCALES) else [None] * len(test_cfg.SCALES)
    out = []
    for i, r in enumerate(rng):
        out.append((i, r, False))
        if test_cfg.FLIP:
            out.append((i, r, True))
    return out


def merge_candidates(per_pass, orig_sizes, test_cfg):
    """per_pass: [(pass_size (w, h), flipped, keep_range, [per image (boxes, scores, labels) in pass coordinates])] ->
    per image (boxes, scores, labels) of the merged result, plus the merged (pre-merge) union per image."""
    B = len(orig_sizes)
    union = []
    for b in range(B):
        parts = [collect_pass(*cands[b], pass_size, orig_sizes[b], flip, rng) for pass_size, flip, rng, cands in per_pass]
        union.append(tuple(torch.cat([p[i] for p in parts]) for i in range(3)))
    mode = "vote" if test_cfg.SPECIAL_NMS == "vote" else "nms"
    res = [merge(*u, class_list(test_cfg), test_cfg.TH, mode, test_cfg.PRE_NMS_TOP_N) for u in union]
    return res, union


def detector_candidates(img, image_size, ids, am, pmap, bank, sd, **kw):
    """The pre-NMS candidates of oracle/restate.py's detector per image — what ATSSPostProcessor returns with
    bbox_aug_enabled (select_over_all_levels skipped): a suppression threshold no IoU exceeds and no per-image cut."""
    from oracle import restate
    return restate.detector(img, image_size, ids, am, pmap, bank, sd, nms_thresh=2.0, max_det=0, **kw)["detections"]


def pad_to(img, div):
    H, W = img.shape[-2:]
    Hp, Wp = (H + div - 1) // div * div, (W + div - 1) // div * div
    out = img.new_zeros(img.shape[:-2] + (Hp, Wp))
    out[..., :H, :W] = img
    return out


def im_detect_bbox_aug(images_by_scale, orig_sizes, ids, am, pmap, bank, sd, test_cfg, div=32, **kw):
    """The whole augmented detection over oracle/restate.py's detector.  images_by_scale[i]: [B, 3, h_i, w_i] normalised,
    un-padded; orig_sizes: per image (w, h)."""
    per_pass = []
    for i, rng, flip in passes(test_cfg):
        x = images_by_scale[i]
        h, w = x.shape[-2:]
        x = torch.flip(x, dims=[-1]) if flip else x
        cands = detector_candidates(pad_to(x, div), (h, w), ids, am, pmap, bank, sd, **kw)
        per_pass.append(((w, h), flip, rng, cands))
    return merge_candidates(per_pass, orig_sizes, test_cfg)


# ---- fixed cases shared by the CPU pinning test and the GPU tests ----------------------------------------------------------
def _objects(g, n_obj, copies, size, n_labels, jitter=6.0):
    """jittered copies of a few objects: boxes [n, 4] inside `size` = (w, h) on a quarter-pixel grid, scores, labels"""
    W, H = size
    cx, cy = torch.rand(n_obj, generator=g) * W, torch.rand(n_obj, generator=g) * H
    bw, bh = 8 + torch.rand(n_obj, generator=g) * W / 3, 8 + torch.rand(n_obj, generator=g) * H / 3
    lab = torch.randint(1, n_labels + 1, (n_obj,), generator=g)
    o = torch.randint(0, n_obj, (n_obj * copies,), generator=g)
    j = (torch.rand(o.numel(), 4, generator=g) - 0.5) * jitter
    b = torch.stack([cx[o] - bw[o] / 2, cy[o] - bh[o] / 2, cx[o] + bw[o] / 2, cy[o] + bh[o] / 2], 1) + j
    b = (b * 4).round() / 4
    b[:, 0::2] = b[:, 0::2].clamp(0, W - 1)
    b[:, 1::2] = b[:, 1::2].clamp(0, H - 1)
    s = 0.05 + 0.9 * torch.rand(o.numel(), generator=g)
    return b.float(), s.float(), lab[o]


def pin_cases():
    """name -> dict(orig_size, passes = [(pass_size, flip, keep_range, boxes, scores, labels)], test = TEST namespace)"""
    from types import SimpleNamespace as NS
    g = torch.Generator().manual_seed(1234)

    def test(**kw):
        d = dict(SPECIAL_NMS="none", TH=0.5, PRE_NMS_TOP_N=1000, NUM_CLASSES=6, SELECT_CLASSES=(), FLIP=False, SCALES=(), RANGES=())
        d.update(kw)
        return NS(**d)

    cases = {}
    # equal ratios; ranges dropping at both ends, areas exactly on a bound (20 x 20 = lo^2, 200 x 200 = hi^2); a flipped pass;
    # labels outside 1..NUM_CLASSES-1; the same box found by a pass and by a flipped pass (an exact score tie)
    b0, s0, l0 = _objects(g, 6, 8, (320, 240), 5)
    edge = torch.tensor([[10., 10., 29., 29.], [5., 5., 204., 204.], [10., 10., 30., 29.], [5., 5., 203., 204.]])
    b0 = torch.cat([b0, edge]); s0 = torch.cat([s0, torch.tensor([0.9, 0.8, 0.7, 0.6])]); l0 = torch.cat([l0, torch.tensor([1, 1, 2, 2])])
    b1, s1, l1 = _objects(g, 6, 8, (640, 480), 5)
    l1[:5] = torch.tensor([0, 7, 6, 0, 9])
    dup = torch.tensor([[100., 50., 180., 140.]])
    dupf = torch.tensor([[640 - 180. - 1, 50., 640 - 100. - 1, 140.]])
    b1 = torch.cat([b1, dupf]); s1 = torch.cat([s1, torch.tensor([0.77])]); l1 = torch.cat([l1, torch.tensor([3])])
    b2, s2, l2 = _objects(g, 6, 8, (960, 720), 5)
    b2 = torch.cat([b2, dup * 1.5]); s2 = torch.cat([s2, torch.tensor([0.77])]); l2 = torch.cat([l2, torch.tensor([3])])
    p = [((320, 240), False, (20, 200), b0, s0, l0), ((640, 480), True, None, b1, s1, l1), ((960, 720), False, (0, 300), b2, s2, l2)]
    cases["equal_nms"] = dict(orig_size=(640, 480), passes=p, test=test())
    cases["equal_vote"] = dict(orig_size=(640, 480), passes=p, test=test(SPECIAL_NMS="vote", TH=0.6))
    cases["th0"] = dict(orig_size=(640, 480), passes=p, test=test(TH=0.0))
    cases["th0_vote"] = dict(orig_size=(640, 480), passes=p, test=test(TH=0.0, SPECIAL_NMS="vote"))
    cases["select_classes"] = dict(orig_size=(640, 480), passes=p, test=test(SELECT_CLASSES=(2, 4)))
    # unequal width / height ratios; a class with exactly one box under vote
    b3, s3, l3 = _objects(g, 5, 10, (333, 250), 4)
    b3 = torch.cat([b3, torch.tensor([[40., 40., 90., 100.]])]); s3 = torch.cat([s3, torch.tensor([0.5])]); l3 = torch.cat([l3, torch.tensor([5])])
    b4, s4, l4 = _objects(g, 5, 10, (667, 500), 4)
    q = [((333, 250), False, None, b3, s3, l3), ((667, 500), True, (16, 400), b4, s4, l4)]
    cases["unequal_vote"] = dict(orig_size=(500, 375), passes=q, test=test(SPECIAL_NMS="vote", TH=0.6))
    cases["unequal_nms"] = dict(orig_size=(500, 375), passes=q, test=test(TH=0.6))
    # more survivors than PRE_NMS_TOP_N with scores tied at the cut (distant boxes: nothing is suppressed)
    n = 12
    bt = torch.stack([torch.arange(n) * 40., torch.zeros(n), torch.arange(n) * 40. + 20, torch.full((n,), 20.)], 1)
    st = torch.tensor([.9, .3, .5, .5, .8, .5, .2, .7, .5, .6, .1, .5])
    lt = torch.tensor([1, 2, 3, 1, 2, 3, 1, 2, 3, 1, 2, 3])
    cases["topn_ties"] = dict(orig_size=(640, 480), passes=[((640, 480), False, None, bt, st, lt)], test=test(PRE_NMS_TOP_N=6))
    cases["empty"] = dict(orig_size=(640, 480), passes=[((640, 480), False, None, torch.zeros(0, 4), torch.zeros(0), torch.zeros(0, dtype=torch.long))],
                          test=test())
    return cases


def run_case(c):
    """-> dict(union = merged candidates (boxes, scores, labels), result = (boxes, scores, labels))"""
    res, union = merge_candidates([(ps, flip, rng, [(b, s, l)]) for ps, flip, rng, b, s, l in c["passes"]], [c["orig_size"]], c["test"])
    return {"union": union[0], "result": res[0]}


def min_iou_margin(boxes, labels, th):
    """min |IoU - th| over same-label pairs (the pinned NMS cases keep it above 1e-6)"""
    b = boxes.numpy().astype(np.float32)
    lab = labels.numpy()
    best = 1.0
    for i in range(b.shape[0]):
        js = np.nonzero(lab == lab[i])[0]
        if js.size:
            best = min(best, float(np.abs(_iou_one(b, i, js).astype(np.float64) - th).min()))
    return best
