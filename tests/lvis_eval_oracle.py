"""Plain numpy restatement of the LVIS box evaluator (maskrcnn_benchmark/data/datasets/evaluation/lvis/lvis_eval.py:
LvisEvaluatorFixedAP, LVISResults, LVISEval; lvis.py: LVIS.get_ann_ids), rules 1-7 of DESIGN.md section 4.

Pinned to the reference code by tests/test_lvis_eval_cpu.py; the GPU evaluator (mqdet_b200/engine/lvis_eval.py) is compared
against it by tests/test_lvis_eval_gpu.py.  Detections carry an arrival number ``seq`` (update order, then image order, then row
order); every stable sort of the reference is a sort by (-score, seq) here."""
import numpy as np

IOU_THRS = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1, endpoint=True)
REC_THRS = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1, endpoint=True)
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]
FREQ_LBL = ["r", "c", "f"]


def convert(boxes_xyxy, in_size, orig_size):
    """Rule 1: fp32 xyxy boxes at the network input size (w, h) -> fp32 xywh at the original size (BoxList.resize with the
    Python-float ratios applied as fp32 multiplies, then convert_to_xywh in fp32)."""
    b = np.asarray(boxes_xyxy, dtype=np.float32).reshape(-1, 4)
    rx = np.float32(float(orig_size[0]) / float(in_size[0]))
    ry = np.float32(float(orig_size[1]) / float(in_size[1]))
    x1, y1, x2, y2 = b[:, 0] * rx, b[:, 1] * ry, b[:, 2] * rx, b[:, 3] * ry
    return np.stack([x1, y1, x2 - x1, y2 - y1], 1).astype(np.float32)


def bb_iou(d, g):
    """pycocotools bbIou on xywh fp64 boxes (no crowd): [len(d), len(g)]."""
    d = np.asarray(d, dtype=np.float64).reshape(-1, 4)
    g = np.asarray(g, dtype=np.float64).reshape(-1, 4)
    out = np.zeros((len(d), len(g)))
    for j in range(len(g)):
        ga = g[j, 2] * g[j, 3]
        for i in range(len(d)):
            da = d[i, 2] * d[i, 3]
            w = min(d[i, 2] + d[i, 0], g[j, 2] + g[j, 0]) - max(d[i, 0], g[j, 0])
            if w <= 0:
                continue
            h = min(d[i, 3] + d[i, 1], g[j, 3] + g[j, 1]) - max(d[i, 1], g[j, 1])
            if h <= 0:
                continue
            i_ = w * h
            out[i, j] = i_ / (da + ga - i_)
    return out


def _order(score, seq):
    return np.lexsort((seq, -np.asarray(score, dtype=np.float64)))


class Detections:
    """Arrived detections in arrival order: image id, category id, fp32 xywh box, fp32 score, arrival number."""

    def __init__(self):
        self.img, self.cat = np.zeros(0, np.int64), np.zeros(0, np.int64)
        self.box, self.score, self.seq = np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int64)

    def take(self, idx):
        d = Detections()
        d.img, d.cat, d.box, d.score, d.seq = self.img[idx], self.cat[idx], self.box[idx], self.score[idx], self.seq[idx]
        return d

    def cat_(self, o):
        d = Detections()
        d.img, d.cat = np.concatenate([self.img, o.img]), np.concatenate([self.cat, o.cat])
        d.box, d.score = np.concatenate([self.box, o.box]), np.concatenate([self.score, o.score])
        d.seq = np.concatenate([self.seq, o.seq])
        return d

    def __len__(self):
        return len(self.seq)


def _top_per_group(d, key, k):
    """Stable top-k by score within every group of ``key`` (ties by arrival), arrival order kept."""
    o = np.lexsort((d.seq, -d.score.astype(np.float64), key))
    ks = key[o]
    start = np.r_[0, np.nonzero(ks[1:] != ks[:-1])[0] + 1] if len(o) else np.zeros(0, np.int64)
    rank = np.arange(len(o)) - np.repeat(start, np.diff(np.r_[start, len(o)]))
    return d.take(np.sort(o[rank < k]))


class Oracle:
    """LvisEvaluatorFixedAP(gt, topk, fixed_ap) followed by LVISEval.run, restated."""

    def __init__(self, gt, topk=10000, fixed_ap=True):
        self.gt, self.topk, self.fixed_ap = gt, topk, fixed_ap
        self.dets = Detections()
        self.next_seq = 0

    def update(self, per_image):
        """per_image: list of (image_id, fp32 xywh [n, 4], fp32 scores [n], category ids [n]) in prediction order."""
        cur = Detections()
        if per_image:
            n = [len(score) for _, _, score, _ in per_image]
            cur.img = np.repeat(np.array([i for i, _, _, _ in per_image], np.int64), n)
            cur.cat = np.concatenate([np.asarray(c, np.int64).reshape(-1) for *_, c in per_image])
            cur.box = np.concatenate([np.asarray(b, np.float32).reshape(-1, 4) for _, b, _, _ in per_image])
            cur.score = np.concatenate([np.asarray(s, np.float32).reshape(-1) for _, _, s, _ in per_image])
            cur.seq = np.arange(self.next_seq, self.next_seq + sum(n), dtype=np.int64)
            self.next_seq += sum(n)
        if self.fixed_ap:   # per update: stable top-k per category, merged with earlier arrivals first on ties
            cur = _top_per_group(cur, cur.cat, self.topk)
            allc = self.dets.cat_(cur)
            self.dets = _top_per_group(allc, allc.cat, self.topk)
        else:               # per update: stable top 300 per image
            self.dets = self.dets.cat_(_top_per_group(cur, cur.img, 300))

    def results(self):
        """The detection list handed to LVISResults, cut (fixed: top-k per category; standard: limit_dets_per_image 300)."""
        if self.fixed_ap:
            return _top_per_group(self.dets, self.dets.cat, self.topk)
        return _top_per_group(self.dets, self.dets.img, 300)

    def evaluate(self):
        gt = self.gt
        img_ids = sorted(im["id"] for im in gt["images"])
        cat_ids = sorted(c["id"] for c in gt["categories"])
        cat_pos = {c: i for i, c in enumerate(cat_ids)}
        neg = {im["id"]: set(im["neg_category_ids"]) for im in gt["images"]}
        nel = {im["id"]: set(im["not_exhaustive_category_ids"]) for im in gt["images"]}
        gts = {}
        present = {i: set() for i in img_ids}
        for a in gt["annotations"]:   # get_ann_ids: listed images and categories, 0 < area < inf
            if a["image_id"] in neg and a["category_id"] in cat_pos and 0 < a["area"] < float("inf"):
                gts.setdefault((a["image_id"], a["category_id"]), []).append(a)
                present[a["image_id"]].add(a["category_id"])
        d = self.results()
        area = d.box[:, 2].astype(np.float64) * d.box[:, 3].astype(np.float64)
        def pair_keys(img, cat):
            return (np.asarray(img, np.int64) << 32) + np.asarray(cat, np.int64)
        neg_keys = pair_keys(*np.array([(i, c) for i, cs in neg.items() for c in cs], np.int64).reshape(-1, 2).T)
        pos_keys = pair_keys(*np.array(list(gts), np.int64).reshape(-1, 2).T)
        dk = pair_keys(d.img, d.cat)
        keep = (np.isin(d.img, img_ids) & np.isin(d.cat, cat_ids) & (area > 0) & (area < np.inf) &
                (np.isin(dk, neg_keys) | np.isin(dk, pos_keys)))
        d = d.take(np.nonzero(keep)[0])
        dts = {}
        for i in _order(d.score, d.seq):  # within a pair: score descending, arrival on ties
            dts.setdefault((int(d.img[i]), int(d.cat[i])), []).append(i)
        T, A = len(IOU_THRS), len(AREA_RNG)
        pairs = {}
        for key in sorted(set(gts) | set(dts)):
            img_id, cat_id = key
            g = gts.get(key, [])
            di = np.array(dts.get(key, []), dtype=np.int64)
            gbox = np.array([a["bbox"] for a in g], dtype=np.float64).reshape(-1, 4)
            ious = bb_iou(d.box[di].astype(np.float64), gbox) if len(g) and len(di) else np.zeros((len(di), len(g)))
            darea = d.box[di, 2].astype(np.float64) * d.box[di, 3].astype(np.float64)
            res = []
            for lo, hi in AREA_RNG:
                g_ig = np.array([1 if (a.get("ignore", 0) or a["area"] < lo or a["area"] > hi) else 0 for a in g], dtype=np.int64)
                gi = np.argsort(g_ig, kind="mergesort")
                g_ig = g_ig[gi]
                gid = np.array([g[j]["id"] for j in gi], dtype=np.int64)
                iou = ious[:, gi]
                dt_m = np.zeros((T, len(di)), dtype=np.int64)
                dt_ig = np.zeros((T, len(di)), dtype=bool)
                for t, thr in enumerate(IOU_THRS):
                    if len(g) == 0:
                        break
                    gt_m = np.zeros(len(g), dtype=bool)
                    for k in range(len(di)):
                        best, m = min(thr, 1 - 1e-10), -1
                        for j in range(len(g)):
                            if gt_m[j]:
                                continue
                            if m > -1 and g_ig[m] == 0 and g_ig[j] == 1:
                                break
                            if iou[k, j] < best:
                                continue
                            best, m = iou[k, j], j
                        if m == -1:
                            continue
                        dt_ig[t, k] = bool(g_ig[m])
                        dt_m[t, k] = gid[m]
                        gt_m[m] = True
                out_rng = (darea < lo) | (darea > hi) | (cat_id in nel[img_id])
                dt_ig = dt_ig | ((dt_m == 0) & out_rng[None, :])
                res.append({"dt_matches": dt_m, "dt_ignore": dt_ig, "gt_ignore": g_ig, "gt_ids": gid,
                            "dt_scores": d.score[di].astype(np.float64), "dt_seq": d.seq[di]})
            pairs[key] = res
        self.pairs, self.dets_eval = pairs, d
        self._accumulate(img_ids, cat_ids)
        return self

    def _accumulate(self, img_ids, cat_ids):
        T, R, K, A = len(IOU_THRS), len(REC_THRS), len(cat_ids), len(AREA_RNG)
        precision, recall = -np.ones((T, R, K, A)), -np.ones((T, K, A))
        by_cat = {}
        for (img_id, cat_id) in sorted(self.pairs, key=lambda p: (p[1], p[0])):   # image-id order within a category
            by_cat.setdefault(cat_id, []).append(self.pairs[img_id, cat_id])
        for k, cat_id in enumerate(cat_ids):
            for a in range(A):
                E = [p[a] for p in by_cat.get(cat_id, [])]
                if not E:
                    continue
                sc = np.concatenate([e["dt_scores"] for e in E])
                o = np.argsort(-sc, kind="mergesort")
                dt_m = np.concatenate([e["dt_matches"] for e in E], axis=1)[:, o]
                dt_ig = np.concatenate([e["dt_ignore"] for e in E], axis=1)[:, o]
                num_gt = int(np.count_nonzero(np.concatenate([e["gt_ignore"] for e in E]) == 0))
                if num_gt == 0:
                    continue
                tps = np.logical_and(dt_m, np.logical_not(dt_ig))
                fps = np.logical_and(np.logical_not(dt_m), np.logical_not(dt_ig))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                for t in range(T):
                    tp, fp = tp_sum[t], fp_sum[t]
                    n = len(tp)
                    rc = tp / num_gt
                    recall[t, k, a] = rc[-1] if n else 0
                    pr = tp / (fp + tp + np.spacing(1))
                    pr = np.maximum.accumulate(pr[::-1])[::-1] if n else pr
                    idx = np.searchsorted(rc, REC_THRS, side="left")
                    q = np.zeros(R)
                    ok = idx < n
                    q[ok] = pr[idx[ok]]
                    precision[t, :, k, a] = q
        self.precision, self.recall = precision, recall
        self.cat_ids = cat_ids

    def summarize(self):
        """-> (results dict in the reference's key order, printed strings)."""
        return summarize(self.precision, self.recall, self.gt, self.cat_ids, 300 if not self.fixed_ap else -1)


def freq_groups(gt, cat_ids):
    freq = {c["id"]: c["frequency"] for c in gt["categories"]}
    groups = [[] for _ in FREQ_LBL]
    for i, c in enumerate(cat_ids):
        groups[FREQ_LBL.index(freq[c])].append(i)
    return groups


def summarize(precision, recall, gt, cat_ids, max_dets):
    """LVISEval.summarize / _summarize / print_results on the accumulated arrays."""
    groups = freq_groups(gt, cat_ids)

    def _s(kind, iou_thr=None, area="all", fg=None):
        aidx = [AREA_LBL.index(area)]
        s = precision if kind == "ap" else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        if kind == "ap":
            s = s[:, :, groups[fg], aidx] if fg is not None else s[:, :, :, aidx]
        else:
            s = s[:, :, aidx]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])

    r = {"AP": _s("ap"), "AP50": _s("ap", 0.50), "AP75": _s("ap", 0.75), "APs": _s("ap", area="small"),
         "APm": _s("ap", area="medium"), "APl": _s("ap", area="large"), "APr": _s("ap", fg=0), "APc": _s("ap", fg=1),
         "APf": _s("ap", fg=2), f"AR@{max_dets}": _s("ar")}
    for area in ["small", "medium", "large"]:
        r[f"AR{area[0]}@{max_dets}"] = _s("ar", area=area)
    tpl = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} catIds={:>3s}] = {:0.3f}"
    lines = []
    for key, value in r.items():
        title, typ = ("Average Precision", "(AP)") if "AP" in key else ("Average Recall", "(AR)")
        iou = "{:0.2f}".format(float(key[2:]) / 100) if len(key) > 2 and key[2].isdigit() else \
            "{:0.2f}:{:0.2f}".format(IOU_THRS[0], IOU_THRS[-1])
        grp = key[2] if len(key) > 2 and key[2] in ["r", "c", "f"] else "all"
        area = key[2] if len(key) > 2 and key[2] in ["s", "m", "l"] else "all"
        lines.append(tpl.format(title, typ, iou, area, max_dets, grp, value))
    return r, lines


# ---- synthetic LVIS-format cases (shared by the CPU pin and the GPU tests) -------------------------------------------------
def synth_gt(seed, n_img=12, n_cat=8, per_img=6):
    """Image ids and category ids with gaps, r / c / f categories (the last one without GTs), an image without GTs, negative and
    not-exhaustive lists, GT boxes in every area range, ``area`` fields exactly on the 32^2 / 96^2 boundaries, and duplicates."""
    rng = np.random.default_rng(seed)
    cats = [{"id": 2 + 3 * k, "frequency": FREQ_LBL[k % 3], "name": f"c{k}"} for k in range(n_cat)]
    cids = [c["id"] for c in cats]
    images, anns = [], []
    for i in range(n_img):
        W, H = int(rng.integers(300, 900)), int(rng.integers(300, 900))
        img_id = 5 + 4 * i
        present = [] if i == 1 else list(rng.choice(cids[:-1], size=min(3, n_cat - 1), replace=False))
        absent = [c for c in cids if c not in present]
        neg = list(rng.choice(absent, size=min(2, len(absent)), replace=False))
        nel = [present[0]] if present and i % 3 == 0 else []
        images.append({"id": img_id, "width": W, "height": H, "neg_category_ids": [int(c) for c in neg],
                       "not_exhaustive_category_ids": [int(c) for c in nel]})
        for j in range(0 if i == 1 else per_img):
            c = int(present[j % len(present)])
            side = float(rng.choice([12.0, 31.0, 32.0, 50.0, 96.0, 140.0, 300.0]))
            w, h = np.float32(side * rng.uniform(0.7, 1.3)), np.float32(side * rng.uniform(0.7, 1.3))
            x, y = np.float32(rng.uniform(0, max(W - w, 1.0))), np.float32(rng.uniform(0, max(H - h, 1.0)))
            area = [float(w) * float(h), float(w) * float(h) * 0.7, 1024.0, 9216.0][j % 4]
            box = [float(x), float(y), float(w), float(h)]
            anns.append({"id": len(anns) + 1, "image_id": img_id, "category_id": c, "bbox": box, "area": area, "iscrowd": 0})
            if j == 2:   # a duplicate
                anns.append({"id": len(anns) + 1, "image_id": img_id, "category_id": c, "bbox": list(box), "area": area,
                             "iscrowd": 0})
    return {"images": images, "annotations": anns, "categories": cats}


def synth_updates(gt, seed, n_upd=3, per_img=40, big_cat=None, big_n=0, extra_cat=99):
    """Detections as the detector emits them: per update a list of (image_id, fp32 xyxy boxes at the network input size,
    (in_w, in_h), (orig_w, orig_h), fp32 scores, category ids).  Scores on a 1/64 grid (ties within and across images), boxes
    near the GTs and elsewhere, one category id outside the GT file, zero-width boxes, an image id outside the GT file and one
    image present in two updates.  ``big_cat`` gets ``big_n`` extra detections per image."""
    rng = np.random.default_rng(seed)
    imgs = list(gt["images"])
    cids = [c["id"] for c in gt["categories"]]
    by_img = {}
    for a in gt["annotations"]:
        by_img.setdefault(a["image_id"], []).append(a)
    chunks = [imgs[k::n_upd] for k in range(n_upd)]
    chunks[-1] = chunks[-1] + [imgs[0]]
    ups = []
    for u, part in enumerate(chunks):
        cur = []
        for im in part + ([{"id": 100000 + u, "width": 400, "height": 300}] if u == 0 else []):
            W, H = im["width"], im["height"]
            s = float(rng.uniform(0.6, 1.6))
            iw, ih = max(1, int(round(W * s))), max(1, int(round(H * s)))
            n = per_img + (big_n if big_cat is not None else 0)
            cat = rng.choice(cids + [extra_cat], size=n).astype(np.int64)
            if big_cat is not None:
                cat[per_img:] = big_cat
            xywh = np.zeros((n, 4), np.float64)
            gts = by_img.get(im["id"], [])
            for k in range(n):
                if gts and rng.random() < 0.6:
                    g = gts[int(rng.integers(len(gts)))]
                    b = np.array(g["bbox"]) + rng.normal(0, 0.08, 4) * max(g["bbox"][2], g["bbox"][3])
                    if rng.random() < 0.7 and big_cat is None:
                        cat[k] = g["category_id"]
                else:
                    wh = rng.uniform(5, 200, 2)
                    b = np.array([rng.uniform(0, W - 5), rng.uniform(0, H - 5), wh[0], wh[1]])
                if k % 17 == 5:
                    b[2] = 0.0
                xywh[k] = b
            xyxy = np.stack([xywh[:, 0], xywh[:, 1], xywh[:, 0] + xywh[:, 2], xywh[:, 1] + xywh[:, 3]], 1) * (iw / W)
            score = (rng.integers(1, 64, n) / 64.0).astype(np.float32)
            cur.append((im["id"], xyxy.astype(np.float32), (iw, ih), (W, H), score, cat))
        ups.append(cur)
    return ups


def pin_cases():
    """name -> (gt, updates, topk, fixed_ap)"""
    g0 = synth_gt(1)
    g1 = synth_gt(2, n_img=6, n_cat=5, per_img=4)
    return {
        "fixed": (g0, synth_updates(g0, 11), 10000, True),
        "fixed_cut": (g0, synth_updates(g0, 12, n_upd=4, per_img=60), 37, True),
        "standard": (g0, synth_updates(g0, 13, per_img=320), 10000, False),
        "fixed_big": (g1, synth_updates(g1, 14, n_upd=2, per_img=10, big_cat=g1["categories"][0]["id"], big_n=1500), 10000, True),
    }


def run_oracle(gt, updates, topk, fixed_ap):
    o = Oracle(gt, topk, fixed_ap)
    for upd in updates:
        o.update([(i, convert(b, s, os_), sc, c) for i, b, s, os_, sc, c in upd])
    return o.evaluate()


def canonical(pairs):
    """Per-(image, category) evaluation arrays in one fixed layout: pair keys [P, 2], int64 (dt_matches, dt_ignore, gt_ignore,
    gt_ids per area range, flattened) and fp64 dt_scores."""
    keys, ints, flts = [], [], []
    for key in sorted(pairs):
        keys.append(key)
        for e in pairs[key]:
            ints += [np.asarray(e["dt_matches"], np.int64).ravel(), np.asarray(e["dt_ignore"], np.int64).ravel(),
                     np.asarray(e["gt_ignore"], np.int64).ravel(), np.asarray(e["gt_ids"], np.int64).ravel()]
            flts.append(np.asarray(e["dt_scores"], np.float64).ravel())
    return (np.array(keys, np.int64).reshape(-1, 2), np.concatenate(ints) if ints else np.zeros(0, np.int64),
            np.concatenate(flts) if flts else np.zeros(0))


# ---- a minival-shaped synthetic set (LVIS minival: 5000 images, 1203 categories, ~50k GTs; 31 chunks x 100 rows per image) -----
def minival_gt(seed, n_img=5000, n_cat=1203, per_img=10):
    """640 x 480 images, six categories present per image, eight negative ones, every fifth image not exhaustive for one."""
    rng = np.random.default_rng(seed)
    cats = [{"id": k + 1, "frequency": FREQ_LBL[k % 3]} for k in range(n_cat)]
    images, anns = [], []
    for i in range(n_img):
        present = rng.choice(n_cat, size=6, replace=False) + 1
        neg = [int(c) for c in rng.choice(n_cat, size=8, replace=False) + 1 if c not in present]
        images.append({"id": i + 1, "width": 640, "height": 480, "neg_category_ids": neg,
                       "not_exhaustive_category_ids": [int(present[0])] if i % 5 == 0 else []})
        for j in range(per_img):
            w, h = rng.uniform(8, 300, 2)
            x, y = rng.uniform(0, 640 - w), rng.uniform(0, 480 - h)
            anns.append({"id": len(anns) + 1, "image_id": i + 1, "category_id": int(present[j % 6]),
                         "bbox": [float(x), float(y), float(w), float(h)], "area": float(w * h), "iscrowd": 0})
    return {"images": images, "annotations": anns, "categories": cats}


MINIVAL_IN_HW, MINIVAL_ORIG_HW = (800, 1066), (480, 640)


def minival_packed(gt, seed, image_ids, rows=100):
    """The chunked detector's packed result fp32 [chunks, B, rows + 1, 6] for ``image_ids`` at a network size of 800 x 1066:
    chunk c holds labels 40c + 1 .. 40c + 40; half the rows lie near a GT of the image (jittered), half anywhere; scores on a
    1/4096 grid (ties within and across images)."""
    rng = np.random.default_rng(seed)
    n_cat = len(gt["categories"])
    chunks = (n_cat + 39) // 40
    by_img = {}
    for a in gt["annotations"]:
        x, y, w, h = a["bbox"]
        by_img.setdefault(a["image_id"], []).append([x, y, x + w, y + h])
    pk = np.zeros((chunks, len(image_ids), rows + 1, 6), np.float32)
    s = MINIVAL_IN_HW[1] / MINIVAL_ORIG_HW[1]
    for b, i in enumerate(image_ids):
        gb = np.array(by_img[i])
        lab = np.minimum(rng.integers(0, 40, (chunks, rows)) + 40 * np.arange(chunks)[:, None] + 1, n_cat)
        xy = rng.uniform(0, 1, (chunks, rows, 2)) * [600.0, 440.0]
        box = np.concatenate([xy, xy + rng.uniform(4, 204, (chunks, rows, 2))], 2)
        near = rng.integers(0, len(gb), (chunks, rows // 2))
        box[:, : rows // 2] = gb[near] + rng.normal(0, 6, (chunks, rows // 2, 4))
        pk[:, b, :rows, :4] = box * s
        pk[:, b, :rows, 4] = rng.integers(1, 4096, (chunks, rows)) / 4096.0
        pk[:, b, :rows, 5] = lab
        pk[:, b, rows, 0] = rows
    return pk


def oracle_update_from_packed(pk, image_ids, in_hw, orig_hw):
    """What the reference's prepare() gets from one packed chunked result: per image the chunks' rows in chunk order."""
    per = []
    for b, i in enumerate(image_ids):
        rows = np.concatenate([pk[c, b, :int(pk[c, b, -1, 0])] for c in range(pk.shape[0])])
        per.append((i, convert(rows[:, :4], (in_hw[1], in_hw[0]), (orig_hw[1], orig_hw[0])), rows[:, 4],
                    rows[:, 5].astype(np.int64)))
    return per
