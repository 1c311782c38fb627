"""Plain numpy restatement of COCO-style box AP as the reference scores ODinW / COCO val
(maskrcnn_benchmark/data/datasets/evaluation/od_to_grounding/od_eval.py: prepare_for_coco_detection, evaluate_predictions_on_coco,
summarize_per_category, COCOResults) through pycocotools (COCO.loadRes; COCOeval, iouType "bbox": _prepare, computeIoU,
evaluateImg, accumulate, summarize).  The rules are DESIGN.md section 4 ("COCO box AP rules").

``COCO`` / ``COCOeval`` keep pycocotools' interface, so the reference's own od_eval.py can run on top of them
(tests/test_coco_eval_cpu.py); the per-pair matching is vectorised over the IoU thresholds and the accumulation over the images
of a category, which computes the same arrays as pycocotools' loops (same fp64 operations, same stable orders).  The GPU evaluator
(mqdet_b200/engine/coco_eval.py) is compared against it by tests/test_coco_eval_gpu.py."""
import copy
import json
from collections import OrderedDict, defaultdict

import numpy as np

IOU_THRS = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1, endpoint=True)
REC_THRS = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1, endpoint=True)
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]
MAX_DETS = [1, 10, 100]


# ---- pycocotools.coco.COCO --------------------------------------------------------------------------------------------------
class COCO:
    def __init__(self, annotation_file=None):
        self.dataset, self.anns, self.cats, self.imgs = {}, {}, {}, {}
        self.imgToAnns, self.catToImgs = defaultdict(list), defaultdict(list)
        if annotation_file is not None:
            if isinstance(annotation_file, str):
                with open(annotation_file) as f:
                    annotation_file = json.load(f)
            self.dataset = annotation_file
            self.createIndex()

    def createIndex(self):
        self.anns, self.cats, self.imgs = {}, {}, {}
        self.imgToAnns, self.catToImgs = defaultdict(list), defaultdict(list)
        for ann in self.dataset.get("annotations", []):
            self.imgToAnns[ann["image_id"]].append(ann)
            self.anns[ann["id"]] = ann
            self.catToImgs[ann["category_id"]].append(ann["image_id"])
        for img in self.dataset.get("images", []):
            self.imgs[img["id"]] = img
        for cat in self.dataset.get("categories", []):
            self.cats[cat["id"]] = cat

    def getAnnIds(self, imgIds=(), catIds=()):
        imgIds, catIds = list(imgIds), set(catIds)
        anns = [a for i in imgIds if i in self.imgToAnns for a in self.imgToAnns[i]] if imgIds else self.dataset["annotations"]
        return [a["id"] for a in anns if not catIds or a["category_id"] in catIds]

    def getCatIds(self):
        return [c["id"] for c in self.dataset.get("categories", [])]

    def getImgIds(self):
        return list(self.imgs.keys())

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def loadRes(self, resFile):
        res = COCO()
        res.dataset["images"] = [img for img in self.dataset["images"]]
        if isinstance(resFile, str):
            with open(resFile) as f:
                anns = json.load(f)
        else:
            anns = resFile
        assert type(anns) == list, "results in not an array of objects"
        ids = [a["image_id"] for a in anns]
        assert set(ids) == (set(ids) & set(self.getImgIds())), "Results do not correspond to current coco set"
        res.dataset["categories"] = copy.deepcopy(self.dataset["categories"])
        for i, ann in enumerate(anns):
            bb = ann["bbox"]
            ann["area"] = bb[2] * bb[3]
            ann["id"] = i + 1
            ann["iscrowd"] = 0
        res.dataset["annotations"] = anns
        res.createIndex()
        return res


# ---- pycocotools.cocoeval.COCOeval (bbox) -----------------------------------------------------------------------------------
class Params:
    def __init__(self, iouType="bbox"):
        self.imgIds, self.catIds = [], []
        self.iouThrs, self.recThrs = IOU_THRS, REC_THRS
        self.maxDets = list(MAX_DETS)
        self.areaRng, self.areaRngLbl = [list(a) for a in AREA_RNG], list(AREA_LBL)
        self.useCats, self.iouType = 1, iouType


def bb_iou(d, g, crowd):
    """pycocotools bbIou on fp64 xywh: [len(d), len(g)]; a crowd GT's union is the detection's area."""
    d = np.asarray(d, np.float64).reshape(-1, 1, 4)
    g = np.asarray(g, np.float64).reshape(1, -1, 4)
    w = np.minimum(d[..., 2] + d[..., 0], g[..., 2] + g[..., 0]) - np.maximum(d[..., 0], g[..., 0])
    h = np.minimum(d[..., 3] + d[..., 1], g[..., 3] + g[..., 1]) - np.maximum(d[..., 1], g[..., 1])
    i = w * h
    da, ga = d[..., 2] * d[..., 3], g[..., 2] * g[..., 3]
    u = np.where(np.asarray(crowd, bool).reshape(1, -1), da, da + ga - i)
    with np.errstate(divide="ignore", invalid="ignore"):
        o = i / u
    return np.where((w > 0) & (h > 0), o, 0.0)


def match_pair(gts, dts, max_det=100):
    """evaluateImg for one (image, category) over the four area ranges: dts sorted by score (stable) and cut to ``max_det``.
    -> per range dict(dtMatches int64 [T, D] (GT ids), dtIgnore bool [T, D], gtIgnore [G] (in the sorted order), dtScores)."""
    T = len(IOU_THRS)
    o = np.argsort([-d["score"] for d in dts], kind="mergesort")[:max_det]
    dt = [dts[i] for i in o]
    D, G = len(dt), len(gts)
    crowd = np.array([int(g["iscrowd"]) for g in gts], bool)
    ious = bb_iou([d["bbox"] for d in dt], [g["bbox"] for g in gts], crowd) if D and G else np.zeros((D, G))
    darea = np.array([d["area"] for d in dt], np.float64)
    garea = np.array([g["area"] for g in gts], np.float64)
    gign = np.array([bool(g["ignore"]) for g in gts], bool)
    gid = np.array([g["id"] for g in gts], np.int64)
    thr = np.minimum(IOU_THRS, 1 - 1e-10)[:, None]
    out = []
    for lo, hi in AREA_RNG:
        ig = (gign | (garea < lo) | (garea > hi)).astype(np.int64)
        gi = np.argsort(ig, kind="mergesort")
        ig, iou, cr, ids = ig[gi], ious[:, gi], crowd[gi], gid[gi]
        gtm = np.zeros((T, G), bool)
        dtm = np.zeros((T, D), np.int64)
        dtig = np.zeros((T, D), bool)
        for k in range(D if G else 0):
            row = iou[k][None, :]
            ok = (~gtm | cr[None, :]) & (row >= thr)
            m = np.full(T, -1)
            for pas in (0, 1):    # the GTs of the range, then (only without a match among them) the ignored ones
                c = ok & (ig == pas)[None, :] & (m < 0)[:, None]
                val = np.where(c, row, -np.inf)
                best = val.max(1)
                last = G - 1 - np.argmax(((val == best[:, None]) & c)[:, ::-1], axis=1)   # a later equal IoU replaces
                m = np.where(c.any(1), last, m)
            t = np.nonzero(m >= 0)[0]
            gtm[t, m[t]] = True
            dtm[t, k] = ids[m[t]]
            dtig[t, k] = ig[m[t]] == 1
        out_rng = (darea < lo) | (darea > hi)
        dtig = dtig | ((dtm == 0) & out_rng[None, :])
        out.append({"dtMatches": dtm, "dtIgnore": dtig, "gtIgnore": ig, "gtIds": ids,
                    "dtScores": np.array([d["score"] for d in dt], np.float64), "dtIds": [d["id"] for d in dt]})
    return out


class COCOeval:
    def __init__(self, cocoGt=None, cocoDt=None, iouType="bbox"):
        assert iouType == "bbox", "the restatement covers box AP only"
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.params = Params(iouType)
        self.eval, self.stats, self.pairs = {}, [], {}
        if cocoGt is not None:
            self.params.imgIds = sorted(cocoGt.getImgIds())
            self.params.catIds = sorted(cocoGt.getCatIds())

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        gts = self.cocoGt.loadAnns(self.cocoGt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        dts = self.cocoDt.loadAnns(self.cocoDt.getAnnIds(imgIds=p.imgIds, catIds=p.catIds))
        for gt in gts:
            gt["ignore"] = "iscrowd" in gt and gt["iscrowd"]
        g, d = defaultdict(list), defaultdict(list)
        for gt in gts:
            g[gt["image_id"], gt["category_id"]].append(gt)
        for dt in dts:
            d[dt["image_id"], dt["category_id"]].append(dt)
        self.pairs = {k: match_pair(g.get(k, []), d.get(k, []), p.maxDets[-1]) for k in sorted(set(g) | set(d))}

    def accumulate(self):
        p = self.params
        T, R, K, A, M = len(p.iouThrs), len(p.recThrs), len(p.catIds), len(p.areaRng), len(p.maxDets)
        precision, recall = -np.ones((T, R, K, A, M)), -np.ones((T, K, A, M))
        by_cat = defaultdict(list)
        for (img, cat) in sorted(self.pairs, key=lambda x: (x[1], x[0])):     # image-id order within a category
            by_cat[cat].append(self.pairs[img, cat])
        for k, cat in enumerate(p.catIds):
            for a in range(A):
                E = [e[a] for e in by_cat.get(cat, [])]
                if not E:
                    continue
                npig = int(np.count_nonzero(np.concatenate([e["gtIgnore"] for e in E]) == 0))
                if npig == 0:
                    continue
                for m, max_det in enumerate(p.maxDets):
                    sc = np.concatenate([e["dtScores"][:max_det] for e in E])
                    o = np.argsort(-sc, kind="mergesort")
                    dtm = np.concatenate([e["dtMatches"][:, :max_det] for e in E], axis=1)[:, o]
                    dtig = np.concatenate([e["dtIgnore"][:, :max_det] for e in E], axis=1)[:, o]
                    tps = np.logical_and(dtm, np.logical_not(dtig))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtig))
                    tp_sum = np.cumsum(tps, axis=1).astype(float)
                    fp_sum = np.cumsum(fps, axis=1).astype(float)
                    nd = tp_sum.shape[1]
                    for t in range(T):
                        tp, fp = tp_sum[t], fp_sum[t]
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = np.maximum.accumulate(pr[::-1])[::-1] if nd else pr
                        idx = np.searchsorted(rc, p.recThrs, side="left")
                        q = np.zeros(R)
                        q[idx < nd] = pr[idx[idx < nd]]
                        precision[t, :, k, a, m] = q
        self.eval = {"params": p, "counts": [T, R, K, A, M], "precision": precision, "recall": recall}

    def summarize(self):
        self.stats, lines = summarize(self.eval["precision"], self.eval["recall"])
        for line in lines:
            print(line)


_SUMMARY = [(1, None, "all", 100), (1, .5, "all", 100), (1, .75, "all", 100), (1, None, "small", 100),
            (1, None, "medium", 100), (1, None, "large", 100), (0, None, "all", 1), (0, None, "all", 10),
            (0, None, "all", 100), (0, None, "small", 100), (0, None, "medium", 100), (0, None, "large", 100)]


def summarize(precision, recall):
    """COCOeval.summarize (_summarizeDets) on the accumulated arrays -> (stats [12], the printed lines)."""
    stats, lines = np.zeros((12,)), []
    for i, (ap, iou_thr, area, max_dets) in enumerate(_SUMMARY):
        s = precision if ap == 1 else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        aind, mind = [AREA_LBL.index(area)], [MAX_DETS.index(max_dets)]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        iou = "{:0.2f}:{:0.2f}".format(IOU_THRS[0], IOU_THRS[-1]) if iou_thr is None else "{:0.2f}".format(iou_thr)
        lines.append(" {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}".format(
            "Average Precision" if ap == 1 else "Average Recall", "(AP)" if ap == 1 else "(AR)", iou, area, max_dets, mean_s))
        stats[i] = mean_s
    return stats, lines


# ---- od_eval.py ------------------------------------------------------------------------------------------------------------
def convert(boxes_xyxy, in_size, orig_size):
    """prepare_for_coco_detection's box conversion: fp32 xyxy at the network input size (w, h) -> fp32 xywh at the GT image
    size: BoxList.resize (the Python-float ratios as fp32 multiplies), then BoxList.convert("xywh") (x2 - x1 + 1 in fp32)."""
    b = np.asarray(boxes_xyxy, dtype=np.float32).reshape(-1, 4)
    rx = np.float32(float(orig_size[0]) / float(in_size[0]))
    ry = np.float32(float(orig_size[1]) / float(in_size[1]))
    x1, y1, x2, y2 = b[:, 0] * rx, b[:, 1] * ry, b[:, 2] * rx, b[:, 3] * ry
    one = np.float32(1)
    return np.stack([x1, y1, (x2 - x1) + one, (y2 - y1) + one], 1).astype(np.float32)


def prepare(gt, per_image, label_to_category=None):
    """prepare_for_coco_detection: per_image = [(image_id, fp32 xyxy at (in_w, in_h), (in_w, in_h), fp32 scores, labels)] in
    prediction order -> the results list (labels outside ``label_to_category`` dropped; images without rows skipped)."""
    imgs = {im["id"]: im for im in gt["images"]}
    res = []
    for img_id, boxes, in_size, scores, labels in per_image:
        if len(scores) == 0:
            continue
        im = imgs.get(img_id)
        orig = (im["width"], im["height"]) if im is not None else in_size
        xywh = convert(boxes, in_size, orig).tolist()
        sc = np.asarray(scores, np.float32).tolist()
        for k, lab in enumerate(np.asarray(labels).tolist()):
            lab = int(lab)
            if label_to_category is not None and lab not in label_to_category:
                continue
            cat = label_to_category[lab] if label_to_category is not None else lab
            res.append({"image_id": img_id, "category_id": cat, "bbox": xywh[k], "score": sc[k]})
    return res


def evaluate(gt, results):
    """evaluate_predictions_on_coco on a results list: -> the COCOeval after accumulate and summarize (quiet)."""
    coco_gt = COCO(copy.deepcopy(gt))
    coco_dt = coco_gt.loadRes(copy.deepcopy(results)) if results else COCO()
    ev = COCOeval(coco_gt, coco_dt, "bbox")
    ev.evaluate()
    ev.accumulate()
    ev.stats, ev.lines = summarize(ev.eval["precision"], ev.eval["recall"])
    return ev


def per_category_csv(precision, cat_ids, cat_names):
    """summarize_per_category's CSV text (per-category means over all entries, -1 included)."""
    def _s(iou_thr=None, area="all", max_dets=100):
        iou = "{:0.2f}:{:0.2f}".format(IOU_THRS[0], IOU_THRS[-1]) if iou_thr is None else "{:0.2f}".format(iou_thr)
        out = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ], ".format("Average Precision", "(AP)", iou, area,
                                                                                    max_dets)
        s = precision
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        s = s[:, :, :, [AREA_LBL.index(area)], [MAX_DETS.index(max_dets)]]
        if len(s[s > -1]) != 0:
            avg = 0.0
            for i in range(len(cat_ids)):
                out += "{}, ".format(np.mean(s[:, :, i, :]))
                avg += np.mean(s[:, :, i, :])
            out += "{} \n".format(avg / len(cat_ids))
        return out

    title = "metric, " + "".join("{}, ".format(cat_names[c]) for c in cat_ids) + "avg \n"
    return "".join([title, _s(), _s(.5), _s(area="small"), _s(area="medium"), _s(area="large")])


def coco_results(stats):
    """COCOResults("bbox") after update: {"bbox": OrderedDict(AP, AP50, AP75, APs, APm, APl)}."""
    return OrderedDict([("bbox", OrderedDict((k, stats[i]) for i, k in enumerate(["AP", "AP50", "AP75", "APs", "APm", "APl"])))])


# ---- synthetic COCO-format cases (shared by the CPU tests and the GPU tests) ---------------------------------------------------
def synth_gt(seed, n_img=12, n_cat=6, per_img=6, crowd_every=0, id0=False):
    """Image and category ids with gaps, the last category without GTs, an image without GTs, GT boxes in every area range,
    ``area`` fields exactly on the 32^2 / 96^2 boundaries, a duplicated GT; crowd GTs every ``crowd_every``-th annotation; with
    ``id0`` the first annotation has id 0."""
    rng = np.random.default_rng(seed)
    cats = [{"id": 2 + 3 * k, "name": f"c{k}"} for k in range(n_cat)]
    cids = [c["id"] for c in cats]
    images, anns = [], []
    for i in range(n_img):
        W, H = int(rng.integers(300, 900)), int(rng.integers(300, 900))
        img_id = 5 + 4 * i
        images.append({"id": img_id, "width": W, "height": H})
        present = [] if i == 1 else list(rng.choice(cids[:-1], size=min(3, n_cat - 1), replace=False))
        for j in range(0 if i == 1 else per_img):
            c = int(present[j % len(present)])
            side = float(rng.choice([12.0, 31.0, 32.0, 50.0, 96.0, 140.0, 300.0]))
            w, h = np.float32(side * rng.uniform(0.7, 1.3)), np.float32(side * rng.uniform(0.7, 1.3))
            x, y = np.float32(rng.uniform(0, max(W - w, 1.0))), np.float32(rng.uniform(0, max(H - h, 1.0)))
            area = [float(w) * float(h), float(w) * float(h) * 0.7, 1024.0, 9216.0][j % 4]
            crowd = int(crowd_every > 0 and len(anns) % crowd_every == crowd_every - 1)
            box = [float(x), float(y), float(w), float(h)]
            anns.append({"id": len(anns) + 1, "image_id": img_id, "category_id": c, "bbox": box, "area": area, "iscrowd": crowd})
            if j == 2:
                anns.append({"id": len(anns) + 1, "image_id": img_id, "category_id": c, "bbox": list(box), "area": area,
                             "iscrowd": 0})
    if id0:
        for a in anns:
            a["id"] -= 1
    return {"images": images, "annotations": anns, "categories": cats}


def synth_updates(gt, seed, n_upd=3, per_img=40, extra_cat=99, pin=False):
    """Detections as the detector emits them: per update a list of (image_id, fp32 xyxy at the network input size, (in_w, in_h),
    fp32 scores, category ids).  Scores on a 1/64 grid (ties within and across images), boxes near the GTs and elsewhere, zero-
    width boxes, a category id outside the GT file, one image in two updates.  ``pin``: the cases where COCO and LVIS standard
    AP coincide (<= 100 per (image, category) and <= 300 per image, positive areas, only GT categories)."""
    rng = np.random.default_rng(seed)
    imgs = list(gt["images"])
    cids = [c["id"] for c in gt["categories"]]
    by_img = defaultdict(list)
    for a in gt["annotations"]:
        by_img[a["image_id"]].append(a)
    chunks = [imgs[k::n_upd] for k in range(n_upd)]
    if not pin:
        chunks[-1] = chunks[-1] + [imgs[0]]
    ups = []
    for part in chunks:
        cur = []
        for im in part:
            W, H = im["width"], im["height"]
            s = float(rng.uniform(0.6, 1.6))
            iw, ih = max(1, int(round(W * s))), max(1, int(round(H * s)))
            cat = rng.choice(cids + ([] if pin else [extra_cat]), size=per_img).astype(np.int64)
            xywh = np.zeros((per_img, 4), np.float64)
            gts = by_img.get(im["id"], [])
            for k in range(per_img):
                if gts and rng.random() < 0.6:
                    g = gts[int(rng.integers(len(gts)))]
                    b = np.array(g["bbox"]) + rng.normal(0, 0.08, 4) * max(g["bbox"][2], g["bbox"][3])
                    b[2:] = np.maximum(b[2:], 2.0)
                    if rng.random() < 0.7:
                        cat[k] = g["category_id"]
                else:
                    wh = rng.uniform(5, 200, 2)
                    b = np.array([rng.uniform(0, W - 5), rng.uniform(0, H - 5), wh[0], wh[1]])
                if k % 17 == 5 and not pin:
                    b[2] = -1.0         # x2 - x1 + 1 = 0: a zero-area detection
                xywh[k] = b
            xyxy = np.stack([xywh[:, 0], xywh[:, 1], xywh[:, 0] + xywh[:, 2], xywh[:, 1] + xywh[:, 3]], 1) * (iw / W)
            score = (rng.integers(1, 64, per_img) / 64.0).astype(np.float32)
            cur.append((im["id"], xyxy.astype(np.float32), (iw, ih), score, cat))
        ups.append(cur)
    return ups


def pin_cases():
    """name -> (gt, updates): the cases pinned to the reference's code."""
    g0 = synth_gt(1)
    g1 = synth_gt(2, n_img=6, n_cat=5, per_img=4)
    g2 = synth_gt(3, n_img=10, n_cat=6, per_img=8, crowd_every=5, id0=True)
    return {"basic": (g0, synth_updates(g0, 11)),
            "dense": (g1, synth_updates(g1, 12, n_upd=2, per_img=260)),
            "crowd_id0": (g2, synth_updates(g2, 13, per_img=60))}


def run_oracle(gt, updates, label_to_category=None):
    res = prepare(gt, [u for upd in updates for u in upd], label_to_category)
    return evaluate(gt, res), res
