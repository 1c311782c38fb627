"""LVIS box AP with the evaluator state on the device: a drop-in for the reference's ``LvisEvaluatorFixedAP``
(maskrcnn_benchmark/data/datasets/evaluation/lvis/lvis_eval.py:766-875), fixed AP (top ``topk`` per category over the dataset)
and standard AP (top 300 per image), fed with the packed results of ``forward_chunked_device`` / ``forward_device`` without a
device-to-host copy.  The rules it reproduces are written out in DESIGN.md section 4 ("LVIS box AP rules"); the kernels are csrc/lvis_eval.cu.

The pool holds one slot per packed row.  When an update would not fit, the pool is cut to its top ``topk`` per category (300
per image) in place of the reference's per-update cut and merge, which keep the same detections (ties by arrival); that cut
reads one count back to the host.  ``update_packed`` does not otherwise synchronise: its two small per-image tables go up
through pinned memory without blocking.

Several ranks: ``synchronize_between_processes`` gathers every rank's (cut) pool with ``parallel.all_gather_rows`` and renumbers
the arrivals rank by rank, which is the reference's rank-order concatenation (lvis_eval.py:800-806); as in the reference, every
rank then holds all detections and only the main process summarises."""
import json

import numpy as np
import torch
import torch.distributed as dist

from .. import ops, parallel
from .._lib import MqdetError

IOU_THRS = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1, endpoint=True)
REC_THRS = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1, endpoint=True)
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]
FREQ_LBL = ["r", "c", "f"]
STANDARD_MAX_DETS = 300


def _pairs(img_idx, cat_idx):
    return (np.asarray(img_idx, np.int64) << 32) | np.asarray(cat_idx, np.int64)


class LvisGroundTruth:
    """An LVIS-format annotation file (path or parsed dict) as device tables, built once.  Only what box AP reads is kept: the
    images with their ``neg_category_ids`` / ``not_exhaustive_category_ids``, the categories with their ``frequency``, and the
    annotations with 0 < area < inf (LVIS.get_ann_ids), in annotation order within each (image, category) pair."""

    def __init__(self, annotations, device=None):
        if isinstance(annotations, str):
            with open(annotations) as f:
                annotations = json.load(f)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.dataset = annotations
        self.img_ids = np.array(sorted(im["id"] for im in annotations["images"]), dtype=np.int64)
        self.cat_ids = np.array(sorted(c["id"] for c in annotations["categories"]), dtype=np.int64)
        self.img_pos = {int(i): k for k, i in enumerate(self.img_ids)}
        cat_pos = {int(c): k for k, c in enumerate(self.cat_ids)}
        freq = {c["id"]: c["frequency"] for c in annotations["categories"]}
        self.freq_groups = [[k for k, c in enumerate(self.cat_ids) if freq[int(c)] == lbl] for lbl in FREQ_LBL]
        rows = []
        for a in annotations["annotations"]:
            if a["image_id"] in self.img_pos and a["category_id"] in cat_pos and 0 < a["area"] < float("inf"):
                if int(a["id"]) < 1:
                    raise ValueError(f"annotation id {a['id']}: LVIS match arrays use 0 for 'unmatched', ids must be >= 1")
                rows.append((self.img_pos[a["image_id"]], cat_pos[a["category_id"]], a))
        neg, nel = [], []
        for im in annotations["images"]:
            k = self.img_pos[im["id"]]
            neg += [(k, cat_pos[c]) for c in im["neg_category_ids"] if c in cat_pos]
            nel += [(k, cat_pos[c]) for c in im["not_exhaustive_category_ids"] if c in cat_pos]

        def table(p):
            p = np.unique(np.array(p, np.int64).reshape(-1, 2), axis=0) if len(p) else np.zeros((0, 2), np.int64)
            return torch.from_numpy(np.sort(_pairs(p[:, 0], p[:, 1]))).to(dev)

        self.dev = gt_tables(rows, len(self.cat_ids), lambda a: a.get("ignore", 0), dev)
        self.dev.update({"cat_ids": torch.from_numpy(self.cat_ids.astype(np.int32)).to(dev),
                         "pos_pairs": torch.unique(self.dev["gt_pair"]), "neg_pairs": table(neg), "nel_pairs": table(nel)})
        self.device = dev
        self.det_area_filter = True


def gt_tables(rows, n_cat, ignore, dev):
    """The GT side of the device evaluation, shared by the LVIS and COCO ground truths.  rows: (image index, category index,
    annotation dict) of the GTs that take part; ``ignore(annotation)`` -> its ignore flag.  -> device tables: gt_pair (image << 32 |
    category, sorted, annotation order within a pair), gt_box fp64 xywh, gt_area fp64 (the ``area`` field), gt_ignore, gt_id,
    num_gt int32 [K, 4] (GTs not ignored per category and area range), and the IoU / recall thresholds and area ranges."""
    order = sorted(range(len(rows)), key=lambda j: (rows[j][0], rows[j][1], j))
    rows = [rows[j] for j in order]
    gi = np.array([r[0] for r in rows], np.int64)
    gc = np.array([r[1] for r in rows], np.int64)
    box = np.array([r[2]["bbox"] for r in rows], np.float64).reshape(-1, 4)
    area = np.array([r[2]["area"] for r in rows], np.float64)
    ign = np.array([1 if ignore(r[2]) else 0 for r in rows], np.int32)
    num_gt = np.zeros((n_cat, 4), np.int32)
    for a, (lo, hi) in enumerate(AREA_RNG):
        ok = (ign == 0) & (area >= lo) & (area <= hi)
        np.add.at(num_gt[:, a], gc[ok], 1)
    return {"gt_pair": torch.from_numpy(_pairs(gi, gc)).to(dev), "gt_box": torch.from_numpy(box).to(dev),
            "gt_area": torch.from_numpy(area).to(dev), "gt_ignore": torch.from_numpy(ign).to(dev),
            "gt_id": torch.tensor([int(r[2]["id"]) for r in rows], dtype=torch.int64).to(dev),
            "num_gt": torch.from_numpy(num_gt).to(dev), "iou_thrs": torch.from_numpy(IOU_THRS).to(dev),
            "rec_thrs": torch.from_numpy(REC_THRS).to(dev), "area_rng": torch.tensor(AREA_RNG, dtype=torch.float64).to(dev)}


class LvisEvaluatorFixedAP:
    """Drop-in for the reference class.  ``update`` takes the reference's input (a list of (image_id, prediction) with
    ``boxes`` xyxy fp32 at the original size, ``scores``, ``labels``: dicts or BoxLists); ``update_packed`` takes the detector's
    packed device result directly.  ``label_to_category`` (int tensor [L]) maps labels to category ids where they differ.
    ``pool_rows`` bounds the device pool; an update larger than the pool after a cut raises."""

    def __init__(self, gt, topk=10000, fixed_ap=True, pool_rows=1 << 24, label_to_category=None):
        if not isinstance(gt, LvisGroundTruth):
            gt = LvisGroundTruth(gt)
        if len(gt.img_ids) >= 1 << 31 or len(gt.cat_ids) >= 1 << 31:
            raise MqdetError("lvis_eval: too many images or categories")
        self.gt, self.topk, self.fixed_ap = gt, int(topk), bool(fixed_ap)
        dev = gt.device
        self.pool = ops.LvisPool(pool_rows, dev)
        self.n = 0              # pool slots in use (host-known; rows of a cut pool are dense)
        self.next_seq = 0
        self.bad = torch.zeros((1,), dtype=torch.int32, device=dev)
        self.label_map = None if label_to_category is None else label_to_category.to(dev, torch.int32).contiguous()
        self.eval, self.results, self.stats = {}, {}, None
        self.last = None

    # -- updates ------------------------------------------------------------------------------------------------------------
    def update(self, predictions, is_cur_results=False):
        if is_cur_results:
            raise NotImplementedError("lvis_eval: result dicts are a debug input of the reference; pass predictions")
        predictions = list(predictions)
        if not predictions:
            return
        rows = []
        for _, p in predictions:
            if isinstance(p, dict):
                b, s, l = p["boxes"], p["scores"], p["labels"]
            else:
                b, s, l = p.bbox, p.get_field("scores"), p.get_field("labels")
            rows.append(torch.cat([b.reshape(-1, 4).float(), s.reshape(-1, 1).float(), l.reshape(-1, 1).float()], 1))
        M = max(max(r.shape[0] for r in rows), 1)
        packed = torch.zeros((1, len(rows), M + 1, 6), dtype=torch.float32, device=self.gt.device)
        for b, r in enumerate(rows):
            packed[0, b, :r.shape[0]] = r
            packed[0, b, M, 0] = r.shape[0]
        ones = [(1, 1)] * len(rows)
        self.update_packed(packed, [i for i, _ in predictions], ones, ones)

    def update_packed(self, det_packed, image_ids, image_sizes, orig_sizes):
        """det_packed: fp32 [B, max_out + 1, 6] (``forward_device``) or [G, B, max_out + 1, 6] (``forward_chunked_device``, a
        chunk's rows after the previous chunk's for each image); image_sizes / orig_sizes: (h, w) of the network input and of
        the original image per image."""
        pk = det_packed if det_packed.dim() == 4 else det_packed.unsqueeze(0)
        G, B, M1, _ = pk.shape
        if len(image_ids) != B or len(image_sizes) != B or len(orig_sizes) != B:
            raise MqdetError(f"lvis_eval: {B} images in the packed result, {len(image_ids)} ids / sizes given")
        rows = G * B * (M1 - 1)
        if self.n + rows > self.pool.cap:
            self._cut()
        if self.n + rows > self.pool.cap:
            raise MqdetError(f"lvis_eval: pool of {self.pool.cap} rows full ({self.n} kept + {rows} arriving); raise pool_rows")
        img_idx = self._upload(torch.tensor([self.gt.img_pos.get(int(i), -1) for i in image_ids], dtype=torch.int32))
        ratios = self._upload(torch.tensor([[np.float32(float(o[1]) / float(s[1])), np.float32(float(o[0]) / float(s[0]))]
                                            for s, o in zip(image_sizes, orig_sizes)], dtype=torch.float32))
        ops.lvis_collect(self.pool, self.n, self.next_seq, pk.contiguous(), img_idx, ratios, self.gt.dev["cat_ids"],
                         label_map=self.label_map, need_img=not self.fixed_ap, bad=self.bad)
        self.n += rows
        self.next_seq += rows
        self.eval = {}

    def _upload(self, t):
        return upload(t, self.gt.device)

    def _cut(self):
        """Keep the top ``topk`` per category (fixed AP) or 300 per image (standard) of the pool, densely."""
        by_image = not self.fixed_ap
        groups = len(self.gt.img_ids) if by_image else len(self.gt.cat_ids)
        dst = ops.LvisPool(self.pool.cap, self.gt.device)
        count = ops.lvis_cut(self.pool, self.n, dst, by_image=by_image, n_groups=groups,
                             k=STANDARD_MAX_DETS if by_image else self.topk)
        self.pool, self.n = dst, int(count.item())

    def synchronize_between_processes(self, group=None):
        """Every rank gets the detections of all ranks, rank 0's first: arrival numbers of rank r are shifted by the arrivals of
        ranks 0 .. r-1.  Identity without an initialised process group of several ranks."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return
        self._cut()
        self.pool, self.n, self.next_seq, (bad,) = gather_pool(self.pool, self.n, self.next_seq, [self.bad], group)
        self.bad.fill_(bad)
        self.eval = {}

    # -- evaluation ---------------------------------------------------------------------------------------------------------
    def accumulate(self, want_match=False):
        if int(self.bad.item()):
            raise MqdetError(f"lvis_eval: {int(self.bad.item())} packed results had a count row outside [0, max_out]")
        self._cut()
        out = ops.lvis_evaluate(self.pool, self.n, self.gt, want_match=want_match)
        self.last = out
        self.eval = {"precision": out["precision"].cpu().numpy(), "recall": out["recall"].cpu().numpy()}
        return self.eval

    def summarize(self):
        """On the main process: prints what the reference prints (fixed AP: the notice on categories with fewer than ``topk``
        detections, the result lines of ``LVISEval.run`` and of its second ``print_results``, the copypaste line; standard: the
        result lines twice) and returns the lines (fixed AP) or None (standard), as the reference does."""
        if dist.is_available() and dist.is_initialized() and dist.get_rank() != 0:
            return None
        if not self.eval:
            self.accumulate()
        max_dets = -1 if self.fixed_ap else STANDARD_MAX_DETS
        self.results, strings = summarize(self.eval["precision"], self.eval["recall"], self.gt.freq_groups, max_dets)
        self.stats = np.array([self.results[k] for k in ("AP", "AP50", "AP75", "APs", "APm", "APl", "APr", "APc", "APf")])
        if self.fixed_ap:
            counts = torch.bincount(self.pool.cat[:self.n].long().clamp(min=-1) + 1, minlength=len(self.gt.cat_ids) + 1)[1:]
            missing = int(((counts > 0) & (counts < self.topk)).sum().item())
            if missing:
                print(f"\n===\n{missing} classes had less than {self.topk} detections!\n"
                      f"Outputting {self.topk} detections for each class will improve AP further.\n"
                      f"If using detectron2, please use the lvdevil/infer_topk.py script to "
                      f"output a results file with {self.topk} detections for each class.\n===")
        for _ in range(2):
            for line in strings:
                print(line)
        if not self.fixed_ap:
            return None
        print("copypaste: %s,%s", ",".join(k for k in self.results if k.startswith("AP")), "path")
        return strings

    def detections(self):
        """The evaluated detections (after the cut) on the host: image id, category id, fp32 xywh, score, arrival number."""
        n = self.n
        img = self.pool.img[:n].cpu().numpy()
        return {"image_id": np.where(img >= 0, self.gt.img_ids[np.maximum(img, 0)], -1),
                "category_id": self.gt.cat_ids[np.maximum(self.pool.cat[:n].cpu().numpy(), 0)],
                "bbox": self.pool.box[:n].cpu().numpy(), "score": self.pool.score[:n].cpu().numpy(),
                "seq": self.pool.seq[:n].cpu().numpy(), "valid": self.pool.cat[:n].cpu().numpy() >= 0}

    def save_instances_results(self, save_path):
        """The kept detections as LVIS result dicts, by image id (then category, score descending, arrival)."""
        if self.fixed_ap:
            self._cut()
        d = self.detections()
        keep = np.nonzero(d["valid"] & (d["image_id"] >= 0))[0]
        keep = keep[np.lexsort((d["seq"][keep], -d["score"][keep].astype(np.float64), d["category_id"][keep], d["image_id"][keep]))]
        inst = [{"image_id": int(d["image_id"][i]), "category_id": int(d["category_id"][i]),
                 "bbox": [float(v) for v in d["bbox"][i]], "score": float(d["score"][i])} for i in keep]
        print("saving instances results to ", save_path)
        with open(save_path, "w") as f:
            json.dump(inst, f)


def upload(t, dev):
    """Host table -> device without a host synchronisation (pinned source, asynchronous copy)."""
    if dev.type == "cuda":
        t = t.pin_memory()
    return t.to(dev, non_blocking=True)


def gather_pool(pool, n, next_seq, counters, group=None):
    """All ranks' pool[:n] rows, rank 0's first, with rank r's arrival numbers shifted by the arrivals of ranks 0 .. r-1, and the
    sums of the int32 [1] ``counters`` over the ranks.  -> (pool, rows, arrivals, [counter sums])."""
    dev = pool.score.device
    rows = torch.cat([pool.score[:n].view(torch.int32)[:, None], pool.box[:n].view(torch.int32), pool.img[:n, None],
                      pool.cat[:n, None], pool.seq[:n].view(torch.int32).view(n, 2)], 1)
    head = torch.tensor([n, next_seq] + [int(c.item()) for c in counters], dtype=torch.int64, device=dev)
    parts, heads = parallel.all_gather_rows(rows, head, group)
    total = sum(int(h[0]) for h in heads)
    out = ops.LvisPool(max(pool.cap, total), dev)
    o = base = 0
    for part, h in zip(parts, heads):
        k = int(h[0])
        out.score[o:o + k] = part[:, 0].view(torch.float32)
        out.box[o:o + k] = part[:, 1:5].contiguous().view(torch.float32)
        out.img[o:o + k], out.cat[o:o + k] = part[:, 5], part[:, 6]
        out.seq[o:o + k] = part[:, 7:9].contiguous().view(torch.int64)[:, 0] + base
        o += k
        base += int(h[1])
    return out, total, base, [sum(int(h[2 + j]) for h in heads) for j in range(len(counters))]


def summarize(precision, recall, freq_groups, max_dets):
    """LVISEval.summarize / print_results on the accumulated host arrays -> (results dict in the reference's key order, the
    printed lines).  Means are numpy's, as in the reference."""

    def _s(kind, iou_thr=None, area="all", fg=None):
        aidx = [AREA_LBL.index(area)]
        s = precision if kind == "ap" else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        if kind == "ap":
            s = s[:, :, freq_groups[fg], aidx] if fg is not None else s[:, :, :, aidx]
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
        if len(key) > 2 and key[2].isdigit():
            iou = "{:0.2f}".format(float(key[2:]) / 100)
        else:
            iou = "{:0.2f}:{:0.2f}".format(IOU_THRS[0], IOU_THRS[-1])
        grp = key[2] if len(key) > 2 and key[2] in ["r", "c", "f"] else "all"
        area = key[2] if len(key) > 2 and key[2] in ["s", "m", "l"] else "all"
        lines.append(tpl.format(title, typ, iou, area, max_dets, grp, value))
    return r, lines
