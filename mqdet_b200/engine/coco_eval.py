"""COCO-style box AP (ODinW, COCO val) with the evaluator state on the device, as the reference scores it: od_to_grounding/od_eval.py
(prepare_for_coco_detection, evaluate_predictions_on_coco, summarize_per_category, COCOResults) through pycocotools' COCOeval
(iouType "bbox").  It is fed with the packed results of ``forward_device`` / ``forward_chunked_device`` without a device-to-host
copy, or with the reference's (image_id, BoxList) list.  The rules are DESIGN.md section 4 ("COCO box AP rules"); the kernels are
the LVIS evaluator's (csrc/lvis_eval.cu), given crowd GTs, no federated filter, no detection area filter and maxDets 1 / 10 / 100.

The pool holds one slot per packed row.  When an update would not fit, the pool is cut to its top 100 per (image, category)
(score descending, arrival on ties), which keeps what pycocotools' evaluateImg keeps; that cut reads one count back to the host.
``update_packed`` does not otherwise synchronise: its two small per-image tables go up through pinned memory without blocking."""
import json
from collections import OrderedDict

import numpy as np
import torch
import torch.distributed as dist

from .. import ops
from .._lib import MqdetError
from .lvis_eval import AREA_LBL, IOU_THRS, gather_pool, gt_tables, upload

MAX_DETS = [1, 10, 100]
_SUMMARY = [(1, None, "all", 100), (1, .5, "all", 100), (1, .75, "all", 100), (1, None, "small", 100),
            (1, None, "medium", 100), (1, None, "large", 100), (0, None, "all", 1), (0, None, "all", 10),
            (0, None, "all", 100), (0, None, "small", 100), (0, None, "medium", 100), (0, None, "large", 100)]


class CocoGroundTruth:
    """A COCO-format annotation file (path or parsed dict) as device tables, built once: the images (with ``width`` /
    ``height``), the categories, and every annotation of a listed image and category with its ``bbox``, ``area``, ``iscrowd``
    and ``id``, in annotation order within each (image, category) pair.  pycocotools sets a GT's ignore flag to ``iscrowd``."""

    def __init__(self, annotations, device=None):
        if isinstance(annotations, str):
            with open(annotations) as f:
                annotations = json.load(f)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.dataset = annotations
        self.img_ids = np.array(sorted(im["id"] for im in annotations["images"]), dtype=np.int64)
        self.cat_ids = np.array(sorted(c["id"] for c in annotations["categories"]), dtype=np.int64)
        self.img_pos = {int(i): k for k, i in enumerate(self.img_ids)}
        self.img_wh = {im["id"]: (im["width"], im["height"]) for im in annotations["images"]}
        self.cat_names = {c["id"]: c["name"] for c in annotations["categories"]}
        cat_pos = {int(c): k for k, c in enumerate(self.cat_ids)}
        rows = [(self.img_pos[a["image_id"]], cat_pos[a["category_id"]], a) for a in annotations["annotations"]
                if a["image_id"] in self.img_pos and a["category_id"] in cat_pos]
        self.dev = gt_tables(rows, len(self.cat_ids), lambda a: a.get("iscrowd", 0), dev)
        self.dev.update({"cat_ids": torch.from_numpy(self.cat_ids.astype(np.int32)).to(dev),
                         "gt_crowd": self.dev["gt_ignore"],      # ignore = iscrowd, so the two flags are one array
                         "max_dets": torch.tensor(MAX_DETS, dtype=torch.int32).to(dev)})
        self.device = dev
        self.det_area_filter = False


class CocoEvaluator:
    """``update`` takes the reference's input, a list of (image_id, prediction): a BoxList (xyxy at ``size``, resized to the GT
    image's width / height as prepare_for_coco_detection does) or a dict with ``boxes`` (xyxy at the GT image's size),
    ``scores`` and ``labels``.  ``update_packed`` takes the detector's packed device result directly.  ``label_to_category``
    (the reference's ``contiguous_category_id_to_json_id``: a dict, or an int tensor [L] with -1 for labels it lacks) maps labels
    to category ids; labels outside it are dropped.  ``pool_rows`` bounds the device pool; an update larger than the pool after
    a cut raises."""

    def __init__(self, gt, label_to_category=None, pool_rows=1 << 22):
        if not isinstance(gt, CocoGroundTruth):
            gt = CocoGroundTruth(gt)
        if len(gt.img_ids) * max(len(gt.cat_ids), 1) >= 1 << 31:
            raise MqdetError("coco_eval: images x categories must stay below 2^31")
        self.gt = gt
        dev = gt.device
        self.pool = ops.LvisPool(pool_rows, dev)
        self.n = 0
        self.next_seq = 0
        self.bad = torch.zeros((1,), dtype=torch.int32, device=dev)
        self.bad_img = torch.zeros((1,), dtype=torch.int32, device=dev)
        if isinstance(label_to_category, dict):
            table = torch.full((max(label_to_category, default=-1) + 1,), -1, dtype=torch.int32)
            for k, v in label_to_category.items():
                if k >= 0:
                    table[k] = v
            label_to_category = table
        self.label_map = None if label_to_category is None else label_to_category.to(dev, torch.int32).contiguous()
        self.eval, self.stats, self.last = {}, None, None

    # -- updates ------------------------------------------------------------------------------------------------------------
    def update(self, predictions):
        predictions = list(predictions)
        if not predictions:
            return
        rows, in_hw, orig_hw = [], [], []
        for img_id, p in predictions:
            wh = self.gt.img_wh.get(int(img_id))
            if isinstance(p, dict):
                b, s, l = p["boxes"], p["scores"], p["labels"]
                size = wh or (1, 1)
            else:
                if p.mode != "xyxy":
                    raise MqdetError("coco_eval: BoxLists in xyxy mode required")
                b, s, l, size = p.bbox, p.get_field("scores"), p.get_field("labels"), p.size
            wh = wh or size
            rows.append(torch.cat([b.reshape(-1, 4).float(), s.reshape(-1, 1).float(), l.reshape(-1, 1).float()], 1))
            in_hw.append((size[1], size[0]))
            orig_hw.append((wh[1], wh[0]))
        M = max(max(r.shape[0] for r in rows), 1)
        packed = torch.zeros((1, len(rows), M + 1, 6), dtype=torch.float32, device=self.gt.device)
        for b, r in enumerate(rows):
            packed[0, b, :r.shape[0]] = r
            packed[0, b, M, 0] = r.shape[0]
        self.update_packed(packed, [i for i, _ in predictions], in_hw, orig_hw)

    def update_packed(self, det_packed, image_ids, image_sizes, orig_sizes):
        """det_packed: fp32 [B, max_out + 1, 6] (``forward_device``) or [G, B, max_out + 1, 6] (``forward_chunked_device``);
        image_sizes / orig_sizes: (h, w) of the network input and of the GT image (its ``height`` / ``width``) per image."""
        pk = det_packed if det_packed.dim() == 4 else det_packed.unsqueeze(0)
        G, B, M1, _ = pk.shape
        if len(image_ids) != B or len(image_sizes) != B or len(orig_sizes) != B:
            raise MqdetError(f"coco_eval: {B} images in the packed result, {len(image_ids)} ids / sizes given")
        rows = G * B * (M1 - 1)
        if self.n + rows > self.pool.cap:
            self._cut()
        if self.n + rows > self.pool.cap:
            raise MqdetError(f"coco_eval: pool of {self.pool.cap} rows full ({self.n} kept + {rows} arriving); raise pool_rows")
        img_idx = self._upload(torch.tensor([self.gt.img_pos.get(int(i), -1) for i in image_ids], dtype=torch.int32))
        ratios = self._upload(torch.tensor([[np.float32(float(o[1]) / float(s[1])), np.float32(float(o[0]) / float(s[0]))]
                                            for s, o in zip(image_sizes, orig_sizes)], dtype=torch.float32))
        ops.lvis_collect(self.pool, self.n, self.next_seq, pk.contiguous(), img_idx, ratios, self.gt.dev["cat_ids"],
                         label_map=self.label_map, need_img=True, need_cat=True, wh_plus_one=True, bad=self.bad,
                         bad_img=self.bad_img)
        self.n += rows
        self.next_seq += rows
        self.eval = {}

    def _upload(self, t):
        return upload(t, self.gt.device)

    def _cut(self):
        """Keep the top 100 per (image, category) of the pool, densely."""
        K = len(self.gt.cat_ids)
        dst = ops.LvisPool(self.pool.cap, self.gt.device)
        count = ops.lvis_cut(self.pool, self.n, dst, group=ops.CUT_BY_PAIR, n_groups=len(self.gt.img_ids) * K, n_cat=K,
                             k=MAX_DETS[-1])
        self.pool, self.n = dst, int(count.item())

    def synchronize_between_processes(self, group=None):
        """Every rank gets the detections of all ranks, rank 0's first (arrivals of rank r after those of ranks 0 .. r-1).
        Identity without an initialised process group of several ranks."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return
        self._cut()
        self.pool, self.n, self.next_seq, (bad, bad_img) = gather_pool(self.pool, self.n, self.next_seq,
                                                                       [self.bad, self.bad_img], group)
        self.bad.fill_(bad)
        self.bad_img.fill_(bad_img)
        self.eval = {}

    # -- evaluation ---------------------------------------------------------------------------------------------------------
    def accumulate(self, want_match=False):
        """-> {"precision" fp64 [10, 101, K, 4, 3], "recall" fp64 [10, K, 4, 3]} (pycocotools' layout) on the host."""
        if int(self.bad.item()):
            raise MqdetError(f"coco_eval: {int(self.bad.item())} packed results had a count row outside [0, max_out]")
        if int(self.bad_img.item()):
            raise MqdetError(f"coco_eval: Results do not correspond to current coco set ({int(self.bad_img.item())} "
                             f"detections on images outside the GT file)")
        self._cut()
        out = ops.lvis_evaluate(self.pool, self.n, self.gt, want_match=want_match)
        self.last = out
        self.eval = {"precision": out["precision"].cpu().numpy(), "recall": out["recall"].cpu().numpy()}
        return self.eval

    def summarize(self):
        """On the main process: prints COCOeval.summarize's 12 lines, sets and returns ``stats`` [12]."""
        if dist.is_available() and dist.is_initialized() and dist.get_rank() != 0:
            return None
        if not self.eval:
            self.accumulate()
        self.stats, lines = summarize(self.eval["precision"], self.eval["recall"])
        for line in lines:
            print(line)
        return self.stats

    def results(self):
        """On the main process: COCOResults("bbox") after update, {"bbox": OrderedDict(AP, AP50, AP75, APs, APm, APl)}; None on
        the other ranks, as ``summarize``."""
        if self.stats is None and self.summarize() is None:
            return None
        return OrderedDict([("bbox", OrderedDict((k, self.stats[i]) for i, k in enumerate(["AP", "AP50", "AP75", "APs", "APm",
                                                                                            "APl"])))])

    def write_per_category_csv(self, path):
        """What summarize_per_category writes: per metric the mean over entries > -1 is only the gate; each category's value
        and their average are means over all its entries, -1 included, as in the reference."""
        if not self.eval:
            self.accumulate()
        text = per_category_csv(self.eval["precision"], [int(c) for c in self.gt.cat_ids], self.gt.cat_names)
        with open(path, "w") as f:
            f.write(text)
        return text

    def detections(self):
        """The evaluated detections (after the cut) on the host: image id, category id, fp32 xywh, score, arrival number."""
        n = self.n
        img = self.pool.img[:n].cpu().numpy()
        return {"image_id": np.where(img >= 0, self.gt.img_ids[np.maximum(img, 0)], -1),
                "category_id": self.gt.cat_ids[np.maximum(self.pool.cat[:n].cpu().numpy(), 0)],
                "bbox": self.pool.box[:n].cpu().numpy(), "score": self.pool.score[:n].cpu().numpy(),
                "seq": self.pool.seq[:n].cpu().numpy()}


def _index(s, iou_thr, area, max_dets, ap):
    if iou_thr is not None:
        s = s[np.where(iou_thr == IOU_THRS)[0]]
    aind, mind = [AREA_LBL.index(area)], [MAX_DETS.index(max_dets)]
    return s[:, :, :, aind, mind] if ap else s[:, :, aind, mind]


def _iou_str(iou_thr):
    return "{:0.2f}:{:0.2f}".format(IOU_THRS[0], IOU_THRS[-1]) if iou_thr is None else "{:0.2f}".format(iou_thr)


def summarize(precision, recall):
    """COCOeval.summarize on the accumulated host arrays -> (stats [12], the printed lines).  Means are numpy's."""
    stats, lines = np.zeros((12,)), []
    for i, (ap, iou_thr, area, max_dets) in enumerate(_SUMMARY):
        s = _index(precision if ap else recall, iou_thr, area, max_dets, ap)
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        lines.append(" {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}".format(
            "Average Precision" if ap else "Average Recall", "(AP)" if ap else "(AR)", _iou_str(iou_thr), area, max_dets, mean_s))
        stats[i] = mean_s
    return stats, lines


def per_category_csv(precision, cat_ids, cat_names):
    """summarize_per_category's text: a title row, then AP, AP50, APs, APm, APl rows (maxDets 100)."""
    out = ["metric, " + "".join("{}, ".format(cat_names[c]) for c in cat_ids) + "avg \n"]
    for iou_thr, area in ((None, "all"), (.5, "all"), (None, "small"), (None, "medium"), (None, "large")):
        row = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ], ".format("Average Precision", "(AP)", _iou_str(iou_thr),
                                                                                    area, 100)
        s = _index(precision, iou_thr, area, 100, True)
        if len(s[s > -1]) != 0:
            avg = 0.0
            for i in range(len(cat_ids)):
                row += "{}, ".format(np.mean(s[:, :, i, :]))
                avg += np.mean(s[:, :, i, :])
            row += "{} \n".format(avg / len(cat_ids))
        out.append(row)
    return "".join(out)
