"""Wall-clock times of the device COCO box AP evaluator (mqdet_b200/engine/coco_eval.py) on a COCO-val-shaped synthetic set:
5000 images, 80 categories, ~37k GTs (~1 % crowd), 100 packed rows per image arriving in updates of --batch images as packed
device results; update_packed over the whole set, then accumulate + summarize, each ended by a device synchronise.  Next to it,
the numpy restatement (tests/coco_eval_oracle.py) on the first --host-images images only.

    python tools/prof_coco_eval.py [--images 5000] [--batch 8] [--host-images 250] [--out FILE.json]

Prints the card's name, power limit and max SM clock with the numbers; needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--host-images", type=int, default=250)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_coco_eval: needs a CUDA device")
    from mqdet_b200.engine.coco_eval import CocoEvaluator, CocoGroundTruth
    import coco_eval_oracle as co
    from test_coco_eval_gpu import IN_HW, ORIG_HW, coco_val_gt, coco_val_packed
    dev = torch.device("cuda:0")
    gt = coco_val_gt(5, a.images)
    ids = [im["id"] for im in gt["images"]]
    batches = [(coco_val_packed(gt, 100 + i0, ids[i0:i0 + a.batch]), ids[i0:i0 + a.batch]) for i0 in range(0, a.images, a.batch)]
    dev_batches = [(torch.from_numpy(pk).to(dev), part) for pk, part in batches]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gtd = CocoGroundTruth(gt, dev)
    torch.cuda.synchronize()
    t_gt = time.perf_counter() - t0
    ev = CocoEvaluator(gtd)
    t0 = time.perf_counter()
    for pk, part in dev_batches:
        ev.update_packed(pk, part, [IN_HW] * len(part), [ORIG_HW] * len(part))
    torch.cuda.synchronize()
    t_upd = time.perf_counter() - t0
    t0 = time.perf_counter()
    ev.accumulate()
    stats = ev.summarize()
    torch.cuda.synchronize()
    t_acc = time.perf_counter() - t0
    host = set(ids[:a.host_images])
    per = []
    for pk, part in batches:
        for b, i in enumerate(part):
            if i in host:
                n = int(pk[0, b, -1, 0])
                per.append((i, pk[0, b, :n, :4], (IN_HW[1], IN_HW[0]), pk[0, b, :n, 4], pk[0, b, :n, 5].astype(np.int64)))
    t0 = time.perf_counter()
    co.evaluate(gt, co.prepare(gt, per))
    t_host = time.perf_counter() - t0
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "images": a.images, "categories": len(gt["categories"]), "gts": len(gt["annotations"]),
           "detections": int(sum(pk[0, :, -1, 0].sum() for pk, _ in batches)), "update_packed_calls": len(batches),
           "gt_load_s": t_gt, "device_update_s": t_upd, "device_accumulate_summarize_s": t_acc, "AP": float(stats[0]),
           "host_restatement_images": a.host_images, "host_restatement_s": t_host,
           "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
