"""Wall-clock times of the device LVIS evaluator (mqdet_b200/engine/lvis_eval.py) on a minival-shaped synthetic set: 5000
images, 1203 categories, ~50k GTs, 31 chunks x 100 detections per image arriving in updates of --batch images as packed
device results; update_packed over the whole set, then accumulate + summarize, each ended by a device synchronise.  Next to it,
the numpy restatement (tests/lvis_eval_oracle.py) on the first --host-images images only (it runs per pair in Python).

    python tools/prof_lvis_eval.py [--images 5000] [--batch 8] [--fixed 1] [--host-images 50] [--out FILE.json]

Prints the card's name and power limit with the numbers; needs a CUDA device.
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
    ap.add_argument("--cats", type=int, default=1203)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--fixed", type=int, default=1)
    ap.add_argument("--host-images", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_lvis_eval: needs a CUDA device")
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    import lvis_eval_oracle as lo
    dev = torch.device("cuda:0")
    gt = lo.minival_gt(5, a.images, a.cats)
    ids = [im["id"] for im in gt["images"]]
    batches = []
    for i0 in range(0, a.images, a.batch):
        part = ids[i0:i0 + a.batch]
        batches.append((lo.minival_packed(gt, 100 + i0, part), part))
    dev_batches = [(torch.from_numpy(pk).to(dev), part) for pk, part in batches]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gtd = LvisGroundTruth(gt, dev)
    torch.cuda.synchronize()
    t_gt = time.perf_counter() - t0
    ev = LvisEvaluatorFixedAP(gtd, fixed_ap=bool(a.fixed))
    t0 = time.perf_counter()
    for pk, part in dev_batches:
        ev.update_packed(pk, part, [lo.MINIVAL_IN_HW] * len(part), [lo.MINIVAL_ORIG_HW] * len(part))
    torch.cuda.synchronize()
    t_upd = time.perf_counter() - t0
    t0 = time.perf_counter()
    ev.accumulate()
    ev.summarize()
    torch.cuda.synchronize()
    t_acc = time.perf_counter() - t0
    # the restatement on the first host-images images
    sub = {"images": gt["images"][: a.host_images], "categories": gt["categories"],
           "annotations": [x for x in gt["annotations"] if x["image_id"] <= a.host_images]}
    t0 = time.perf_counter()
    o = lo.Oracle(sub, 10000, bool(a.fixed))
    for pk, part in batches:
        if part[0] > a.host_images:
            break
        keep = [k for k, i in enumerate(part) if i <= a.host_images]
        o.update(lo.oracle_update_from_packed(pk[:, keep], [part[k] for k in keep], lo.MINIVAL_IN_HW, lo.MINIVAL_ORIG_HW))
    o.evaluate()
    o.summarize()
    t_host = time.perf_counter() - t0
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "images": a.images, "categories": a.cats, "gts": len(gt["annotations"]), "fixed_ap": bool(a.fixed),
           "rows": a.images * ((a.cats + 39) // 40) * 100,
           "gt_load_s": t_gt, "device_update_s": t_upd, "device_accumulate_summarize_s": t_acc,
           "AP": float(ev.results["AP"]), "host_restatement_images": a.host_images, "host_restatement_s": t_host,
           "peak_alloc_gb": torch.cuda.max_memory_allocated() / 1e9}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
