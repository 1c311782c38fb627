"""Wall time of multi-scale + flip test-time augmentation for MQ-GroundingDINO-T (engine/bbox_aug.py), next to one
``forward_chunked_device`` at the test size, measured alternately in one process; and CUDA-event times of the collect + merge
alone (``ops.bbox_aug_collect_packed`` for every pass + ``ops.nms_by_class``) on the passes' own packed rows.

    python tools/prof_bbox_aug_gdino.py [--reps 3] [--classes 80] [--out FILE.json]

Model: the full MQ-GroundingDINO-T shape (Swin-T, 6 + 6 layers, 900 queries) with synthetic weights, an 80-class prompt with
five vision queries per class; one decoded 800 x 1333 uint8 image; the default ``TEST.SCALES`` / ``TEST.RANGES`` /
``TEST.MAX_SIZE`` and ``TEST.FLIP`` (24 passes).  Wall times end with the device->host copy of the result.  Prints the card's
name and power limit with the numbers; needs a CUDA device.
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
import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--classes", type=int, default=80)
    ap.add_argument("--merge-reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_bbox_aug_gdino: a CUDA device is required (nothing is measured on the CPU)")
    from mqdet_b200 import ops
    from mqdet_b200.engine import bbox_aug
    from mqdet_b200.engine.transforms import TestTransform, upload
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    from test_gdino_asm_gpu import _build_model
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    gen = synth.Gen(7)
    model = _build_model(synth.gdino_sd(gen, 6, 6, 900), 6, 6, 900, dev)
    ids, am, pmap = synth.prompt(a.classes, 2, 256, gen)
    model.query_selector.set_query_bank(synth.query_bank(pmap, 5, gen))
    caps = {"input_ids": ids, "attention_mask": am}
    t = model.cfg.TEST
    img = upload([torch.randint(0, 256, (800, 1333, 3), generator=gen.g, dtype=torch.uint8)], dev)

    def tta():
        return bbox_aug.im_detect_bbox_aug_images(model, img, caps, pmap)

    il, _ = TestTransform(model.cfg)(img, dev)

    def single():
        out = model.forward_chunked_device(il, [caps], [pmap], chunks_per_pass=1)
        return out["det_packed"].cpu()

    res = tta()   # warm-up: every pass geometry, the prompt state, module loads
    single()
    torch.cuda.synchronize()
    times = {"tta": [], "forward_chunked_device": []}
    for _ in range(a.reps):
        for name, fn in (("tta", tta), ("forward_chunked_device", single)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            times[name].append((time.perf_counter() - t0) * 1e3)

    # collect + merge alone, on the packed rows of every pass of the image
    passes = []
    for i, rng, flip in ((i, r, f) for i, r in enumerate(t.RANGES) for f in ((False, True) if t.FLIP else (False,))):
        x = TestTransform(model.cfg, t.SCALES[i], t.MAX_SIZE)(img, dev, pad=False)[0].tensors
        h, w = x.shape[-2:]
        H, W = -(-h // 32) * 32, -(-w // 32) * 32
        if flip:
            batch = ops.hflip_pad(x, (H, W))
        else:
            batch = x.new_zeros((1, 3, H, W))
            batch[..., :h, :w] = x
        det = model.forward_chunked_device(ImageList(batch, [(h, w)]), [caps], [pmap], chunks_per_pass=1)["det_packed"][0]
        passes.append((det.clone(), (w, h), flip, rng))
    merged = ops.MergedBoxes(1, len(passes) * 900, dev)
    classes = torch.arange(1, int(t.NUM_CLASSES), dtype=torch.int32, device=dev)

    def collect_merge():
        merged.count.zero_()
        merged.overflow.zero_()
        for det, size, flip, rng in passes:
            ops.bbox_aug_collect_packed(merged, det, size, (1333, 800), flip=flip, keep_range=rng)
        return ops.nms_by_class(merged.boxes, merged.scores, merged.labels, merged.count, classes, float(t.TH), top_n=int(t.PRE_NMS_TOP_N),
                                max_out=bbox_aug.result_rows(t, merged.cap), overflow=merged.overflow)

    collect_merge()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.merge_reps):
        collect_merge()
    e1.record()
    torch.cuda.synchronize()
    rows = sum(int(d[0, -1, 0]) for d, *_ in passes)
    result = {"card": card, "passes": len(passes), "scales": list(t.SCALES), "max_size": t.MAX_SIZE, "classes": a.classes,
              "rows_collected": rows, "merged": int(merged.count[0]), "detections": len(res[0]),
              "ms_per_image": {k: v for k, v in times.items()},
              "collect_merge_ms": e0.elapsed_time(e1) / a.merge_reps}
    print(f"card (name, power limit, max SM clock): {card}")
    print(f"{len(passes)} passes, {rows} packed rows collected, {result['merged']} merged, {len(res[0])} detections")
    for k, v in times.items():
        print(f"  {k:28s} " + "  ".join(f"{x:9.1f}" for x in v) + "  ms per image")
    print(f"  {'collect + merge (events)':28s} {result['collect_merge_ms']:9.3f} ms")
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
