"""Throughput of MQ-GLIP-T evaluation on images of many sizes: batches that split at every target-size change (the default of
``online_update.make_batches`` and the only form before padded batches) against the reference's test-loader batches
(``reference_test_batches(..., TEST.IMS_PER_BATCH = 8, ASPECT_RATIO_GROUPING)``, each padded to its largest image).
    python tools/prof_mixed_batches.py [--images 256] [--rounds 3] [--reps 20] [--out FILE]
Synthetic MQ-GLIP-T (80-class prompt, K = 5) at MIN_SIZE_TEST 800 / MAX_SIZE_TEST 1333; decoded uint8 images drawn (fixed seed)
from a list of COCO-like original sizes.  Each batch goes through ``TestTransform`` (``mixed_sizes=True`` for the padded batches),
``forward_device`` and one device-to-host copy of the packed detections; the two batchings alternate within every round and each
is timed over the whole set (host clock around work ending in a device synchronise, after a warm-up pass over the set).  The
mixed ``test_transform`` launch is also timed alone (CUDA events around ``reps`` launches, one padded batch of 8).

The CUDA-graph engine runs the same reference batches twice: ``InferenceEngine.run_batches`` over the transformed batches
(device ImageLists) and ``run_images`` over the decoded images (upload and transform on its copy stream).  Its first pass captures
one graph per padded shape and is reported apart (captures, capture seconds, distinct shapes); the timed rounds replay only.
MQ-GroundingDINO-T runs ``--gdino-images`` COCO-like images at one image per batch, as the reference's GroundingDINO test loader
does, through eager ``forward_device`` and through ``GroundingDINOEngine.run_batches``.  Each engine row reports peak
``max_memory_allocated`` and the device memory held per live graph (allocated and reserved growth over the capture pass, less the
staging buffers, divided by the graphs captured).  The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout (and to
--out)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from mqdet_b200 import _lib, ops
from mqdet_b200.config import mq_glip_t_cfg
from mqdet_b200.engine.batches import reference_test_batches
from mqdet_b200.engine.transforms import TestTransform, upload
from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
from tools import synth
from tools.prof_gcp_queries import card, timed

# (height, width) of COCO-like originals: the common 640-wide landscapes and portraits, squares, and a few odd ones
SIZES = [(480, 640), (427, 640), (424, 640), (640, 480), (640, 427), (612, 612), (640, 640), (375, 500), (500, 375), (333, 500),
         (360, 640), (640, 360), (512, 640), (640, 512), (478, 640), (481, 640)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--gdino-images", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_mixed_batches: needs a CUDA device")
    _lib.load()
    dev = torch.device("cuda:0")
    info = card()
    gen = synth.Gen(99)
    sd = synth.detector_sd(gen)
    cfg = mq_glip_t_cfg()
    model = GeneralizedVLRCNN_New(cfg)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            sd[k] = v
    model.load_state_dict(sd, strict=True)
    del sd
    model = model.to(dev).eval()
    ids, am, pmap = synth.prompt(80, 2, 256, gen)
    model.query_selector.set_query_bank(synth.query_bank(pmap, 5, gen))
    caps = {"input_ids": ids, "attention_mask": am}
    rng = np.random.default_rng(7)
    hw = [SIZES[i] for i in rng.integers(0, len(SIZES), args.images)]
    images = upload([rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in hw], dev)   # decoded images already on the device
    tf = TestTransform(cfg)

    split, cur = [], []                       # consecutive images of one target size, at most 8 per batch
    for i, (h, w) in enumerate(hw):
        if cur and (len(cur) == 8 or tf.target_size(*hw[cur[0]]) != tf.target_size(h, w)):
            split.append(cur)
            cur = []
        cur.append(i)
    split.append(cur)
    ref = reference_test_batches(hw, cfg.TEST.IMS_PER_BATCH, cfg.DATALOADER.ASPECT_RATIO_GROUPING)
    plans = {"size_split": (split, False), "reference_batches": (ref, True)}

    def run(batches, mixed):
        for idx in batches:
            il, _ = tf([images[i] for i in idx], dev, mixed_sizes=mixed)
            model.forward_device(il, caps, pmap)["det_packed"].cpu()

    for batches, mixed in plans.values():    # warm-up: every batch shape of both plans
        run(batches, mixed)
    secs = {k: [] for k in plans}
    for _ in range(args.rounds):
        for name, (batches, mixed) in plans.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(batches, mixed)
            torch.cuda.synchronize()
            secs[name].append(time.perf_counter() - t0)
    first = ref[0]
    xt = [ops.resize_coeffs(hw[i][1], tf.target_size(*hw[i])[1], dev) for i in first]
    yt = [ops.resize_coeffs(hw[i][0], tf.target_size(*hw[i])[0], dev) for i in first]
    out_hw = [tf.target_size(*hw[i]) for i in first]
    Hp, Wp = (-(-max(h for h, _ in out_hw) // 32) * 32, -(-max(w for _, w in out_hw) // 32) * 32)
    us = timed(lambda: ops.test_transform([images[i] for i in first], xt, yt, out_hw, (Hp, Wp), tf.mean, tf.std, bgr=tf.bgr,
                                          times255=tf.times255), args.reps) * 1e3
    # the CUDA-graph engine over the same reference batches: run_batches (transformed device batches) and run_images (uint8)
    from mqdet_b200.engine.inference import InferenceEngine
    pre = [tf([images[i] for i in idx], dev, mixed_sizes=True)[0] for idx in ref]
    eng = InferenceEngine(model, caps, pmap)
    engine_rows = {"engine_run_batches": lambda: eng.run_batches(pre), "engine_run_images": lambda: eng.run_images(images, ref)}
    capture = engine_capture(eng, engine_rows["engine_run_batches"], len(ref))
    for _ in range(args.rounds):
        for name, fn in engine_rows.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in fn():
                pass
            torch.cuda.synchronize()
            secs.setdefault(name, []).append(time.perf_counter() - t0)
            plans.setdefault(name, (ref, True))
    capture.update(eng.batches.stats(), peak_gb=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))
    print(f"engine: {capture}", flush=True)
    eng.close()
    del eng, pre, model
    torch.cuda.empty_cache()
    gd = gdino_rows(args, dev)

    rows = []
    for name, v in secs.items():
        batches = plans[name][0]
        rows.append({"batching": name, "batches": len(batches), "s": [round(t, 3) for t in v],
                     "images_per_s": [round(args.images / t, 2) for t in v]})
        print(f"{name:18s} {len(batches):4d} batches: " + " ".join(f"{args.images / t:8.2f}" for t in v) + " images/s", flush=True)
    print(f"mixed test_transform, one padded batch of {len(first)} ({Hp} x {Wp}): {us:.1f} us per launch")
    line = json.dumps({"card": info, "images": args.images, "rows": rows, "engine_capture": capture, "gdino": gd,
                       "mixed_transform": {"batch": len(first), "padded_hw": [Hp, Wp], "us": round(us, 1)}})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


def engine_capture(eng, run, n_batches):
    """The engine's first pass over the set (every new padded shape warmed up and captured), timed apart from the steady state,
    and the device memory each captured graph holds."""
    torch.cuda.synchronize()
    a0, r0 = torch.cuda.memory_allocated(), torch.cuda.memory_reserved()
    t0 = time.perf_counter()
    for _ in run():
        pass
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    st = eng.batches.stats()
    n, buf = max(st["captures"], 1), eng.batches.buffer_bytes       # the staging buffers are not part of any graph
    return {"first_pass_s": round(wall, 3), "batches": n_batches, "buffers_mb": round(buf / 2 ** 20, 1),
            "alloc_mb_per_graph": round((torch.cuda.memory_allocated() - a0 - buf) / n / 2 ** 20, 1),
            "reserved_mb_per_graph": round((torch.cuda.memory_reserved() - r0 - buf) / n / 2 ** 20, 1)}


def gdino_rows(args, dev):
    """MQ-GroundingDINO-T at one image per batch: eager forward_device (+ one device-to-host copy per image) against
    GroundingDINOEngine.run_batches, alternating, on the same transformed images."""
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.engine.inference import GroundingDINOEngine
    from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO
    gen = synth.Gen(1238)
    ids, am, pmap = synth.prompt(13, 2, 256, gen)
    sd = synth.gdino_sd(synth.Gen(99))
    cfg = mq_groundingdino_t_cfg()
    model = GroundingDINO(cfg)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            sd[k] = v
    model.load_state_dict(sd, strict=True)
    del sd
    model = model.to(dev).eval()
    model.query_selector.set_query_bank(synth.query_bank(pmap, 5, gen))
    caps = {"input_ids": ids, "attention_mask": am}
    rng = np.random.default_rng(11)
    hw = [SIZES[i] for i in rng.integers(0, len(SIZES), args.gdino_images)]
    tf = TestTransform(cfg)
    images = upload([rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in hw], dev)
    batches = [tf([im], dev)[0] for im in images]
    torch.cuda.reset_peak_memory_stats(dev)
    eng = GroundingDINOEngine(model, caps, pmap)
    capture = engine_capture(eng, lambda: eng.run_batches(batches), len(batches))

    def eager():
        for il in batches:
            model.forward_device(il, caps, pmap)["det_packed"].cpu()

    eager()
    secs = {"eager_forward_device": [], "engine_run_batches": []}
    for _ in range(args.rounds):
        for name, fn in (("eager_forward_device", eager), ("engine_run_batches", lambda: [None for _ in eng.run_batches(batches)])):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            secs[name].append(time.perf_counter() - t0)
    capture.update(eng.batches.stats(), peak_gb=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
                   padded_shapes=len({tuple(il.tensors.shape[-2:]) for il in batches}))
    for name, v in secs.items():
        print(f"gdino {name:22s} {len(batches):4d} images: " + " ".join(f"{len(batches) / t:8.2f}" for t in v) + " images/s",
              flush=True)
    print(f"gdino engine: {capture}", flush=True)
    eng.close()
    return {"images": len(batches), "capture": capture,
            "rows": [{"path": k, "s": [round(t, 3) for t in v], "images_per_s": [round(len(batches) / t, 2) for t in v]}
                     for k, v in secs.items()]}


if __name__ == "__main__":
    main()
