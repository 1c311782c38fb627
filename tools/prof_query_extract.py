"""Cost of building a vision-query bank over a dataset (tools/train_net.py --extract_query) on synthetic MQ-GLIP-T and
MQ-GroundingDINO-T: ``--images`` decoded uint8 images of 16 COCO-like sizes, about 7 ground-truth boxes per image over 80 labels,
TEST.IMS_PER_BATCH = 8 with aspect grouping, MIN_SIZE_TEST / MAX_SIZE_TEST = 800 / 1333, MAX_QUERY_NUMBER 5 (the LVIS / ODinW banks)
and 5000 (COCO / Objects365).
    python tools/prof_query_extract.py [--images 192] [--runs 3] [--out FILE]
For each detector and cap, ``engine.query_extract.extract_query_bank`` and the reference's host loop (per batch the device test
transform, BoxList.resize on the host, ``model.extract_query``, which copies the pooled features to the host and appends box by box)
run alternately, ``--runs`` times each after one warm-up of both; the host clock around each call ends in a device synchronise.
Reports images/s per run, whether the two banks are identical, and the card's name, power limit and max SM clock read in the same run.
One JSON line on stdout (and to --out)."""
import argparse
import json
import os
import sys
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from mqdet_b200 import _lib
from mqdet_b200.engine.batches import reference_test_batches
from mqdet_b200.engine.query_extract import extract_query_bank
from mqdet_b200.engine.transforms import TestTransform
from mqdet_b200.structures.bounding_box import BoxList
from tools import synth
from tools.prof_gcp_queries import card

SIZES = [(480, 640), (427, 640), (640, 480), (375, 500), (333, 500), (612, 612), (640, 427), (500, 375), (424, 640), (360, 640),
         (640, 512), (500, 333), (426, 640), (480, 600), (512, 640), (640, 640)]


def dataset(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    imgs, targets = [], []
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        imgs.append(torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy())
        k = int(torch.randint(3, 12, (1,), generator=g))
        x1, y1 = torch.rand(k, generator=g) * w * 0.8, torch.rand(k, generator=g) * h * 0.8
        b = torch.stack([x1, y1, x1 + 8 + torch.rand(k, generator=g) * w * 0.3, y1 + 8 + torch.rand(k, generator=g) * h * 0.3], 1)
        t = BoxList(b, (w, h), mode="xyxy")
        t.add_field("labels", torch.randint(1, 81, (k,), generator=g))
        targets.append(t)
    return imgs, targets


def model_of(kind, dev):
    """The synthetic detectors of the GPU tests: MQ-GLIP-T, and MQ-GroundingDINO-T with 2 + 2 transformer layers (the extraction
    runs only the backbone and input_proj, which the layer counts do not change)."""
    if kind == "glip":
        from test_gcp_many_queries_gpu import _glip
        model = _glip(synth.detector_sd(synth.Gen(2024), bias0=-1.5), dev, 5)
    else:
        from test_gdino_asm_gpu import _build_model, _gdino_case
        model = _build_model(_gdino_case(3033, 1, 160, 224, 13, 2, 2, 100)[0], 2, 2, 100, dev)
    model.cfg.TEST.IMS_PER_BATCH = 8
    return model


def host_loop(model, imgs, targets, batches, dev):
    bank, tt = defaultdict(list), TestTransform(model.cfg)
    for idx in batches:
        il, _ = tt([imgs[i] for i in idx], dev, mixed_sizes=True)
        tg = [targets[i].resize((w, h)) for i, (h, w) in zip(idx, il.image_sizes)]
        bank = model.extract_query(il, tg, bank)
    return bank


def timed(fn, n_images):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, n_images / (time.perf_counter() - t0)


def same(a, b):
    ka, kb = sorted(k for k, v in a.items() if len(v)), sorted(k for k, v in b.items() if len(v))
    return ka == kb and all(torch.equal(a[k].cpu(), b[k].cpu()) for k in ka)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=192)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_query_extract: needs a CUDA device")
    _lib.load()
    dev = torch.device("cuda:0")
    imgs, targets = dataset(args.images)
    batches = reference_test_batches([im.shape[:2] for im in imgs], 8, True)
    res = {"card": card(), "images": args.images, "boxes": sum(len(t) for t in targets), "ims_per_batch": 8, "results": {}}
    for kind in ("glip", "gdino"):
        model = model_of(kind, dev)
        for K in (5, 5000):
            model.cfg.VISION_QUERY.MAX_QUERY_NUMBER = K
            engine = lambda: extract_query_bank(model, imgs, targets, model.cfg)
            host = lambda: host_loop(model, imgs, targets, batches, dev)
            a, b = engine(), host()                                       # warm-up of both
            ok = same(a, b)
            eng, hst = [], []
            for _ in range(args.runs):
                a, r = timed(engine, args.images)
                eng.append(round(r, 1))
                b, r = timed(host, args.images)
                hst.append(round(r, 1))
                ok = ok and same(a, b)
            res["results"][f"{kind}_K{K}"] = {"engine_images_per_s": eng, "host_loop_images_per_s": hst, "identical": ok,
                                              "speedup_median": round(float(np.median(eng) / np.median(hst)), 3)}
        del model
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
