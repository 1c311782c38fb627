"""LVIS-protocol evaluation through ``ChunkedEngine``: 1203 classes as 31 prompts of 40 (TEST.CHUNKED_EVALUATION 40), K = 5 vision
queries per class, one image per batch (TEST.IMS_PER_BATCH 1) over COCO-like original sizes at MIN_SIZE_TEST 800 / MAX_SIZE_TEST
1333, for MQ-GLIP-T, MQ-GLIP-L and MQ-GroundingDINO-T at full depth with random-init weights (``synth``).
    python tools/prof_chunked_engine.py [--images 12] [--rounds 3] [--chunks-per-pass 8] [--models glip_t glip_l gdino_t] [--all-shapes]
                                        [--out FILE]
``--all-shapes`` replaces the random draw by one image per padded shape of a COCO-like set at 800 / 1333 (one side at 800, the
other from 800 to 1333 in 32-pixel steps, both orientations, plus originals whose long side is capped at 1333: 43 shapes), so
the capture pass shows whether the default graph limit holds them all, and what they hold in memory.
Per model, alternating within every round and each timed over the whole set (host clock around work that ends in a device
synchronise, after a warm-up pass that also captures the engine's graphs):
  * ``eager``: eager ``forward_chunked`` of the transformed image (one device-to-host copy of its packed detections, then BoxLists);
  * ``run_batches``: ``ChunkedEngine.run_batches`` over the same transformed images (device ImageLists);
  * ``run_images``: ``ChunkedEngine.run_images`` over the decoded uint8 images (upload and transform on its copy stream).
Reports images/s and chunk-forwards/s per round, the engine's capture pass apart (captures, seconds, evictions, device memory per
graph beyond the staging buffers, peak ``max_memory_allocated``), and the largest difference between the engine's and the eager
detections (counts, boxes, scores, labels; must be 0).  The card's name, power limit and max SM clock are read in the same run.
One JSON line on stdout (and to --out)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from mqdet_b200 import _lib
from mqdet_b200.engine.inference import ChunkedEngine
from mqdet_b200.engine.transforms import TestTransform, upload
from tools import synth
from tools.prof_gcp_queries import card
from tools.prof_mixed_batches import SIZES, engine_capture

NCLS, CHUNK, K = 1203, 40, 5


def all_shape_sizes():
    """Originals whose test-transform targets cover every padded shape: (800, w) for w in 800..1333 by 32, their transposes,
    and (h, 1333) for h in 672..800 by 32 (the long side capped) with their transposes."""
    land = [(800, w) for w in list(range(800, 1333, 32)) + [1333]] + [(h, 1333) for h in range(672, 800, 32)]
    return land + [(w, h) for h, w in land if h != w]


def build(name, dev):
    from mqdet_b200.config import mq_glip_l_cfg, mq_glip_t_cfg, mq_groundingdino_t_cfg
    gen = synth.Gen(1203)
    chunks = synth.chunked_prompts(NCLS, CHUNK, 256, gen)
    bank = {}
    for _, _, pm in chunks:
        bank.update(synth.query_bank(pm, K, gen))
    if name == "gdino_t":
        from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO
        sd = synth.gdino_sd(synth.Gen(99))
        model = GroundingDINO(mq_groundingdino_t_cfg(**{"MODEL.DYHEAD.NUM_CLASSES": NCLS + 1}))
    else:
        from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
        if name == "glip_l":
            sd = synth.detector_sd(synth.Gen(98), num_convs=8, swin=dict(depths=(2, 2, 18, 2), heads=(6, 12, 24, 48), embed=192, ws=12))
            cfg = mq_glip_l_cfg()
        else:
            sd = synth.detector_sd(synth.Gen(98))
            cfg = mq_glip_t_cfg(**{"MODEL.ATSS.DETECTIONS_PER_IMG": 300})
        model = GeneralizedVLRCNN_New(cfg)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            sd[k] = v
    model.load_state_dict(sd, strict=True)
    del sd
    model = model.to(dev).eval()
    model.query_selector.set_query_bank(bank)
    return model, [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks], [pm for _, _, pm in chunks]


def max_diff(got, want):
    d = 0.0
    for g, w in zip(got, want):
        if len(g) != len(w):
            return float("inf")
        if len(g):
            d = max(d, float((g.bbox - w.bbox).abs().max()), float((g.get_field("scores") - w.get_field("scores")).abs().max()),
                    float((g.get_field("labels") != w.get_field("labels")).sum()))
    return d


def profile(name, args, dev):
    model, caps, pmaps = build(name, dev)
    cfg = model.cfg
    rng = np.random.default_rng(7)
    hw = all_shape_sizes() if args.all_shapes else [SIZES[i] for i in rng.integers(0, len(SIZES), args.images)]
    images = upload([rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in hw], dev)
    tf = TestTransform(cfg)
    pre = [tf([im], dev, mixed_sizes=True)[0] for im in images]
    idx = [[i] for i in range(len(images))]
    n = len(caps)
    cpp = args.chunks_per_pass

    def eager():
        res = []
        for il in pre:
            res.append(model.forward_chunked(il, caps, pmaps, cpp)[0])
        return res

    want = eager()
    torch.cuda.reset_peak_memory_stats(dev)
    eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=cpp)
    capture = engine_capture(eng, lambda: eng.run_batches(pre), len(pre))
    got = [r[0] for r in eng.run_batches(pre)]
    diff = max_diff(got, want)
    rows = {"eager": lambda: eager(), "run_batches": lambda: [None for _ in eng.run_batches(pre)],
            "run_images": lambda: [None for _ in eng.run_images(images, idx)]}
    rows["run_images"]()
    secs = {k: [] for k in rows}
    for _ in range(args.rounds):
        for k, fn in rows.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            secs[k].append(time.perf_counter() - t0)
    capture.update(eng.stats(), peak_gb=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
                   padded_shapes=len({tuple(il.tensors.shape[-2:]) for il in pre}))
    eng.close()
    out = {"model": name, "images": len(pre), "chunks": n, "chunks_per_pass": cpp, "max_abs_diff": diff, "capture": capture,
           "rows": [{"path": k, "s": [round(t, 3) for t in v], "images_per_s": [round(len(pre) / t, 3) for t in v],
                     "chunk_forwards_per_s": [round(len(pre) * n / t, 1) for t in v]} for k, v in secs.items()]}
    for r in out["rows"]:
        print(f"{name:8s} {r['path']:12s} images/s " + " ".join(f"{v:7.3f}" for v in r["images_per_s"]), flush=True)
    print(f"{name:8s} capture {capture} max_abs_diff {diff}", flush=True)
    del eng, model, pre, images
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunks-per-pass", type=int, default=8)
    ap.add_argument("--models", nargs="+", default=["glip_t", "glip_l", "gdino_t"], choices=["glip_t", "glip_l", "gdino_t"])
    ap.add_argument("--all-shapes", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_chunked_engine: needs a CUDA device")
    _lib.load()
    dev = torch.device("cuda:0")
    info = card()
    res = [profile(m, args, dev) for m in args.models]
    line = json.dumps({"card": info, "classes": NCLS, "chunk": CHUNK, "K": K, "models": res})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
