"""Cost of vision-only evaluation (VISION_QUERY.MASK_DURING_INFERENCE) on synthetic MQ-GLIP-T at 800 x 1333, K = 5:
forward_device with an 80-class prompt at B = 8, and forward_chunked_device over two 40-class chunks at B = 1 (LVIS-shaped).
    python tools/prof_vision_only.py [--rounds 3] [--steps 5] [--reps 500] [--out FILE]
For each input, modes off / TEXT_DROPOUT 1.0 / TEXT_DROPOUT 0.5 alternate within every round (ms per call from CUDA events around
``steps`` calls after a warm-up call).  The ``ops.mask_prompt_tokens`` launch is timed alone at the shapes the two paths hand it
(CUDA events around ``reps`` launches).  The card's name, power limit and max SM clock are read in the same run.  One JSON line
on stdout (and to --out)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from mqdet_b200 import _lib, ops
from mqdet_b200.config import mq_glip_t_cfg
from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
from mqdet_b200.structures.image_list import ImageList
from tools import synth
from tools.prof_gcp_queries import card, timed

H_IMG, W_IMG = 800, 1333
MODES = {"off": (False, 1.0), "p1.0": (True, 1.0), "p0.5": (True, 0.5)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_vision_only: needs a CUDA device")
    _lib.load()
    dev = torch.device("cuda:0")
    info = card()
    sd = synth.detector_sd(synth.Gen(99))
    model = GeneralizedVLRCNN_New(mq_glip_t_cfg())
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            sd[k] = v
    model.load_state_dict(sd, strict=True)
    del sd
    model = model.to(dev).eval()
    gen = synth.Gen(7)
    ids, am, pmap = synth.prompt(80, 2, 256, gen)
    chunks = synth.chunked_prompts(80, 40, 256, gen)
    bank = synth.query_bank(pmap, 5, gen)
    model.query_selector.set_query_bank(bank)
    img8 = ImageList(synth.images(gen, 8, H_IMG, W_IMG).to(dev), [(H_IMG, W_IMG)] * 8)
    img1 = ImageList(synth.images(gen, 1, H_IMG, W_IMG).to(dev), [(H_IMG, W_IMG)])
    caps = {"input_ids": ids, "attention_mask": am}
    ccaps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    cmaps = [pm for _, _, pm in chunks]
    calls = {"forward_device_80cls_b8": (8, lambda: model.forward_device(img8, caps, pmap)),
             "forward_chunked_device_2x40cls_b1": (1, lambda: model.forward_chunked_device(img1, ccaps, cmaps, chunks_per_pass=8))}
    ms = {(name, mode): [] for name in calls for mode in MODES}
    for _ in range(args.rounds):
        for name, (_, fn) in calls.items():
            for mode, (on, rate) in MODES.items():
                model.cfg.VISION_QUERY.MASK_DURING_INFERENCE, model.cfg.VISION_QUERY.TEXT_DROPOUT = on, rate
                ms[(name, mode)].append(timed(fn, args.steps))
    kernel = {}
    for E, C in ((8, 80), (2, 40)):
        x = torch.randint(1000, 29000, (E, 256), device=dev)
        cat = torch.randint(-1, C, (E, 256), device=dev, dtype=torch.int32)
        fl = torch.randint(0, 2, (E, C), device=dev, dtype=torch.uint8)
        kernel[f"E{E}_C{C}"] = round(timed(lambda: ops.mask_prompt_tokens(x, cat, fl, 103), args.reps) * 1e3, 2)
    rows = []
    for (name, mode), v in ms.items():
        B = calls[name][0]
        rows.append({"call": name, "mode": mode, "ms": [round(t, 3) for t in v], "images_per_s": [round(B / t * 1e3, 2) for t in v]})
        print(f"{name:36s} {mode:5s}: " + " ".join(f"{t:8.3f}" for t in v) + " ms", flush=True)
    print("mask_prompt_tokens alone (us per launch): " + ", ".join(f"{k} {v}" for k, v in kernel.items()))
    line = json.dumps({"card": info, "rows": rows, "mask_prompt_tokens_us": kernel})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
