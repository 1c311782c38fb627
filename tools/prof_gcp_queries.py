"""Cost of the vision-query count K (VISION_QUERY.NUM_QUERY_PER_CLASS) on the GCP path of synthetic MQ-GLIP-T, for two inputs:
an 80-class prompt at B = 8 (COCO-shaped) and a 40-class chunk at B = 1 (one LVIS chunk), T = 256, two tokens per class, so
S = K queries per class token.
    python tools/prof_gcp_queries.py [--ks 5,16,32,100] [--reps 200] [--steps 5] [--out FILE]
For every (input, K) it reports:
1. ops.gcp_sparse_attn alone: ms per launch from CUDA events around `reps` launches, and the K / V rows it gathers through L2,
   B * T * S * 2 * 1 KB (every slot of every token reads one 512-dim fp16 K row and one V row, padding slots included), over that time.
2. ops.gcp_build_index (counts and the [B, T, S] index table from the [B, V, T] mask; sparse_index runs it twice per distinct mask):
   ms per call, CUDA events around `reps` calls.
3. The whole QVBertModel forward of the detector (embeddings, PreSelect over the 5577 pooled image tokens of an 800 x 1333 image, 12
   BERT layers with the six GCP blocks): ms per call, CUDA events around `steps` calls.
4. forward_device of the detector at 800 x 1333 (padded to 800 x 1344): images/s over `steps` eager calls ending in a synchronise.
The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout (and to --out)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from mqdet_b200 import _lib, ops
from mqdet_b200.config import mq_glip_t_cfg
from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
from mqdet_b200.structures.image_list import ImageList
from tools import synth

INPUTS = {"prompt80_b8": (80, 8), "chunk40_b1": (40, 1)}
H_IMG, W_IMG, I_POOLED = 800, 1333, 5577


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, n):
    """ms per call of fn() from CUDA events around n calls (after one warm-up call)."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="5,16,32,100")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_gcp_queries: needs a CUDA device")
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
    lang = model.language_backbone.body.model
    rows = []
    for name, (ncls, B) in INPUTS.items():
        gen = synth.Gen(7 + ncls)
        ids, am, pmap = synth.prompt(ncls, 2, 256, gen)
        img = synth.images(gen, B, H_IMG, W_IMG).to(dev)
        il = ImageList(img, [(H_IMG, W_IMG)] * B)
        caps = {"input_ids": ids, "attention_mask": am}
        images = gen.randn(B, I_POOLED, 256).to(dev)
        ids_d, am_d = ids.expand(B, -1).contiguous().to(dev), am.expand(B, -1).contiguous().to(dev)
        for K in (int(k) for k in args.ks.split(",")):
            T = ids.shape[1]
            vision, vmask = synth.vision_queries(pmap, K, T, 256, gen)
            V = vision.shape[1]
            vision = vision.expand(B, -1, -1).contiguous().to(dev)
            vmask = vmask.expand(B, -1, -1).contiguous().to(dev)
            idx, _ = ops.gcp_build_index(vmask, K)
            q = (gen.randn(B, T, 512) * 0.125).half().to(dev)
            kv = gen.randn(B, V + 1, 1024).half().to(dev)
            ms_index = timed(lambda: ops.gcp_build_index(vmask, K), args.reps)
            ms_attn = timed(lambda: ops.gcp_sparse_attn(q, kv, idx, 8, 64), args.reps)
            gathered = B * T * K * 2 * 1024
            ms_lang = timed(lambda: lang(input_ids=ids_d, attention_mask=am_d, vision=vision, images=images,
                                         vision_attention_mask=vmask), args.steps)
            model.query_selector.num_query_per_class = K
            model.query_selector.set_query_bank(synth.query_bank(pmap, K, gen))
            ms_fwd = timed(lambda: model.forward_device(il, caps, pmap), args.steps)
            row = {"input": name, "B": B, "classes": ncls, "K": K, "V": V, "gcp_sparse_attn_ms": round(ms_attn, 4),
                   "gcp_build_index_ms": round(ms_index, 4), "gathered_MB": round(gathered / 1e6, 2), "gathered_GB_per_s": round(gathered / ms_attn / 1e6, 1),
                   "qvbert_forward_ms": round(ms_lang, 3), "forward_device_images_per_s": round(B / ms_fwd * 1e3, 2)}
            rows.append(row)
            print(f"{name} K={K:4d}: gcp_sparse_attn {ms_attn * 1e3:8.1f} us ({row['gathered_GB_per_s']:7.1f} GB/s of K/V rows), "
                  f"gcp_build_index {ms_index * 1e3:8.1f} us, "
                  f"QVBertModel {ms_lang:7.2f} ms, forward_device {row['forward_device_images_per_s']:6.2f} images/s", flush=True)
            del q, kv, idx, vision, vmask
            torch.cuda.empty_cache()
    res = {"card": info, "rows": rows}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
