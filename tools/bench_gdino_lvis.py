"""LVIS-style chunked evaluation of MQ-GroundingDINO-T: 1203 classes as 31 prompts of 40 (TEST.CHUNKED_EVALUATION 40 of
configs/vision_query_5shot/lvis_*_groundingdino-T.yaml), K = 5 vision queries per class, full depth (6 + 6 layers, 900 queries),
synthetic 800x1333 images and random-init weights (``synth.gdino_sd``).

Times, alternating and ``--repeats`` times (device-synchronised host clock, every shape warmed up first):
  (i)  ``GroundingDINO.forward_chunked_device`` at each ``--chunks-per-pass`` (Swin-T + input_proj once per image batch);
  (ii) the loop a user runs without it: one ``forward_device`` per chunk (31 per image batch).
Prints ONE JSON line: images/s and chunk-forwards/s (median over the repeats) and peak ``torch.cuda.max_memory_allocated`` per
variant, the largest difference between the packed detections of (i) and (ii), and the card name, power limit and max SM clock
read in the same run (``nvidia-smi --query-gpu``, read-only).  ``--out FILE`` also writes the line to FILE.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.prof_atss_loss import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1, help="images per batch (TEST.IMS_PER_BATCH of the LVIS configs: 1)")
    ap.add_argument("--chunks-per-pass", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--classes", type=int, default=1203)
    ap.add_argument("--chunk", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from mqdet_b200 import _lib
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    from util import load_sd
    if not torch.cuda.is_available():
        raise SystemExit("bench_gdino_lvis: needs a CUDA device")
    _lib.load()
    dev = torch.device("cuda:0")
    gen = synth.Gen(1203)
    sd = synth.gdino_sd(gen, 6, 6, 900)
    chunks = synth.chunked_prompts(args.classes, args.chunk, 256, gen)
    bank = {}
    for _, _, pm in chunks:
        bank.update(synth.query_bank(pm, 5, gen))
    B, h, w = args.images, 800, 1333
    img = synth.rgb_images(gen, B, h, w)
    model = GroundingDINO(mq_groundingdino_t_cfg(**{"MODEL.DYHEAD.NUM_CLASSES": args.classes + 1}))
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    model = load_sd(model, full).to(dev).eval()
    model.query_selector.set_query_bank(bank)
    il = ImageList(img.to(dev), [(h, w)] * B)
    caps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    pmaps = [pm for _, _, pm in chunks]
    nc = len(chunks)

    def loop():   # (ii): one whole forward per chunk
        return torch.stack([model.forward_device(il, cap, pm)["det_packed"] for cap, pm in zip(caps, pmaps)])

    variants = {f"chunked_{c}": (lambda c=c: model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=c)["det_packed"])
                for c in args.chunks_per_pass}
    variants["per_chunk_forward_device"] = loop
    outs, peak = {}, {}
    for name, fn in variants.items():   # warm-up of every shape (and the prompt / geometry caches), peak memory per variant
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        outs[name] = fn()
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated(dev)
    times = {name: [] for name in variants}
    for _ in range(args.repeats):
        for name, fn in variants.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    ref = outs["per_chunk_forward_device"]
    res = {"workload": f"MQ-GroundingDINO-T 6+6 layers, 900 queries, {B} x 800x1333, {args.classes} classes as {nc} chunks of "
                       f"{args.chunk}, K=5", "repeats": args.repeats, "variants": {}}
    for name in variants:
        t = sorted(times[name])[len(times[name]) // 2]
        d = outs[name]
        res["variants"][name] = {"seconds_per_batch": t, "seconds_all": times[name], "images_per_s": B / t,
                                 "chunk_forwards_per_s": B * nc / t, "max_memory_allocated_bytes": int(peak[name]),
                                 "max_abs_diff_vs_per_chunk": float((d - ref).abs().max()),
                                 "detections": int(d[:, :, -1, 0].sum())}
    res["gpu"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
