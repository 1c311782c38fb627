"""Cost of the test-time vision-query update (VISION_QUERY.NUM_TURNS) on synthetic MQ-GLIP-T over an ODinW-sized test set:
``--images`` images at two sizes in runs of 40 (so batches break where the size changes), a 13-class prompt, a 5-shot starting bank,
NUM_QUERY_PER_CLASS = MAX_TEST_QUERY_NUMBER = 100, 3 turns.
    python tools/prof_online_update.py [--images 160] [--batch 8] [--out FILE]
Reports seconds per turn (host clock around each turn, which ends in the turn's device->host copy) for the turn loop of
``engine.online_update`` at
B = ``--batch`` and B = 1, and for the host loop of the reference (one-image forward, BoxLists on the host, ``extract_query
(exclude_similar=True)`` with the bank on the host), whether the three give the same banks, and the card's name, power limit and max SM
clock read in the same run.  The synthetic detector scores lower than a trained one, so SCORE_THRESHOLD is set to keep about ten
boxes of the first image.  One JSON line on stdout (and to --out)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

from mqdet_b200 import _lib
from mqdet_b200.config import mq_glip_t_cfg
from mqdet_b200.engine.online_update import make_batches, update_turn
from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
from mqdet_b200.structures.bounding_box import BoxList
from mqdet_b200.structures.image_list import to_image_list
from tools import synth
from tools.prof_gcp_queries import card

SIZES = ((480, 640), (512, 683))


def host_loop(model, imgs, caps, pmap, start, turns):
    """The reference's loop, timed per turn: -> (banks, seconds per turn)."""
    import online_update_oracle as ou
    vq = model.cfg.VISION_QUERY
    bank, banks, secs = ou.copy_bank(start), [], []
    for turn in range(turns):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if turn > 0:
            model.set_query_bank({k: v.clone() for k, v in banks[-1].items()})
        for im in imgs:
            il = to_image_list([im], 32)
            out = model.forward_device(il, caps, pmap)
            pk, pyr = out["det_packed"][0].cpu(), out["pyramid16"]
            off, maps = 0, []
            for h, w in out["levels"].sizes:
                maps.append(pyr[:, off:off + h * w].float().transpose(1, 2).reshape(1, -1, h, w).contiguous())
                off += h * w
            h, w = il.image_sizes[0]
            n = int(pk[-1, 0])
            bl = BoxList(pk[:n, :4].clone(), (w, h), mode="xyxy")
            bl.add_field("scores", pk[:n, 4].clone())
            bl.add_field("labels", pk[:n, 5].long())
            bank = model.extract_query(targets=[bl[bl.get_field("scores") > vq.SCORE_THRESHOLD]], query_images=bank, visual_features=maps,
                                       exclude_similar=True, max_query_number=vq.MAX_TEST_QUERY_NUMBER)
        banks.append(ou.copy_bank(bank))
        secs.append(time.perf_counter() - t0)
    return banks, secs


def device_path(model, imgs, caps, pmap, start, turns, B):
    """``engine.online_update``'s turn loop (``update_turn`` + the turn's one device->host copy), timed per turn."""
    from mqdet_b200 import ops
    batches = make_batches(imgs, B)
    qb = ops.QueryBank.from_dict(start, max(int(k) for k in pmap) + 1, model.cfg.VISION_QUERY.MAX_TEST_QUERY_NUMBER, 256, imgs[0].device)
    bad = torch.zeros((1,), dtype=torch.int32, device=imgs[0].device)
    banks, secs = [], []
    for turn in range(turns):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if turn > 0:
            model.set_query_bank(banks[-1])
        update_turn(model, batches, caps, pmap, qb, model.cfg, bad)
        host = torch.cat([qb.count, bad]).cpu()
        banks.append(qb.as_dict(host[:-1]))
        secs.append(time.perf_counter() - t0)
    assert int(host[-1]) == 0
    return banks, secs


def same(a, b):
    ka = sorted(int(k) for k, v in a.items() if len(v))
    kb = sorted(int(k) for k, v in b.items() if len(v))
    return ka == kb and all(torch.equal(a[k].cpu(), b[k].cpu()) for k in ka)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=160)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prof_online_update: needs a CUDA device")
    _lib.load()
    dev = torch.device("cuda:0")
    info = card()
    sd = synth.detector_sd(synth.Gen(99), bias0=-1.5)
    model = GeneralizedVLRCNN_New(mq_glip_t_cfg(**{"VISION_QUERY.NUM_QUERY_PER_CLASS": 100}))
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            sd[k] = v
    model.load_state_dict(sd, strict=True)
    del sd
    model = model.to(dev).eval()
    gen = synth.Gen(7)
    ids, am, pmap = synth.prompt(13, 2, 256, gen)
    caps = {"input_ids": ids, "attention_mask": am}
    start = synth.query_bank(pmap, 5, gen)
    imgs = [synth.images(gen, 1, *SIZES[(i // 40) % 2])[0].to(dev) for i in range(args.images)]
    model.set_query_bank({k: v.clone() for k, v in start.items()})
    pk = model.forward_device(to_image_list([imgs[0]], 32), caps, pmap)["det_packed"][0].cpu()
    scores = pk[:int(pk[-1, 0]), 4].sort(descending=True)[0]
    vq = model.cfg.VISION_QUERY
    vq.SCORE_THRESHOLD = float(scores[min(9, len(scores) - 1)]) - 1e-4
    vq.MAX_TEST_QUERY_NUMBER = 100
    turns = 3
    rows = {}
    for name, fn in ((f"device_b{args.batch}", lambda: device_path(model, imgs, caps, pmap, start, turns, args.batch)),
                     ("device_b1", lambda: device_path(model, imgs, caps, pmap, start, turns, 1)),
                     ("host_loop", lambda: host_loop(model, imgs, caps, pmap, start, turns))):
        model.set_query_bank({k: v.clone() for k, v in start.items()})
        r = fn()
        rows[name] = r
        print(f"{name:10s}: s per turn " + " ".join(f"{s:7.3f}" for s in r[1]), flush=True)
    ref = rows["host_loop"][0]
    equal = {k: all(same(a, b) for a, b in zip(v[0], ref)) for k, v in rows.items() if k != "host_loop"}
    line = json.dumps({"card": info, "images": args.images, "sizes": SIZES, "turns": turns, "score_threshold": vq.SCORE_THRESHOLD,
                       "bank_rows_per_turn": [sum(len(v) for v in b.values()) for b in ref],
                       "s_per_turn": {k: [round(s, 3) for s in v[1]] for k, v in rows.items()}, "banks_equal_host_loop": equal})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
