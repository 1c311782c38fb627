"""CUDA-event times of the test-time-augmentation merge (csrc/bbox_aug.cu): 24 passes x 5000 candidates per image appended by
``ops.bbox_aug_collect`` and merged by ``ops.nms_by_class`` (``nms`` and ``vote``), graph-replayed, next to the host-side path
of the reference's box_aug.py on the same CUDA tensors (a Python loop over the classes, every class copied to the host and
merged there by tests/bbox_aug_oracle.py, the per-image cut after a ``.cpu()``).

    python tools/prof_bbox_aug.py [--batch 2] [--passes 24] [--cand 5000] [--reps 20] [--out FILE.json]

Boxes: jittered copies of a few hundred objects over 80 classes, the classes skewed (a quarter of the objects in one class).
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
import torch  # noqa: E402


def make_pass(g, n_obj, n, size, objects):
    cx, cy, bw, bh, lab = objects
    o = torch.randint(0, n_obj, (n,), generator=g)
    j = (torch.rand(n, 4, generator=g) - 0.5) * 12
    b = torch.stack([cx[o] - bw[o] / 2, cy[o] - bh[o] / 2, cx[o] + bw[o] / 2, cy[o] + bh[o] / 2], 1) + j
    b[:, 0::2] = b[:, 0::2].clamp(0, size[0] - 1)
    b[:, 1::2] = b[:, 1::2].clamp(0, size[1] - 1)
    return b.float(), (0.05 + 0.9 * torch.rand(n, generator=g)).float(), lab[o].float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--passes", type=int, default=24)
    ap.add_argument("--cand", type=int, default=5000)
    ap.add_argument("--objects", type=int, default=300)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_bbox_aug: a CUDA device is required (nothing is measured on the CPU)")
    import bbox_aug_oracle as bo
    from mqdet_b200 import ops
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()
    g = torch.Generator().manual_seed(5)
    size = (1333, 800)
    B, P, S = a.batch, a.passes, (a.cand + 255) // 256 * 256
    lab = torch.randint(1, 81, (a.objects,), generator=g)
    lab[: a.objects // 4] = 1
    objects = (torch.rand(a.objects, generator=g) * size[0], torch.rand(a.objects, generator=g) * size[1],
               20 + torch.rand(a.objects, generator=g) * 300, 20 + torch.rand(a.objects, generator=g) * 300, lab)
    cands = []
    for p in range(P):
        cb, cs, cl = torch.zeros(B, S, 4), torch.zeros(B, S), torch.zeros(B, S)
        for b in range(B):
            cb[b, :a.cand], cs[b, :a.cand], cl[b, :a.cand] = make_pass(g, a.objects, a.cand, size, objects)
        cands.append((cb.to(dev), cs.to(dev), cl.to(dev), torch.full((B,), a.cand, dtype=torch.int32, device=dev), p % 2 == 1))
    classes = torch.arange(1, 81, dtype=torch.int32, device=dev)
    merged = ops.MergedBoxes(B, min(P * S, ops.BBOX_AUG_MAX_CAP), dev)
    result = {"card": card, "batch": B, "passes": P, "candidates_per_pass": a.cand, "merged_per_image": P * a.cand, "ms": {}}

    def collect():
        merged.count.zero_()
        merged.overflow.zero_()
        for cb, cs, cl, tot, flip in cands:
            ops.bbox_aug_collect(merged, cb, cs, cl, tot, size, size, flip=flip, keep_range=(0, 10000))

    def timed(fn, name):
        fn()                                             # warm-up (module load, allocator)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            fn()
            with torch.cuda.graph(graph, stream=s):
                fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
        result["ms"][name] = e0.elapsed_time(e1) / a.reps

    timed(collect, "collect (all passes)")
    collect()
    for mode in ("nms", "vote"):
        timed(lambda: ops.nms_by_class(merged.boxes, merged.scores, merged.labels, merged.count, classes, 0.6, mode=mode, top_n=1000,
                                       max_out=1056), f"nms_by_class {mode}")
    torch.cuda.synchronize()
    n = int(merged.count[0])
    for mode in ("nms", "vote"):   # the reference-style path: per image, per class, through the host
        t0 = time.perf_counter()
        for b in range(B):
            parts = []
            for c in range(1, 81):
                inds = (merged.labels[b, :n] == c).nonzero().view(-1)
                if inds.numel() == 0:
                    continue
                parts.append(bo.merge(merged.boxes[b, :n][inds].cpu(), merged.scores[b, :n][inds].cpu(),
                                      torch.full((inds.numel(),), c), [c], 0.6, mode, 0))
            sc = torch.cat([p[1] for p in parts]).to(dev)
            if sc.numel() > 1000:
                thr = torch.kthvalue(sc.cpu(), sc.numel() - 1000 + 1)[0].item()
                (sc >= thr).nonzero()
        torch.cuda.synchronize()
        result["ms"][f"host-side per-class loop {mode}"] = (time.perf_counter() - t0) * 1e3
    print(f"card: {card}")
    print(f"B = {B}, {P} passes x {a.cand} candidates = {P * a.cand} merged boxes per image, 80 classes")
    for k, v in result["ms"].items():
        print(f"  {k:36s} {v:10.3f} ms")
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
