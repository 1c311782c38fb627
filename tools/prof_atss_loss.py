"""CUDA-event timing of the ATSS assignment + pre-training losses at the bench shape (B = 8, 800x1344 -> N = 22400 anchors, T = 256).

    python tools/prof_atss_loss.py [--gts 10 50 200] [--reps 20] [--out DIR]

For each GT count G: ``ops.atss_loss`` with the assignment included (``atss_targets`` + the loss kernels, one launch sequence),
warmed up, then ``--reps`` launches between two CUDA events; the fp32 torch restatement (tests/atss_oracle.py) with autograd on
the same CUDA tensors as the comparator.  The HBM bound is the traffic the losses need at least: logits read once and d_logits
written once (B*N*T*4 bytes each) plus reg_ctr / d_reg_ctr and the match map; the fraction reported is bound / measured time at
3.35 TB/s (H100 SXM data sheet).  The card name and power limit are read in the same run.  JSON -> DIR/atss_loss.json (default: a
directory under the system temp dir).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BPS = 3.35e12


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"error": str(e)}


def inputs(B, G, T, dev, seed=0):
    import torch
    import atss_oracle as ao
    gen = torch.Generator().manual_seed(seed)
    h, w = 800, 1344
    sizes = ao.level_sizes(h, w)
    N = sum(a * b for a, b in sizes)
    boxes = torch.stack([ao._boxes(gen, G, h, w) for _ in range(B)])
    labels = torch.randint(1, 81, (B, G), generator=gen, dtype=torch.int32)
    tokens = torch.zeros(B, G, T)
    tokens[..., 5:8] = 1.0
    return {"sizes": sizes, "gt_boxes": boxes.to(dev), "gt_labels": labels.to(dev),
            "gt_count": torch.full((B,), G, dtype=torch.int32).to(dev), "gt_tokens": tokens.to(dev),
            "logits": (torch.randn(B, N, T, generator=gen) * 2 - 3).to(dev), "reg_ctr": (torch.randn(B, N, 5, generator=gen) * 0.5).to(dev),
            "text_mask": torch.ones(B, T).to(dev)}


def time_ms(fn, reps):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--gts", type=int, nargs="+", default=[10, 50, 200])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prof_atss_loss: needs a CUDA device")
    import atss_oracle as ao
    from mqdet_b200 import _lib, ops
    _lib.load()
    dev = torch.device("cuda:0")
    info = gpu_info()
    rows = []
    for G in a.gts:
        d = inputs(a.batch, G, a.tokens, dev)
        lv = ops.get_levels(d["sizes"], dev)
        B, N, T = d["logits"].shape

        def ours():
            return ops.atss_loss(d["logits"], d["reg_ctr"], d["gt_boxes"], d["gt_labels"], d["gt_count"], d["gt_tokens"], lv, ao.STRIDES,
                                 ao.SIZES, ao.REG_SCALES, d["text_mask"])

        def restated():
            import atss_oracle
            match = torch.stack([atss_oracle.assign_image(*[x.to(dev) for x in atss_oracle.anchors(d["sizes"])], d["gt_boxes"][b])[0]
                                 for b in range(B)])
            return atss_oracle.losses_and_grads(d["logits"], d["reg_ctr"], match, d["sizes"], d["gt_boxes"], d["gt_labels"], d["gt_tokens"],
                                                ao.REG_SCALES, d["text_mask"])

        t_ours = time_ms(ours, a.reps)
        try:
            t_ref = time_ms(restated, max(2, a.reps // 10))
        except Exception as e:  # noqa: BLE001 - the comparator's device placement is reported, not fatal
            t_ref = None
            print(f"G={G}: restatement on CUDA failed: {type(e).__name__}: {e}")
        nbytes = 2.0 * B * N * T * 4 + 2.0 * B * N * 5 * 4 + B * N * 4
        bound_ms = nbytes / HBM_BPS * 1e3
        row = {"G": G, "B": B, "N": N, "T": T, "atss_loss_ms": t_ours, "restatement_autograd_ms": t_ref, "hbm_bound_ms": bound_ms,
               "fraction_of_hbm_bound": bound_ms / t_ours}
        rows.append(row)
        print(json.dumps(row))
    res = {"gpu": info, "rows": rows}
    print(json.dumps({"gpu": info}))
    out = a.out or tempfile.mkdtemp(prefix="prof_atss_loss_")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "atss_loss.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"wrote {os.path.join(out, 'atss_loss.json')}")


if __name__ == "__main__":
    main()
