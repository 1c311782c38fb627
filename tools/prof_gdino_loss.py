"""Timing of the GroundingDINO training losses at config 4's per-GPU shape (B = 2, Q = 900, T = 256, L = 6 decoder layers).

    python tools/prof_gdino_loss.py [--gts 10 50 200] [--reps 20] [--out DIR]

For each GT count G per image:
  * ``step``: ``GroundingDINO.decoder_outputs_flat`` (the six layers' boxes and class logits from their hidden states) + the
    matching cost + the linear sum assignment + the losses and gradients (``SetCriterion.forward_flat``), captured once in a CUDA
    graph and replayed ``--reps`` times between two CUDA events;
  * ``solver``: ``ops.linear_sum_assignment`` alone on the twelve [900 x G] problems of that step (one warp per problem);
  * ``reference_style``: the path of the reference on the same CUDA tensors: the restatement's torch ops for the cost
    (tests/gdino_loss_oracle.py, the reference's matcher arithmetic), ``.cpu()`` and scipy per image and layer, then the losses
    and their autograd gradients (wall time per step, it synchronises by construction).
The card name and power limit are read in the same run.  JSON -> DIR/gdino_loss.json (default: a directory under the system temp
dir).  The decoder hidden states are synthetic: the timing does not depend on their values.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from tools.prof_atss_loss import gpu_info, time_ms  # noqa: E402


def decoder_state(model, B, Q, T, L, dev, seed=0):
    """what ``forward_device(..., all_layers=True)`` hands to ``decoder_outputs``: normed hidden states and references of every
    layer, valid ratios, the enhanced text and its mask."""
    import torch
    from mqdet_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    E = model.hidden_dim
    hs = [torch.randn(B, Q, E, generator=gen).to(dev) for _ in range(L)]
    refs = [torch.sigmoid(torch.randn(B, Q, 4, generator=gen) - 1.0).to(dev) for _ in range(L + 1)]
    text = torch.randn(B, T, E, generator=gen).to(dev)
    mask = torch.zeros(B, T, dtype=torch.bool)
    mask[0, :200], mask[1, :150] = True, True
    return {"hs": hs, "references": refs, "valid_ratios": torch.ones(B, 4, 2, device=dev),
            "transformer": {"memory_text": text, "memory_text16": ops.cast_f16(text)}, "text_token_mask": mask.to(dev)}


def gt_pack(B, G, T, dev, seed=0):
    import torch
    import gdino_loss_oracle as go
    gen = torch.Generator().manual_seed(seed)
    boxes = torch.stack([go._gt_boxes(gen, G) for _ in range(B)])
    tokens = torch.zeros(B, G, T)
    for b in range(B):
        for g in range(G):
            s = int(torch.randint(1, 140, (1,), generator=gen))
            tokens[b, g, s:s + 1 + g % 3] = 1.0
    return boxes.to(dev), torch.full((B,), G, dtype=torch.int32, device=dev), tokens.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gts", type=int, nargs="+", default=[10, 50, 200])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prof_gdino_loss: needs a CUDA device")
    import gdino_loss_oracle as go
    from mqdet_b200 import _lib, ops
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO
    _lib.load()
    dev = torch.device("cuda:0")
    info = gpu_info()
    model = GroundingDINO(mq_groundingdino_t_cfg()).to(dev).eval()
    B, Q, T, L = 2, model.num_queries, model.max_text_len, len(model.bbox_embed)
    st = decoder_state(model, B, Q, T, L, dev)
    rows = []
    for G in a.gts:
        pack = gt_pack(B, G, T, dev, seed=G)
        text_mask = torch.zeros(B, T, device=dev)
        text_mask[:, :st["text_token_mask"].shape[1]] = st["text_token_mask"].float()

        def step():
            logits, boxes = model.decoder_outputs_flat(st)
            return model.loss_evaluator.forward_flat(logits, boxes, pack, text_mask)

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            r = step()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            r = step()
        t_step = time_ms(g.replay, a.reps)
        cost = r["cost"].view(L * B, Q, G).clone()
        counts = pack[1].repeat(L)
        t_solver = time_ms(lambda: ops.linear_sum_assignment(cost, counts), a.reps)
        logits, boxes = model.decoder_outputs_flat(st)

        def reference_style():
            _, match = go.match_layers(logits, boxes, *pack)
            return go.losses_and_grads(logits, boxes, match, *pack, text_mask)

        reference_style()
        torch.cuda.synchronize()
        n = max(2, a.reps // 10)
        t0 = time.perf_counter()
        for _ in range(n):
            reference_style()
        torch.cuda.synchronize()
        t_ref = (time.perf_counter() - t0) / n * 1e3
        row = {"G": G, "B": B, "Q": Q, "T": T, "L": L, "step_graph_ms": t_step, "solver_ms": t_solver, "reference_style_ms": t_ref}
        rows.append(row)
        print(json.dumps(row))
    res = {"gpu": info, "rows": rows}
    print(json.dumps({"gpu": info}))
    out = a.out or tempfile.mkdtemp(prefix="prof_gdino_loss_")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "gdino_loss.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"wrote {os.path.join(out, 'gdino_loss.json')}")


if __name__ == "__main__":
    main()
