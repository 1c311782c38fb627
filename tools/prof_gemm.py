"""Per-shape profile of the GEMM launches of one MQ-GLIP-T forward at the bench shape (B = 8, 800x1333, 80-class prompt).

    python tools/prof_gemm.py [--batch 8] [--out DIR] [--reps 20]

One eager ``forward_device`` (stream overlap off, as bench.py's roofline pass) is recorded with ``ops.GEMM_PROFILE`` and every
``ops.gemm`` call's arguments: M, N, K, batch, output dtype and epilogue (bias, activation, gate, fp16 / fp32 residual).  Each
distinct launch is then replayed from a CUDA graph of ``--reps`` back-to-back launches on the operands the forward used, with
the product kernel and, as a yardstick only, ``torch.matmul`` (cuBLAS, fp16 out, no epilogue) on the same A and B.

Per shape: count per step, us per launch, the lower bound max(bytes / 3.35 TB/s, flops / (0.7 * 989 TFLOP/s)) with bytes and
flops computed from the shape (every operand once, the output, the residual), the fraction of that bound reached, and ms per
step (count x us).  The card name, power limit and max SM clock are read in the same run.  JSON -> DIR/gemm_shapes.json.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12           # H100 SXM data sheet, HBM3
TENSOR_FLOPS = 0.7 * 989e12  # 70 % of the dense fp16 data-sheet rate


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"error": str(e)}


def epilogue_tag(kw):
    from mqdet_b200._lib import ACT_GELU, ACT_RELU, VEC_PER_COL, VEC_PER_ROW, VEC_SCALAR
    t = []
    if kw.get("bias") is not None:
        t.append("bias_col" if kw.get("bias_mode", VEC_PER_COL) == VEC_PER_COL else "bias_row")
    act = kw.get("act", 0)
    if act == ACT_GELU:
        t.append("gelu")
    elif act == ACT_RELU:
        t.append("relu")
    if kw.get("clamp", 0.0):
        t.append("clamp")
    if kw.get("gate") is not None:
        t.append({VEC_SCALAR: "gate_s", VEC_PER_COL: "gate_col", VEC_PER_ROW: "gate_row"}.get(kw.get("gate_mode"), "gate"))
    r = kw.get("residual")
    if r is not None:
        t.append("res_f32" if r.element_size() == 4 else "res_f16")
    return "+".join(t) or "-"


def shape_cost(M, N, K, nb, a, b, out, kw):
    es_o = out.element_size()
    na = a.numel() // (M * K) if a.dim() > 2 else 1
    nbw = b.numel() // (N * K) if b.dim() > 2 else 1
    by = 2.0 * M * K * na + 2.0 * N * K * nbw + es_o * M * N * nb
    if kw.get("residual") is not None:
        by += kw["residual"].element_size() * M * N * nb
    fl = 2.0 * M * N * K * nb
    return by, fl, max(by / HBM_BPS, fl / TENSOR_FLOPS) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "mqdet_prof_gemm"),
                    help="directory of the JSON result (default: a directory under the system temp dir)")
    ap.add_argument("--tag", default="", help="label stored with the results (e.g. the build)")
    args = ap.parse_args()

    import torch
    import bench
    from mqdet_b200 import _lib, ops
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
    from mqdet_b200.structures.image_list import ImageList
    from tools import synth

    _lib.load()
    dev = torch.device("cuda:0")
    B = args.batch
    _, ids, am, pmap, bank, img = bench.build_inputs(B, 1235)
    sd = synth.detector_sd(synth.Gen(99), bias0=-math.log((1 - 0.01) / 0.01))  # bench.py's default
    model = GeneralizedVLRCNN_New(mq_glip_t_cfg())
    own = model.state_dict()
    for k in own:
        if k.endswith("relative_position_index"):
            sd[k] = own[k]
    model.load_state_dict(sd, strict=True)
    del sd
    model = model.to(dev).eval()
    model.query_selector.set_query_bank(bank)
    caps = {"input_ids": ids, "attention_mask": am}
    il = ImageList(img.to(dev), [(bench.H_IMG, bench.W_IMG)] * B)
    model.rpn.head.overlap_text_stream = model.overlap_text_prefix = False
    model.forward_device(il, caps, pmap)  # warm-up: caches, tensor maps, module loads
    torch.cuda.synchronize()

    # ---- record one forward: every ops.gemm call with its operands, timed by ops.GEMM_PROFILE ----
    calls = []
    orig = ops.gemm

    def rec(a, b, out=None, **kw):
        o = orig(a, b, out, **kw)
        calls.append((a, b, o, kw))
        return o

    ops.gemm = rec
    ops.GEMM_PROFILE = []
    model.forward_device(il, caps, pmap)
    torch.cuda.synchronize()
    prof, ops.GEMM_PROFILE, ops.gemm = ops.GEMM_PROFILE, None, orig
    assert len(prof) == len(calls), (len(prof), len(calls))

    groups = {}
    for (e0, e1, _, (M, N, K, nb)), (a, b, o, kw) in zip(prof, calls):
        key = (M, N, K, nb, str(o.dtype).replace("torch.", ""), epilogue_tag(kw))
        g = groups.setdefault(key, {"count": 0, "eager_ms": 0.0, "args": (a, b, o, kw)})
        g["count"] += 1
        g["eager_ms"] += e0.elapsed_time(e1)
    del calls

    def graph_us(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                for _ in range(args.reps):
                    fn()
        torch.cuda.synchronize()
        g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (3 * args.reps)

    rows = []
    for (M, N, K, nb, odt, epi), g in groups.items():
        a, b, o, kw = g["args"]
        us = graph_us(lambda: orig(a, b, o, **kw))
        bt = b.transpose(-1, -2)
        try:
            cu = graph_us(lambda: torch.matmul(a, bt))
        except RuntimeError:  # a view torch.matmul cannot take as is
            cu = float("nan")
        by, fl, bound = shape_cost(M, N, K, nb, a, b, o, kw)
        rows.append({"M": M, "N": N, "K": K, "batch": nb, "out": odt, "epilogue": epi, "count": g["count"],
                     "us": round(us, 2), "cublas_us": round(cu, 2), "bound_us": round(bound, 2),
                     "frac_of_bound": round(bound / us, 3), "ms_per_step": round(g["count"] * us / 1e3, 3),
                     "eager_ms_per_step": round(g["eager_ms"], 3), "gbytes": round(by / 1e9, 4), "gflop": round(fl / 1e9, 2)})
        del g["args"]
    rows.sort(key=lambda r: -r["ms_per_step"])
    tot = sum(r["ms_per_step"] for r in rows)
    totb = sum(r["count"] * r["bound_us"] for r in rows) / 1e3
    info = gpu_info()
    print(f"# {info}  batch {B}  launches {sum(r['count'] for r in rows)}  distinct {len(rows)}  {args.tag}")
    print(f"{'M':>7} {'N':>5} {'K':>5} {'nb':>4} {'out':>7} {'epilogue':<22} {'cnt':>4} {'us':>9} {'cublas':>9} {'bound':>8} "
          f"{'frac':>6} {'ms/step':>8}")
    for r in rows:
        print(f"{r['M']:>7} {r['N']:>5} {r['K']:>5} {r['batch']:>4} {r['out']:>7} {r['epilogue']:<22} {r['count']:>4} "
              f"{r['us']:>9.2f} {r['cublas_us']:>9.2f} {r['bound_us']:>8.2f} {r['frac_of_bound']:>6.3f} {r['ms_per_step']:>8.3f}")
    print(f"# total {tot:.2f} ms/step (graph-replayed, summed per shape), bound {totb:.2f} ms/step, "
          f"eager {sum(r['eager_ms_per_step'] for r in rows):.2f} ms/step")
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"gemm_shapes{('_' + args.tag) if args.tag else ''}.json")
    print(f"# -> {path}")
    with open(path, "w") as f:
        json.dump({"gpu": info, "batch": B, "tag": args.tag, "total_ms_per_step": tot, "bound_ms_per_step": totb,
                   "shapes": rows}, f, indent=1)


if __name__ == "__main__":
    main()
