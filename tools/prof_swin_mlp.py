"""The fused Swin MLP kernel against the three launches it replaces, at the bench's shapes (B = 8, 800x1333 padded to
800x1344: stage 1 = 537600 x 96, stage 2 = 134400 x 192, two blocks each).

    python tools/prof_swin_mlp.py [--batch 8] [--reps 20] [--out DIR]

Per shape, on the same seeded inputs: ``ops.swin_mlp`` and the unfused chain (``layernorm`` -> fc1 ``gemm`` with bias + GELU ->
fc2 ``gemm`` with bias + fp32 residual), each replayed from a CUDA graph of ``--reps`` back-to-back launches after a warm-up.
Reported: us per block, the bound max(bytes / 3.35 TB/s, flops / (0.7 * 989 TFLOP/s)) and the fraction of it reached.  The fused
kernel's bytes are the fp32 rows in and out and the weights; the chain's add the fp16 LN output and the fp16 hidden activation
written and read back.  Both outputs are compared bit for bit.  The card name, power limit and max SM clock are read in the
same run.  JSON -> DIR/swin_mlp.json.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.prof_gemm import HBM_BPS, TENSOR_FLOPS, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "mqdet_prof_swin_mlp"),
                    help="directory of the JSON result (default: a directory under the system temp dir)")
    args = ap.parse_args()

    import torch
    from mqdet_b200 import _lib, ops
    from mqdet_b200._lib import ACT_GELU

    _lib.load()
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(0)
    tokens1 = args.batch * (800 // 4) * (1344 // 4)

    def graph_us(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(gr, stream=s):
                for _ in range(args.reps):
                    fn()
        torch.cuda.synchronize()
        gr.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            gr.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (3 * args.reps)

    rows = []
    for stage, (M, C) in enumerate([(tokens1, 96), (tokens1 // 4, 192)], start=1):
        H = 4 * C
        x = (torch.randn(M, C, generator=g)).to(dev)
        ln_w, ln_b = (1 + 0.1 * torch.randn(C, generator=g)).to(dev), (0.1 * torch.randn(C, generator=g)).to(dev)
        w1, b1 = (0.1 * torch.randn(H, C, generator=g)).half().to(dev), (0.5 * torch.randn(H, generator=g)).to(dev)
        w2, b2 = (0.05 * torch.randn(C, H, generator=g)).half().to(dev), (0.5 * torch.randn(C, generator=g)).to(dev)
        xn = torch.empty(M, C, dtype=torch.float16, device=dev)
        h = torch.empty(M, H, dtype=torch.float16, device=dev)
        y_chain = torch.empty(M, C, dtype=torch.float32, device=dev)
        out = {}

        def chain():  # as SwinTransformerBlock.forward_flat runs it with fused_mlp off
            xn_ = ops.layernorm(x, ln_w, ln_b, 1e-5)
            h_ = ops.gemm(xn_, w1, bias=b1, act=ACT_GELU)
            out["chain"] = ops.gemm(h_, w2, bias=b2, out_dtype=torch.float32, residual=x)

        def fused():
            out["y"] = ops.swin_mlp(x, ln_w, ln_b, 1e-5, w1, b1, w2, b2)

        def chain_parts():
            return (graph_us(lambda: ops.layernorm(x, ln_w, ln_b, 1e-5)),
                    graph_us(lambda: ops.gemm(xn, w1, h, bias=b1, act=ACT_GELU)),
                    graph_us(lambda: ops.gemm(h, w2, y_chain, bias=b2, out_dtype=torch.float32, residual=x)))

        us_f = graph_us(fused)
        us_c = graph_us(chain)
        parts = chain_parts()
        chain()
        fused()
        torch.cuda.synchronize()
        equal = bool(torch.equal(out["y"], out["chain"]))
        fl = 2.0 * 2.0 * M * C * H
        by_w = 2.0 * 2.0 * H * C
        by_f = 4.0 * 2 * M * C + by_w
        by_c = by_f + 2.0 * 2 * M * C + 2.0 * 2 * M * H  # + xn written and read, + h written and read
        bound_f = max(by_f / HBM_BPS, fl / TENSOR_FLOPS) * 1e6
        bound_c = max(by_c / HBM_BPS, fl / TENSOR_FLOPS) * 1e6
        rows.append({"stage": stage, "M": M, "C": C, "fused_us": round(us_f, 2), "chain_us": round(us_c, 2),
                     "chain_parts_us": {"layernorm": round(parts[0], 2), "fc1_gelu": round(parts[1], 2),
                                        "fc2_residual": round(parts[2], 2)},
                     "fused_over_chain": round(us_f / us_c, 3), "fused_bound_us": round(bound_f, 2),
                     "fused_frac_of_bound": round(bound_f / us_f, 3), "chain_bound_us": round(bound_c, 2),
                     "chain_frac_of_bound": round(bound_c / us_c, 3), "bit_identical": equal,
                     "gbytes_fused": round(by_f / 1e9, 4), "gbytes_chain": round(by_c / 1e9, 4), "gflop": round(fl / 1e9, 2)})
        del x, xn, h, y_chain, out

    info = gpu_info()
    print(f"# {info}  batch {args.batch}  reps {args.reps}")
    print(f"{'stage':>5} {'M':>7} {'C':>4} {'fused us':>9} {'chain us':>9} {'LN':>7} {'fc1':>7} {'fc2':>7} {'ratio':>6} "
          f"{'bound':>7} {'frac':>6} {'equal':>6}")
    for r in rows:
        p = r["chain_parts_us"]
        print(f"{r['stage']:>5} {r['M']:>7} {r['C']:>4} {r['fused_us']:>9.2f} {r['chain_us']:>9.2f} {p['layernorm']:>7.1f} "
              f"{p['fc1_gelu']:>7.1f} {p['fc2_residual']:>7.1f} {r['fused_over_chain']:>6.3f} {r['fused_bound_us']:>7.1f} "
              f"{r['fused_frac_of_bound']:>6.3f} {str(r['bit_identical']):>6}")
    per_step_f = 2 * sum(r["fused_us"] for r in rows) / 1e3
    per_step_c = 2 * sum(r["chain_us"] for r in rows) / 1e3
    print(f"# per step (two blocks per stage): fused {per_step_f:.3f} ms, chain {per_step_c:.3f} ms")
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "swin_mlp.json")
    print(f"# -> {path}")
    with open(path, "w") as f:
        json.dump({"gpu": info, "batch": args.batch, "reps": args.reps, "per_step_ms": {"fused": per_step_f, "chain": per_step_c},
                   "shapes": rows}, f, indent=1)


if __name__ == "__main__":
    main()
