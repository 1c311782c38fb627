"""DyConv's three DCNv2 convolutions at the bench shape: implicit GEMM (mqdet_dcn_conv, one launch) against the sampling
kernel + GEMM pair it replaces (3 x mqdet_dcn_cols + 3 x mqdet_gemm_f16).  Prints one JSON line, with the weight bytes the
implicit kernel streams from L2 into shared memory per launch (every 64-row tile reads the 36 k-blocks of 32 KB of its
branch's weight) and the card's name and power limit read in the same run.

    python tools/bench_dcn.py [--batch 8] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TILE_ROWS = 64                   # output rows per dcn_conv_kernel tile (dcnconv.cu DC_BM)
WEIGHT_TILE_BYTES = 36 * 32768   # 36 k-blocks of [256 x 64] fp16 per tile


def main():
    import torch
    from mqdet_b200 import ops
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    sizes = [(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)]
    lv = ops.Levels(sizes, dev)
    g = torch.Generator().manual_seed(0)
    B = a.batch
    x16 = torch.randn(B, lv.N, 256, generator=g).half().to(dev)
    om = (torch.randn(B, lv.N, 32, generator=g) * 0.5).to(dev)
    ks = [1, 2, 0]
    ws = [(torch.randn(256, 2304, generator=g) * 0.02).half().to(dev) for _ in ks]
    bs = [torch.randn(256, generator=g).to(dev) for _ in ks]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.iters):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2]

    t_imp = timed(lambda: ops.dcn_conv(x16, om, lv, ks, ws, bs))
    t_col = timed(lambda: [ops.gemm(ops.dcn_cols(x16, om, lv, k), w, bias=b) for k, w, b in zip(ks, ws, bs)])
    rows = B * (lv.N + 2 * lv.N1)
    flop = 2.0 * rows * 256 * 2304
    tiles = sum((B * r + TILE_ROWS - 1) // TILE_ROWS for r in (lv.N, lv.N1, lv.N1))
    w_bytes = tiles * WEIGHT_TILE_BYTES
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    card = q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)
    print(json.dumps({"shape": f"B={B}, rows {rows} x K 2304 x N 256 (three branches)", "implicit_ms": t_imp, "cols_gemm_ms": t_col,
                      "implicit_tflops": flop / t_imp / 1e9, "speedup": t_col / t_imp, "tiles": tiles,
                      "weight_gb_per_launch": w_bytes / 1e9, "weight_tb_per_s": w_bytes / t_imp / 1e9, "card": card,
                      "timing": "median of CUDA-event times, 256 MiB L2 flush between iterations"}))


if __name__ == "__main__":
    main()
