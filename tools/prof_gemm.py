"""GEMM shapes of the MQ-GLIP-T forward, timed with CUDA events (CUDA-graph replay to take the Python/ctypes launch
path out of the measurement) or run once each for ncu."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from mqdet_b200 import ops

dev = torch.device("cuda:0")
SHAPES = [  # (M, N, K, what)
    (179200, 2048, 256, "BiAttn v_proj / values_v (B=8)"),
    (179200, 256, 2048, "BiAttn out_v_proj (B=8)"),
    (179200, 256, 2304, "DyConv DCN conv (B=8)"),
    (2048, 3072, 768, "GCP/BERT FFN up (B=8)"),
    (2048, 768, 3072, "GCP/BERT FFN down (B=8)"),
    (2048, 512, 768, "GCP to_q (B=8)"),
    (8192, 8192, 8192, "square"),
]
mode = sys.argv[1] if len(sys.argv) > 1 else "time"
only = int(sys.argv[2]) if len(sys.argv) > 2 else None
res = {}
for i, (M, N, K, what) in enumerate(SHAPES):
    if only is not None and i != only:
        continue
    a = torch.randn(M, K, device=dev).half()
    b = torch.randn(N, K, device=dev).half()
    c = torch.empty(M, N, device=dev, dtype=torch.float16)
    if mode == "ncu":
        ops.gemm(a, b, out=c)
        torch.cuda.synchronize()
        continue
    for _ in range(3):
        ops.gemm(a, b, out=c)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for _ in range(10):
                ops.gemm(a, b, out=c)
    torch.cuda.synchronize()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    if mode == "timeonly":
        print(f"{M}x{N}x{K} ms={ms:.4f} tflops={2 * M * N * K / ms / 1e9:.1f}", flush=True)
        continue
    for _ in range(3):
        torch.matmul(a, b.T, out=c)
    e0.record()
    for _ in range(10):
        torch.matmul(a, b.T, out=c)
    e1.record()
    torch.cuda.synchronize()
    cms = e0.elapsed_time(e1) / 10
    for _ in range(3):
        ops.gemm(a, b, out=c, impl=ops.IMPL_TC_ONESHOT)
    e0.record()
    for _ in range(10):
        ops.gemm(a, b, out=c, impl=ops.IMPL_TC_ONESHOT)
    e1.record()
    torch.cuda.synchronize()
    oms = e0.elapsed_time(e1) / 10
    res[f"{M}x{N}x{K}"] = dict(what=what, ms=round(ms, 4), oneshot_ms=round(oms, 4), tflops=round(2 * M * N * K / ms / 1e9, 1), cublas_ms=round(cms, 4),
                               cublas_tflops=round(2 * M * N * K / cms / 1e9, 1),
                               out_gbs=round(M * N * 2 / ms / 1e6, 1))
    print(f"{M}x{N}x{K}", res[f"{M}x{N}x{K}"], flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
if mode == "time":
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", "gemm_shapes.json"), "w"), indent=1)
