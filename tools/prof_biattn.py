"""The BiAttention fusion at the bench size (B=8, N=22400 image tokens, T=256, H=8).
    python tools/prof_biattn.py [reps]
1. One BiAttention fusion layer (BiAttentionBlockForCheckpoint.forward_flat) on the product path: the layer norms, the small
   projection GEMMs, biattn_image_kernel and biattn_text_kernel.  It runs `reps` times (default 1) and, for reps > 1, prints its
   mean time per call from CUDA events.
2. For reps > 1, the image side alone: one ops.biattn_image call (biattn_image_kernel and its colmax_reduce_kernel) captured in a
   CUDA graph 20 times and replayed `reps` times.  It prints ms per call, the executed tensor TFLOP/s (S and P.mT per head), the
   rate at which the kernel feeds shared memory from L2 (per tile: the image-token tile once, then 8 k-blocks of 32 KB per
   head), and the card's name and power limit read in the same run.
3. For reps > 1, the text side alone: one ops.biattn_text_vn call (biattn_text_kernel) as the fusion layer issues it -- q is the
   image tokens broadcast over the heads, colmax comes from the image side -- timed the same way.  It prints ms per call, the
   executed TFLOP/s (S^T and P.vn per head) and the L2 -> shared rate from the kernel's own loads (per CTA of 128 text tokens:
   the two K tiles once, then one [64 x 256] image-token tile per step of 64 image tokens)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from mqdet_b200 import ops
from mqdet_b200.config import mq_glip_t_cfg
from mqdet_b200.utils.fuse_helper import BiAttentionBlockForCheckpoint
from tools import synth

dev = torch.device("cuda:0")
gen = synth.Gen(5)
blk = BiAttentionBlockForCheckpoint(v_dim=256, l_dim=768, embed_dim=2048, num_heads=8, hidden_dim=3072, dropout=0.1,
                                    drop_path=0.0, init_values=1.0 / 6, cfg=mq_glip_t_cfg())
blk.load_state_dict(synth.bi_attention_sd(gen), strict=True)
blk = blk.to(dev).eval()
B, N, T, H = 8, 22400, 256, 8
v16 = gen.randn(B, N, 256).half().to(dev)
l32 = gen.randn(B, T, 768).to(dev)
mask = torch.ones(B, T, dtype=torch.long, device=dev)
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 1
for _ in range(reps):
    blk.forward_flat(v16, l32, mask)
torch.cuda.synchronize()
if reps > 1:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        blk.forward_flat(v16, l32, mask)
    e1.record()
    torch.cuda.synchronize()
    print(f"BiAttention layer: {e0.elapsed_time(e1) / reps:.3f} ms")

    def graph_ms(call, per_graph=20):
        """ms per call of `call`, captured per_graph times in one CUDA graph and replayed reps times"""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(per_graph):
                call()
        g.replay()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (reps * per_graph)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    card = q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)

    args = dict(vn16=v16, gT=(gen.randn(B, H, T, 256) * 0.2).half().to(dev), gbias=gen.randn(B, H, T, 8).to(dev),
                mT=(gen.randn(B, H, 256, T) * 0.25).half().to(dev), bias=gen.randn(256).to(dev), gamma=gen.randn(256).to(dev),
                residual=gen.randn(B, N, 256).half().to(dev), mask=mask.float(), clamp=5.0e4, heads=H)
    ms = graph_ms(lambda: ops.biattn_image(**args))
    tiles = B * ((N + 63) // 64)
    executed = B * H * 2.0 * (2.0 * N * T * 256)
    l2_bytes = tiles * (64 * 256 * 2 + H * 8 * 256 * 64 * 2)
    print(f"biattn_image (B={B} N={N} T={T} H={H}): {ms:.3f} ms per call, {executed / ms / 1e9:.1f} TFLOP/s executed, "
          f"{l2_bytes / ms / 1e6:.0f} GB/s L2 -> shared, on {card}")

    _, colmax = ops.biattn_image(**args)
    u = torch.empty((B, H, T, 256), dtype=torch.float16, device=dev)
    qh = v16.view(B, 1, N, 256).expand(B, H, N, 256)
    ms = graph_ms(lambda: ops.biattn_text_vn(args["gT"], qh, v16, colmax, 5.0e4, u, rowbias=args["gbias"]))
    ctas = B * H * ((T + 127) // 128)
    l2_bytes = ctas * (min(T, 128) * 256 * 2 + ((N + 63) // 64) * 64 * 256 * 2)
    print(f"biattn_text (B={B} N={N} T={T} H={H}): {ms:.3f} ms per call, {executed / ms / 1e9:.1f} TFLOP/s executed, "
          f"{l2_bytes / ms / 1e6:.0f} GB/s L2 -> shared, on {card}")
