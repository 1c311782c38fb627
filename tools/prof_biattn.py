"""One BiAttention fusion layer (BiAttentionBlockForCheckpoint.forward_flat) at the bench size (B=8, N=22400 image tokens,
T=256) on the product path: the layer norms, the small projection GEMMs, biattn_image_kernel and biattn_text_kernel.
    python tools/prof_biattn.py [reps]
runs the layer `reps` times (default 1) and, for reps > 1, prints its mean time per call from CUDA events."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from mqdet_b200.config import mq_glip_t_cfg
from mqdet_b200.utils.fuse_helper import BiAttentionBlockForCheckpoint
from tools import synth

dev = torch.device("cuda:0")
gen = synth.Gen(5)
blk = BiAttentionBlockForCheckpoint(v_dim=256, l_dim=768, embed_dim=2048, num_heads=8, hidden_dim=3072, dropout=0.1,
                                    drop_path=0.0, init_values=1.0 / 6, cfg=mq_glip_t_cfg())
blk.load_state_dict(synth.bi_attention_sd(gen), strict=True)
blk = blk.to(dev).eval()
B, N, T = 8, 22400, 256
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
