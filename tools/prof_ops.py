"""Single hot operators at the bench shape (B=8, 800x1344), for ncu captures and CUDA-event timings:

    python tools/prof_ops.py swin_fc1|swin_fc2|swin_qkv|swin_proj|dcn|conv_off|ln1 [reps]
    ncu --set full --import-source on --clock-control none -k regex:gemm_wg -c 1 -o prof_swin_fc1 python tools/prof_ops.py swin_fc1 1

Prints the median CUDA-event time per call (256 MiB L2 flush between calls) with the algorithmic GB/s and TFLOP/s.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from mqdet_b200 import ops
from mqdet_b200._lib import ACT_GELU, ACT_NONE

dev = torch.device("cuda:0")
which = sys.argv[1] if len(sys.argv) > 1 else "swin_fc1"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 7
g = torch.Generator().manual_seed(0)
M1 = 8 * 200 * 336  # stage-1 tokens


def rnd(*s, scale=1.0):
    return (torch.randn(*s, generator=g) * scale).half().to(dev)


GEMMS = {  # name: (M, N, K, act, residual)
    "swin_fc1": (M1, 384, 96, ACT_GELU, False), "swin_fc2": (M1, 96, 384, ACT_NONE, True),
    "swin_qkv": (M1, 288, 96, ACT_NONE, False), "swin_proj": (M1, 96, 96, ACT_NONE, True),
    "s2_fc1": (M1 // 4, 768, 192, ACT_GELU, False), "s3_fc1": (M1 // 16, 1536, 384, ACT_GELU, False),
    "s3_fc2": (M1 // 16, 384, 1536, ACT_NONE, True),
}
if which in GEMMS:
    M, N, K, act, res = GEMMS[which]
    a, w = rnd(M, K), rnd(N, K, scale=0.05)
    bias = torch.randn(N, generator=g).to(dev)
    r = rnd(M, N) if res else None
    fn = lambda: ops.gemm(a, w, bias=bias, act=act, residual=r)  # noqa: E731
    byt = 2.0 * (M * K + N * K + M * N * (2 if res else 1))
    flop = 2.0 * M * N * K
elif which == "dcn":
    lv = ops.Levels([(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)], dev)
    x16 = rnd(8, lv.N, 256)
    om = (torch.randn(8, lv.N, 32, generator=g) * 0.5).to(dev)
    ws = [rnd(256, 2304, scale=0.02) for _ in range(3)]
    bs = [torch.randn(256, generator=g).to(dev) for _ in range(3)]
    fn = lambda: ops.dcn_conv(x16, om, lv, [1, 2, 0], ws, bs)  # noqa: E731
    rows = 8 * (lv.N + 2 * lv.N1)
    byt = 2.0 * (8 * lv.N * 256 + rows * 256) + 3 * 2.0 * 256 * 2304
    flop = 2.0 * rows * 256 * 2304
elif which == "dyconv":
    # one whole DyConv layer (offset conv, dcn_conv, chan_stats, gn_attn, combine, DyReLU) for multi-kernel ncu captures
    from mqdet_b200.modeling.rpn.vldyhead import Conv3x3Norm, DyConv
    from tools import synth
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from util import load_sd
    gen = synth.Gen(3)
    conv_func = lambda i, o, s: Conv3x3Norm(i, o, s, deformable=True, bn_type=["gn", 16])  # noqa: E731
    mod = load_sd(DyConv(256, 256, conv_func=conv_func, use_dyrelu=True, use_dyfuse=True, use_deform=True), synth.dyconv_sd(gen))
    mod = mod.to(dev).eval()
    lv = ops.Levels([(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)], dev)
    x16 = rnd(8, lv.N, 256)
    fn = lambda: mod.forward_flat(x16, lv)  # noqa: E731
    byt, flop = 2.0 * 2 * 8 * lv.N * 256, 2.0 * 8 * (lv.N + 2 * lv.N1) * 256 * 2304
elif which == "conv_off":
    lv = ops.Levels([(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)], dev)
    x16 = rnd(8, lv.N, 256)
    w = rnd(27, 2304, scale=0.02)
    b = torch.randn(27, generator=g).to(dev)
    fn = lambda: ops.conv3x3_small(x16, w, b, lv)  # noqa: E731
    byt = 2.0 * 8 * lv.N * 256 + 4.0 * 8 * lv.N * 32
    flop = 2.0 * 8 * lv.N * 27 * 2304
elif which == "ln1":
    x = rnd(M1, 96)
    wt, bt = torch.ones(96, device=dev), torch.zeros(96, device=dev)
    fn = lambda: ops.layernorm(x, wt, bt, 1e-5)  # noqa: E731
    byt, flop = 4.0 * M1 * 96, 0.0
else:
    raise SystemExit(f"unknown op {which}")

flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
fn()
torch.cuda.synchronize()
ts = []
for _ in range(reps):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
ts.sort()
t = ts[len(ts) // 2]
print(f"{which}: {t:.4f} ms  {byt / t / 1e6:.0f} GB/s algorithmic  {flop / t / 1e9:.1f} TFLOP/s")
