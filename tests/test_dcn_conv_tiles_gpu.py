"""dcn_conv_kernel's tile edges and its split of the gather over four threads per pixel.  Shapes that put the edges of 64-
and 128-row tiles everywhere: rows per job not a multiple of the tile, a job shorter than one tile, tiles straddling levels
and images, B = 1, one level (branch 1 only), no offset/mask tensor.  Checked against the sampling kernel + GEMM pair, and
for bit-identical reruns and CUDA-graph replays."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _case(sizes, B, with_om, dev, seed):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(seed)
    lv = ops.Levels(sizes, dev)
    x16 = torch.randn(B, lv.N, 256, generator=g).half().to(dev)
    om = None
    if with_om:
        om = torch.randn(B, lv.N, 32, generator=g)
        om[..., :18] *= 2.5
        om = om.to(dev).contiguous()
    ks = [1, 2, 0] if len(sizes) > 1 else [1]
    ws = [(torch.randn(256, 2304, generator=g) * 0.03).half().to(dev) for _ in ks]
    bs = [torch.randn(256, generator=g).to(dev) for _ in ks]
    return lv, x16, om, ks, ws, bs


@pytest.mark.parametrize("sizes,B,with_om", [
    ([(13, 17), (7, 9), (4, 5), (2, 3), (1, 1)], 3, True),    # 933 / 270 rows: ragged last tiles, tiles across images
    ([(13, 17), (7, 9), (4, 5), (2, 3), (1, 1)], 3, False),   # the same without offsets / mask
    ([(9, 11), (3, 4), (2, 2)], 1, True),                     # B = 1; 115 and 16 rows: every job shorter than one tile
    ([(9, 11), (3, 4), (2, 2)], 1, False),
    ([(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)], 2, True),  # 1502 / 382 rows: tiles straddle levels and images
    ([(16, 24)], 1, True),                                    # one level, branch 1 only: exactly three tiles
    ([(11, 13)], 3, False),                                   # one level, 429 rows, no offsets / mask
])
def test_dcn_conv_128_row_tiles_equal_cols_gemm(dev, sizes, B, with_om):
    from mqdet_b200 import ops
    lv, x16, om, ks, ws, bs = _case(sizes, B, with_om, dev, 17)
    ys = ops.dcn_conv(x16, om, lv, ks, ws, bs)
    for k, w, b, y in zip(ks, ws, bs, ys):
        ref = ops.gemm(ops.dcn_cols(x16, om, lv, k), w, bias=b)
        assert y.shape == ref.shape
        err = (y.float() - ref.float()).abs().max().item()
        assert err <= 2e-3 * ref.float().abs().max().item(), (k, err, ref.float().abs().max().item())


def test_dcn_conv_reruns_and_graph_replay_bit_identical(dev):
    from mqdet_b200 import ops
    lv, x16, om, ks, ws, bs = _case([(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)], 3, True, dev, 23)
    y1 = ops.dcn_conv(x16, om, lv, ks, ws, bs)
    y2 = ops.dcn_conv(x16, om, lv, ks, ws, bs)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.dcn_conv(x16, om, lv, ks, ws, bs)   # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = ops.dcn_conv(x16, om, lv, ks, ws, bs)
    for y in yg:
        y.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, b, c in zip(y1, y2, yg):
        assert torch.equal(a, b)
        assert torch.equal(a, c)
