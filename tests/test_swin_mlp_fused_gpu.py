"""GPU checks of the fused Swin MLP kernel (ops.swin_mlp: LN2 -> fc1 -> GELU -> fc2 -> residual in one launch) against the
three-launch chain it replaces (layernorm -> gemm with bias + GELU -> gemm with bias + fp32 residual) on identical inputs.
The two must be bit-identical: the LN arithmetic, the k16 wgmma chains and the epilogue operation order are the same.
Covered: the bench's stage-1 / stage-2 shapes, ragged row counts, a single tile, fewer tiles than SMs, one reserved SM,
graph replay with new inputs, and the whole Swin-T backbone with the fused path on and off."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(g, *shape, s=0.5):
    return torch.randn(*shape, generator=g) * s


def _params(dev, g, C):
    H = 4 * C
    return dict(ln_w=(1 + _mk(g, C, s=0.1)).to(dev), ln_b=_mk(g, C, s=0.1).to(dev), eps=1e-5,
                w1=_mk(g, H, C, s=0.1).half().to(dev), b1=_mk(g, H, s=0.5).to(dev),
                w2=_mk(g, C, H, s=0.05).half().to(dev), b2=_mk(g, C, s=0.5).to(dev))


def _chain(x, p):
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU
    xn = ops.layernorm(x, p["ln_w"], p["ln_b"], p["eps"])
    h = ops.gemm(xn, p["w1"], bias=p["b1"], act=ACT_GELU)
    return ops.gemm(h, p["w2"], bias=p["b2"], out_dtype=torch.float32, residual=x)


def _fused(x, p):
    from mqdet_b200 import ops
    return ops.swin_mlp(x, p["ln_w"], p["ln_b"], p["eps"], p["w1"], p["b1"], p["w2"], p["b2"])


# (rows, C): the bench's stage-1 / stage-2 shapes (B = 8), ragged rows (not a multiple of the 64-row tile, and an odd tile
# count, so one consumer warpgroup idles in the last round), a single (partial) tile, fewer tiles than SMs
SHAPES = [(537600, 96), (134400, 192), (64 * 1001 + 37, 96), (64 * 333 + 1, 192), (40, 96), (64, 192), (64 * 50 + 5, 96),
          (64 * 7, 192)]


@pytest.mark.parametrize("rows,C", SHAPES)
def test_fused_equals_chain(dev, rows, C):
    g = torch.Generator(device="cpu").manual_seed(rows + C)
    p = _params(dev, g, C)
    x = _mk(g, rows, C, s=1.0).to(dev)
    ref = _chain(x, p)
    out = _fused(x, p)
    assert torch.equal(out, ref), (out - ref).abs().max().item()


def test_reserved_sm(dev):
    """131 CTAs: tile schedules with a remainder on some CTAs."""
    from mqdet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(5)
    try:
        _lib.check(lib.mqdet_reserve_sms(1), "reserve_sms")
        for rows, C in [(64 * 1000 + 9, 96), (64 * 263, 192)]:
            p = _params(dev, g, C)
            x = _mk(g, rows, C, s=1.0).to(dev)
            assert torch.equal(_fused(x, p), _chain(x, p)), (rows, C)
    finally:
        _lib.check(lib.mqdet_reserve_sms(0), "reserve_sms")


def test_graph_replay_new_inputs(dev):
    """Two dependent fused launches (stage-1 then stage-2 width) captured once and replayed with new input contents equal
    eager launches on those contents."""
    g = torch.Generator(device="cpu").manual_seed(9)
    p1, p2 = _params(dev, g, 96), _params(dev, g, 192)
    x1 = torch.empty(64 * 900 + 3, 96, device=dev)
    x2 = torch.empty(64 * 400 + 17, 192, device=dev)
    x1.copy_(_mk(g, *x1.shape, s=1.0))
    x2.copy_(_mk(g, *x2.shape, s=1.0))
    _fused(x1, p1), _fused(x2, p2)  # warm-up: tensor maps and the shared-memory opt-in outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y1 = _fused(x1, p1)
        y2 = _fused(x2 + 0.0, p2)
    for seed in (1, 2):
        gg = torch.Generator(device="cpu").manual_seed(100 + seed)
        x1.copy_(_mk(gg, *x1.shape, s=1.0))
        x2.copy_(_mk(gg, *x2.shape, s=1.0))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y1, _chain(x1, p1))
        assert torch.equal(y2, _chain(x2, p2))


def test_bad_arguments(dev):
    from mqdet_b200 import ops
    from mqdet_b200._lib import MqdetError
    g = torch.Generator(device="cpu").manual_seed(3)
    p = _params(dev, g, 128 // 32 * 32)  # C = 128 is not supported
    with pytest.raises(MqdetError):
        _fused(torch.zeros(64, 128, device=dev), p)
    p = _params(dev, g, 96)
    with pytest.raises(MqdetError):
        ops.swin_mlp(torch.zeros(64, 96, device=dev), p["ln_w"], p["ln_b"], 1e-5, p["w2"], p["b1"], p["w1"], p["b2"])


def test_backbone_fused_equals_unfused(dev):
    """The whole Swin-T backbone (stages 1-2 fused) gives the same bits with the fused MLP on and off."""
    from mqdet_b200.modeling.backbone.swint import SwinTransformer, SwinTransformerBlock
    torch.manual_seed(0)
    m = SwinTransformer().to(dev).eval()
    with torch.no_grad():
        for prm in m.parameters():
            prm.add_(torch.randn_like(prm) * 0.02)
    g = torch.Generator(device="cpu").manual_seed(7)
    img = _mk(g, 2, 3, 480, 640, s=1.0).to(dev)
    assert SwinTransformerBlock.fused_mlp
    on = m.forward_flat(img, want=(0, 1, 2, 3))
    try:
        SwinTransformerBlock.fused_mlp = False
        off = m.forward_flat(img, want=(0, 1, 2, 3))
    finally:
        SwinTransformerBlock.fused_mlp = True
    for i in on:
        assert torch.equal(on[i][0], off[i][0]), i
