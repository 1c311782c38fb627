"""GPU parity of the persistent wgmma GEMM: the Swin / FPN shapes of the B = 8 forward, tile counts that are not a multiple of
the grid, ragged edges, outputs that take no paired stores, the one-tile-per-CTA launch and graph replay.  Reference: the same op in
torch fp32, tolerances of test_gemm_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _check(out, ref, out_is_f16):
    out = out.float()
    scale = ref.abs().max().item() + 1e-6
    err = (out - ref).abs().max().item()
    tol = scale * (1.5e-3 if out_is_f16 else 2e-5)
    assert err <= tol, f"max err {err:.3e} > tol {tol:.3e} (scale {scale:.3e})"


def _mk(g, *shape, s=0.5):
    return torch.randn(*shape, generator=g) * s


def _ref(a, b, bias=None, gelu=False, residual=None):
    v = a.float() @ b.float().transpose(-1, -2)
    if bias is not None:
        v = v + bias
    if gelu:
        v = torch.nn.functional.gelu(v)
    if residual is not None:
        v = v + residual.float()
    return v


@pytest.mark.parametrize("M,N,K,kind", [
    (537600, 288, 96, "qkv"),          # Swin stage 1 at B = 8: qkv, full M
    (537600, 96, 96, "proj"),          # window-attention projection + fp32 residual
    (537600, 384, 96, "fc1"),          # MLP up + GELU
    (134400, 96, 384, "fc2"),          # MLP down (stage-2 sized M) + fp32 residual
    (33600, 384, 384, "qkv"),          # stage 3
    (8400, 256, 768, "fpn"),           # FPN 1x1
])
def test_swin_fpn_shapes(dev, M, N, K, kind):
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = _mk(g, M, K).half().to(dev)
    b = _mk(g, N, K, s=0.1).half().to(dev)
    bias = _mk(g, N, s=1).to(dev)
    if kind in ("proj", "fc2"):
        r = _mk(g, M, N, s=1).to(dev)
        out = ops.gemm(a, b, bias=bias, residual=r, out_dtype=torch.float32)
        _check(out, _ref(a, b, bias, residual=r), False)
    elif kind == "fc1":
        _check(ops.gemm(a, b, bias=bias, act=ACT_GELU), _ref(a, b, bias, gelu=True), True)
    else:
        _check(ops.gemm(a, b, bias=bias), _ref(a, b, bias), True)


@pytest.mark.parametrize("M,N,K", [(128 * 133, 128, 64), (128 * 131 + 1, 200, 96), (128 * 265, 72, 136), (1000, 1000, 64),
                                   (128 * 7 + 65, 129, 256), (65, 8, 8)])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
def test_ragged_and_grid_remainders(dev, M, N, K, out_dtype):
    """Tile counts one above / below a multiple of the grid, ragged last m- and n-tiles (including a last m-tile whose
    second 64-row half is empty), K not a multiple of the 64-wide k-block."""
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M * 3 + N + K)
    a = _mk(g, M, K).half().to(dev)
    b = _mk(g, N, K).half().to(dev)
    bias = _mk(g, N, s=1).to(dev)
    _check(ops.gemm(a, b, bias=bias, out_dtype=out_dtype), _ref(a, b, bias), out_dtype == torch.float16)


def test_many_tiles_per_cta_small_k(dev):
    """K <= 256 with dozens of tiles per CTA: the ring wraps many times over tiles and the staging buffer is reused."""
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(3)
    for (M, N, K) in [(128 * 132 * 40 + 17, 96, 96), (128 * 132 * 20, 192, 256), (128 * 132 * 9 + 100, 64, 32)]:
        a = _mk(g, M, K).half().to(dev)
        b = _mk(g, N, K, s=0.2).half().to(dev)
        _check(ops.gemm(a, b), _ref(a, b), True)


def test_unaligned_outputs(dev):
    """Outputs with odd row / batch strides or a base off by one element: scalar stores, nothing written outside the view."""
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(4)
    Bz, M, N, K = 3, 1000, 100, 128
    a = _mk(g, Bz, M, K).half().to(dev)
    b = _mk(g, Bz, N, K).half().to(dev)
    ref = _ref(a, b)
    # row stride 101 elements: neither 16-byte aligned for fp16 nor for fp32
    for dt, f16 in ((torch.float16, True), (torch.float32, False)):
        buf = torch.zeros(Bz, M, N + 1, dtype=dt, device=dev)
        ops.gemm(a, b, out=buf[..., :N])
        _check(buf[..., :N], ref, f16)
        assert buf[..., N].abs().max().item() == 0.0
        # base shifted by one element
        buf2 = torch.zeros(Bz * M * N + 1, dtype=dt, device=dev)
        o = buf2[1:].view(Bz, M, N)
        ops.gemm(a, b, out=o)
        _check(o, ref, f16)
        assert buf2[0].item() == 0.0


def test_oneshot_bitwise_equal(dev):
    """MQDET_GEMM_IMPL_TC_ONESHOT is the same kernel with one tile per CTA: bit-identical outputs."""
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU
    g = torch.Generator(device="cpu").manual_seed(5)
    for (M, N, K) in [(128 * 300 + 40, 384, 96), (5000, 96, 384), (777, 40, 64)]:
        a = _mk(g, M, K).half().to(dev)
        b = _mk(g, N, K, s=0.2).half().to(dev)
        bias = _mk(g, N, s=1).to(dev)
        r = _mk(g, M, N, s=1).to(dev)
        for kw in (dict(bias=bias, act=ACT_GELU), dict(bias=bias, residual=r, out_dtype=torch.float32)):
            x = ops.gemm(a, b, **kw)
            y = ops.gemm(a, b, impl=ops.IMPL_TC_ONESHOT, **kw)
            assert torch.equal(x, y)


def test_graph_replay_back_to_back(dev):
    """Several dependent launches captured in one CUDA graph (no per-launch device state to reset), checked after replay."""
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU
    g = torch.Generator(device="cpu").manual_seed(6)
    M, C, H = 128 * 500 + 3, 96, 384
    x = _mk(g, M, C, s=1).half().to(dev)
    w1 = _mk(g, H, C, s=0.1).half().to(dev)
    w2 = _mk(g, C, H, s=0.05).half().to(dev)
    b1, b2 = _mk(g, H, s=1).to(dev), _mk(g, C, s=1).to(dev)
    res = _mk(g, M, C, s=1).to(dev)
    h = torch.empty(M, H, dtype=torch.float16, device=dev)
    y = torch.empty(M, C, dtype=torch.float32, device=dev)

    def step():
        ops.gemm(x, w1, out=h, bias=b1, act=ACT_GELU)
        ops.gemm(h, w2, out=y, bias=b2, residual=res)

    step()
    torch.cuda.synchronize()
    h_ref, y_ref = h.clone(), y.clone()
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            step()
    h.zero_()
    y.zero_()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(h, h_ref) and torch.equal(y, y_ref)
    _check(h, _ref(x, w1, b1, gelu=True), True)
    _check(y, _ref(h, w2, b2, residual=res), False)
