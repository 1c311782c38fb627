"""GPU checks of the GEMM's specialised epilogues (no epilogue / bias / bias + GELU in fp16, bias + fp32 residual in fp32) and
their TMA-store output path, against the generic epilogue with pointer stores, which the same product takes when C cannot
be addressed by a tensor map (base not 16-byte aligned).  Also: ragged edges and strided / batched outputs clipped by the
TMA unit, the ping-pong persistent kernel against the one-tile-per-CTA launch (also with one SM reserved, so that a CTA's
consecutive tiles change n-tile), and graph replay."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(g, *shape, s=0.5):
    return torch.randn(*shape, generator=g) * s


def _variants(dev, g, M, N):
    """kwargs per epilogue variant: the four specialised ones and a generic one (per-column gate + clamp)."""
    from mqdet_b200._lib import ACT_GELU, VEC_PER_COL
    bias = _mk(g, N, s=1).to(dev)
    res = _mk(g, M, N, s=1).to(dev)
    gate = _mk(g, N, s=1).to(dev)
    return {
        "none_f16": dict(),
        "bias_f16": dict(bias=bias),
        "bias_gelu_f16": dict(bias=bias, act=ACT_GELU),
        "bias_res_f32": dict(bias=bias, residual=res, out_dtype=torch.float32),
        "generic_gate_clamp": dict(bias=bias, gate=gate, gate_mode=VEC_PER_COL, clamp=0.7),
    }


def _shifted_out(M, N, dtype, dev):
    """An [M, N] output whose base is one element past a 16-byte boundary (no tensor map): the pointer-store path."""
    buf = torch.zeros(M * N + 1, dtype=dtype, device=dev)
    return buf, buf[1:].view(M, N)


@pytest.mark.parametrize("M,N,K", [(128 * 300 + 40, 384, 96), (128 * 50 + 3, 288, 192), (5000, 96, 384), (777, 40, 64)])
def test_store_paths_agree(dev, M, N, K):
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = _mk(g, M, K).half().to(dev)
    b = _mk(g, N, K, s=0.2).half().to(dev)
    for name, kw in _variants(dev, g, M, N).items():
        x = ops.gemm(a, b, **kw)
        assert x.data_ptr() % 16 == 0
        buf, y = _shifted_out(M, N, x.dtype, dev)
        ops.gemm(a, b, out=y, **kw)
        assert torch.equal(x, y), name
        assert buf[0].item() == 0.0, name


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
def test_edge_clipping_strided_batched(dev, out_dtype):
    """Ragged M and N, nb1 = 3 and nb2 = 2 batches, ldc > N views (16-byte multiples, so the TMA path is taken) inside a
    zeroed larger buffer: the view equals the pointer-store result and nothing outside it is written."""
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU
    g = torch.Generator(device="cpu").manual_seed(11)
    nb2, nb1, M, N, K = 2, 3, 128 * 3 + 17, 200, 96
    a = _mk(g, nb2, nb1, M, K).half().to(dev)
    b = _mk(g, nb2, nb1, N, K, s=0.2).half().to(dev)
    bias = _mk(g, N, s=1).to(dev)
    kws = [dict(bias=bias)]
    if out_dtype == torch.float16:
        kws += [dict(), dict(bias=bias, act=ACT_GELU)]
    else:
        kws += [dict(bias=bias, residual=_mk(g, nb2, nb1, M, N, s=1).to(dev))]
    for kw in kws:
        ref = torch.zeros(nb2, nb1, M, N + 1, dtype=out_dtype, device=dev)[..., :N]  # odd ldc: pointer stores
        ops.gemm(a, b, out=ref, **kw)
        big = torch.zeros(nb2, nb1 + 1, M + 5, N + 24, dtype=out_dtype, device=dev)
        view = big[:, :nb1, 2:M + 2, 8:N + 8]
        assert view.data_ptr() % 16 == 0 and (view.stride(2) * view.element_size()) % 16 == 0
        ops.gemm(a, b, out=view, **kw)
        assert torch.equal(view, ref)
        mask = torch.ones_like(big, dtype=torch.bool)
        mask[:, :nb1, 2:M + 2, 8:N + 8] = False
        assert big[mask].abs().max().item() == 0.0


@pytest.mark.parametrize("M,N,K", [(537600, 384, 96), (537600, 96, 96), (134400, 192, 192), (128 * 131 + 1, 200, 96),
                                   (5000, 96, 384), (2048, 768, 768)])
def test_persistent_equals_oneshot(dev, M, N, K):
    """Swin stage-1 M gives dozens of tiles per CTA, so the ping-pong turns and the output staging wrap many times."""
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M + 7 * N + K)
    a = _mk(g, M, K).half().to(dev)
    b = _mk(g, N, K, s=0.2).half().to(dev)
    for name, kw in _variants(dev, g, M, N).items():
        x = ops.gemm(a, b, **kw)
        y = ops.gemm(a, b, impl=ops.IMPL_TC_ONESHOT, **kw)
        assert torch.equal(x, y), name


def test_reserved_sm_equals_oneshot(dev):
    """131 CTAs: a CTA's consecutive tiles no longer share an n-tile."""
    from mqdet_b200 import _lib, ops
    g = torch.Generator(device="cpu").manual_seed(21)
    lib = _lib.load()
    try:
        _lib.check(lib.mqdet_reserve_sms(1), "reserve_sms")
        for (M, N, K) in [(128 * 1000 + 5, 384, 96), (128 * 500, 288, 96), (20000, 96, 384)]:
            a = _mk(g, M, K).half().to(dev)
            b = _mk(g, N, K, s=0.2).half().to(dev)
            for name, kw in _variants(dev, g, M, N).items():
                x = ops.gemm(a, b, **kw)
                y = ops.gemm(a, b, impl=ops.IMPL_TC_ONESHOT, **kw)
                assert torch.equal(x, y), name
    finally:
        _lib.check(lib.mqdet_reserve_sms(0), "reserve_sms")


def test_graph_replay_new_inputs(dev):
    """A captured chain of dependent launches (qkv-like, fc1 + GELU, fc2 + residual, a plain product) replayed with new input
    contents equals the same launches run eagerly on those contents."""
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU
    g = torch.Generator(device="cpu").manual_seed(31)
    M, C, H = 128 * 700 + 9, 96, 384
    x = _mk(g, M, C, s=1).half().to(dev)
    res = _mk(g, M, C, s=1).to(dev)
    w0 = _mk(g, 3 * C, C, s=0.1).half().to(dev)
    w1 = _mk(g, H, C, s=0.1).half().to(dev)
    w2 = _mk(g, C, H, s=0.05).half().to(dev)
    b0, b1, b2 = _mk(g, 3 * C, s=1).to(dev), _mk(g, H, s=1).to(dev), _mk(g, C, s=1).to(dev)
    q = torch.empty(M, 3 * C, dtype=torch.float16, device=dev)
    h = torch.empty(M, H, dtype=torch.float16, device=dev)
    y = torch.empty(M, C, dtype=torch.float32, device=dev)
    z = torch.empty(M, C, dtype=torch.float16, device=dev)

    def step():
        ops.gemm(x, w0, out=q, bias=b0)
        ops.gemm(x, w1, out=h, bias=b1, act=ACT_GELU)
        ops.gemm(h, w2, out=y, bias=b2, residual=res)
        ops.gemm(q[:, :C], w2[:, :C], out=z)

    step()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            step()
    torch.cuda.synchronize()
    for seed in (1, 2):
        gg = torch.Generator(device="cpu").manual_seed(100 + seed)
        x.copy_(_mk(gg, M, C, s=1).half())
        res.copy_(_mk(gg, M, C, s=1))
        for t in (q, h, y, z):
            t.zero_()
        graph.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in (q, h, y, z)]
        step()
        torch.cuda.synchronize()
        for t0, t1 in zip(got, (q, h, y, z)):
            assert torch.equal(t0, t1)
