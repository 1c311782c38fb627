"""GPU parity of the wgmma GEMM (through the C ABI) against a plain PyTorch fp32 reference of the same op and
against the SIMT validation kernel.  Tolerance: fp32 accumulation of fp16-exact products, so only summation order
differs: |err| <= 2e-3*|ref|_max*sqrt(K)/sqrt(K) ~ rtol 1e-4; fp16 outputs add one fp16 rounding (2^-11 relative)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, *, alpha=1.0, bias=None, bias_mode=None, scale_after_bias=False, act=None, clamp=0.0, gate=None,
         gate_tanh=False, residual=None):
    acc = a.float() @ b.float().transpose(-1, -2)
    if bias is not None:
        bb = bias.unsqueeze(-2) if bias_mode == "col" else bias.unsqueeze(-1)
    else:
        bb = 0.0
    v = alpha * (acc + bb) if scale_after_bias else alpha * acc + bb
    if act == "gelu":
        v = torch.nn.functional.gelu(v)
    elif act == "relu":
        v = torch.relu(v)
    if clamp > 0:
        v = v.clamp(-clamp, clamp)
    if gate is not None:
        g = gate.tanh() if gate_tanh else gate
        v = v * g
    if residual is not None:
        v = v + residual.float()
    return v


def _check(out, ref, out_is_f16):
    out = out.float()
    scale = ref.abs().max().item() + 1e-6
    err = (out - ref).abs().max().item()
    tol = scale * (1.5e-3 if out_is_f16 else 2e-5)
    assert err <= tol, f"max err {err:.3e} > tol {tol:.3e} (scale {scale:.3e})"


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 512, 768), (2048, 3072, 768), (300, 200, 136), (77, 50, 256),
                                   (2048, 768, 3072), (1, 768, 768), (4096, 32, 64), (129, 257, 72), (22400, 256, 256)])
@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
def test_plain(dev, M, N, K, out_dtype):
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(dev)
    b = (torch.randn(N, K, generator=g) * 0.5).half().to(dev)
    out = ops.gemm(a, b, out_dtype=out_dtype)
    ref = _ref(a, b)
    _check(out, ref, out_dtype == torch.float16)
    simt = ops.gemm(a, b, out_dtype=out_dtype, impl=ops.IMPL_SIMT)
    _check(simt, ref, out_dtype == torch.float16)
    oneshot = ops.gemm(a, b, out_dtype=out_dtype, impl=ops.IMPL_TC_ONESHOT)
    _check(oneshot, ref, out_dtype == torch.float16)


def test_persistent_many_tiles_per_cta(dev):
    """Many more tiles than SMs (several waves of CTAs, 128- and 64-wide tiles, K from one k-block to a wrapping ring), with a
    ragged last M tile and batches."""
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(77)
    for (Bz, M, N, K) in [(1, 128 * 40 + 37, 512, 256), (5, 1000, 384, 192), (1, 70000, 128, 64), (1, 128 * 100 + 5, 512, 256),
                          (6, 128 * 30, 256, 192), (3, 22400, 256, 256)]:
        a = (torch.randn(Bz, M, K, generator=g) * 0.5).half().to(dev)
        b = (torch.randn(Bz, N, K, generator=g) * 0.5).half().to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        res = torch.randn(Bz, M, N, generator=g).to(dev)
        ref = torch.einsum("zmk,znk->zmn", a.float(), b.float())
        _check(ops.gemm(a, b, bias=bias), ref + bias, True)                                   # TMA-store epilogue
        _check(ops.gemm(a, b, bias=bias, residual=res, out_dtype=torch.float32), ref + bias + res, False)  # fallback epilogue


def test_persistent_epilogue_modes(dev):
    """Every epilogue combination the forward uses (scale / bias folding, per-row and per-column vectors, gates, residuals,
    clamp, GELU), at sizes with several tiles per SM and long K."""
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU, VEC_PER_COL, VEC_PER_ROW, VEC_SCALAR
    g = torch.Generator(device="cpu").manual_seed(21)

    def mk(*shape, s=0.3):
        return (torch.randn(*shape, generator=g) * s)

    # K <= 256 (B-resident tiles), N = 512: 256-wide tile when the output is fp16 + TMA-storable
    M, N, K = 128 * 300 + 40, 512, 256
    a, b = mk(M, K).half().to(dev), mk(N, K).half().to(dev)
    bc, br, gc = mk(N, s=1).to(dev), mk(M, s=1).to(dev), mk(N, s=1).to(dev)
    r16, r32 = mk(M, N, s=1).half().to(dev), mk(M, N, s=1).to(dev)
    gs = torch.tensor([0.4], device=dev)
    _check(ops.gemm(a, b, bias=bc, alpha=0.25, scale_after_bias=True), _ref(a, b, bias=bc, bias_mode="col", alpha=0.25, scale_after_bias=True), True)
    _check(ops.gemm(a, b, bias=br, bias_mode=VEC_PER_ROW), _ref(a, b, bias=br, bias_mode="row"), True)
    _check(ops.gemm(a, b, clamp=2.0), _ref(a, b, clamp=2.0), True)
    _check(ops.gemm(a, b, bias=bc, act=ACT_GELU), _ref(a, b, bias=bc, bias_mode="col", act="gelu"), True)
    _check(ops.gemm(a, b, bias=bc, gate=gc, gate_mode=VEC_PER_COL, residual=r16),
           _ref(a, b, bias=bc, bias_mode="col", gate=gc, residual=r16), True)
    _check(ops.gemm(a, b, bias=bc, residual=r32, out_dtype=torch.float32), _ref(a, b, bias=bc, bias_mode="col", residual=r32), False)
    _check(ops.gemm(a, b, gate=gs, gate_mode=VEC_SCALAR, gate_tanh=True, residual=r32, out_dtype=torch.float32),
           _ref(a, b, gate=gs, gate_tanh=True, residual=r32), False)
    _check(ops.gemm(a, b, bias=bc, gate=br, gate_mode=VEC_PER_ROW, out_dtype=torch.float32),   # col bias + row gate: generic
           _ref(a, b, bias=bc, bias_mode="col") * br[:, None], False)
    # long K (ring-streamed 128x256 tile), gamma * (acc + b) + fp16 residual = the BiAttention out-projection
    M, N, K = 128 * 200 + 8, 256, 1024
    a, b = mk(M, K).half().to(dev), mk(N, K, s=0.1).half().to(dev)
    bc, gc = mk(N, s=1).to(dev), mk(N, s=1).to(dev)
    r16 = mk(M, N, s=1).half().to(dev)
    _check(ops.gemm(a, b, bias=bc, gate=gc, gate_mode=VEC_PER_COL, residual=r16),
           _ref(a, b, bias=bc, bias_mode="col", gate=gc, residual=r16), True)
    _check(ops.gemm(a, b, bias=bc, act=ACT_GELU), _ref(a, b, bias=bc, bias_mode="col", act="gelu"), True)
    # batched, per-batch bias rows, narrow tile (N = 64) fast epilogue
    Bz, M, N, K = 3, 128 * 120, 64, 128
    a, b = mk(Bz, M, K).half().to(dev), mk(Bz, N, K).half().to(dev)
    r32 = mk(Bz, M, N, s=1).to(dev)
    ref = torch.einsum("zmk,znk->zmn", a.float(), b.float())
    _check(ops.gemm(a, b, residual=r32, out_dtype=torch.float32), ref + r32, False)
    _check(ops.gemm(a, b, alpha=0.5), 0.5 * ref, True)


def test_epilogues(dev):
    from mqdet_b200 import ops
    from mqdet_b200._lib import ACT_GELU, ACT_RELU, VEC_PER_COL, VEC_PER_ROW, VEC_SCALAR
    g = torch.Generator(device="cpu").manual_seed(5)
    M, N, K = 384, 320, 256
    a = (torch.randn(M, K, generator=g) * 0.3).half().to(dev)
    b = (torch.randn(N, K, generator=g) * 0.3).half().to(dev)
    bc = torch.randn(N, generator=g).to(dev)
    br = torch.randn(M, generator=g).to(dev)
    res32 = torch.randn(M, N, generator=g).to(dev)
    res16 = res32.half()
    gs = torch.tensor([0.3], device=dev)
    gc = torch.randn(N, generator=g).to(dev)
    # bias per column + GELU, fp16 out
    _check(ops.gemm(a, b, bias=bc, act=ACT_GELU), _ref(a, b, bias=bc, bias_mode="col", act="gelu"), True)
    # bias per row + ReLU + clamp
    _check(ops.gemm(a, b, bias=br, bias_mode=VEC_PER_ROW, act=ACT_RELU, clamp=1.0, out_dtype=torch.float32),
           _ref(a, b, bias=br, bias_mode="row", act="relu", clamp=1.0), False)
    # alpha after bias (BiAttention query projection, fuse_helper.py:221)
    _check(ops.gemm(a, b, bias=bc, alpha=0.0625, scale_after_bias=True, out_dtype=torch.float32),
           _ref(a, b, bias=bc, bias_mode="col", alpha=0.0625, scale_after_bias=True), False)
    # tanh(scalar gate) * acc + fp32 residual (GCP FFN output, modeling_bert_new.py:372)
    _check(ops.gemm(a, b, gate=gs, gate_mode=VEC_SCALAR, gate_tanh=True, residual=res32, out_dtype=torch.float32),
           _ref(a, b, gate=gs, gate_tanh=True, residual=res32), False)
    # per-column gamma * (acc + bias) + fp16 residual (BiAttention layer-scale, fuse_helper.py:423-424)
    _check(ops.gemm(a, b, bias=bc, gate=gc, gate_mode=VEC_PER_COL, residual=res16),
           _ref(a, b, bias=bc, bias_mode="col", gate=gc, residual=res16), True)


def test_batched_strided_heads(dev):
    """Attention-shaped batched products on head-strided views: scores = q k^T, ctx = p v with v pre-transposed."""
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(11)
    B, T, H, d = 3, 200, 12, 64
    qk = (torch.randn(B, T, 2, H, d, generator=g) * 0.5).half().to(dev)
    q, k = qk[:, :, 0], qk[:, :, 1]
    scores = torch.empty(B, H, T, T, dtype=torch.float32, device=dev)
    ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=scores, alpha=d ** -0.5)
    ref = torch.einsum("bthd,bshd->bhts", q.float(), k.float()) * d ** -0.5
    _check(scores, ref, False)
    p = torch.softmax(ref, -1).half()
    vT = (torch.randn(B, H, d, T, generator=g) * 0.5).half().to(dev)
    ctx = torch.empty(B, T, H, d, dtype=torch.float16, device=dev)
    ops.gemm(p, vT, out=ctx.permute(0, 2, 1, 3))
    ref2 = torch.einsum("bhts,bhds->bthd", p.float(), vT.float())
    _check(ctx, ref2, True)


def test_broadcast_weight_transposed_product(dev):
    """vT[b] = W . x[b]^T + bias_row : A broadcast over the batch, K = 256, ragged N (= 5577 image tokens)."""
    from mqdet_b200 import ops
    from mqdet_b200._lib import VEC_PER_ROW
    g = torch.Generator(device="cpu").manual_seed(13)
    B, I, D, O = 2, 5577, 256, 256
    Ipad = (I + 7) // 8 * 8
    w = (torch.randn(O, D, generator=g) * 0.1).half().to(dev)
    x = (torch.randn(B, I, D, generator=g)).half().to(dev)
    bias = torch.randn(O, generator=g).to(dev)
    out = torch.zeros(B, O, Ipad, dtype=torch.float16, device=dev)
    ops.gemm(w, x, out=out[:, :, :I], bias=bias, bias_mode=VEC_PER_ROW)
    ref = torch.einsum("od,bid->boi", w.float(), x.float()) + bias[None, :, None]
    _check(out[:, :, :I], ref, True)
    assert out[:, :, I:].abs().max().item() == 0.0


def test_small_k32_heads(dev):
    """PreSelect heads have dim 32 < the 64-wide K tile: TMA zero-fills the rest of the box."""
    from mqdet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(17)
    B, V, I, H, d = 2, 50, 1050, 8, 32
    q = (torch.randn(B, V, H, d, generator=g)).half().to(dev)
    k = (torch.randn(B, I, H, d, generator=g)).half().to(dev)
    Ipad = (I + 7) // 8 * 8
    s = torch.empty(B, H, V, Ipad, dtype=torch.float32, device=dev)
    ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=s[..., :I])
    ref = torch.einsum("bvhd,bihd->bhvi", q.float(), k.float())
    _check(s[..., :I], ref, False)


def test_bad_args_raise(dev):
    from mqdet_b200 import ops
    from mqdet_b200._lib import MqdetError
    a = torch.zeros(16, 12, dtype=torch.float16, device=dev)  # K % 8 != 0
    b = torch.zeros(16, 12, dtype=torch.float16, device=dev)
    with pytest.raises(MqdetError):
        ops.gemm(a, b)
    with pytest.raises(MqdetError):
        ops.gemm(torch.zeros(4, 8, dtype=torch.float16), torch.zeros(4, 8, dtype=torch.float16))  # CPU tensors
