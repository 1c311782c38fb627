"""GPU parity of the GCP path (through the C ABI) against the CPU oracle (oracle/restate.py) on seeded inputs.

Cases follow SURVEY.md §7 "minimum slice": ncls in {10, 80}, K=5, T=256, B in {1, 8}, plus ragged edge cases
(classes with fewer than K queries, tokens with no class, a batch item without any query)."""
import pytest
import torch

from util import assert_close, load_sd, vq_cfg

pytestmark = pytest.mark.gpu


def _inputs(seed, B, ncls, K=5, T=256, D=768, ragged=False):
    from oracle import synth
    gen = synth.Gen(seed)
    _, _, pmap = synth.prompt(ncls, 2, T, gen)
    q, m = synth.vision_queries(pmap, K, T, D, gen)
    vision = gen.randn(B, q.shape[1], D)
    mask = m.expand(B, -1, -1).clone()
    if ragged:
        mask[0, 3] = 0  # class 0 keeps 4 queries in image 0
        mask[0, 7:10] = 0  # class 1 keeps 2
        if B > 1:
            mask[1] = 0  # image 1: no query at all -> output must equal the FFN of x only
    x = gen.randn(B, T, D)
    return x, vision, mask


@pytest.mark.parametrize("D,rows,dt", [(96, 4099, torch.float32), (192, 4097, torch.float32), (96, 5003, torch.float16),
                                       (192, 4100, torch.float16)])
def test_layernorm_narrow_rows(dev, D, rows, dt):
    """Swin stage 1 / 2 widths take the several-rows-per-warp kernel (rows >= 4096): ragged row counts, both input types."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(D + rows)
    x = (torch.randn(rows, D, generator=g) * 2.0 + 0.7).to(dt)
    w, b = torch.randn(D, generator=g), torch.randn(D, generator=g)
    ref = torch.nn.functional.layer_norm(x.float(), (D,), w, b, 1e-5)
    o16, o32 = ops.layernorm(x.to(dev), w.to(dev), b.to(dev), 1e-5, out16=True, out32=True)
    assert_close(o32, ref, 1e-5, "narrow layernorm fp32 out")
    assert_close(o16, ref, 1e-3, "narrow layernorm fp16 out")


def test_layernorm_and_softmax(dev):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(3)
    x = torch.randn(37, 768, generator=g) * 2 + 0.5
    w, b = torch.randn(768, generator=g), torch.randn(768, generator=g)
    ref = torch.nn.functional.layer_norm(x, (768,), w, b, 1e-5)
    o16, o32 = ops.layernorm(x.to(dev), w.to(dev), b.to(dev), 1e-5, out16=True, out32=True)
    assert_close(o32, ref, 1e-5, "layernorm fp32")
    assert_close(o16, ref, 1e-3, "layernorm fp16")
    # zero padding row: LN(0) = beta exactly
    xz = x.view(1, 37, 768).clone()
    oz = ops.layernorm(xz.to(dev), w.to(dev), b.to(dev), 1e-5, out16=False, out32=True, zero_row_period=37)
    assert torch.equal(oz[0, 36].cpu(), b)
    assert_close(oz[0, :36], ref[:36], 1e-5, "layernorm non-pad rows")
    # add + LN
    y = torch.randn(37, 768, generator=g)
    a16, a32 = ops.add_layernorm(x.to(dev), y.to(dev), w.to(dev), b.to(dev), 1e-12)
    assert_close(a32, torch.nn.functional.layer_norm(x + y, (768,), w, b, 1e-12), 1e-5, "add_layernorm")
    # masked softmax with padding columns
    s = torch.randn(2, 4, 19, 24, generator=g) * 3
    cm = torch.ones(2, 21)
    cm[0, 15:] = 0
    cm[1, 3] = 0
    p = ops.softmax_rows(s.to(dev), n=21, colmask=cm.to(dev), rows_per_batch=4 * 19, mask_value=-10000.0)
    ref = torch.softmax(s[..., :21] + (1 - cm)[:, None, None, :] * -10000.0, -1)
    assert_close(p[..., :21], ref, 1e-3, "softmax")
    assert p[..., 21:].abs().max().item() == 0


def test_build_index(dev):
    from mqdet_b200 import ops
    from oracle import restate
    x, vision, mask = _inputs(21, 2, 10, ragged=True)
    idx_ref = restate.gcp_index(mask)
    idx, counts = ops.gcp_build_index(mask.to(dev), idx_ref.shape[2])
    assert torch.equal(idx.cpu().long(), idx_ref)
    assert torch.equal(counts.cpu().long(), (mask != 0).sum(1))


@pytest.mark.parametrize("B,ncls,ragged", [(1, 10, False), (2, 10, True), (1, 80, False), (8, 80, False)])
def test_gcp_block(dev, B, ncls, ragged):
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import GatedCrossAttentionBlock
    from oracle import restate, synth
    sd = synth.gcp_block_sd(synth.Gen(100 + ncls))
    x, vision, mask = _inputs(200 + ncls + B, B, ncls, ragged=ragged)
    ref, gate = restate.gcp_block(x, vision, mask, sd, return_gate=True)
    blk = load_sd(GatedCrossAttentionBlock(dim=768, cfg=vq_cfg()), sd).to(dev).eval()
    out = blk(x.to(dev), vision.to(dev), mask.to(dev))
    assert out.dtype == torch.float32 and out.shape == x.shape
    assert_close(out, ref, what=f"GCP block B={B} ncls={ncls}")
    # sparse attention sub-op on its own (drop-in MaskedCrossAttention surface)
    s_ref = restate.gcp_sparse_attention(x, vision, mask, sd, "attn.")
    s = blk.attn(x.to(dev), vision.to(dev), mask.to(dev))
    assert_close(s, s_ref, what="sparse attention")
    # tokens without any class get EXACTLY zero attention output (modeling_bert_new.py:227-231)
    no_cls = (mask.sum(1) == 0)
    assert s.cpu()[no_cls].abs().max().item() == 0.0


def test_gcp_block_tensor_core_matches_simt(dev):
    """Same block with the GEMMs routed through the plain FMA kernel: isolates tensor-core/TMA addressing errors."""
    from mqdet_b200 import ops
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import GatedCrossAttentionBlock
    from oracle import synth
    sd = synth.gcp_block_sd(synth.Gen(7))
    x, vision, mask = _inputs(8, 2, 10)
    blk = load_sd(GatedCrossAttentionBlock(dim=768, cfg=vq_cfg()), sd).to(dev).eval()
    a = blk(x.to(dev), vision.to(dev), mask.to(dev))
    try:
        ops.DEFAULT_GEMM_IMPL = ops.IMPL_SIMT
        b = blk(x.to(dev), vision.to(dev), mask.to(dev))
    finally:
        ops.DEFAULT_GEMM_IMPL = ops.IMPL_TC
    assert_close(a, b, 2e-4, "tensor-core vs simt")


@pytest.mark.parametrize("B,ncls", [(1, 10), (2, 80)])
def test_preselect(dev, B, ncls):
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import PreSelectModule
    from oracle import restate, synth
    gen = synth.Gen(300 + ncls)
    sd = synth.preselect_sd(gen)
    V, I = ncls * 5, 1100 + 17  # ragged image-token count (not a multiple of 8); full size 5577 is covered in bench
    vision = gen.randn(B, V, 256, scale=0.5)
    image = gen.randn(B, I, 256)
    ref = restate.preselect(vision, image, sd)
    mod = load_sd(PreSelectModule(dim=256, out_dim=768, cfg=vq_cfg()), sd).to(dev).eval()
    out = mod(vision.to(dev), image.to(dev))["vision"]
    assert_close(out, ref, what="PreSelect")


def test_bert_layer(dev):
    from mqdet_b200 import ops
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import BertLayer
    from oracle import restate, synth
    gen = synth.Gen(41)
    sd = synth.bert_layer_sd(gen, "")
    B, T, D = 2, 256, 768
    h = gen.randn(B, T, D)
    am = torch.ones(B, T)
    am[0, 200:] = 0
    am[1, 33:] = 0
    ref = restate.bert_layer(h, restate.extended_mask(am), sd, "")
    layer = load_sd(BertLayer(D, 12, 3072), sd).to(dev).eval()
    h32 = h.to(dev)
    o32, o16 = layer(h32, ops.cast_f16(h32), am.to(dev))
    assert_close(o32, ref, what="BERT layer")
    assert_close(o16, ref, 2e-3, "BERT layer fp16 copy")


def test_gcp_block_vs_reference_golden(dev):
    """CUDA path vs the vectors recorded from the reference's own GatedCrossAttentionBlock (tests/golden/gcp_block.pt)."""
    import os
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import GatedCrossAttentionBlock
    from oracle import make_golden
    from util import ROOT, FP16_TOL
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "gcp_block.pt"))
    c = make_golden.case_inputs("gcp_block")
    blk = load_sd(GatedCrossAttentionBlock(dim=768, cfg=vq_cfg()), c["sd"]).to(dev).eval()
    y = blk(c["x"].to(dev), c["vision"].to(dev), c["mask"].to(dev))
    got = make_golden.sub(y.float().cpu(), *fx["subsample"]["y"])
    err = (got - fx["y"]).abs().max().item()
    assert err <= FP16_TOL * fx["y_absmax"] + FP16_TOL, err


def test_preselect_vs_reference_golden(dev):
    import os
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import PreSelectModule
    from oracle import make_golden
    from util import ROOT, FP16_TOL
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "preselect.pt"))
    c = make_golden.case_inputs("preselect")
    mod = load_sd(PreSelectModule(dim=256, out_dim=768, cfg=vq_cfg()), c["sd"]).to(dev).eval()
    v = mod(c["vision"].to(dev), c["image"].to(dev))["vision"]
    got = make_golden.sub(v.float().cpu(), *fx["subsample"]["vision"])
    err = (got - fx["vision"]).abs().max().item()
    assert err <= FP16_TOL * fx["vision_absmax"] + FP16_TOL, err


def test_dense_cross_attention_flash_equals_unfused(dev):
    """PreSelect's dense MaskedCrossAttention: the flash-style kernel (online softmax over 64-token chunks, scores never in
    HBM) against the unfused GEMM / softmax_rows / GEMM path and plain torch, ragged query and key counts."""
    from mqdet_b200 import ops
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import PreSelectModule
    from oracle import synth
    g = torch.Generator().manual_seed(12)
    for (B, Tq, I) in [(2, 50, 1117), (1, 400, 5577), (3, 7, 64), (1, 65, 63)]:
        q = (torch.randn(B, Tq, 256, generator=g) * 0.5).half()
        kv = torch.randn(B, I, 512, generator=g).half()
        out = ops.dense_cross_attn(q.to(dev), kv.to(dev), 8, 32).float().cpu()
        qf = q.float().view(B, Tq, 8, 32).transpose(1, 2)
        kf = kv.float()[..., :256].reshape(B, I, 8, 32).transpose(1, 2)
        vf = kv.float()[..., 256:].reshape(B, I, 8, 32).transpose(1, 2)
        ref = (torch.softmax(qf @ kf.transpose(-1, -2), dim=-1) @ vf).transpose(1, 2).reshape(B, Tq, 256)
        assert_close(out, ref, 1e-3, f"dense_cross_attn {B, Tq, I}")
    gen = synth.Gen(301)
    sd = synth.preselect_sd(gen)
    mod = load_sd(PreSelectModule(dim=256, out_dim=768, cfg=vq_cfg()), sd).to(dev).eval()
    vision, image = gen.randn(2, 50, 256, scale=0.5).to(dev), gen.randn(2, 1117, 256).to(dev)
    a = mod(vision, image)["vision"]
    for blk in mod.layers:
        blk.image_condition.flash = False
    b = mod(vision, image)["vision"]
    assert_close(a, b, 1e-3, "PreSelect: flash vs unfused attention")
