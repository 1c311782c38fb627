"""GPU parity of the VL deep-fusion tower: BiAttention fusion, DyConv (DCNv2 + GN + scale attention + DyReLU) and the
full VLDyHead (6 x [fusion, BERT layer, DyConv] + dot-product token head) against the CPU oracle."""
import os

import pytest
import torch

from util import FP16_TOL, ROOT, assert_close, load_sd

pytestmark = pytest.mark.gpu

SIZES = [(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)]


def test_bi_attention_vs_oracle_and_golden(dev):
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.utils.fuse_helper import BiAttentionBlockForCheckpoint
    from oracle import make_golden, restate
    c = make_golden.case_inputs("bi_attention")
    blk = BiAttentionBlockForCheckpoint(v_dim=256, l_dim=768, embed_dim=2048, num_heads=8, hidden_dim=3072, dropout=0.1,
                                        drop_path=0.0, init_values=1.0 / 6, cfg=mq_glip_t_cfg())
    blk = load_sd(blk, c["sd"]).to(dev).eval()
    v = restate.flatten_levels(c["feats"])
    v_ref, l_ref = restate.bi_attention(v, c["l"], c["mask"], c["sd"])
    out = blk(*[f.to(dev) for f in c["feats"]], c["l"].to(dev), c["mask"].to(dev), None)
    v_out = restate.flatten_levels([o.cpu() for o in out[:5]])
    assert_close(v_out, v_ref, what="fusion: visual stream")
    assert_close(out[5], l_ref, what="fusion: language stream")
    assert out[6] is None and len(out) == 10
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "bi_attention.pt"))
    for key, got in (("v", v_out), ("l", out[5].cpu())):
        g = make_golden.sub(got.float(), *fx["subsample"][key])
        err = (g - fx[key]).abs().max().item()
        assert err <= FP16_TOL * fx[key + "_absmax"] + FP16_TOL, (key, err)


def test_bi_attention_fused_equals_f32_scores(dev):
    """The product path (image-side kernel: scores in registers -> softmax -> P.V_l -> out-projection -> layer scale + residual;
    text-side kernel on the image tokens with in-kernel column sums) against the explicit "f32" path (fp32 score matrices in
    HBM, softmax_rows, plain GEMMs).  Ragged N (not a multiple of 64 / 128), T < 256, masks.  An unknown score_precision
    raises instead of selecting some path."""
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.utils.fuse_helper import BiAttentionBlockForCheckpoint
    from oracle import synth
    gen = synth.Gen(31)
    sd = synth.bi_attention_sd(gen)
    blk = BiAttentionBlockForCheckpoint(v_dim=256, l_dim=768, embed_dim=2048, num_heads=8, hidden_dim=3072, dropout=0.1,
                                        drop_path=0.0, init_values=1.0 / 6, cfg=mq_glip_t_cfg())
    blk = load_sd(blk, sd).to(dev).eval()
    for (B, N, T) in [(2, 1000, 256), (1, 333, 256), (2, 520, 64), (3, 128, 256), (1, 2600, 200)]:
        v16 = gen.randn(B, N, 256).half().to(dev)
        l32 = gen.randn(B, T, 768).to(dev)
        mask = torch.ones(B, T, dtype=torch.long)
        mask[0, T // 3:] = 0
        mask = mask.to(dev)
        blk.attn.score_precision = "fused"
        v1, l1 = blk.forward_flat(v16, l32, mask)
        blk.attn.score_precision = "f32"
        v0, l0 = blk.forward_flat(v16, l32, mask)
        assert_close(v1, v0, 1e-3, f"fused vs f32-score visual stream {B, N, T}")
        assert_close(l1, l0, 1e-3, f"fused vs f32-score language stream {B, N, T}")
        blk.attn.score_precision = "fused"
    # no mask at all, and an image whose tokens are ALL masked (uniform probabilities, like the reference's fp32 -9e15 sum)
    v16 = gen.randn(2, 300, 256).half().to(dev)
    l32 = gen.randn(2, 256, 768).to(dev)
    va, la = blk.forward_flat(v16, l32, None)
    blk.attn.score_precision = "f32"
    vb, lb = blk.forward_flat(v16, l32, None)
    assert_close(va, vb, 1e-3, "fused vs f32, no mask")
    # an image whose tokens are ALL masked: the reference's fp32 sum A + (-9e15) swallows A, so its softmax is uniform over
    # the T tokens (fuse_helper.py:277-287); checked against the oracle, which adds the mask exactly like the reference
    from oracle import restate
    mask = torch.ones(2, 256, dtype=torch.long)
    mask[1] = 0
    blk.attn.score_precision = "fused"
    vc, lc = blk.forward_flat(v16, l32, mask.to(dev))
    v_ref, l_ref = restate.bi_attention(v16.float().cpu(), l32.cpu(), mask, sd)
    assert_close(vc, v_ref, 1e-3, "fused vs oracle, fully masked image")
    assert_close(lc, l_ref, 1e-3, "fused vs oracle, fully masked image (language)")
    blk.attn.score_precision = "f16"
    with pytest.raises(ValueError, match="score_precision"):
        blk.forward_flat(v16, l32, None)
    with pytest.raises(ValueError, match="score_precision"):
        blk.forward_flat_split(v16, l32, None)
    blk.attn.score_precision = "fused"


def test_dcn_cols_plain_equals_unfold(dev):
    """om == NULL: the sampling stage is a plain 3x3/pad-1 im2col with k = tap*C + c."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(2)
    feats = [torch.randn(2, 256, h, w, generator=g) for h, w in SIZES]
    lv = ops.Levels(SIZES, dev)
    x16 = torch.cat([f.flatten(2).transpose(1, 2) for f in feats], 1).half().to(dev).contiguous()
    cols = ops.dcn_cols(x16, None, lv, 1).float().cpu().view(2, lv.N, 9, 256)
    for l, f in enumerate(feats):
        h, w = SIZES[l]
        u = torch.nn.functional.unfold(f.half().float(), 3, padding=1).view(2, 256, 9, h * w).permute(0, 3, 2, 1)
        assert torch.equal(cols[:, lv.off[l]:lv.off[l + 1]], u)


def test_conv3x3_small_equals_conv2d(dev):
    """The column-matrix-free 27-channel offset conv (implicit GEMM on mma.sync) == F.conv2d on the fp16-rounded operands;
    level sizes chosen so that warps straddle level and image boundaries and the last pixel tile is ragged."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(4)
    sizes = [(13, 17), (7, 9), (4, 5), (2, 3), (1, 1)]
    B, O = 3, 27
    feats = [torch.randn(B, 256, h, w, generator=g) for h, w in sizes]
    wt = torch.randn(O, 256, 3, 3, generator=g) * 0.05
    bias = torch.randn(O, generator=g)
    lv = ops.Levels(sizes, dev)
    x16 = torch.cat([f.flatten(2).transpose(1, 2) for f in feats], 1).half().to(dev).contiguous()
    w16 = wt.permute(0, 2, 3, 1).reshape(O, -1).half().to(dev).contiguous()   # k = tap*C + c
    out = ops.conv3x3_small(x16, w16, bias.to(dev), lv).view(B, lv.N, 32)[..., :O].cpu()
    for l, f in enumerate(feats):
        ref = torch.nn.functional.conv2d(f.half().float(), wt.half().float(), bias, padding=1)   # [B,O,h,w]
        ref = ref.flatten(2).transpose(1, 2)
        got = out[:, lv.off[l]:lv.off[l + 1]]
        err = (got - ref).abs().max().item()
        assert err <= 2e-4 * ref.abs().max().item() + 1e-5, (l, err)     # fp32 accumulation of fp16-exact products


@pytest.mark.parametrize("sizes,B,with_om", [([(13, 17), (7, 9), (4, 5), (2, 3), (1, 1)], 3, True),
                                             ([(40, 56), (20, 28), (10, 14), (5, 7), (3, 4)], 2, True),
                                             ([(13, 17), (7, 9), (4, 5)], 2, False), ([(9, 11)], 2, True)])
def test_dcn_conv_implicit_equals_cols_gemm(dev, sizes, B, with_om):
    """mqdet_dcn_conv (sampling fused into the wgmma mainloop, three branches in one launch) against the sampling kernel +
    GEMM pair it replaces: same fp16 operands, same fp32 accumulation, the mask folded into the corner weights (one fp32
    rounding apart) -> equal up to an fp16 ulp of the column values.  Sizes make tiles straddle levels, images and the ragged
    last tile; large offsets push samples outside the maps."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(11)
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
    ys = ops.dcn_conv(x16, om, lv, ks, ws, bs)
    for k, w, b, y in zip(ks, ws, bs, ys):
        ref = ops.gemm(ops.dcn_cols(x16, om, lv, k), w, bias=b)
        assert y.shape == ref.shape
        err = (y.float() - ref.float()).abs().max().item()
        assert err <= 2e-3 * ref.float().abs().max().item(), (k, err, ref.float().abs().max().item())
    # no bias pointer
    y0 = ops.dcn_conv(x16, om, lv, [1], ws[:1], [None])[0]
    ref0 = ops.gemm(ops.dcn_cols(x16, om, lv, 1), ws[0])
    assert (y0.float() - ref0.float()).abs().max().item() <= 2e-3 * ref0.float().abs().max().item()


def test_dyconv(dev):
    from mqdet_b200 import ops
    from mqdet_b200.modeling.rpn.vldyhead import Conv3x3Norm, DyConv
    from oracle import restate, synth
    gen = synth.Gen(77)
    sd = synth.dyconv_sd(gen)
    feats = [gen.randn(2, 256, h, w) for h, w in SIZES]
    ref = restate.flatten_levels(restate.dyconv(feats, sd))
    conv_func = lambda i, o, s: Conv3x3Norm(i, o, s, deformable=True, bn_type=["gn", 16])  # noqa: E731
    mod = load_sd(DyConv(256, 256, conv_func=conv_func, use_dyrelu=True, use_dyfuse=True, use_deform=True), sd)
    mod = mod.to(dev).eval()
    lv = ops.Levels(SIZES, dev)
    x16 = restate.flatten_levels(feats).half().to(dev).contiguous()
    out = mod.forward_flat(x16, lv)
    assert_close(out, ref, 3e-3, "DyConv (fp16 activations)")
    mod.implicit_dcn = False   # sampling kernel + GEMM pair instead of the implicit GEMM
    assert_close(mod.forward_flat(x16, lv), ref, 3e-3, "DyConv (column-matrix path)")
    mod.implicit_dcn = True
    # the same inputs through the REFERENCE's own DyConv.forward (fixture recorded by oracle/make_golden.py)
    from oracle import make_golden
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "dyconv.pt"))
    g = make_golden.sub(out.float().cpu(), *fx["subsample"]["v"])
    assert (g - fx["v"]).abs().max().item() <= 3e-3 * fx["v_absmax"] + 3e-3
    # reference-facing dict API
    o2 = mod({"visual": [f.to(dev) for f in feats], "lang": None})["visual"]
    assert [tuple(o.shape) for o in o2] == [tuple(f.shape) for f in feats]
    assert_close(restate.flatten_levels([o.cpu() for o in o2]), ref, 3e-3, "DyConv dict API")


def test_vldyhead_tower(dev):
    from mqdet_b200 import ops
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.rpn.vldyhead import VLDyHead
    from oracle import restate, synth
    gen = synth.Gen(78)
    nconv = 6
    sd = synth.vldyhead_sd(gen, nconv)
    B, T = 2, 256
    feats = [gen.randn(B, 256, h, w) for h, w in SIZES]
    hidden = gen.randn(B, T, 768)
    masks = torch.ones(B, T, dtype=torch.long)
    masks[0, 120:] = 0
    masks[1, 31:] = 0
    ref = restate.vl_dyhead(feats, hidden, masks, sd, nconv)
    head = load_sd(VLDyHead(mq_glip_t_cfg()), sd).to(dev).eval()
    lv = ops.Levels(SIZES, dev)
    v16 = restate.flatten_levels(feats).half().to(dev).contiguous()
    r = head.forward_flat(v16, lv, hidden.to(dev), masks.to(dev))
    # 18 chained stages with fp16 operands; DCNv2 sampling positions and DyReLU branch choices depend on the features,
    # so rounding noise (~5e-4 per fp16-operand product, the per-operator tests above) is amplified layer over layer —
    # by ~1.5x per layer with these deliberately lively synthetic weights (offsets of whole pixels, x20 token projection).
    # Attribution (tests/test_parity_experiment_gpu.py): every stage fed the oracle's input stays at the per-operator scale on
    # its own; keeping the attention scores in fp32 does not change the end-to-end figure; and the fp32 CPU oracle ITSELF moves
    # by 1.4e-2 (logits) when nothing but its inter-stage visual stream is rounded to fp16 (tools/fp16_storage_experiment.py).
    # The end-to-end deviation is therefore the chaotic amplification of fp16 STORAGE noise by these weights — it moves between
    # bit-different but equally accurate kernel variants — and not a defect of a stage; test_tower_reference_like_init checks the same tower at 3e-3 with
    # weights scaled like the reference's initialisation.  The per-operator bound stays at the north-star 1e-3.
    bad = []
    assert_close(r["hidden"], ref["hidden"], 4e-3, "tower: language stream", defer=bad)
    vis_ref = restate.flatten_levels(ref["visual"])
    assert_close(r["visual"], vis_ref, 3e-2, "tower: visual stream", defer=bad)
    mean_rel = (r["visual"].float().cpu() - vis_ref).abs().mean().item() / vis_ref.abs().mean().item()
    if mean_rel > 1e-2:
        bad.append(f"tower: visual stream mean relative error {mean_rel:.3e}")
    assert_close(r["dot_product_logits"], ref["dot_product_logits"], 2.5e-2, "tower: dot-product logits", defer=bad)
    ref_reg = restate.flatten_levels(ref["bbox_reg"])
    scale = torch.cat([torch.full((h * w,), float(sd[f"scales.{l}.scale"])) for l, (h, w) in enumerate(SIZES)])
    assert_close(r["reg_ctr"][..., :4].cpu() * scale[None, :, None], ref_reg, 3e-2, "tower: bbox regression", defer=bad)
    assert_close(r["reg_ctr"][..., 4].cpu(), restate.flatten_levels(ref["centerness"])[..., 0], 3e-2, "tower: centerness",
                 defer=bad)
    # reference-facing tuple API
    out = head([f.to(dev) for f in feats], {"hidden": hidden.to(dev), "masks": masks.to(dev)})
    assert len(out) == 10 and len(out[6]) == 5 and out[6][0].shape == (B, 20 * 28, T)
    assert_close(torch.cat([o.cpu() for o in out[6]], 1), ref["dot_product_logits"], 2.5e-2, "tuple API logits", defer=bad)
    assert_close(restate.flatten_levels([o.cpu() for o in out[1]]), ref_reg, 3e-2, "tuple API bbox_reg", defer=bad)
    # the same inputs through the REFERENCE's own VLDyHead.forward (fixture recorded by oracle/make_golden.py), same bounds
    from oracle import make_golden
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "vldyhead.pt"))
    for key, got_t, tol in (("logits", r["dot_product_logits"], 2.5e-2), ("hidden", r["hidden"], 4e-3)):
        g = make_golden.sub(got_t.float().cpu(), *fx["subsample"][key])
        err = (g - fx[key]).abs().max().item()
        if err > tol * fx[key + "_absmax"] + tol:
            bad.append(f"golden {key}: {err:.3e}")
    assert not bad, bad


def test_tower_reference_like_init(dev):
    """The same 6-layer tower with weights scaled like the reference's own initialisation (DyConv convs N(0, 0.01),
    vldyhead.py:184-203; unscaled 768->256 token projection) instead of the deliberately lively test weights: without the
    ~1.5x per-layer amplification the end-to-end logits stay within 3e-3 of max|ref| (VERDICT round 1, item 1c)."""
    from mqdet_b200 import ops
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.rpn.vldyhead import VLDyHead
    from oracle import restate, synth
    gen = synth.Gen(79)
    nconv = 6
    sd = synth.vldyhead_sd(gen, nconv)
    for k in list(sd):
        if ".DyConv." in k and k.endswith("conv.weight"):
            sd[k] = sd[k] / 3.0                      # N(0, 0.03) -> N(0, 0.01)
        if k.endswith("offset.weight"):
            sd[k] = sd[k] / 4.0
        if k.endswith("offset.bias"):
            sd[k] = sd[k] / 5.0
    sd["dot_product_projection_text.weight"] = sd["dot_product_projection_text.weight"] / 20.0
    B, T = 2, 256
    feats = [gen.randn(B, 256, h, w) for h, w in SIZES]
    hidden = gen.randn(B, T, 768)
    masks = torch.ones(B, T, dtype=torch.long)
    masks[0, 120:] = 0
    masks[1, 31:] = 0
    ref = restate.vl_dyhead(feats, hidden, masks, sd, nconv)
    head = load_sd(VLDyHead(mq_glip_t_cfg()), sd).to(dev).eval()
    lv = ops.Levels(SIZES, dev)
    r = head.forward_flat(restate.flatten_levels(feats).half().to(dev).contiguous(), lv, hidden.to(dev), masks.to(dev))
    bad = []
    assert_close(r["hidden"], ref["hidden"], 3e-3, "reference-like tower: language stream", defer=bad)
    assert_close(r["visual"], restate.flatten_levels(ref["visual"]), 6e-3, "reference-like tower: visual stream", defer=bad)
    assert_close(r["dot_product_logits"], ref["dot_product_logits"], 3e-3, "reference-like tower: dot-product logits", defer=bad)
    assert not bad, bad


def test_tower_two_streams_equal_single_stream(dev):
    """The tower with the text branch on a second stream (fork / join per layer) must return exactly what the single-stream
    order returns — same kernels, same inputs, only the interleaving changes — also when replayed from a CUDA graph."""
    from mqdet_b200 import ops
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.rpn.vldyhead import VLDyHead
    from oracle import restate, synth
    gen = synth.Gen(80)
    sd = synth.vldyhead_sd(gen, 6)
    B, T = 2, 256
    sizes = [(40, 56), (20, 28), (10, 14), (5, 7), (3, 4)]
    feats = [gen.randn(B, 256, h, w) for h, w in sizes]
    hidden = gen.randn(B, T, 768).to(dev)
    masks = torch.ones(B, T, dtype=torch.long)
    masks[0, 100:] = 0
    masks = masks.to(dev)
    head = load_sd(VLDyHead(mq_glip_t_cfg()), sd).to(dev).eval()
    lv = ops.Levels(sizes, dev)
    v16 = restate.flatten_levels(feats).half().to(dev).contiguous()
    head.overlap_text_stream = False
    a = head.forward_flat(v16, lv, hidden, masks)
    a = {k: a[k].clone() for k in ("dot_product_logits", "reg_ctr", "hidden", "visual")}
    head.overlap_text_stream = True
    for _ in range(3):   # repeated: a lifetime / ordering bug between the streams would show up as run-to-run differences
        b = head.forward_flat(v16, lv, hidden, masks)
        torch.cuda.synchronize()
        for k in a:
            assert torch.equal(a[k], b[k]), f"two-stream tower differs in {k}"
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = head.forward_flat(v16, lv, hidden, masks)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for k in a:
            assert torch.equal(a[k], c[k]), f"captured two-stream tower differs in {k}"
