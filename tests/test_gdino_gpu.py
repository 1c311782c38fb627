"""GPU parity of the GroundingDINO reuse row (SURVEY.md §8 a18): ContrastiveEmbed through the C ABI (wgmma product +
mask/pad kernel) against the CPU oracle and the golden vectors recorded from the reference's own class."""
import os

import pytest
import torch

from util import FP16_TOL, ROOT

pytestmark = pytest.mark.gpu


def _check(out, ref, absmax):
    out = out.cpu()
    assert out.shape == ref.shape
    assert torch.equal(torch.isinf(out) & (out < 0), torch.isinf(ref))      # exact -inf pattern (index work: bit-exact)
    fin = torch.isfinite(ref)
    assert (out[fin] - ref[fin]).abs().max().item() <= FP16_TOL * absmax + FP16_TOL


def test_contrastive_embed_vs_oracle_and_golden(dev):
    from mqdet_b200.modeling.groundingdino.utils import ContrastiveEmbed
    from oracle import make_golden, restate
    c = make_golden.case_inputs("contrastive_embed")
    ref = restate.contrastive_embed(c["x"], c["y"], c["mask"], 256)
    mod = ContrastiveEmbed(max_text_len=256)
    out = mod(c["x"].to(dev), {"encoded_text": c["y"].to(dev), "text_token_mask": c["mask"].to(dev)})
    _check(out, ref, ref[torch.isfinite(ref)].abs().max().item())
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "contrastive_embed.pt"))
    _check(make_golden.sub(out.cpu(), *fx["subsample"]["logits"]), fx["logits"], fx["logits_absmax"])


def test_contrastive_embed_encoder_memory_shape(dev):
    """Two-stage proposal scoring (transformer.py:288-303): 22323 memory tokens x 195 text tokens, batch 2."""
    from mqdet_b200.modeling.groundingdino.utils import ContrastiveEmbed
    from oracle import restate
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 22323, 256, generator=g)
    y = torch.randn(2, 195, 256, generator=g)
    mask = torch.ones(2, 195, dtype=torch.bool)
    mask[1, 40:] = False
    ref = restate.contrastive_embed(x, y, mask, 256)
    out = ContrastiveEmbed(256)(x.to(dev), {"encoded_text": y.to(dev), "text_token_mask": mask.to(dev)})
    _check(out, ref, ref[torch.isfinite(ref)].abs().max().item())
    # the two-stage selection consumes the row maximum: same top-900 set up to fp16 ties
    top_ref = ref.max(-1)[0].topk(900, dim=1)[1]
    top_out = out.cpu().max(-1)[0].topk(900, dim=1)[1]
    for b in range(2):
        inter = len(set(top_ref[b].tolist()) & set(top_out[b].tolist()))
        assert inter >= 890, inter


@pytest.mark.parametrize("ref_dim,Q", [(2, 1750), (4, 900)])
def test_ms_deform_attn_vs_oracle(dev, ref_dim, Q):
    """MultiScaleDeformableAttention (SURVEY.md §8f rank 1): encoder-style call (queries == the flattened pyramid, 2-d
    reference points) and decoder-style call (900 queries, 4-d reference boxes), padding mask, batch_first False and True."""
    from mqdet_b200.modeling.groundingdino.ms_deform_attn import MultiScaleDeformableAttention
    from oracle import restate, synth
    from util import assert_close, load_sd
    gen = synth.Gen(1310 + ref_dim)
    sd = synth.msda_sd(gen)
    shapes = [(40, 30), (20, 15), (10, 8), (5, 4)]
    B, E = 2, 256
    nv = sum(h * w for h, w in shapes)
    if ref_dim == 2:
        Q = nv
    query, value = gen.randn(B, Q, E), gen.randn(B, nv, E)
    pos = gen.randn(B, Q, E, scale=0.3)
    ref_pts = torch.rand(B, Q, 4, ref_dim, generator=gen.g)
    if ref_dim == 4:
        ref_pts[..., 2:] = ref_pts[..., 2:] * 0.3 + 0.05
    mask = torch.zeros(B, nv, dtype=torch.bool)
    mask[1, -77:] = True
    ref = restate.ms_deform_attn(query, value, ref_pts, shapes, sd, key_padding_mask=mask, query_pos=pos)
    ss = torch.tensor(shapes)
    lsi = torch.cat([ss.new_zeros(1), (ss[:, 0] * ss[:, 1]).cumsum(0)[:-1]])
    for batch_first in (True, False):
        mod = load_sd(MultiScaleDeformableAttention(embed_dim=E, num_heads=8, num_levels=4, num_points=4, batch_first=batch_first), sd)
        mod = mod.to(dev).eval()
        q, v, p = query.to(dev), value.to(dev), pos.to(dev)
        if not batch_first:
            q, v, p = q.transpose(0, 1), v.transpose(0, 1), p.transpose(0, 1)
        out = mod(q, value=v, query_pos=p, key_padding_mask=mask.to(dev), reference_points=ref_pts.to(dev), spatial_shapes=ss.to(dev),
                  level_start_index=lsi.to(dev))
        if not batch_first:
            out = out.transpose(0, 1)
        assert_close(out, ref, 2e-3, f"MultiScaleDeformableAttention ref_dim={ref_dim} batch_first={batch_first}")


def test_global_max_shift_clamp_row_max(dev):
    """The three small ops of STABLE_SOFTMAX_2D / the two-stage selection, exactly against torch (sizes off the vector width)."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(31)
    for n in (1, 7, 1024 * 1024 + 3):
        x = (torch.randn(n, generator=g) * 1000).to(dev)
        gm = ops.global_max(x)
        assert gm.item() == x.max().item()
        y = x.clone()
        ops.shift_clamp_(y, gm, -500.0, 500.0)
        assert torch.equal(y, (x - x.max()).clamp(-500.0, 500.0))
    x = torch.randn(5003, 256, generator=g)
    x[:, 200:] = float("-inf")
    x[17] = float("-inf")
    assert torch.equal(ops.row_max(x.to(dev)).cpu(), x.max(-1)[0])


@pytest.mark.parametrize("masks", [False, True])
def test_gdino_bi_attention_block(dev, masks):
    """GroundingDINO BiAttentionBlock (fuse_modules.py:257-296; stable_softmax_2d, -inf boolean masks for text AND image tokens)
    at the MQ-GroundingDINO-T encoder dimensions (256 / 256 / 1024, 4 heads), N not a multiple of 8."""
    from mqdet_b200.modeling.groundingdino.fuse_modules import BiAttentionBlock
    from oracle import restate, synth
    from util import assert_close, load_sd
    gen = synth.Gen(1410)
    sd = synth.bi_attention_sd(gen, v_dim=256, l_dim=256, embed=1024)
    B, N, T = 2, 1003, 64
    v, l = gen.randn(B, N, 256), gen.randn(B, T, 256)
    mask_v = mask_l = None
    if masks:
        mask_v = torch.zeros(B, N, dtype=torch.bool)
        mask_v[1, -131:] = True
        mask_l = torch.zeros(B, T, dtype=torch.bool)
        mask_l[0, -9:] = True
    ref_v, ref_l = restate.gdino_bi_attention(v, l, sd, mask_v=mask_v, mask_l=mask_l)
    mod = load_sd(BiAttentionBlock(v_dim=256, l_dim=256, embed_dim=1024, num_heads=4), sd).to(dev).eval()
    out_v, out_l = mod(v.to(dev), l.to(dev), attention_mask_v=None if mask_v is None else mask_v.to(dev),
                       attention_mask_l=None if mask_l is None else mask_l.to(dev))
    assert out_v.dtype == torch.float32 and out_l.dtype == torch.float32
    assert_close(out_v, ref_v, 1e-3, "GroundingDINO BiAttentionBlock: image side")
    assert_close(out_l, ref_l, 1e-3, "GroundingDINO BiAttentionBlock: text side")


def test_gdino_two_stage_select(dev):
    """Two-stage query selection (transformer.py:297-318) at the encoder size of config 4 (22323 positions, 256 text tokens with
    -inf padding, 900 queries): indices identical to torch.topk, gathers exact; ties resolve towards the lower index."""
    from mqdet_b200.modeling.groundingdino.two_stage import select_queries
    from oracle import restate
    g = torch.Generator().manual_seed(77)
    B, Q, T, C, k = 2, 22323, 256, 256, 900
    logits = torch.randn(B, Q, T, generator=g) * 3.0
    logits[:, :, 40:] = float("-inf")          # padded text tokens (ContrastiveEmbed fills -inf)
    coord = torch.randn(B, Q, 4, generator=g)
    prop = torch.randn(B, Q, 4, generator=g) * 2.0
    mem = torch.randn(B, Q, C, generator=g)
    ref = restate.gdino_two_stage_select(logits, coord, prop, mem, k)
    out = select_queries(logits.to(dev), coord.to(dev), prop.to(dev), mem.to(dev), k)
    assert torch.equal(out["topk_logits"].cpu(), ref["topk_logits"])
    assert torch.equal(out["topk_proposals"].cpu(), ref["idx"])
    assert torch.equal(out["refpoint_embed"].cpu(), ref["refpoint_embed"]) and torch.equal(out["tgt"].cpu(), ref["tgt"])
    assert (out["init_box_proposal"].cpu() - ref["init_box_proposal"]).abs().max().item() <= 2e-7
    # ties: equal keys come out in index order; k == n; a row of -inf
    from mqdet_b200 import ops
    keys = torch.zeros(3, 1500)
    keys[1, 100:] = -1.0
    keys[2] = float("-inf")
    idx = ops.topk_desc(keys.to(dev), 1000).cpu()
    assert torch.equal(idx[0], torch.arange(1000)) and torch.equal(idx[1], torch.arange(1000)) and torch.equal(idx[2], torch.arange(1000))
    small = torch.tensor([[3.0, -1.0, 7.0, 7.0, 0.5]])
    assert ops.topk_desc(small.to(dev), 5).cpu().tolist() == [[2, 3, 0, 4, 1]]
