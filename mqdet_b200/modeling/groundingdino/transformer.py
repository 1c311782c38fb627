"""GroundingDINO's encoder / decoder on sm_90a kernels, drop-in for groundingdino_new/models/GroundingDINO/transformer.py
(``Transformer`` :40-403, ``TransformerEncoder`` :406-590, ``TransformerDecoder`` :593-716, ``DeformableTransformerEncoderLayer``
:719-760, ``DeformableTransformerDecoderLayer`` :763-878) and transformer_vanilla.py:72-123 (``TransformerEncoderLayer``, the text
enhancer) under the shipped MQ-GroundingDINO-T settings (config/defaults.py:944-987: two_stage_type "standard", embed_init_tgt,
text enhancer, fusion layers, text cross-attention, post-norm, relu, dropout 0), inference only.

Same constructor arguments and ``state_dict`` keys as the reference (``nn.MultiheadAttention`` / ``nn.Linear`` / ``nn.LayerNorm``
objects are parameter containers); all arithmetic runs in libmqdet_b200.so:

  * every Linear / attention product: the wgmma GEMM (fp16 operands, fp32 accumulation, fused bias / relu / residual epilogues);
  * ``nn.MultiheadAttention`` (text enhancer with the per-category block mask, decoder self-attention over the 900 queries, decoder
    text cross-attention with the padding mask): Q|K|V^T projections, scores laid out [B, Lq, H, Lk] so one mask row serves the H
    heads of a query, ``softmax_rows`` with the mask folded in, P.V, output projection;
  * multi-scale deformable attention: ``MultiScaleDeformableAttention.core`` (``mqdet_ms_deform_attn``);
  * vision-language fusion: ``BiAttentionBlock`` (``stable_softmax_2d``);
  * ``with_pos_embed`` adds, masked memory: ``mqdet_add_cast``; residual + LayerNorm: ``mqdet_add_layernorm``;
  * decoder box refinement + conditional-query sine embedding: ``mqdet_box_refine_sine``;
  * two-stage query selection: ``ContrastiveEmbed`` + ``select_queries`` (row max, radix-select top-900, row gathers).

Geometry that depends only on the padding masks and the prompt (level position embeddings, encoder reference points, valid ratios,
anchor proposals, text position embeddings) is built once per input geometry by ``Transformer.prepare`` (host / torch index
arithmetic, like the anchors of the GLIP path) and reused by every forward of that geometry.
"""
import math

import torch
from torch import nn

from ... import ops
from ..._lib import ACT_RELU, VEC_PER_ROW, MqdetError
from ...utils.weights import f32, w16
from .fuse_modules import BiAttentionBlock
from .ms_deform_attn import MultiScaleDeformableAttention as MSDeformAttn
from .two_stage import select_queries
from .utils import MLP, ContrastiveEmbed, gen_encoder_output_proposals, get_sine_pos_embed


def _ln(a32, b32, norm):
    """LN(a + b) -> (fp16, fp32)."""
    return ops.add_layernorm(a32, b32, f32(norm.weight), f32(norm.bias), norm.eps)


def _ffn(x16, x32, linear1, linear2, norm):
    """x = LN(x + linear2(relu(linear1(x)))) (transformer.py:745-749,861-866) -> (fp16, fp32)."""
    shp = x32.shape
    h = ops.gemm(x16.view(-1, shp[-1]), w16(linear1.weight), bias=f32(linear1.bias), act=ACT_RELU)
    f = ops.gemm(h, w16(linear2.weight), bias=f32(linear2.bias), out_dtype=torch.float32)
    o16, o32 = _ln(x32.view(-1, shp[-1]), f, norm)
    return o16.view(shp), o32.view(shp)


def multihead_attention(m, q16, k16, v16, *, mask2d=None, keymask=None):
    """torch.nn.MultiheadAttention.forward at eval on the parameters of ``m`` (in_proj_weight / in_proj_bias / out_proj), batch
    first: q16 [B,Lq,E], k16 / v16 [B,Lk,E] fp16; mask2d fp32 [B,Lq,Lk] (1 = may attend, 0 = -inf; shared by the heads) or keymask
    fp32 [B,Lk] (1 = keep, 0 = -inf) -> fp32 [B*Lq, E] (the out_proj output, before the residual)."""
    B, Lq, E = q16.shape
    Lk = k16.shape[1]
    H = m.num_heads
    d = E // H
    Lkp = (Lk + 7) // 8 * 8
    bias = f32(m.in_proj_bias)
    dev = q16.device
    if q16 is k16:  # self-attention: Q | K in one product
        qk = ops.gemm(q16.view(B * Lq, E), w16(m.in_proj_weight, rows=(0, 2 * E)), bias=bias[: 2 * E]).view(B, Lq, 2, H, d)
        q, k = qk[:, :, 0], qk[:, :, 1]
    else:
        q = ops.gemm(q16.view(B * Lq, E), w16(m.in_proj_weight, rows=(0, E)), bias=bias[:E]).view(B, Lq, H, d)
        k = ops.gemm(k16.view(B * Lk, E), w16(m.in_proj_weight, rows=(E, 2 * E)), bias=bias[E: 2 * E]).view(B, Lk, H, d)
    # V^T[b] = W_v . v[b]^T + b_v -> [B, E, Lkp]: P.V is then K-major x K-major; the padding columns stay zero
    vT = torch.zeros((B, E, Lkp), dtype=torch.float16, device=dev)
    ops.gemm(w16(m.in_proj_weight, rows=(2 * E, 3 * E)), v16, out=vT[:, :, :Lk], bias=bias[2 * E:], bias_mode=VEC_PER_ROW)
    scores = torch.empty((B, Lq, H, Lkp), dtype=torch.float32, device=dev)
    ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=scores.permute(0, 2, 1, 3)[..., :Lk], alpha=d ** -0.5)
    if mask2d is not None:
        p = ops.softmax_rows(scores, n=Lk, colmask=mask2d, rows_per_batch=H, mask_value=float("-inf"))
    elif keymask is not None:
        p = ops.softmax_rows(scores, n=Lk, colmask=keymask, rows_per_batch=Lq * H, mask_value=float("-inf"))
    else:
        p = ops.softmax_rows(scores, n=Lk)
    ctx = torch.empty((B, Lq, H, d), dtype=torch.float16, device=dev)
    ops.gemm(p.permute(0, 2, 1, 3), vT.view(B, H, d, Lkp), out=ctx.permute(0, 2, 1, 3))
    return ops.gemm(ctx.view(B * Lq, E), w16(m.out_proj.weight), bias=f32(m.out_proj.bias), out_dtype=torch.float32)


class TransformerEncoderLayer(nn.Module):
    """transformer_vanilla.py:72-123 — the text enhancer layer (post-norm, relu; the key padding mask is NOT applied, :114)."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation="relu", normalize_before=False):
        super().__init__()
        if activation != "relu" or normalize_before:
            raise NotImplementedError("text enhancer: post-norm relu only (the shipped configuration)")
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.nhead = nhead

    @torch.no_grad()
    def forward_flat(self, src16, src32, pos32, mask2d):
        """src [B,T,E] (fp16 + fp32), pos32 [B,T,E], mask2d fp32 [B,T,T] (1 = may attend) -> (fp16, fp32)."""
        B, T, E = src32.shape
        q16 = ops.add_cast(src32, pos32)
        a = multihead_attention(self.self_attn, q16, q16, src16, mask2d=mask2d)
        s16, s32 = _ln(src32.view(B * T, E), a, self.norm1)
        return _ffn(s16.view(B, T, E), s32.view(B, T, E), self.linear1, self.linear2, self.norm2)

    def forward(self, src, src_mask=None, src_key_padding_mask=None, pos=None):
        """Reference signature: src [T,B,E], src_mask bool [B,T,T] (True = NOT allowed), pos [T,B,E] -> [T,B,E]."""
        if not src.is_cuda:
            raise MqdetError("TransformerEncoderLayer: CUDA tensors required (no CPU fallback)")
        s32 = src.transpose(0, 1).float().contiguous()
        p32 = torch.zeros_like(s32) if pos is None else pos.transpose(0, 1).float().contiguous()
        m = (~src_mask.bool()).float().contiguous()
        return self.forward_flat(ops.cast_f16(s32), s32, p32, m)[1].transpose(0, 1)


class DeformableTransformerEncoderLayer(nn.Module):
    """transformer.py:719-760."""

    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8, n_points=4):
        super().__init__()
        if activation != "relu":
            raise NotImplementedError("relu only (transformer_activation of the shipped configuration)")
        self.self_attn = MSDeformAttn(embed_dim=d_model, num_levels=n_levels, num_heads=n_heads, num_points=n_points, batch_first=True)
        self.norm1 = nn.LayerNorm(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.norm2 = nn.LayerNorm(d_model)

    @torch.no_grad()
    def forward_flat(self, src16, src32, pos32, reference_points, spatial_shapes, keep):
        B, N, E = src32.shape
        q16 = ops.add_cast(src32, pos32)
        a = self.self_attn.core(q16, src16, keep, reference_points, spatial_shapes)
        s16, s32 = _ln(src32.view(B * N, E), a.view(B * N, E), self.norm1)
        return _ffn(s16.view(B, N, E), s32.view(B, N, E), self.linear1, self.linear2, self.norm2)

    def forward(self, src, pos, reference_points, spatial_shapes, level_start_index, key_padding_mask=None):
        if not src.is_cuda:
            raise MqdetError("DeformableTransformerEncoderLayer: CUDA tensors required (no CPU fallback)")
        s32 = src.float().contiguous()
        keep = None if key_padding_mask is None else (~key_padding_mask.bool()).reshape(-1).float().contiguous()
        return self.forward_flat(ops.cast_f16(s32), s32, pos.float().contiguous(), reference_points, spatial_shapes, keep)[1]


class DeformableTransformerDecoderLayer(nn.Module):
    """transformer.py:763-878 with use_text_cross_attention."""

    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8, n_points=4,
                 use_text_feat_guide=False, use_text_cross_attention=False):
        super().__init__()
        if activation != "relu" or use_text_feat_guide:
            raise NotImplementedError("relu, no text-feature guide (the shipped configuration)")
        self.cross_attn = MSDeformAttn(embed_dim=d_model, num_levels=n_levels, num_heads=n_heads, num_points=n_points, batch_first=True)
        self.norm1 = nn.LayerNorm(d_model)
        self.use_text_cross_attention = use_text_cross_attention
        if use_text_cross_attention:
            self.ca_text = nn.MultiheadAttention(d_model, n_heads, dropout=dropout)
            self.catext_norm = nn.LayerNorm(d_model)
        self.self_attn = nn.MultiheadAttention(d_model, n_heads, dropout=dropout)
        self.norm2 = nn.LayerNorm(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.norm3 = nn.LayerNorm(d_model)

    @torch.no_grad()
    def forward_flat(self, tgt16, tgt32, qpos32, ref_input, memory16, keep_mem, spatial_shapes, text16, text_keep):
        """tgt [B,nq,E]; qpos32 [B,nq,E]; ref_input fp32 [B,nq,L,4]; memory16 [B,N,E]; text16 [B,T,E]; text_keep fp32 [B,T]."""
        B, nq, E = tgt32.shape
        q16 = ops.add_cast(tgt32, qpos32)
        a = multihead_attention(self.self_attn, q16, q16, tgt16)
        t16, t32 = _ln(tgt32.view(B * nq, E), a, self.norm2)
        if self.use_text_cross_attention:
            q16 = ops.add_cast(t32.view(B, nq, E), qpos32)
            a = multihead_attention(self.ca_text, q16, text16, text16, keymask=text_keep)
            t16, t32 = _ln(t32, a, self.catext_norm)
        q16 = ops.add_cast(t32.view(B, nq, E), qpos32)
        a = self.cross_attn.core(q16, memory16, keep_mem, ref_input, spatial_shapes)
        t16, t32 = _ln(t32, a.view(B * nq, E), self.norm1)
        return _ffn(t16.view(B, nq, E), t32.view(B, nq, E), self.linear1, self.linear2, self.norm3)


class TransformerEncoder(nn.Module):
    """transformer.py:406-590: per layer  fusion (BiAttentionBlock) -> text enhancer -> deformable encoder layer."""

    def __init__(self, encoder_layer_args, num_layers, d_model=256, num_queries=300, text_enhance_args=None, fusion_args=None):
        super().__init__()
        self.layers = nn.ModuleList([DeformableTransformerEncoderLayer(*encoder_layer_args) for _ in range(num_layers)])
        self.text_layers = nn.ModuleList([TransformerEncoderLayer(**text_enhance_args) for _ in range(num_layers)]) \
            if text_enhance_args is not None else []
        self.fusion_layers = nn.ModuleList([BiAttentionBlock(**fusion_args) for _ in range(num_layers)]) \
            if fusion_args is not None else []
        self.num_layers, self.d_model, self.num_queries = num_layers, d_model, num_queries

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        """transformer.py:473-489 (geometry only)."""
        refs = []
        for lvl, (H_, W_) in enumerate(spatial_shapes):
            ref_y, ref_x = torch.meshgrid(torch.linspace(0.5, H_ - 0.5, H_, dtype=torch.float32, device=device),
                                          torch.linspace(0.5, W_ - 0.5, W_, dtype=torch.float32, device=device), indexing="ij")
            ref_y = ref_y.reshape(-1)[None] / (valid_ratios[:, None, lvl, 1] * H_)
            ref_x = ref_x.reshape(-1)[None] / (valid_ratios[:, None, lvl, 0] * W_)
            refs.append(torch.stack((ref_x, ref_y), -1))
        return torch.cat(refs, 1)[:, :, None] * valid_ratios[:, None]

    @torch.no_grad()
    def forward_flat(self, src32, geo, text32):
        """src32 [B,N,E] fp32, text32 [B,T,E] fp32, geo = Transformer.prepare(...) -> (memory16, memory32, text16, text32)."""
        out32, out16 = src32, None
        t32, t16 = text32, None
        for i, layer in enumerate(self.layers):
            if len(self.fusion_layers):
                out32, t32 = self.fusion_layers[i](out32, t32, keep_v=geo["keep_mem2d"], keep_l=geo["text_keep"],
                                                   per_element_max=geo.get("per_element_max", False))
                out16 = t16 = None
            if len(self.text_layers):
                t16 = ops.cast_f16(t32) if t16 is None else t16
                t16, t32 = self.text_layers[i].forward_flat(t16, t32, geo["pos_text"], geo["text_self_mask"])
            out16 = ops.cast_f16(out32) if out16 is None else out16
            out16, out32 = layer.forward_flat(out16, out32, geo["pos"], geo["ref_enc"], geo["spatial_shapes"], geo["keep_mem"])
        if out16 is None:
            out16 = ops.cast_f16(out32)
        if t16 is None:
            t16 = ops.cast_f16(t32)
        return out16, out32, t16, t32


class TransformerDecoder(nn.Module):
    """transformer.py:593-716 (return_intermediate, query_dim 4, iterative box refinement)."""

    def __init__(self, decoder_layer_args, num_layers, norm=None, return_intermediate=True, d_model=256, query_dim=4,
                 num_feature_levels=1):
        super().__init__()
        assert return_intermediate and query_dim == 4
        self.layers = nn.ModuleList([DeformableTransformerDecoderLayer(**decoder_layer_args) for _ in range(num_layers)])
        self.num_layers, self.norm, self.d_model = num_layers, norm, d_model
        self.ref_point_head = MLP(query_dim // 2 * d_model, d_model, d_model, 2)
        self.bbox_embed = None
        self.class_embed = None

    @torch.no_grad()
    def forward_flat(self, tgt32, refpoints_unsigmoid, memory16, geo, text16, all_layers=False):
        """tgt32 [B,nq,E]; refpoints_unsigmoid fp32 [B,nq,4] -> (hs: list of fp32 [B,nq,E] (the last layer only unless
        ``all_layers``), references: list of sigmoid boxes fp32 [B,nq,4] (num_layers + 1 entries))."""
        B, nq, E = tgt32.shape
        out32, out16 = tgt32.contiguous(), ops.cast_f16(tgt32.contiguous())
        ref, ref_input, sine = ops.box_refine_sine(refpoints_unsigmoid, geo["valid_ratios"], ref_is_logit=True)
        refs, hs = [ref], []
        for i, layer in enumerate(self.layers):
            qpos = self.ref_point_head(sine.view(B * nq, -1), out_dtype=torch.float32).view(B, nq, E)
            out16, out32 = layer.forward_flat(out16, out32, qpos, ref_input, memory16, geo["keep_mem"], geo["spatial_shapes"],
                                              text16, geo["text_keep"])
            delta = self.bbox_embed[i](out16.view(B * nq, E), out_dtype=torch.float32)  # [B*nq, 8] (4 used)
            ref, ref_input, sine = ops.box_refine_sine(ref, geo["valid_ratios"], delta=delta.view(B, nq, -1),
                                                       want_sine=i + 1 < self.num_layers)
            refs.append(ref)
            if all_layers or i + 1 == self.num_layers:
                hs.append(ops.layernorm(out32, f32(self.norm.weight), f32(self.norm.bias), self.norm.eps, out16=False, out32=True))
        return hs, refs


class Transformer(nn.Module):
    """transformer.py:40-403.  ``forward`` keeps the reference signature; ``forward_flat`` is the fp16 / flat-row path."""

    def __init__(self, d_model=256, nhead=8, num_queries=300, num_encoder_layers=6, num_unicoder_layers=0, num_decoder_layers=6,
                 dim_feedforward=2048, dropout=0.0, activation="relu", normalize_before=False, return_intermediate_dec=False,
                 query_dim=4, num_patterns=0, num_feature_levels=1, enc_n_points=4, dec_n_points=4, learnable_tgt_init=False,
                 two_stage_type="no", embed_init_tgt=False, use_text_enhancer=False, use_fusion_layer=False, use_checkpoint=False,
                 use_transformer_ckpt=False, use_text_cross_attention=False, text_dropout=0.1, fusion_dropout=0.1,
                 fusion_droppath=0.0):
        super().__init__()
        if two_stage_type != "standard" or not embed_init_tgt or not learnable_tgt_init or normalize_before or num_patterns:
            raise NotImplementedError("two_stage_type='standard' + embed_init_tgt + learnable_tgt_init, post-norm, no patterns "
                                      "(the shipped MQ-GroundingDINO-T configuration)")
        self.num_feature_levels, self.num_queries, self.d_model, self.nhead = num_feature_levels, num_queries, d_model, nhead
        self.num_encoder_layers, self.num_decoder_layers = num_encoder_layers, num_decoder_layers
        enc_args = (d_model, dim_feedforward, dropout, activation, num_feature_levels, nhead, enc_n_points)
        text_args = dict(d_model=d_model, nhead=nhead // 2, dim_feedforward=dim_feedforward // 2, dropout=text_dropout) \
            if use_text_enhancer else None
        fusion_args = dict(v_dim=d_model, l_dim=d_model, embed_dim=dim_feedforward // 2, num_heads=nhead // 2, dropout=fusion_dropout,
                           drop_path=fusion_droppath) if use_fusion_layer else None
        self.encoder = TransformerEncoder(enc_args, num_encoder_layers, d_model=d_model, num_queries=num_queries,
                                          text_enhance_args=text_args, fusion_args=fusion_args)
        dec_args = dict(d_model=d_model, d_ffn=dim_feedforward, dropout=dropout, activation=activation, n_levels=num_feature_levels,
                        n_heads=nhead, n_points=dec_n_points, use_text_cross_attention=use_text_cross_attention)
        self.decoder = TransformerDecoder(dec_args, num_decoder_layers, nn.LayerNorm(d_model), return_intermediate=True,
                                          d_model=d_model, query_dim=query_dim, num_feature_levels=num_feature_levels)
        self.level_embed = nn.Parameter(torch.Tensor(num_feature_levels, d_model))
        self.tgt_embed = nn.Embedding(num_queries, d_model)
        nn.init.normal_(self.tgt_embed.weight.data)
        self.two_stage_type, self.embed_init_tgt = two_stage_type, embed_init_tgt
        self.enc_output = nn.Linear(d_model, d_model)
        self.enc_output_norm = nn.LayerNorm(d_model)
        self.enc_out_class_embed = None
        self.enc_out_bbox_embed = None
        self._reset_parameters()
        self._geo = {}

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, MSDeformAttn):
                m.init_weights()
        nn.init.normal_(self.level_embed)

    @staticmethod
    def get_valid_ratio(mask):
        """transformer.py:194-201."""
        _, H, W = mask.shape
        valid_H = torch.sum(~mask[:, :, 0], 1)
        valid_W = torch.sum(~mask[:, 0, :], 1)
        return torch.stack([valid_W.float() / W, valid_H.float() / H], -1)

    @torch.no_grad()
    def prepare(self, masks, pos_embeds, text_token_mask, position_ids, text_self_attention_masks):
        """Everything that depends only on the padding masks and on the prompt (transformer.py:222-250,473-489,516-530;
        utils.py:59-107): cached by the caller per input geometry.  masks: list of bool [B,h,w] (True = padding); pos_embeds: list
        of [B,C,h,w]; text_token_mask bool [B,T] (True = token in use); position_ids int64 [B,T]; text_self_attention_masks bool
        [B,T,T] (True = may attend)."""
        return {**self.prepare_image(masks, pos_embeds), **self.prepare_text(text_token_mask, position_ids, text_self_attention_masks)}

    IMAGE_GEOMETRY_KEYS = ("mask_flat", "pos", "valid_ratios", "ref_enc", "keep_mem2d", "output_proposals")

    @torch.no_grad()
    def prepare_image(self, masks, pos_embeds):
        """The image half of ``prepare``: level masks, level position embeddings, valid ratios, encoder reference points, anchor
        proposals.  Batched tensors are under ``IMAGE_GEOMETRY_KEYS`` (plus the flat views ``keep_mem`` / ``proposal_keep``)."""
        dev = masks[0].device
        shapes = [tuple(int(x) for x in m.shape[-2:]) for m in masks]
        mask_flat = torch.cat([m.flatten(1) for m in masks], 1)
        pos = torch.cat([p.flatten(2).transpose(1, 2).float() + self.level_embed[l].detach().float().view(1, 1, -1)
                         for l, p in enumerate(pos_embeds)], 1).contiguous()
        valid_ratios = torch.stack([self.get_valid_ratio(m) for m in masks], 1).float().contiguous()
        ref_enc = TransformerEncoder.get_reference_points(shapes, valid_ratios, dev).contiguous()
        valid, proposals = gen_encoder_output_proposals(mask_flat, shapes)
        keep = (~mask_flat).float().contiguous()
        return {"spatial_shapes": shapes, "mask_flat": mask_flat, "pos": pos, "valid_ratios": valid_ratios, "ref_enc": ref_enc,
                "keep_mem": keep.reshape(-1), "keep_mem2d": keep,
                "proposal_keep": (valid & ~mask_flat).float().reshape(-1).contiguous(), "output_proposals": proposals.contiguous()}

    @staticmethod
    def repeat_image_geometry(img_geo, times):
        """``prepare_image`` output for a batch that holds the same images ``times`` times over (element e = k * B + image)."""
        out = dict(img_geo)
        for k in Transformer.IMAGE_GEOMETRY_KEYS:
            t = img_geo[k]
            out[k] = t.repeat(times, *([1] * (t.dim() - 1))).contiguous()
        out["keep_mem"] = out["keep_mem2d"].reshape(-1)
        out["proposal_keep"] = img_geo["proposal_keep"].repeat(times).contiguous()
        return out

    @torch.no_grad()
    def prepare_text(self, text_token_mask, position_ids, text_self_attention_masks):
        """The prompt half of ``prepare``: text position embeddings, token and self-attention masks."""
        pos_text = get_sine_pos_embed(position_ids[..., None].float(), num_pos_feats=256, exchange_xy=False).contiguous()
        return {"pos_text": pos_text, "text_keep": text_token_mask.float().contiguous(), "text_token_mask": text_token_mask,
                "text_self_mask": text_self_attention_masks.float().contiguous()}

    @torch.no_grad()
    def forward_flat(self, src32, geo, text32, all_layers=False, proposals=None):
        """src32 fp32 [B,N,E] (levels concatenated), text32 fp32 [B,T,E] -> dict(hs, references, memory, memory_text, ...).
        ``proposals``: see ``select_queries`` (parity tests only)."""
        B, N, E = src32.shape
        mem16, mem32, text16, text32 = self.encoder.forward_flat(src32, geo, text32)
        # two-stage query selection (:272-318)
        om16 = ops.add_cast(mem32, None, geo["proposal_keep"])
        eo = ops.gemm(om16.view(B * N, E), w16(self.enc_output.weight), bias=f32(self.enc_output.bias), out_dtype=torch.float32)
        n = self.enc_output_norm
        o16, o32 = ops.layernorm(eo, f32(n.weight), f32(n.bias), n.eps, out16=True, out32=True)
        text_dict = {"encoded_text": text32, "encoded_text16": text16, "text_token_mask": geo["text_token_mask"]}
        enc_class = self.enc_out_class_embed(o16.view(B, N, E), text_dict)
        coord = self.enc_out_bbox_embed(o16, out_dtype=torch.float32, residual=geo["output_proposals"].view(B * N, 4))
        sel = select_queries(enc_class, coord.view(B, N, -1)[..., :4], geo["output_proposals"], o32.view(B, N, E), self.num_queries,
                             proposals=proposals)
        tgt = self.tgt_embed.weight.detach().float()[None].expand(B, -1, -1).contiguous()
        hs, refs = self.decoder.forward_flat(tgt, sel["refpoint_embed"], mem16, geo, text16, all_layers=all_layers)
        return {"hs": hs, "references": refs, "memory": mem32, "memory_text": text32, "memory_text16": text16,
                "enc_class": enc_class, "topk_proposals": sel["topk_proposals"], "init_box_proposal": sel["init_box_proposal"],
                "hs_enc": sel["tgt"], "ref_enc": sel["refpoint_embed"]}

    def forward(self, srcs, masks, refpoint_embed, pos_embeds, tgt, attn_mask=None, text_dict=None):
        """Reference signature (:206-403): srcs / pos_embeds lists of [B,C,h,w], masks list of bool [B,h,w]; text_dict with
        encoded_text, text_token_mask, position_ids, text_self_attention_masks -> (hs, references, hs_enc, ref_enc,
        init_box_proposal); ``text_dict['encoded_text']`` is replaced by the enhanced text like the reference does."""
        if refpoint_embed is not None or tgt is not None or attn_mask is not None:
            raise NotImplementedError("denoising queries (training) are not part of the inference path")
        if not srcs[0].is_cuda:
            raise MqdetError("Transformer: CUDA tensors required (no CPU fallback)")
        geo = self.prepare(masks, pos_embeds, text_dict["text_token_mask"], text_dict["position_ids"],
                           text_dict["text_self_attention_masks"])
        src = torch.cat([s.flatten(2).transpose(1, 2) for s in srcs], 1).float().contiguous()
        out = self.forward_flat(src, geo, text_dict["encoded_text"].float().contiguous(), all_layers=True)
        text_dict["encoded_text"] = out["memory_text"]
        return out["hs"], out["references"], out["hs_enc"].unsqueeze(0), out["ref_enc"].sigmoid().unsqueeze(0), out["init_box_proposal"]
