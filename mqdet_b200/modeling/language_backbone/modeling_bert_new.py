"""Vision-conditioned BERT: Gated Class-scalable Perceiver (GCP) blocks + PreSelect + BERT layers on sm_90a kernels.

Drop-in for maskrcnn_benchmark/modeling/language_backbone/modeling_bert_new.py: same class names, constructor
arguments, parameter names (``attn.norm``, ``attn.norm_kv``, ``attn.to_q``, ``attn.to_kv``, ``attn.to_out``,
``attn_gate.{norm,linear1,linear2}``, ``ff.{norm,linear1,linear2}``, ``ff_gate``, ``encoder.qv_layer.N``,
``pre_select.layers.N`` ...) and forward signatures, inference only (no autograd; backward is SURVEY.md §8f).
nn.LayerNorm / nn.Linear objects are parameter containers; all arithmetic runs in libmqdet_b200.so.

Data layout: text stream fp32 [B,T,768] in HBM (residual accuracy), every GEMM operand fp16, fp32 accumulation.
"""
from collections import OrderedDict

import torch
from torch import nn

from ... import ops
from ..._lib import ACT_GELU, VEC_PER_ROW, VEC_SCALAR, MqdetError
from ...utils.weights import f32, w16


def exists(val):
    """modeling_bert_new.py:106-113."""
    return val is not None and len(val) > 0


def FeedForward(dim, mult=4, out_dim=None):
    """Parameter container with the reference's names (modeling_bert_new.py:115-126): LN -> Linear -> GELU -> Linear."""
    inner_dim = int(dim * mult)
    out_dim = dim if out_dim is None else out_dim
    return nn.Sequential(OrderedDict([
        ("norm", nn.LayerNorm(dim)),
        ("linear1", nn.Linear(dim, inner_dim, bias=False)),
        ("gelu", nn.GELU()),
        ("linear2", nn.Linear(inner_dim, out_dim, bias=False)),
    ]))


def _ln16(x, norm, **kw):
    return ops.layernorm(x, f32(norm.weight), f32(norm.bias), norm.eps, **kw)


def _as_f32(x):
    return ops.cast_f32(x) if x.dtype == torch.float16 else x.float().contiguous()


# one-entry caches: the index table / padded vision tensor are identical for the 6 GCP blocks of a forward
_idx_cache = {}
_pad_cache = {}


def cache_entries():
    """The current entries of the two caches, for a holder that must keep them alive (a captured CUDA graph reads them)."""
    return (_idx_cache.get("e"), _pad_cache.get("e"))


def sparse_index(attention_mask):
    """[B,V,T] 0/1 mask -> int32 [B,T,S] ascending query indices padded with V (get_index_with_padding_batch :40-63).
    S = the global max count; computing it needs one device->host read, done once per distinct mask tensor.
    The cache holds the tensor itself (identity + version), never a bare data_ptr that the allocator could recycle."""
    ent = _idx_cache.get("e")
    if ent is not None and ent[0] is attention_mask and ent[1] == attention_mask._version:
        return ent[2]
    m = attention_mask if attention_mask.dtype == torch.float32 else attention_mask.float()
    _, counts = ops.gcp_build_index(m, 1)
    S = int(counts.max().item())
    idx, _ = ops.gcp_build_index(m, max(S, 1))
    _idx_cache["e"] = (attention_mask, attention_mask._version, idx)
    return idx


def use_sparse_index(attention_mask, idx):
    """Make ``idx`` (``sparse_index(attention_mask)``, kept by the caller) the current entry: a forward that alternates between
    several masks (one per pass of a chunked forward) then reads no count on the host, and can be captured in a CUDA graph."""
    _idx_cache["e"] = (attention_mask, attention_mask._version, idx)


def padded_vision(vision):
    """cat(vision, zero row) -> fp32 [B, V+1, D] (modeling_bert_new.py:176-177); cached per vision tensor object."""
    ent = _pad_cache.get("e")
    if ent is not None and ent[0] is vision and ent[1] == vision._version:
        return ent[2]
    B, V, D = vision.shape
    buf = torch.zeros((B, V + 1, D), dtype=torch.float32, device=vision.device)
    buf[:, :V].copy_(vision)
    _pad_cache["e"] = (vision, vision._version, buf)
    return buf


class MaskedCrossAttention(nn.Module):
    """modeling_bert_new.py:128-248.  ``spase_forward=True``: sparse GCP attention (each text token attends to the <=S
    queries of its class); ``False``: dense cross-attention (PreSelect).  Linear layers are bias-free."""

    def __init__(self, *, input_dim, output_dim=None, dim_head=64, heads=8, norm_kv=False, share_kv=False, cfg=None,
                 spase_forward=False):
        super().__init__()
        if share_kv:
            raise NotImplementedError("share_kv=True is not used by any MQ config (VISION_QUERY.SHARE_KV False)")
        self.spase_forward = spase_forward
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.dim_head = dim_head
        self.share_kv = share_kv
        inner_dim = dim_head * heads
        self.inner_dim = inner_dim
        output_dim = input_dim if output_dim is None else output_dim
        self.norm = nn.LayerNorm(input_dim)
        self.norm_kv = nn.LayerNorm(input_dim) if norm_kv else None
        self.to_q = nn.Linear(input_dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(input_dim, inner_dim * 2, bias=False)
        self.to_out = nn.Linear(inner_dim, output_dim, bias=False)
        self.flash = True  # dense path: fused attention kernel (False: the unfused GEMM / softmax_rows path, kept for A/B tests)

    # -- sparse (GCP) ------------------------------------------------------------------------------------------
    def _sparse(self, x32, vision, attention_mask, out_residual=None):
        B, T, D = x32.shape
        V = vision.shape[1]
        idx = sparse_index(attention_mask)
        vis_pad = padded_vision(vision)
        xn = _ln16(x32, self.norm)
        q = ops.gemm(xn.view(B * T, D), w16(self.to_q.weight), alpha=self.scale)
        kn = _ln16(vis_pad, self.norm_kv) if self.norm_kv is not None else ops.cast_f16(vis_pad)
        kv = ops.gemm(kn.view(B * (V + 1), D), w16(self.to_kv.weight))  # K|V once per unique query
        o = ops.gcp_sparse_attn(q.view(B, T, self.inner_dim), kv.view(B, V + 1, 2 * self.inner_dim), idx, self.heads,
                                self.dim_head)
        s = ops.gemm(o.view(B * T, self.inner_dim), w16(self.to_out.weight), out_dtype=torch.float32)
        return s.view(B, T, -1)

    # -- dense (PreSelect) -------------------------------------------------------------------------------------
    def _dense(self, x32, ctx, residual):
        """x32 [B,Tq,D] fp32 attends to ctx [B,I,D]; returns to_out(attn) + residual as fp32 [B,Tq,out]."""
        B, Tq, D = x32.shape
        I = ctx.shape[1]
        H, d, inner = self.heads, self.dim_head, self.inner_dim
        Ipad = (I + 7) // 8 * 8
        xn = _ln16(x32, self.norm)
        cn = _ln16(ctx, self.norm_kv) if self.norm_kv is not None else ops.cast_f16(ctx)
        if d == 32 and self.flash:
            # ONE projection for K | V (the to_kv Linear as is) and ONE flash-style attention kernel: the fp32 score tensor
            # [B, H, Tq, I] (571 MB at B = 8, 80 classes) is never written
            q = ops.gemm(xn.view(B * Tq, D), w16(self.to_q.weight), alpha=self.scale).view(B, Tq, inner)
            kv = ops.gemm(cn.view(B * I, D), w16(self.to_kv.weight)).view(B, I, 2 * inner)
            o = ops.dense_cross_attn(q, kv, H, d)
            out = ops.gemm(o.view(B * Tq, inner), w16(self.to_out.weight), out_dtype=torch.float32,
                           residual=residual.reshape(B * Tq, -1) if residual is not None else None)
            return out.view(B, Tq, -1)
        q = ops.gemm(xn.view(B * Tq, D), w16(self.to_q.weight), alpha=self.scale).view(B, Tq, H, d)
        k = ops.gemm(cn.view(B * I, D), w16(self.to_kv.weight, rows=(0, inner))).view(B, I, H, d)
        # V^T[b] = W_v . cn[b]^T  -> [B, inner, Ipad] so that P.V is again a K-major x K-major product
        vT = torch.zeros((B, inner, Ipad), dtype=torch.float16, device=x32.device)
        ops.gemm(w16(self.to_kv.weight, rows=(inner, 2 * inner)), cn, out=vT[:, :, :I])
        scores = torch.empty((B, H, Tq, Ipad), dtype=torch.float32, device=x32.device)
        ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=scores[..., :I])
        p = ops.softmax_rows(scores, n=I)
        o = torch.empty((B, Tq, H, d), dtype=torch.float16, device=x32.device)
        ops.gemm(p, vT.view(B, H, d, Ipad), out=o.permute(0, 2, 1, 3))
        out = ops.gemm(o.view(B * Tq, inner), w16(self.to_out.weight), out_dtype=torch.float32,
                       residual=residual.reshape(B * Tq, -1) if residual is not None else None)
        return out.view(B, Tq, -1)

    def forward(self, x, vision, attention_mask=None):
        if not x.is_cuda:
            raise MqdetError("MaskedCrossAttention: CUDA tensors required (no CPU fallback)")
        x32 = _as_f32(x)
        if self.spase_forward:
            return self._sparse(x32, vision, attention_mask)
        if exists(attention_mask):
            raise NotImplementedError("dense MaskedCrossAttention with a mask is not on the MQ-Det path")
        return self._dense(x32, _as_f32(vision) if vision.dtype != torch.float32 else vision, None)


class GatedCrossAttentionBlock(nn.Module):
    """modeling_bert_new.py:250-374 under the shipped flags (CONDITION_GATE, NONLINEAR_GATE, NO_CAT, FIX_ATTN_GATE=-1,
    no ADAPT layer; configs/pretrain/mq-glip-t.yaml:132-141):
        s = attn(x, vision, mask);  g = tanh(MLP(s));  x1 = s*g + x;  y = FF(x1)*tanh(ff_gate) + x1
    """

    def __init__(self, *, dim, dim_head=64, heads=8, ff_mult=4, share_kv=False, cfg=None, enable_ffn=True):
        super().__init__()
        vq = cfg.VISION_QUERY
        if not (vq.FIX_ATTN_GATE == -1.0 and vq.CONDITION_GATE and vq.NONLINEAR_GATE and vq.NO_CAT) or \
                getattr(vq, "ADD_ADAPT_LAYER", False):
            raise NotImplementedError("only the shipped gate configuration (CONDITION_GATE+NONLINEAR_GATE+NO_CAT, "
                                      "FIX_ATTN_GATE=-1, no ADAPT layer) is implemented")
        self.attn = MaskedCrossAttention(input_dim=dim, dim_head=dim_head, heads=heads, share_kv=share_kv, cfg=cfg,
                                         norm_kv=True, spase_forward=True)
        self.attn_gate = FeedForward(dim=dim, mult=0.5, out_dim=1)
        torch.nn.init.constant_(self.attn_gate.linear2.weight, 0)
        self.enable_ffn = enable_ffn
        if enable_ffn:
            self.ff = FeedForward(dim, mult=ff_mult)
            self.ff_gate = nn.Parameter(torch.tensor([0.]))
        self.cfg = cfg
        self.attn_gate_value = 0.

    @torch.no_grad()
    def forward(self, x, vision, attention_mask=None, batched_positive_label_position=None):
        if not x.is_cuda:
            raise MqdetError("GatedCrossAttentionBlock: CUDA tensors required (no CPU fallback)")
        B, T, D = x.shape
        x32 = _as_f32(x)
        s = self.attn._sparse(x32, vision, attention_mask)  # fp32 [B,T,D]
        sn = _ln16(s, self.attn_gate.norm)
        h1 = ops.gemm(sn.view(B * T, D), w16(self.attn_gate.linear1.weight), act=ACT_GELU)
        want_gate = bool(getattr(self.cfg.VISION_QUERY, "RETURN_ATTN_GATE_VALUE", False))
        norm = self.ff.norm if self.enable_ffn else self.attn_gate.norm
        res = ops.gcp_gate_residual_ln(h1, f32(self.attn_gate.linear2.weight).view(-1), s, x32, f32(norm.weight),
                                       f32(norm.bias), norm.eps, want_gate=want_gate)
        x1, x1n = res[0], res[1]
        if want_gate:
            self.attn_gate_value = res[2].mean().item()
        if not self.enable_ffn:
            return x1
        h2 = ops.gemm(x1n.view(B * T, D), w16(self.ff.linear1.weight), act=ACT_GELU)
        y = ops.gemm(h2, w16(self.ff.linear2.weight), out_dtype=torch.float32, gate=f32(self.ff_gate),
                     gate_mode=VEC_SCALAR, gate_tanh=True, residual=x1.view(B * T, D))
        return y.view(B, T, D)


class PreSelectBlock(nn.Module):
    """modeling_bert_new.py:377-409: v <- CA(LN(v), LN_kv(img)) + res_mapping(v);  v <- FF(v) + v."""

    def __init__(self, *, dim, out_dim=None, dim_head=32, heads=8, ff_mult=4, share_kv=False, cfg=None):
        super().__init__()
        self.image_condition = MaskedCrossAttention(input_dim=dim, output_dim=out_dim, dim_head=dim_head, heads=heads,
                                                    norm_kv=True, share_kv=share_kv, cfg=cfg, spase_forward=False)
        self.ff = FeedForward(out_dim, mult=ff_mult)
        self.res_mapping = nn.Linear(dim, out_dim, bias=False) if dim != out_dim else nn.Identity()

    @torch.no_grad()
    def forward(self, x):
        vision, image = x["vision"], x["image"]
        v32 = _as_f32(vision)
        B, V, D = v32.shape
        if isinstance(self.res_mapping, nn.Linear):
            res = ops.gemm(ops.cast_f16(v32).view(B * V, D), w16(self.res_mapping.weight), out_dtype=torch.float32)
            res = res.view(B, V, -1)
        else:
            res = v32
        img32 = image if image.dtype == torch.float32 else _as_f32(image)
        v = self.image_condition._dense(v32, img32, res)  # fp32 [B,V,out]
        Do = v.shape[-1]
        vn = _ln16(v, self.ff.norm)
        h = ops.gemm(vn.view(B * V, Do), w16(self.ff.linear1.weight), act=ACT_GELU)
        v = ops.gemm(h, w16(self.ff.linear2.weight), out_dtype=torch.float32, residual=v.view(B * V, Do))
        return {"vision": v.view(B, V, Do), "image": image}


class PreSelectModule(nn.Module):
    """modeling_bert_new.py:412-448."""

    def __init__(self, *, dim, out_dim, dim_head=32, heads=8, ff_mult=4, num_layers=2, share_kv=False, cfg=None):
        super().__init__()
        layers = [PreSelectBlock(dim=dim, out_dim=dim, dim_head=dim_head, heads=heads, ff_mult=ff_mult,
                                 share_kv=share_kv, cfg=cfg) for _ in range(num_layers - 1)]
        layers.append(PreSelectBlock(dim=dim, out_dim=out_dim, dim_head=dim_head, heads=heads, ff_mult=ff_mult,
                                     share_kv=share_kv, cfg=cfg))
        self.layers = nn.Sequential(*layers)
        self.scale = cfg.VISION_QUERY.VISION_SCALE
        self.augment_image_with_query = getattr(cfg.VISION_QUERY, "AUGMENT_IMAGE_WITH_QUERY", False)
        if self.augment_image_with_query:
            raise NotImplementedError("AUGMENT_IMAGE_WITH_QUERY is False in every shipped MQ config")

    @torch.no_grad()
    def forward(self, vision, image):
        if self.scale != 1.0:
            vision, image = vision * self.scale, image * self.scale
        return self.layers({"vision": vision, "image": image})


# ----------------------------------------------------------------------------------------------------------------------
# BERT (HF key names so bert-base-uncased checkpoints load unchanged)
# ----------------------------------------------------------------------------------------------------------------------
class _SelfAttn(nn.Module):
    def __init__(self, D):
        super().__init__()
        self.query, self.key, self.value = nn.Linear(D, D), nn.Linear(D, D), nn.Linear(D, D)


class _SelfOutput(nn.Module):
    def __init__(self, D_in, D, eps):
        super().__init__()
        self.dense = nn.Linear(D_in, D)
        self.LayerNorm = nn.LayerNorm(D, eps=eps)


class _Attention(nn.Module):
    def __init__(self, D, eps):
        super().__init__()
        self.self = _SelfAttn(D)
        self.output = _SelfOutput(D, D, eps)


class _Intermediate(nn.Module):
    def __init__(self, D, I):
        super().__init__()
        self.dense = nn.Linear(D, I)


class BertLayer(nn.Module):
    """Post-LN BERT layer (HF BertLayer as called by QVBertEncoder.forward, modeling_bert_new.py:600-608; in-repo copy
    with +-5e4 clamps: modeling/rpn/modeling_bert.py:39-270).  ``clamp`` > 0 applies the clamps."""

    def __init__(self, hidden, heads, intermediate, eps=1e-12, clamp=0.0):
        super().__init__()
        self.attention = _Attention(hidden, eps)
        self.intermediate = _Intermediate(hidden, intermediate)
        self.output = _SelfOutput(intermediate, hidden, eps)
        self.heads = heads
        self.clamp = clamp
        self._qkv = None

    def _qk16(self):
        sa = self.attention.self
        key = tuple((p.data_ptr(), p._version) for p in (sa.query.weight, sa.key.weight, sa.query.bias, sa.key.bias))
        if self._qkv is None or self._qkv[0] != key:
            w = ops.cast_f16(torch.cat([sa.query.weight, sa.key.weight], 0).detach().float().contiguous())
            b = torch.cat([sa.query.bias, sa.key.bias], 0).detach().float().contiguous()
            self._qkv = (key, w, b)
        return self._qkv[1], self._qkv[2]

    @torch.no_grad()
    def forward(self, h32, h16, colmask):
        """h32 fp32 [B,T,D] (+ its fp16 copy h16), colmask fp32 [B,T] (1 keep / 0 pad; or [B,T,T] per query) -> (fp32, fp16)
        outputs."""
        B, T, D = h32.shape
        H = self.heads
        d = D // H
        sa = self.attention.self
        w, b = self._qk16()
        qk = ops.gemm(h16.view(B * T, D), w, bias=b).view(B, T, 2, H, d)  # fused Q|K projection
        q, k = qk[:, :, 0], qk[:, :, 1]
        # V^T[b] = W_v . h[b]^T + b_v  -> [B, H, d, T]: P.V below is then K-major x K-major, no transpose kernel
        vT = ops.gemm(w16(sa.value.weight), h16, bias=f32(sa.value.bias), bias_mode=VEC_PER_ROW).view(B, H, d, T)
        ctx = torch.empty((B, T, H, d), dtype=torch.float16, device=h32.device)
        if colmask.dim() == 3:
            # per-query mask [B, T, T] (GroundingDINO's per-category block-diagonal text mask, bertwarper.py:271-320): scores laid
            # out [B, T, H, T] so that the H rows of one (image, query) are consecutive and share one mask row
            scores = torch.empty((B, T, H, T), dtype=torch.float32, device=h32.device)
            ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=scores.permute(0, 2, 1, 3), alpha=d ** -0.5, clamp=self.clamp)
            p = ops.softmax_rows(scores, colmask=colmask, rows_per_batch=H, mask_value=-10000.0)
            ops.gemm(p.permute(0, 2, 1, 3), vT, out=ctx.permute(0, 2, 1, 3))
        else:
            scores = torch.empty((B, H, T, T), dtype=torch.float32, device=h32.device)
            ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=scores, alpha=d ** -0.5, clamp=self.clamp)
            p = ops.softmax_rows(scores, colmask=colmask, rows_per_batch=H * T, mask_value=-10000.0)
            ops.gemm(p, vT, out=ctx.permute(0, 2, 1, 3))
        ao = self.attention.output
        # BertSelfOutput has no clamp_values (rpn/modeling_bert.py:186-190); only the attention scores, BertIntermediate
        # (before and after the GELU: same result as one clamp after it) and BertOutput are clamped (:140-143, 250-271)
        a = ops.gemm(ctx.view(B * T, D), w16(ao.dense.weight), bias=f32(ao.dense.bias), out_dtype=torch.float32)
        a16, a32 = ops.add_layernorm(a, h32.view(B * T, D), f32(ao.LayerNorm.weight), f32(ao.LayerNorm.bias),
                                     ao.LayerNorm.eps)
        it = ops.gemm(a16, w16(self.intermediate.dense.weight), bias=f32(self.intermediate.dense.bias), act=ACT_GELU,
                      clamp=self.clamp)
        o = ops.gemm(it, w16(self.output.dense.weight), bias=f32(self.output.dense.bias), out_dtype=torch.float32,
                     clamp=self.clamp)
        o16, o32 = ops.add_layernorm(o, a32, f32(self.output.LayerNorm.weight), f32(self.output.LayerNorm.bias),
                                     self.output.LayerNorm.eps, clamp=self.clamp)
        return o32.view(B, T, D), o16.view(B, T, D)


class QVBertEmbeddings(nn.Module):
    """modeling_bert_new.py:450-519 at eval: word + token_type(0) + absolute position embeddings, LayerNorm."""

    def __init__(self, config, cfg=None):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size, padding_idx=getattr(config, "pad_token_id", 0))
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=config.layer_norm_eps)
        self.cfg = cfg

    @torch.no_grad()
    def forward(self, input_ids, token_type_ids=None, position_ids=None):
        B, T = input_ids.shape
        # row gathers (index plumbing); the arithmetic (3-way add + LN) runs in add_layernorm
        w = self.word_embeddings.weight.detach()[input_ids].float().contiguous()
        pos = self.position_embeddings.weight.detach()[:T] if position_ids is None else \
            self.position_embeddings.weight.detach()[position_ids]
        tt = self.token_type_embeddings.weight.detach()[0] if token_type_ids is None else \
            self.token_type_embeddings.weight.detach()[token_type_ids]
        other = (pos + tt).float().expand(B, T, -1).contiguous()
        e16, e32 = ops.add_layernorm(w, other, f32(self.LayerNorm.weight), f32(self.LayerNorm.bias), self.LayerNorm.eps)
        return e32, e16


class ModelOutput(dict):
    """dict with attribute access, standing in for HF's BaseModelOutputWithPoolingAndCrossAttentions."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


class QVBertEncoder(nn.Module):
    """modeling_bert_new.py:522-639: GCP block i-start applied BEFORE BERT layer i for i >= start_qv_layer_index."""

    def __init__(self, config, dim, dim_head=64, heads=8, ff_mult=4, start_qv_layer_index=6, share_kv=False, cfg=None):
        super().__init__()
        self.start_qv_layer_index = start_qv_layer_index
        n = config.num_hidden_layers
        assert start_qv_layer_index < n
        self.layer = nn.ModuleList([BertLayer(config.hidden_size, config.num_attention_heads, config.intermediate_size,
                                              config.layer_norm_eps) for _ in range(n)])
        self.qv_layer = nn.ModuleList([GatedCrossAttentionBlock(dim=dim, dim_head=dim_head, heads=heads, ff_mult=ff_mult,
                                                                share_kv=share_kv, cfg=cfg)
                                       for _ in range(n - start_qv_layer_index)])

    @torch.no_grad()
    def forward_prefix(self, h32, h16, colmask, output_hidden_states=False):
        """BERT layers 0 .. start_qv_layer_index-1: they depend on the prompt only, not on the image, so the detector runs them
        on a second stream next to the visual backbone.  Returns the state ``forward(..., prefix=state)`` continues from."""
        all_h = () if output_hidden_states else None
        for i in range(self.start_qv_layer_index):
            if output_hidden_states:
                all_h = all_h + (h32,)
            h32, h16 = self.layer[i](h32, h16, colmask)
        return dict(h32=h32, h16=h16, all_h=all_h, next=self.start_qv_layer_index)

    @torch.no_grad()
    def forward(self, h32, h16, colmask, vision=None, vision_attention_mask=None, batched_pos_category_map=None,
                output_hidden_states=False, prefix=None):
        all_h = () if output_hidden_states else None
        first = 0
        if prefix is not None:
            h32, h16, first = prefix["h32"], prefix["h16"], prefix["next"]
            if output_hidden_states:
                all_h = prefix["all_h"]
        for i, layer in enumerate(self.layer):
            if i < first:
                continue
            if output_hidden_states:
                all_h = all_h + (h32,)
            if i >= self.start_qv_layer_index and exists(vision):
                h32 = self.qv_layer[i - self.start_qv_layer_index](h32, vision, vision_attention_mask,
                                                                   batched_pos_category_map)
                h16 = ops.cast_f16(h32)
            h32, h16 = layer(h32, h16, colmask)
        if output_hidden_states:
            all_h = all_h + (h32,)
        return h32, all_h


class QVBertModel(nn.Module):
    """modeling_bert_new.py:642-848 (inference).  ``config``: an HF-BertConfig-like object (hidden_size,
    num_hidden_layers, num_attention_heads, intermediate_size, vocab_size, max_position_embeddings, type_vocab_size,
    layer_norm_eps)."""

    def __init__(self, config, dim_t, dim_v, dim_head_t=64, dim_head_v=32, heads=8, ff_mult=4, num_pre_select_layers=2,
                 share_kv=False, cfg=None, **kwargs):
        super().__init__()
        self.config = config
        self.cfg = cfg
        self.embeddings = QVBertEmbeddings(config, cfg)
        self.encoder = QVBertEncoder(config=config, dim=dim_t, dim_head=dim_head_t, heads=heads, ff_mult=ff_mult,
                                     share_kv=share_kv, cfg=cfg)
        self.pre_select = PreSelectModule(dim=dim_v, out_dim=dim_t, dim_head=dim_head_v, heads=heads, ff_mult=ff_mult,
                                          num_layers=num_pre_select_layers, share_kv=share_kv, cfg=cfg)
        self.pooler = None  # add_pooling_layer=False at the only call site (bert_model_new.py:24)

    def get_gate_value(self):
        """modeling_bert_new.py:662-684 under CONDITION_GATE: ffn gates always, attn gates only when returned."""
        attn_gates, ff_gates = [], []
        for blk in self.encoder.qv_layer:
            if getattr(self.cfg.VISION_QUERY, "RETURN_ATTN_GATE_VALUE", False):
                attn_gates.append(blk.attn_gate_value)
            ff_gates.append(blk.ff_gate)
        return {"attn_gates": attn_gates, "ffn_gates": ff_gates}

    def prefix_weights_key(self):
        """(data_ptr, _version) of every parameter ``text_prefix`` reads: a cached prefix is valid while this is unchanged
        (``load_state_dict`` and in-place updates bump the versions)."""
        mods = [self.embeddings] + [self.encoder.layer[i] for i in range(self.encoder.start_qv_layer_index)]
        return tuple((p.data_ptr(), p._version) for m in mods for p in m.parameters())

    @torch.no_grad()
    def text_prefix(self, input_ids, attention_mask=None, token_type_ids=None, position_ids=None, output_hidden_states=True):
        """Embeddings + the BERT layers that precede the first GCP block (image-independent part of ``forward``)."""
        if input_ids is None or not input_ids.is_cuda:
            raise MqdetError("QVBertModel: CUDA input_ids required (no CPU fallback)")
        B, T = input_ids.shape
        if attention_mask is None:
            attention_mask = torch.ones((B, T), device=input_ids.device)
        colmask = attention_mask.float().contiguous()
        h32, h16 = self.embeddings(input_ids, token_type_ids, position_ids)
        st = self.encoder.forward_prefix(h32, h16, colmask, output_hidden_states=bool(output_hidden_states))
        st["colmask"] = colmask
        return st

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, token_type_ids=None, position_ids=None, head_mask=None,
                inputs_embeds=None, output_hidden_states=None, return_dict=True, vision=None, images=None,
                vision_attention_mask=None, batched_pos_category_map=None, text_prefix=None, **unused):
        if input_ids is None or not input_ids.is_cuda:
            raise MqdetError("QVBertModel: CUDA input_ids required (no CPU fallback)")
        B, T = input_ids.shape
        if attention_mask is None:
            attention_mask = torch.ones((B, T), device=input_ids.device)
        if text_prefix is not None:
            colmask, h32, h16 = text_prefix["colmask"], None, None
        else:
            colmask = attention_mask.float().contiguous()
            h32, h16 = self.embeddings(input_ids, token_type_ids, position_ids)
        augmented_vision = None
        if exists(images) and exists(vision):
            vision = self.pre_select(vision, images)["vision"]
            augmented_vision = vision
        h32, all_h = self.encoder(h32, h16, colmask, vision=vision, vision_attention_mask=vision_attention_mask,
                                  batched_pos_category_map=batched_pos_category_map,
                                  output_hidden_states=bool(output_hidden_states), prefix=text_prefix)
        out = ModelOutput(last_hidden_state=h32, pooler_output=None, hidden_states=all_h)
        out["vision_query_gates"] = self.get_gate_value()
        if getattr(self.cfg.VISION_QUERY, "QUERY_FUSION", False):
            out["augmented_vision"] = augmented_vision
            out["vision_attention_mask"] = vision_attention_mask
        return out
