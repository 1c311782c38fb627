"""GroundingDINO's vision-language fusion block, drop-in for groundingdino_new/models/GroundingDINO/fuse_modules.py:99-297
(``BiMultiHeadAttention`` / ``BiAttentionBlock``: v_dim = l_dim = 256, embed 1024, 4 heads of 256 in the MQ-GroundingDINO-T
encoder, transformer.py:171-180).

Same parameters (``state_dict`` keys) and arithmetic as the reference; it differs from the GLIP block (utils/fuse_helper.py) in
three places, all handled by the shared implementation:
  * ``stable_softmax_2d = True``: the GLOBAL maximum of the score tensor is subtracted before the +-5e4 clamps (:177-187) —
    ``mqdet_global_max_f32`` + ``mqdet_shift_clamp_f32`` on the fp32 scores, the maximum never leaves the device; batched prompt
    chunks (``GroundingDINO.forward_chunked_device``) take one maximum per batch element, since the reference sees one chunk per
    forward;
  * masks are boolean with True = padding and are filled with -inf (:201-214), for the text tokens AND for the image tokens;
  * the block takes / returns flat ``[B, N, C]`` tensors (no FPN-level lists).
The scores are materialised in fp32 here (the global maximum is needed before either softmax), i.e. this is the explicit path,
not the fused wgmma attention kernels of the GLIP tower.
"""
import torch
from torch import nn

from ... import ops
from ..._lib import MqdetError
from ...utils import fuse_helper
from ...utils.weights import f32


class BiMultiHeadAttention(fuse_helper.BiMultiHeadAttention):
    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, cfg=None):
        super().__init__(v_dim, l_dim, embed_dim, num_heads, dropout=dropout, cfg=None, stable_softmax_2d=True,
                         clamp_min_for_underflow=True, clamp_max_for_overflow=True, mask_fill=(float("-inf"), 0.0))

    @staticmethod
    def _keep(mask):
        """bool [B, n] with True = padding -> fp32 1 keep / 0 padding (None stays None)."""
        return None if mask is None else (~mask.bool()).float().contiguous()

    @torch.no_grad()
    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None):
        """Reference signature (:147): v [B,N,v_dim], l [B,T,l_dim] (both already layer-normed by the block) ->
        (attn_output_v [B,N,v_dim], attn_output_l [B,T,l_dim]) fp32."""
        if not v.is_cuda:
            raise MqdetError("BiMultiHeadAttention: CUDA tensors required (no CPU fallback)")
        dv, dl = self._attend(ops.cast_f16(v.float().contiguous()), ops.cast_f16(l.float().contiguous()),
                              self._keep(attention_mask_l), mask_v=self._keep(attention_mask_v))
        return ops.cast_f32(dv), dl


class BiAttentionBlock(nn.Module):
    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, drop_path=0.0, init_values=1e-4, cfg=None):
        super().__init__()
        self.layer_norm_v = nn.LayerNorm(v_dim)
        self.layer_norm_l = nn.LayerNorm(l_dim)
        self.attn = BiMultiHeadAttention(v_dim=v_dim, l_dim=l_dim, embed_dim=embed_dim, num_heads=num_heads, dropout=dropout)
        self.drop_path = nn.Identity()  # eval
        self.gamma_v = nn.Parameter(init_values * torch.ones((v_dim)), requires_grad=True)
        self.gamma_l = nn.Parameter(init_values * torch.ones((l_dim)), requires_grad=True)

    @torch.no_grad()
    def forward(self, v, l, attention_mask_v=None, attention_mask_l=None, keep_v=None, keep_l=None, per_element_max=False):
        """v [B,N,v_dim], l [B,T,l_dim] fp32 -> (v', l') fp32:  x' = LN(x) + gamma * delta  (residual on the NORMALISED inputs,
        :286-296).  ``keep_v`` / ``keep_l``: the masks already as fp32 1 keep / 0 padding (the assembly builds them once).
        ``per_element_max``: the stable-softmax maximum of each batch element alone (batched prompt chunks)."""
        if not v.is_cuda:
            raise MqdetError("BiAttentionBlock: CUDA tensors required (no CPU fallback)")
        nv, nl = self.layer_norm_v, self.layer_norm_l
        vn16, vn32 = ops.layernorm(v.float().contiguous(), f32(nv.weight), f32(nv.bias), nv.eps, out16=True, out32=True)
        ln16, ln32 = ops.layernorm(l.float().contiguous(), f32(nl.weight), f32(nl.bias), nl.eps, out16=True, out32=True)
        a = self.attn
        keep_l = a._keep(attention_mask_l) if keep_l is None else keep_l
        keep_v = a._keep(attention_mask_v) if keep_v is None else keep_v
        dv, dl = a._attend(vn16, ln16, keep_l, mask_v=keep_v, per_element_max=per_element_max,
                           v_epilogue=dict(gate=f32(self.gamma_v), residual=vn32, out_dtype=torch.float32),
                           l_epilogue=dict(gate=f32(self.gamma_l), residual=ln32))
        return dv, dl
