"""Multi-scale deformable attention of the GroundingDINO encoder / decoder on sm_90a kernels.

Drop-in for groundingdino_new/models/GroundingDINO/ms_deform_attn.py:136-352 (``MultiScaleDeformableAttention``): same
constructor arguments, parameter names (``sampling_offsets``, ``attention_weights``, ``value_proj``, ``output_proj``) and forward
signature, inference only.  Two GEMMs (value projection with the padding mask as a per-row gate; sampling offsets and attention
logits as ONE product over the concatenated weights), one fused kernel (softmax over the L*P logits, sampling locations,
bilinear gathers, weighted sum — ``mqdet_ms_deform_attn``) and the output projection.
"""
import math

import torch
from torch import nn

from ... import ops
from ..._lib import VEC_PER_ROW, MqdetError
from ...utils.weights import f32, w16


class MultiScaleDeformableAttention(nn.Module):
    def __init__(self, embed_dim=256, num_heads=8, num_levels=4, num_points=4, img2col_step=64, batch_first=False):
        super().__init__()
        if embed_dim % num_heads != 0:
            raise ValueError("embed_dim must be divisible by num_heads, but got {} and {}".format(embed_dim, num_heads))
        self.batch_first = batch_first
        self.im2col_step = img2col_step
        self.embed_dim, self.num_heads, self.num_levels, self.num_points = embed_dim, num_heads, num_levels, num_points
        self.sampling_offsets = nn.Linear(embed_dim, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dim, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dim, embed_dim)
        self.output_proj = nn.Linear(embed_dim, embed_dim)
        self._cat = None
        self.init_weights()

    def init_weights(self):
        """ms_deform_attn.py:196-220."""
        nn.init.constant_(self.sampling_offsets.weight.data, 0.0)
        thetas = torch.arange(self.num_heads, dtype=torch.float32) * (2.0 * math.pi / self.num_heads)
        grid = torch.stack([thetas.cos(), thetas.sin()], -1)
        grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(self.num_heads, 1, 1, 2).repeat(1, self.num_levels, self.num_points, 1)
        for i in range(self.num_points):
            grid[:, :, i, :] *= i + 1
        with torch.no_grad():
            self.sampling_offsets.bias = nn.Parameter(grid.view(-1))
        nn.init.constant_(self.attention_weights.weight.data, 0.0)
        nn.init.constant_(self.attention_weights.bias.data, 0.0)
        nn.init.xavier_uniform_(self.value_proj.weight.data)
        nn.init.constant_(self.value_proj.bias.data, 0.0)
        nn.init.xavier_uniform_(self.output_proj.weight.data)
        nn.init.constant_(self.output_proj.bias.data, 0.0)

    def _offsets_and_logits_weights(self):
        ps = (self.sampling_offsets.weight, self.attention_weights.weight, self.sampling_offsets.bias, self.attention_weights.bias)
        key = tuple((p.data_ptr(), p._version) for p in ps)
        if self._cat is None or self._cat[0] != key:
            w = ops.cast_f16(torch.cat([ps[0], ps[1]], 0).detach().float().contiguous())
            b = torch.cat([ps[2], ps[3]], 0).detach().float().contiguous()
            self._cat = (key, w, b)
        return self._cat[1], self._cat[2]

    @torch.no_grad()
    def forward(self, query, key=None, value=None, query_pos=None, key_padding_mask=None, reference_points=None,
                spatial_shapes=None, level_start_index=None, **kwargs):
        if not query.is_cuda:
            raise MqdetError("MultiScaleDeformableAttention: CUDA tensors required (no CPU fallback)")
        if value is None:
            value = query
        if query_pos is not None:
            query = query + query_pos
        if not self.batch_first:
            query, value = query.permute(1, 0, 2), value.permute(1, 0, 2)
        keep = None
        if key_padding_mask is not None:   # value.masked_fill(mask, 0) as a per-row gate of the projection (:282-283)
            keep = (~key_padding_mask.bool()).reshape(-1).float().contiguous()
        out = self.core(ops.cast_f16(query.contiguous()), ops.cast_f16(value.contiguous()), keep, reference_points, spatial_shapes)
        return out if self.batch_first else out.permute(1, 0, 2)

    @torch.no_grad()
    def core(self, q16, v16_in, keep, reference_points, spatial_shapes, residual=None):
        """Batch-first fp16 operands: q16 [bs, nq, E] (query + query_pos already added), v16_in [bs, nv, E] (un-projected value),
        keep fp32 [bs*nv] (1 = valid, 0 = padding) or None -> fp32 [bs, nq, E] (+ ``residual`` fp32 when given)."""
        bs, nq, E = q16.shape
        nv = v16_in.shape[1]
        sizes = [(int(h), int(w)) for h, w in (spatial_shapes.tolist() if torch.is_tensor(spatial_shapes) else spatial_shapes)]
        assert sum(h * w for h, w in sizes) == nv
        levels = ops.get_levels(sizes, q16.device)
        H, L, P = self.num_heads, self.num_levels, self.num_points
        v16 = ops.gemm(v16_in.view(bs * nv, E), w16(self.value_proj.weight), bias=f32(self.value_proj.bias),
                       gate=keep, gate_mode=VEC_PER_ROW if keep is not None else 0).view(bs, nv, E)
        wc, bc = self._offsets_and_logits_weights()
        proj = ops.gemm(q16.view(bs * nq, E), wc, bias=bc, out_dtype=torch.float32)  # [bs*nq, H*L*P*3]
        out16 = ops.ms_deform_attn(v16, proj, H * L * P * 2, reference_points.float().contiguous(), levels, H, P)
        out = ops.gemm(out16.view(bs * nq, E), w16(self.output_proj.weight), bias=f32(self.output_proj.bias),
                       out_dtype=torch.float32, residual=None if residual is None else residual.view(bs * nq, E))
        return out.view(bs, nq, E)
