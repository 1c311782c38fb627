"""GroundingDINO pieces on the MQ-Det hot path (SURVEY.md §8 a18).

Drop-in for ``groundingdino_new/models/GroundingDINO/utils.py:233-268`` (``ContrastiveEmbed``): the query x token
similarity that scores the 900 decoder queries of every decoder layer and the encoder memory tokens of the two-stage
proposal selection (``transformer.py:288-303``), plus the small helpers of the encoder / decoder assembly (``MLP`` :171-185,
``get_sine_pos_embed`` :24-56, ``gen_encoder_output_proposals`` :59-118).
"""
import math

import torch
from torch import nn

from ... import ops
from ..._lib import ACT_RELU, MqdetError
from ...utils.weights import f32, w16


class MLP(nn.Module):
    """utils.py:171-185 — Linear + relu ... Linear; parameter names ``layers.N``.  Every layer is one wgmma GEMM with the bias /
    relu (and, on the last layer, an optional residual) in the epilogue."""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))

    @torch.no_grad()
    def forward(self, x, out_dtype=torch.float32, residual=None):
        """x [..., input_dim] (fp16, or fp32 which is cast) -> [..., output_dim] in ``out_dtype`` (+ residual fp32)."""
        if not x.is_cuda:
            raise MqdetError("MLP: CUDA tensors required (no CPU fallback)")
        lead = x.shape[:-1]
        x = x.reshape(-1, x.shape[-1])
        x = x if x.dtype == torch.float16 else ops.cast_f16(x.float().contiguous())
        for i, layer in enumerate(self.layers):
            last = i == self.num_layers - 1
            x = ops.gemm(x, w16(layer.weight), bias=f32(layer.bias), act=0 if last else ACT_RELU,
                         out_dtype=out_dtype if last else torch.float16, residual=residual if last else None)
        return x.view(*lead, -1)


def get_sine_pos_embed(pos_tensor, num_pos_feats=128, temperature=10000, exchange_xy=True):
    """utils.py:24-56: pos_tensor [B, n, k] -> [B, n, k * num_pos_feats].  Prompt geometry (the text position ids), computed once
    per prompt by ``Transformer.prepare``."""
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=pos_tensor.device)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    res = []
    for x in pos_tensor.split([1] * pos_tensor.shape[-1], dim=-1):
        s = x * (2 * math.pi) / dim_t
        res.append(torch.stack((s[..., 0::2].sin(), s[..., 1::2].cos()), dim=3).flatten(2))
    if exchange_xy:
        res[0], res[1] = res[1], res[0]
    return torch.cat(res, dim=-1)


def gen_encoder_output_proposals(memory_padding_mask, spatial_shapes):
    """The geometry half of utils.py:59-118 (learnedwh=None): memory_padding_mask bool [B, sum(hw)] (True = padding) ->
    (valid bool [B, sum(hw)], output_proposals fp32 [B, sum(hw), 4] un-sigmoided, +inf on padded / invalid positions).  The memory
    half (``output_memory`` = memory zeroed where padded or invalid) is ``mqdet_add_cast`` with ``valid & ~mask`` as the row gate."""
    N_ = memory_padding_mask.shape[0]
    dev = memory_padding_mask.device
    proposals, cur = [], 0
    for lvl, (H_, W_) in enumerate(spatial_shapes):
        m = memory_padding_mask[:, cur:cur + H_ * W_].view(N_, H_, W_, 1)
        valid_H = torch.sum(~m[:, :, 0, 0], 1)
        valid_W = torch.sum(~m[:, 0, :, 0], 1)
        gy, gx = torch.meshgrid(torch.linspace(0, H_ - 1, H_, dtype=torch.float32, device=dev),
                                torch.linspace(0, W_ - 1, W_, dtype=torch.float32, device=dev), indexing="ij")
        grid = torch.cat([gx.unsqueeze(-1), gy.unsqueeze(-1)], -1)
        scale = torch.cat([valid_W.unsqueeze(-1), valid_H.unsqueeze(-1)], 1).view(N_, 1, 1, 2)
        grid = (grid.unsqueeze(0).expand(N_, -1, -1, -1) + 0.5) / scale
        wh = torch.ones_like(grid) * 0.05 * (2.0 ** lvl)
        proposals.append(torch.cat((grid, wh), -1).view(N_, -1, 4))
        cur += H_ * W_
    prop = torch.cat(proposals, 1)
    valid = ((prop > 0.01) & (prop < 0.99)).all(-1)
    prop = torch.log(prop / (1 - prop))
    prop = prop.masked_fill(memory_padding_mask.unsqueeze(-1), float("inf")).masked_fill(~valid.unsqueeze(-1), float("inf"))
    return valid, prop


class ContrastiveEmbed(nn.Module):
    def __init__(self, max_text_len=256):
        super().__init__()
        self.max_text_len = max_text_len

    @torch.no_grad()
    def forward(self, x, text_dict):
        """x [bs, nq, d_model]; text_dict = {'encoded_text': [bs, T, d_model], 'text_token_mask': [bs, T] bool (True =
        token in use)} -> [bs, nq, max_text_len] fp32, -inf on padding and beyond T.  One wgmma product (fp16 operands,
        fp32 accumulate/output) + the in-place mask/pad kernel."""
        assert isinstance(text_dict, dict)
        y = text_dict["encoded_text"]
        mask = text_dict["text_token_mask"]
        if not x.is_cuda:
            raise MqdetError("ContrastiveEmbed: CUDA tensors required (no CPU fallback)")
        lead = x.shape[:-2]
        x3 = x.reshape(-1, x.shape[-2], x.shape[-1])
        if y.shape[-1] % 8:
            raise MqdetError("ContrastiveEmbed: d_model must be a multiple of 8")
        x16 = x3.contiguous() if x3.dtype == torch.float16 else ops.cast_f16(x3.float().contiguous())
        y16 = text_dict.get("encoded_text16")  # optional fp16 copy of encoded_text (the assembly keeps one)
        if y16 is None:
            y16 = y.contiguous() if y.dtype == torch.float16 else ops.cast_f16(y.float().contiguous())
        out = ops.contrastive_embed(x16, y16, mask, self.max_text_len)
        return out.reshape(*lead, x.shape[-2], self.max_text_len)
