"""Swin Transformer backbone on sm_90a kernels.

Drop-in for maskrcnn_benchmark/modeling/backbone/swint.py (``SwinTransformer`` :434-615, ``SwinTransformerBlock``
:145-242, ``WindowAttention`` :64-142, ``PatchMerging`` :245-284, ``PatchEmbed`` :393-431) with the reference's
parameter names, inference only.  Tokens are kept as [B, H*W, C] rows: residual stream fp32, GEMM operands fp16.
Window partition / cyclic shift / padding / region mask are index arithmetic inside the window-attention kernel.
"""
import torch
from torch import nn

from ... import ops
from ..._lib import ACT_GELU, MqdetError
from ...utils.weights import f32, w16


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.fc2 = nn.Linear(hidden_features, in_features)


class WindowAttention(nn.Module):
    def __init__(self, dim, window_size, num_heads):
        super().__init__()
        self.dim, self.window_size, self.num_heads = dim, window_size, num_heads
        self.scale = (dim // num_heads) ** -0.5
        ws = window_size
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws - 1) * (2 * ws - 1), num_heads))
        coords = torch.stack(torch.meshgrid([torch.arange(ws), torch.arange(ws)], indexing="ij"))
        cf = torch.flatten(coords, 1)
        rel = (cf[:, :, None] - cf[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += ws - 1
        rel[:, :, 1] += ws - 1
        rel[:, :, 0] *= 2 * ws - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.proj = nn.Linear(dim, dim)
        nn.init.trunc_normal_(self.relative_position_bias_table, std=.02)
        self._dense = None

    def dense_bias(self):
        """Relative position bias (swint.py:124-127) as the padded table ``mqdet_swin_window_attn`` reads: fp32 [heads, NP, NP],
        NP = N rounded up to 16, = log2(e) * bias inside [N, N] and -inf outside; cached per table version."""
        t = self.relative_position_bias_table
        key = (t.data_ptr(), t._version)
        if self._dense is None or self._dense[0] != key:
            N = self.window_size * self.window_size
            NP = (N + 15) // 16 * 16
            d = t.detach()[self.relative_position_index.view(-1)].view(N, N, -1).permute(2, 0, 1).float()
            pad = torch.full((d.shape[0], NP, NP), float("-inf"), dtype=torch.float32, device=d.device)
            pad[:, :N, :N] = d * 1.4426950408889634
            self._dense = (key, pad.contiguous())
        return self._dense[1]


class SwinTransformerBlock(nn.Module):
    # C = 96 / 192 (Swin-T stages 1-2, Swin-L stage 1): LN2 -> fc1 -> GELU -> fc2 -> residual in one kernel (ops.swin_mlp,
    # bit-identical); False keeps the three launches, for A/B runs
    fused_mlp = True

    def __init__(self, dim, num_heads, window_size=7, shift_size=0, mlp_ratio=4.):
        super().__init__()
        self.dim, self.num_heads, self.window_size, self.shift_size = dim, num_heads, window_size, shift_size
        self.norm1 = nn.LayerNorm(dim)
        self.attn = WindowAttention(dim, window_size, num_heads)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))
        self.H = self.W = None

    @torch.no_grad()
    def forward_flat(self, x32, B, H, W):
        """x32 fp32 [B*H*W, C] -> fp32 [B*H*W, C] (swint.py:186-242)."""
        a = self.attn
        xn = ops.layernorm(x32, f32(self.norm1.weight), f32(self.norm1.bias), self.norm1.eps)
        qkv = ops.gemm(xn, w16(a.qkv.weight), bias=f32(a.qkv.bias))
        o = ops.swin_window_attn(qkv, f32(a.qkv.bias), a.dense_bias(), B, H, W, self.num_heads, self.window_size,
                                 self.shift_size, a.scale)
        x32 = ops.gemm(o, w16(a.proj.weight), bias=f32(a.proj.bias), out_dtype=torch.float32, residual=x32)
        if self.fused_mlp and self.dim in (96, 192) and self.mlp.fc1.out_features == 4 * self.dim:
            return ops.swin_mlp(x32, f32(self.norm2.weight), f32(self.norm2.bias), self.norm2.eps, w16(self.mlp.fc1.weight),
                                f32(self.mlp.fc1.bias), w16(self.mlp.fc2.weight), f32(self.mlp.fc2.bias))
        xn = ops.layernorm(x32, f32(self.norm2.weight), f32(self.norm2.bias), self.norm2.eps)
        h = ops.gemm(xn, w16(self.mlp.fc1.weight), bias=f32(self.mlp.fc1.bias), act=ACT_GELU)
        return ops.gemm(h, w16(self.mlp.fc2.weight), bias=f32(self.mlp.fc2.bias), out_dtype=torch.float32, residual=x32)

    def forward(self, x, mask_matrix=None):
        """Reference signature: x [B, H*W, C] with self.H / self.W set by the caller; the mask is recomputed in-kernel."""
        if not x.is_cuda:
            raise MqdetError("SwinTransformerBlock: CUDA tensors required (no CPU fallback)")
        B, L, C = x.shape
        return self.forward_flat(x.float().contiguous().view(B * L, C), B, self.H, self.W).view(B, L, C)


class PatchMerging(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.dim = dim
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = nn.LayerNorm(4 * dim)

    @torch.no_grad()
    def forward_flat(self, x32, B, H, W):
        xn, H2, W2 = ops.patch_merge_ln(x32, B, H, W, f32(self.norm.weight), f32(self.norm.bias), self.norm.eps)
        return ops.gemm(xn, w16(self.reduction.weight), out_dtype=torch.float32), H2, W2


class BasicLayer(nn.Module):
    def __init__(self, dim, depth, num_heads, window_size=7, mlp_ratio=4., downsample=True):
        super().__init__()
        self.window_size, self.shift_size, self.depth = window_size, window_size // 2, depth
        self.blocks = nn.ModuleList([SwinTransformerBlock(dim, num_heads, window_size,
                                                          0 if (i % 2 == 0) else window_size // 2, mlp_ratio)
                                     for i in range(depth)])
        self.downsample = PatchMerging(dim) if downsample else None


class PatchEmbed(nn.Module):
    def __init__(self, patch_size=4, in_chans=3, embed_dim=96):
        super().__init__()
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm = nn.LayerNorm(embed_dim)


class SwinTransformer(nn.Module):
    """swint.py:434-615 with ape=False, patch_norm=True, out_features stage2..stage5."""

    def __init__(self, embed_dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24), window_size=7, mlp_ratio=4.,
                 out_features=("stage2", "stage3", "stage4", "stage5")):
        super().__init__()
        if window_size not in (7, 12) or any((embed_dim * 2 ** i) // h != 32 for i, h in enumerate(num_heads)):
            raise NotImplementedError("window 7 (Swin-T, MQ-GLIP-T) or 12 (Swin-L, MQ-GLIP-L) with head_dim 32 only")
        self.num_layers = len(depths)
        self.embed_dim = embed_dim
        self.out_features = out_features
        self.patch_embed = PatchEmbed(4, 3, embed_dim)
        self.layers = nn.ModuleList([BasicLayer(int(embed_dim * 2 ** i), depths[i], num_heads[i], window_size, mlp_ratio,
                                                downsample=(i < self.num_layers - 1)) for i in range(self.num_layers)])
        self.num_features = [int(embed_dim * 2 ** i) for i in range(self.num_layers)]
        for i in range(self.num_layers):
            if f"stage{i + 2}" in out_features:
                # norm0 is nn.Identity for *-RETINANET backbones (swint.py:547-548)
                self.add_module(f"norm{i}", nn.Identity() if i == 0 else nn.LayerNorm(self.num_features[i]))

    @torch.no_grad()
    def forward_flat(self, img, want=(1, 2, 3)):
        """img [B,3,H,W] fp32 -> {stage index: (tokens fp16 [B, h*w, C], h, w)} for the stages FPN consumes."""
        if not img.is_cuda:
            raise MqdetError("SwinTransformer: CUDA tensors required (no CPU fallback)")
        B = img.shape[0]
        pe = self.patch_embed
        patches, H, W = ops.patchify4(img)
        x16 = ops.gemm(patches, w16(pe.proj.weight, view=(self.embed_dim, -1)), bias=f32(pe.proj.bias))
        x32 = ops.layernorm(x16, f32(pe.norm.weight), f32(pe.norm.bias), pe.norm.eps, out16=False, out32=True)
        outs = {}
        for i, layer in enumerate(self.layers):
            for blk in layer.blocks:
                x32 = blk.forward_flat(x32, B, H, W)
            if i in want and f"stage{i + 2}" in self.out_features:
                n = getattr(self, f"norm{i}")
                t16 = ops.cast_f16(x32) if isinstance(n, nn.Identity) else ops.layernorm(x32, f32(n.weight), f32(n.bias), n.eps)
                outs[i] = (t16.view(B, H * W, -1), H, W)
            if layer.downsample is not None:
                x32, H, W = layer.downsample.forward_flat(x32, B, H, W)
        return outs

    def forward(self, x):
        """Reference signature: returns the list of [B, C, H, W] fp32 stage outputs (all out_features)."""
        outs = self.forward_flat(x, want=tuple(range(self.num_layers)))
        res = []
        for i in sorted(outs):
            t, h, w = outs[i]
            res.append(ops.cast_f32(t).transpose(1, 2).reshape(t.shape[0], -1, h, w).contiguous())
        return res
