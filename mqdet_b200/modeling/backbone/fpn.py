"""FPN (P3-P5 + conv P6/P7) on sm_90a kernels.

Drop-in for maskrcnn_benchmark/modeling/backbone/fpn.py (``FPN`` :6-129 in the SWINT-FPN-RETINANET configuration of
modeling/backbone/__init__.py:37-80: in_channels_list [0, C3, C4, C5], plain convs with bias, ``LastLevelP6P7``
:137-154 fed by P5) with the reference's parameter names (``fpn_inner{2,3,4}``, ``fpn_layer{2,3,4}``, ``top_blocks.p6/p7``).
The pyramid is written directly into the concatenated fp16 tensor [B, N, 256] the head consumes.
"""
import torch
from torch import nn

from ... import ops
from ..._lib import MqdetError
from ...utils.weights import f32, w16
from ..rpn.vldyhead import _conv_w16


class LastLevelP6P7(nn.Module):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.p6 = nn.Conv2d(in_channels, out_channels, 3, 2, 1)
        self.p7 = nn.Conv2d(out_channels, out_channels, 3, 2, 1)
        for m in (self.p6, self.p7):
            nn.init.kaiming_uniform_(m.weight, a=1)
            nn.init.constant_(m.bias, 0)
        self.use_P5 = in_channels == out_channels


class FPN(nn.Module):
    def __init__(self, in_channels_list, out_channels, top_blocks=None):
        super().__init__()
        self.inner_blocks, self.layer_blocks = [], []
        for idx, c in enumerate(in_channels_list, 1):
            if c == 0:
                continue
            inner, layer = f"fpn_inner{idx}", f"fpn_layer{idx}"
            self.add_module(inner, nn.Conv2d(c, out_channels, 1))
            self.add_module(layer, nn.Conv2d(out_channels, out_channels, 3, 1, 1))
            for m in (getattr(self, inner), getattr(self, layer)):
                nn.init.kaiming_uniform_(m.weight, a=1)
                nn.init.constant_(m.bias, 0)
            self.inner_blocks.append(inner)
            self.layer_blocks.append(layer)
        self.top_blocks = top_blocks
        self.out_channels = out_channels
        if not (isinstance(top_blocks, LastLevelP6P7) and top_blocks.use_P5):
            raise NotImplementedError("only the RetinaNet-style top block fed by P5 (MQ-GLIP configs)")

    @torch.no_grad()
    def forward_flat(self, feats):
        """feats: list of (tokens fp16 [B, h*w, C_i], h, w) for C3, C4, C5 -> (pyramid fp16 [B, N, 256], Levels)."""
        B = feats[0][0].shape[0]
        dev = feats[0][0].device
        C = self.out_channels
        sizes = [(h, w) for _, h, w in feats]
        h5, w5 = sizes[-1]
        h6, w6 = (h5 + 2 - 3) // 2 + 1, (w5 + 2 - 3) // 2 + 1
        h7, w7 = (h6 + 2 - 3) // 2 + 1, (w6 + 2 - 3) // 2 + 1
        levels = ops.get_levels(sizes + [(h6, w6), (h7, w7)], dev)
        pyr = torch.empty((B, levels.N, C), dtype=torch.float16, device=dev)

        def conv1x1(name, t):
            m = getattr(self, name)
            return ops.gemm(t.reshape(-1, t.shape[-1]), w16(m.weight, view=(C, -1)), bias=f32(m.bias)).view(B, -1, C)

        def conv3x3(m, t, h, w, out_view, stride=1, relu_in=False):
            cols, ho, wo = ops.im2col3x3(t, B, h, w, stride, relu_in)
            ops.gemm(cols.view(B, ho * wo, -1), _conv_w16(m.weight), out=out_view, bias=f32(m.bias))
            return ho, wo

        # top-down pathway (fpn.py:78-102)
        n = len(feats)
        last = conv1x1(self.inner_blocks[-1], feats[-1][0])
        conv3x3(getattr(self, self.layer_blocks[-1]), last, *sizes[-1], pyr[:, levels.off[n - 1]:levels.off[n]])
        for i in range(n - 2, -1, -1):
            lat = conv1x1(self.inner_blocks[i], feats[i][0])
            last = ops.upsample_add(lat, last, B, sizes[i][0], sizes[i][1], sizes[i + 1][0], sizes[i + 1][1])
            conv3x3(getattr(self, self.layer_blocks[i]), last, *sizes[i], pyr[:, levels.off[i]:levels.off[i + 1]])
        # P6 = conv(P5), P7 = conv(relu(P6))   (fpn.py:137-154)
        p5 = pyr[:, levels.off[n - 1]:levels.off[n]]
        conv3x3(self.top_blocks.p6, p5, h5, w5, pyr[:, levels.off[n]:levels.off[n + 1]], stride=2)
        p6 = pyr[:, levels.off[n]:levels.off[n + 1]]
        conv3x3(self.top_blocks.p7, p6, h6, w6, pyr[:, levels.off[n + 1]:levels.off[n + 2]], stride=2, relu_in=True)
        return pyr, levels

    def forward(self, x):
        """Reference signature: list of [B, C_i, H_i, W_i] maps (4 stages; the first is ignored) -> tuple of 5 maps."""
        if not x[-1].is_cuda:
            raise MqdetError("FPN: CUDA tensors required (no CPU fallback)")
        use = x[-len(self.inner_blocks):]
        feats = [(ops.cast_f16(f.flatten(2).transpose(1, 2).contiguous()), f.shape[2], f.shape[3]) for f in use]
        pyr, levels = self.forward_flat(feats)
        p32 = ops.cast_f32(pyr)
        B = p32.shape[0]
        return tuple(p32[:, levels.off[l]:levels.off[l + 1]].transpose(1, 2).reshape(B, -1, h, w).contiguous()
                     for l, (h, w) in enumerate(levels.sizes))
