"""Training forward / backward of PreSelect (modeling_bert_new.py:377-448) on sm_90a kernels — with the GCP blocks the only trainable
parameters of the modulated pre-training (``'pre_select' in key``: tools/train_net.py:70-77, solver/build.py:46-49).

    PreSelectTrain(module).forward(vision, image)   -> vision' fp32 [B,V,out_dim]  (the input of every GCP block)
    PreSelectTrain(module).backward(dvision')       -> {parameter name: fp32 gradient} (names as in module.state_dict())

The training forward materialises the attention probabilities (the inference path's flash-style ``mqdet_dense_cross_attn`` keeps none);
the image tokens come from the frozen FPN, so no gradient flows into them.  As in gcp_backward.py every dX = dY W / dW = dY^T X /
attention-backward product is a wgmma GEMM and the K-major operands come from ``mqdet_transpose_cast(_batched)``.
"""
import torch
from torch import nn

from ... import ops
from ..._lib import ACT_GELU, MqdetError
from ...utils.weights import f32, w16
from .gcp_backward import _wT16
from .modeling_bert_new import _ln16


class _BlockTrain:
    def __init__(self, blk):
        self.blk = blk
        self.c = None

    def forward(self, v32, img32, cn16):
        blk, a = self.blk, self.blk.image_condition
        B, V, Din = v32.shape
        I = img32.shape[1]
        H, d, inner = a.heads, a.dim_head, a.inner_dim
        Ip = (I + 7) // 8 * 8
        dev = v32.device
        v16 = ops.cast_f16(v32)
        lin = isinstance(blk.res_mapping, nn.Linear)
        res = ops.gemm(v16.view(B * V, Din), w16(blk.res_mapping.weight), out_dtype=torch.float32) if lin else v32.view(B * V, Din)
        xn = _ln16(v32, a.norm)
        if cn16 is None:
            cn16 = _ln16(img32, a.norm_kv)
        q = ops.gemm(xn.view(B * V, Din), w16(a.to_q.weight), alpha=a.scale).view(B, V, H, d)
        kv = ops.gemm(cn16.view(B * I, -1), w16(a.to_kv.weight)).view(B, I, 2, H, d)
        k, v = kv[:, :, 0], kv[:, :, 1]
        scores = torch.zeros((B, H, V, Ip), dtype=torch.float32, device=dev)
        ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=scores[..., :I])
        p = ops.softmax_rows(scores, n=I)
        del scores
        vT = ops.transpose_cast_batched(v.permute(0, 2, 1, 3))                      # [B,H,d,Ip]
        o = torch.empty((B, V, H, d), dtype=torch.float16, device=dev)
        ops.gemm(p, vT, out=o.permute(0, 2, 1, 3))
        v1 = ops.gemm(o.view(B * V, inner), w16(a.to_out.weight), out_dtype=torch.float32, residual=res)
        vn = _ln16(v1, blk.ff.norm)
        h = ops.gemm(vn, w16(blk.ff.linear1.weight), act=ACT_GELU)
        v2 = ops.gemm(h, w16(blk.ff.linear2.weight), out_dtype=torch.float32, residual=v1)
        self.c = dict(B=B, V=V, I=I, Ip=Ip, Din=Din, v32=v32.contiguous().view(B * V, Din), v16=v16.view(B * V, Din), img32=img32,
                      xn=xn.view(B * V, Din), cn=cn16.view(B * I, -1), q=q, k=k, v=v, p=p, o=o.view(B * V, inner), v1=v1, vn=vn, h=h, lin=lin)
        return v2.view(B, V, -1)

    def backward(self, dv2):
        c, blk, a = self.c, self.blk, self.blk.image_condition
        B, V, I, Ip, Din = c["B"], c["V"], c["I"], c["Ip"], c["Din"]
        H, d, inner = a.heads, a.dim_head, a.inner_dim
        dev = dv2.device
        tr, trb = ops.transpose_cast, ops.transpose_cast_batched
        g = {}
        dv2 = dv2.float().contiguous().view(B * V, -1)
        ff = blk.ff
        # ---- v2 = v1 + FF(v1)
        dv2_16 = ops.cast_f16(dv2)
        g["ff.linear2.weight"] = ops.gemm(tr(dv2_16), tr(c["h"]), out_dtype=torch.float32)
        dh = ops.gemm(dv2_16, _wT16(ff.linear2.weight))
        z = ops.gemm(c["vn"], w16(ff.linear1.weight))
        dz = ops.gelu_bwd(z, dh)
        g["ff.linear1.weight"] = ops.gemm(tr(dz), tr(c["vn"]), out_dtype=torch.float32)
        dvn = ops.gemm(dz, _wT16(ff.linear1.weight), out_dtype=torch.float32)
        dv1 = dv2.clone()
        _, g["ff.norm.weight"], g["ff.norm.bias"] = ops.layernorm_bwd(dvn, c["v1"], f32(ff.norm.weight), ff.norm.eps, dx=dv1)
        # ---- v1 = o Wout^T + res_mapping(v)
        dv1_16 = ops.cast_f16(dv1)
        g["image_condition.to_out.weight"] = ops.gemm(tr(dv1_16), tr(c["o"]), out_dtype=torch.float32)
        do = ops.gemm(dv1_16, _wT16(a.to_out.weight)).view(B, V, H, d)
        if c["lin"]:
            g["res_mapping.weight"] = ops.gemm(tr(dv1_16), tr(c["v16"]), out_dtype=torch.float32)
            dvin = ops.gemm(dv1_16, _wT16(blk.res_mapping.weight), out_dtype=torch.float32)
        else:
            dvin = dv1.clone()
        # ---- dense cross-attention over the I image tokens
        dp = torch.zeros((B, H, V, Ip), dtype=torch.float32, device=dev)
        ops.gemm(do.permute(0, 2, 1, 3), c["v"].permute(0, 2, 1, 3), out=dp[..., :I])
        ds = ops.softmax_bwd_rows(c["p"], dp)                                            # [B,H,V,Ip], padding columns 0
        del dp
        dq = torch.empty((B, V, H, d), dtype=torch.float16, device=dev)
        # q is stored pre-scaled (scores = q . k), so dq = dS K and dk = dS^T q carry no extra factor; the scale returns in dWq / dxn
        ops.gemm(ds, trb(c["k"].permute(0, 2, 1, 3)), out=dq.permute(0, 2, 1, 3))
        dkv = torch.empty((B, I, 2, H, d), dtype=torch.float16, device=dev)
        ops.gemm(trb(ds)[:, :, :I], trb(c["q"].permute(0, 2, 1, 3)), out=dkv[:, :, 0].permute(0, 2, 1, 3))
        ops.gemm(trb(c["p"])[:, :, :I], trb(do.permute(0, 2, 1, 3)), out=dkv[:, :, 1].permute(0, 2, 1, 3))
        # ---- projections and the two LayerNorms
        dq2 = dq.view(B * V, inner)
        g["image_condition.to_q.weight"] = ops.gemm(tr(dq2), tr(c["xn"]), out_dtype=torch.float32, alpha=a.scale)
        dxn = ops.gemm(dq2, _wT16(a.to_q.weight), out_dtype=torch.float32, alpha=a.scale)
        _, g["image_condition.norm.weight"], g["image_condition.norm.bias"] = ops.layernorm_bwd(dxn, c["v32"], f32(a.norm.weight), a.norm.eps,
                                                                                              dx=dvin)
        dkv2 = dkv.view(B * I, 2 * inner)
        g["image_condition.to_kv.weight"] = ops.gemm(tr(dkv2), tr(c["cn"]), out_dtype=torch.float32)
        dcn = ops.gemm(dkv2, _wT16(a.to_kv.weight), out_dtype=torch.float32)
        _, g["image_condition.norm_kv.weight"], g["image_condition.norm_kv.bias"] = ops.layernorm_bwd(
            dcn, c["img32"].contiguous().view(B * I, -1), f32(a.norm_kv.weight), a.norm_kv.eps)   # d(image tokens) is discarded: FPN is frozen
        self.c = None
        return dvin.view(B, V, Din), g


class PreSelectTrain:
    def __init__(self, module):
        if module.scale != 1.0:
            raise NotImplementedError("VISION_QUERY.VISION_SCALE is 1.0 in every MQ config")
        self.module = module
        self.blocks = [_BlockTrain(b) for b in module.layers]

    @torch.no_grad()
    def forward(self, vision, image):
        if not vision.is_cuda:
            raise MqdetError("PreSelectTrain: CUDA tensors required (no CPU fallback)")
        v = vision.float().contiguous()
        img = image.float().contiguous()
        for b in self.blocks:
            v = b.forward(v, img, None)
        return v

    @torch.no_grad()
    def backward(self, dvision):
        grads = {}
        d = dvision
        for i in range(len(self.blocks) - 1, -1, -1):
            d, g = self.blocks[i].backward(d)
            grads.update({f"layers.{i}.{k}": v for k, v in g.items()})
        return d, grads
