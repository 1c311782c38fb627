"""Activation backward of a (frozen) post-LN BERT layer on sm_90a kernels — the part of the modulated pre-training backward that
carries the loss gradient through ``encoder.layer.N`` between two Gated Class-scalable Perceiver blocks (QVBertEncoder.forward,
modeling_bert_new.py:566-610: GCP block i-6 sits BEFORE BERT layer i, so the gradient of block i-6 needs the backward of layers i..11).
BERT itself is frozen in the MQ pre-training (tools/train_net.py:70-77): only dL/d(input) is produced, no weight gradients.

    BertLayerTrain(layer).forward(h32, h16, colmask)   the inference kernels, keeping the activations the backward needs
    BertLayerTrain(layer).backward(dout)               dL/dh, fp32 [B,T,D]

Every product of the backward is a wgmma GEMM: dX = dY W with the cached transposed weight (``wT16``); the attention backward
(dP = dC V^T, dQ = dS K, dK = dS^T Q, dV = P^T dC) takes its K-major operands from operand-swapped projections (K^T = W_k h^T, like
the forward's V^T) or from ``mqdet_transpose_cast_batched``; softmax / LayerNorm / GELU backward are the kernels of csrc/train.cu.
Pre-activations of the GELU and the V / K^T / Q^T projections are recomputed rather than stored.
"""
import torch

from ... import ops
from ..._lib import VEC_PER_ROW, MqdetError
from ...utils.weights import f32, w16, wT16


class BertLayerTrain:
    def __init__(self, layer):
        if layer.clamp:
            raise NotImplementedError("the +-5e4 clamps of BertEncoderLayer are not differentiated (QVBert's layers carry none)")
        self.layer = layer
        self.ctx = None

    @torch.no_grad()
    def forward(self, h32, h16, colmask):
        """BertLayer.forward (same kernels and order), 2-D padding mask, keeping p / ctx / the LayerNorm addends."""
        L = self.layer
        if not h32.is_cuda:
            raise MqdetError("BertLayerTrain: CUDA tensors required (no CPU fallback)")
        if colmask.dim() != 2:
            raise NotImplementedError("per-query masks are an inference feature of the GroundingDINO text encoder")
        B, T, D = h32.shape
        H = L.heads
        d = D // H
        sa = L.attention.self
        w, b = L._qk16()
        qk = ops.gemm(h16.view(B * T, D), w, bias=b).view(B, T, 2, H, d)
        q, k = qk[:, :, 0], qk[:, :, 1]
        vT = ops.gemm(w16(sa.value.weight), h16, bias=f32(sa.value.bias), bias_mode=VEC_PER_ROW).view(B, H, d, T)
        scores = torch.empty((B, H, T, T), dtype=torch.float32, device=h32.device)
        ops.gemm(q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3), out=scores, alpha=d ** -0.5)
        p = ops.softmax_rows(scores, colmask=colmask, rows_per_batch=H * T, mask_value=-10000.0)
        ctx = torch.empty((B, T, H, d), dtype=torch.float16, device=h32.device)
        ops.gemm(p, vT, out=ctx.permute(0, 2, 1, 3))
        ao = L.attention.output
        a = ops.gemm(ctx.view(B * T, D), w16(ao.dense.weight), bias=f32(ao.dense.bias), out_dtype=torch.float32)
        a16, a32 = ops.add_layernorm(a, h32.view(B * T, D), f32(ao.LayerNorm.weight), f32(ao.LayerNorm.bias), ao.LayerNorm.eps)
        it = ops.gemm(a16, w16(L.intermediate.dense.weight), bias=f32(L.intermediate.dense.bias), act=1)
        o = ops.gemm(it, w16(L.output.dense.weight), bias=f32(L.output.dense.bias), out_dtype=torch.float32)
        o16, o32 = ops.add_layernorm(o, a32, f32(L.output.LayerNorm.weight), f32(L.output.LayerNorm.bias), L.output.LayerNorm.eps)
        self.ctx = dict(B=B, T=T, D=D, h32=h32.contiguous().view(B * T, D), h16=h16.contiguous(), q=q, k=k, p=p, a=a, a16=a16, a32=a32, o=o)
        return o32.view(B, T, D), o16.view(B, T, D)

    @torch.no_grad()
    def backward(self, dout):
        """dout fp32 [B,T,D] (gradient w.r.t. the layer output) -> dL/dh fp32 [B,T,D]."""
        c, L = self.ctx, self.layer
        if c is None:
            raise MqdetError("BertLayerTrain.backward before forward")
        B, T, D = c["B"], c["T"], c["D"]
        H = L.heads
        d = D // H
        M = B * T
        sa, ao, mid, out = L.attention.self, L.attention.output, L.intermediate, L.output
        dout = dout.float().contiguous().view(M, D)
        # ---- out = LN(it Wout^T + b + a)
        ds2, _, _ = ops.layernorm_bwd(dout, c["o"], f32(out.LayerNorm.weight), out.LayerNorm.eps, want_param_grads=False, x2=c["a32"])
        dit = ops.gemm(ops.cast_f16(ds2), wT16(out.dense.weight))
        zi = ops.gemm(c["a16"], w16(mid.dense.weight), bias=f32(mid.dense.bias))
        dzi = ops.gelu_bwd(zi, dit)
        da = ops.gemm(dzi, wT16(mid.dense.weight), out_dtype=torch.float32, residual=ds2)
        # ---- a = LN(ctx Wo^T + b + h)
        ds1, _, _ = ops.layernorm_bwd(da, c["a"], f32(ao.LayerNorm.weight), ao.LayerNorm.eps, want_param_grads=False, x2=c["h32"])
        dctx = ops.gemm(ops.cast_f16(ds1), wT16(ao.dense.weight)).view(B, T, H, d)
        # ---- attention: ctx = P V, P = softmax(Q K^T / sqrt(d) + mask)
        h16 = c["h16"]
        v = ops.gemm(h16.view(M, D), w16(sa.value.weight), bias=f32(sa.value.bias)).view(B, T, H, d)
        dp = torch.empty((B, H, T, T), dtype=torch.float32, device=dout.device)
        ops.gemm(dctx.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3), out=dp)
        ds = ops.softmax_bwd_rows(c["p"], dp)                                         # [B,H,T,Tk] fp16
        scale = d ** -0.5
        kT = ops.gemm(w16(sa.key.weight), h16, bias=f32(sa.key.bias), bias_mode=VEC_PER_ROW).view(B, H, d, T)
        qT = ops.gemm(w16(sa.query.weight), h16, bias=f32(sa.query.bias), bias_mode=VEC_PER_ROW).view(B, H, d, T)
        dq = torch.empty((B, T, H, d), dtype=torch.float16, device=dout.device)
        ops.gemm(ds, kT, out=dq.permute(0, 2, 1, 3), alpha=scale)
        dk = torch.empty((B, T, H, d), dtype=torch.float16, device=dout.device)
        ops.gemm(ops.transpose_cast_batched(ds), qT, out=dk.permute(0, 2, 1, 3), alpha=scale)
        dv = torch.empty((B, T, H, d), dtype=torch.float16, device=dout.device)
        ops.gemm(ops.transpose_cast_batched(c["p"]), ops.transpose_cast_batched(dctx.permute(0, 2, 1, 3)), out=dv.permute(0, 2, 1, 3))
        # ---- projections: dh = ds1 (residual) + dq Wq + dk Wk + dv Wv
        dh = ops.gemm(dq.view(M, D), wT16(sa.query.weight), out_dtype=torch.float32, residual=ds1)
        dh = ops.gemm(dk.view(M, D), wT16(sa.key.weight), out_dtype=torch.float32, residual=dh)
        dh = ops.gemm(dv.view(M, D), wT16(sa.value.weight), out_dtype=torch.float32, residual=dh)
        self.ctx = None
        return dh.view(B, T, D)
