"""Training forward / backward of the Gated Class-scalable Perceiver block on sm_90a kernels — SURVEY.md §8(b2)'s ``gcp_block_fwd`` /
``gcp_block_bwd`` (BASELINE config 5: "GCP backward kernel").  In the reference these blocks (``encoder.qv_layer.N``) and PreSelect are
the ONLY trainable parameters of the modulated pre-training (tools/train_net.py:70-77, solver/build.py:46-49); their backward is
autograd over modeling_bert_new.py:186-248,298-374.  Here:

    ctx = GCPBlockTrain(block).forward(x, vision, mask)      the inference kernels, keeping what the backward needs
    dx, dvision, grads = GCPBlockTrain(block).backward(dy)   grads: {parameter name -> fp32 gradient}, names as in block.state_dict()

Forward arithmetic is the inference path (same kernels, same order).  Backward: every activation gradient dX = dY W and weight
gradient dW = dY^T X is one wgmma GEMM (fp16 operands, fp32 accumulation; both operands of a weight gradient are brought to
K-major by ``mqdet_transpose_cast``); LayerNorm / GELU / gate / sparse-attention backward, the scalar ff_gate gradient and the scatter
of dK / dV onto the unique query rows are the kernels of csrc/train.cu.  Pre-activations of the two GELUs are recomputed (one GEMM
each) instead of being stored.  Gradients w.r.t. the text stream are fp32; fp16 intermediates (dq, d(out), dz) can underflow for tiny
upstream gradients — scale the loss like the reference's GradScaler does (engine/trainer.py:119-140).
"""
import torch

from ... import ops
from ..._lib import ACT_GELU, VEC_SCALAR, MqdetError
from ...utils.weights import f32, w16
from .modeling_bert_new import _ln16, padded_vision, sparse_index


# Most vision queries per text token the sparse-attention backward takes (GCPB_MAX_S in csrc/train.cu); inference takes up to
# ops.GCP_MAX_S.  MQ-Det pre-trains with 5 queries per class and finetunes with 1 to 10.
GCP_TRAIN_MAX_S = 16


def _train_index(attention_mask):
    """sparse_index(attention_mask), rejected above GCP_TRAIN_MAX_S queries per token before any training compute is launched."""
    idx = sparse_index(attention_mask)
    if idx.shape[2] > GCP_TRAIN_MAX_S:
        raise MqdetError(f"GCP training: a text token has {idx.shape[2]} vision queries; the GCP backward takes at most "
                         f"GCP_TRAIN_MAX_S = {GCP_TRAIN_MAX_S} (set VISION_QUERY.NUM_QUERY_PER_CLASS so that no token exceeds it)")
    return idx


def _wT16(weight):
    """[out, in] parameter -> fp16 [in, out_p]: the B operand of dX = dY W (K = out)."""
    return ops.transpose_cast(weight.detach().float().contiguous())


class GCPBlockTrain:
    def __init__(self, block):
        if not block.enable_ffn:
            raise NotImplementedError("GCP blocks carry the gated FFN in every MQ config")
        self.block = block
        self.ctx = None

    @torch.no_grad()
    def forward(self, x, vision, attention_mask):
        """x fp32 [B,T,D], vision fp32 [B,V,D] (PreSelect output), attention_mask [B,V,T] -> y fp32 [B,T,D]."""
        blk, a = self.block, self.block.attn
        if not x.is_cuda:
            raise MqdetError("GCPBlockTrain: CUDA tensors required (no CPU fallback)")
        B, T, D = x.shape
        V = vision.shape[1]
        idx = _train_index(attention_mask)
        x32 = x.float().contiguous()
        vis_pad = padded_vision(vision)
        xn = _ln16(x32, a.norm)
        q = ops.gemm(xn.view(B * T, D), w16(a.to_q.weight), alpha=a.scale)
        kn = _ln16(vis_pad, a.norm_kv)
        kv = ops.gemm(kn.view(B * (V + 1), D), w16(a.to_kv.weight))
        o = ops.gcp_sparse_attn(q.view(B, T, a.inner_dim), kv.view(B, V + 1, 2 * a.inner_dim), idx, a.heads, a.dim_head)
        s = ops.gemm(o.view(B * T, a.inner_dim), w16(a.to_out.weight), out_dtype=torch.float32)
        sn = _ln16(s, blk.attn_gate.norm)
        h1 = ops.gemm(sn, w16(blk.attn_gate.linear1.weight), act=ACT_GELU)
        x1, x1n, g = ops.gcp_gate_residual_ln(h1, f32(blk.attn_gate.linear2.weight).view(-1), s, x32.view(B * T, D),
                                              f32(blk.ff.norm.weight), f32(blk.ff.norm.bias), blk.ff.norm.eps, want_gate=True)
        h2 = ops.gemm(x1n.view(B * T, D), w16(blk.ff.linear1.weight), act=ACT_GELU)
        y = ops.gemm(h2, w16(blk.ff.linear2.weight), out_dtype=torch.float32, gate=f32(blk.ff_gate), gate_mode=VEC_SCALAR,
                     gate_tanh=True, residual=x1.view(B * T, D))
        self.ctx = dict(B=B, T=T, D=D, V=V, x32=x32, idx=idx, vis_pad=vis_pad, xn=xn.view(B * T, D), q=q, kn=kn.view(B * (V + 1), D),
                        kv=kv, o=o.view(B * T, a.inner_dim), s=s, sn=sn, h1=h1, g=g.view(-1), x1=x1.view(B * T, D),
                        x1n=x1n.view(B * T, D), h2=h2)
        return y.view(B, T, D)

    @torch.no_grad()
    def backward(self, dy):
        """dy fp32 [B,T,D] -> (dx fp32 [B,T,D], dvision fp32 [B,V,D], {parameter name: fp32 gradient})."""
        c, blk, a = self.ctx, self.block, self.block.attn
        if c is None:
            raise MqdetError("GCPBlockTrain.backward before forward")
        B, T, D, V = c["B"], c["T"], c["D"], c["V"]
        M = B * T
        dy = dy.float().contiguous().view(M, D)
        grads = {}
        tr = ops.transpose_cast
        # ---- y = x1 + tanh(ff_gate) * (h2 W4^T)                                              (modeling_bert_new.py:366-372)
        ff = blk.ff
        u = ops.gemm(c["h2"], w16(ff.linear2.weight), out_dtype=torch.float32)
        grads["ff_gate"] = ops.dot_sum(dy, u, one_minus_tanh2_of=f32(blk.ff_gate))
        du16 = ops.scale_cast(dy, f32(blk.ff_gate), tanh_scalar=True)
        grads["ff.linear2.weight"] = ops.gemm(tr(du16), tr(c["h2"]), out_dtype=torch.float32)
        dh2 = ops.gemm(du16, _wT16(ff.linear2.weight))
        z2 = ops.gemm(c["x1n"], w16(ff.linear1.weight))
        dz2 = ops.gelu_bwd(z2, dh2)
        grads["ff.linear1.weight"] = ops.gemm(tr(dz2), tr(c["x1n"]), out_dtype=torch.float32)
        dx1n = ops.gemm(dz2, _wT16(ff.linear1.weight), out_dtype=torch.float32)
        dx1 = dy.clone()
        _, grads["ff.norm.weight"], grads["ff.norm.bias"] = ops.layernorm_bwd(dx1n, c["x1"], f32(ff.norm.weight), ff.norm.eps, dx=dx1)
        # ---- x1 = s * tanh(MLP_gate(LN(s))) + x                                              (:355-361)
        ag = blk.attn_gate
        w2 = f32(ag.linear2.weight).view(-1)
        ds, dgpre, dh1 = ops.gcp_gate_bwd(dx1, c["s"], c["g"], w2)
        grads["attn_gate.linear2.weight"] = ops.colsum_weighted(c["h1"], dgpre).view(1, -1)
        z1 = ops.gemm(c["sn"], w16(ag.linear1.weight))
        dz1 = ops.gelu_bwd(z1, dh1)
        grads["attn_gate.linear1.weight"] = ops.gemm(tr(dz1), tr(c["sn"]), out_dtype=torch.float32)
        dsn = ops.gemm(dz1, _wT16(ag.linear1.weight), out_dtype=torch.float32)
        _, grads["attn_gate.norm.weight"], grads["attn_gate.norm.bias"] = ops.layernorm_bwd(dsn, c["s"], f32(ag.norm.weight), ag.norm.eps,
                                                                                            dx=ds)
        # ---- s = o Wout^T                                                                     (:236-240)
        ds16 = ops.cast_f16(ds)
        grads["attn.to_out.weight"] = ops.gemm(tr(ds16), tr(c["o"]), out_dtype=torch.float32)
        do16 = ops.gemm(ds16, _wT16(a.to_out.weight))
        # ---- sparse masked cross-attention                                                    (:215-233)
        inner = a.inner_dim
        dq16, dkv = ops.gcp_sparse_attn_bwd(c["q"].view(B, T, inner), c["kv"].view(B, V + 1, 2 * inner), c["idx"], do16.view(B, T, inner),
                                            a.heads, a.dim_head)
        # ---- q = scale * LN(x) Wq^T                                                           (:200-206)
        dq2 = dq16.view(M, inner)
        grads["attn.to_q.weight"] = ops.gemm(tr(dq2), tr(c["xn"]), out_dtype=torch.float32, alpha=a.scale)
        dxn = ops.gemm(dq2, _wT16(a.to_q.weight), out_dtype=torch.float32, alpha=a.scale)
        dx, grads["attn.norm.weight"], grads["attn.norm.bias"] = ops.layernorm_bwd(dxn, c["x32"].view(M, D), f32(a.norm.weight), a.norm.eps,
                                                                                  dx=dx1)
        # ---- [k | v] = LN_kv(cat(vision, 0)) Wkv^T, once per unique query                     (:176-213)
        dkv16 = ops.cast_f16(dkv.view(B * (V + 1), 2 * inner))
        grads["attn.to_kv.weight"] = ops.gemm(tr(dkv16), tr(c["kn"]), out_dtype=torch.float32)
        dkn = ops.gemm(dkv16, _wT16(a.to_kv.weight), out_dtype=torch.float32)
        dvis, grads["attn.norm_kv.weight"], grads["attn.norm_kv.bias"] = ops.layernorm_bwd(dkn, c["vis_pad"].view(B * (V + 1), D),
                                                                                          f32(a.norm_kv.weight), a.norm_kv.eps)
        dvision = dvis.view(B, V + 1, D)[:, :V].contiguous()   # the zero padding row is a constant
        self.ctx = None
        return dx.view(B, T, D), dvision, grads


class QVBertEncoderTrain:
    """Training forward / backward of the vision-conditioned half of ``QVBertEncoder`` (modeling_bert_new.py:566-610): for
    i = start_qv .. last:  h <- GCP_{i-start}(h, vision, mask);  h <- BertLayer_i(h).  ``backward(dh)`` runs the chain in reverse and
    returns dL/dh at the entry of the first GCP block, dL/d(vision) summed over the blocks (the gradient PreSelect receives) and the
    gradients of every ``qv_layer.N.*`` parameter.  BERT layers are frozen (activation backward only); the layers before the first GCP
    block see no trainable parameter and are not differentiated."""

    def __init__(self, encoder):
        from .bert_backward import BertLayerTrain
        self.encoder = encoder
        s = encoder.start_qv_layer_index
        self.gcp = [GCPBlockTrain(b) for b in encoder.qv_layer]
        self.bert = [BertLayerTrain(encoder.layer[i]) for i in range(s, len(encoder.layer))]

    @torch.no_grad()
    def forward(self, h32, colmask, vision, vision_attention_mask):
        """h32 fp32 [B,T,D] = output of BERT layer start_qv-1; vision fp32 [B,V,D] (PreSelect output) -> final hidden state."""
        for g, b in zip(self.gcp, self.bert):
            h32 = g.forward(h32, vision, vision_attention_mask)
            h32, _ = b.forward(h32, ops.cast_f16(h32.contiguous()), colmask)
        return h32

    @torch.no_grad()
    def backward(self, dh):
        grads, dvision = {}, None
        for i in range(len(self.gcp) - 1, -1, -1):
            dh = self.bert[i].backward(dh)
            dh, dv, g = self.gcp[i].backward(dh)
            dvision = dv if dvision is None else dvision.add_(dv)   # plain accumulation of six [B,V,D] tensors (torch add)
            grads.update({f"qv_layer.{i}.{k}": v for k, v in g.items()})
        return dh, dvision, grads


class QVBertModelTrain:
    """Training forward / backward of ``QVBertModel`` (modeling_bert_new.py:690-848) restricted to what the modulated pre-training
    updates: every ``encoder.qv_layer.N.*`` and ``pre_select.*`` parameter (45.66 M parameters; BERT, embeddings frozen).

        hidden = forward(input_ids, attention_mask, vision, images, vision_attention_mask)     fp32 [B,T,768]
        grads  = backward(d_hidden)     {"encoder.qv_layer.N...": g, "pre_select.layers.N...": g}, names as in model.state_dict()

    The embeddings and the BERT layers before the first GCP block run on the inference path (no trainable parameter upstream of them);
    PreSelect, the GCP blocks and the BERT layers between them run their training forwards.  ``backward`` is the complete gradient of
    the trainable half of the language backbone GIVEN dL/d(hidden) — producing that input gradient from the detection loss needs the
    backward of the frozen fusion tower, which is not built (DESIGN.md)."""

    def __init__(self, model):
        from .preselect_backward import PreSelectTrain
        self.model = model
        self.pre = PreSelectTrain(model.pre_select)
        self.enc = QVBertEncoderTrain(model.encoder)

    @torch.no_grad()
    def forward(self, input_ids, attention_mask, vision, images, vision_attention_mask):
        _train_index(vision_attention_mask)
        st = self.model.text_prefix(input_ids, attention_mask, output_hidden_states=False)
        vq = self.pre.forward(vision, images)
        return self.enc.forward(st["h32"], st["colmask"], vq, vision_attention_mask)

    @torch.no_grad()
    def backward(self, d_hidden):
        _, dvq, g = self.enc.backward(d_hidden)
        _, gp = self.pre.backward(dvq)
        grads = {"encoder." + k: v for k, v in g.items()}
        grads.update({"pre_select." + k: v for k, v in gp.items()})
        return grads
