"""TEST DOUBLE — torch-CPU stand-ins for the C-ABI entry points of ``mqdet_b200.ops``, used ONLY by tests/test_host_logic_cpu.py
(in a subprocess) to exercise the HOST-SIDE logic of the drop-in modules without a GPU: views / strides / batch layouts handed to the
GEMM, mask conventions, cached geometry, the composition of the training backward.  Each stand-in restates what the corresponding kernel is
specified to compute in include/mqdet_b200.h, with fp16 rounding where the kernel rounds, so the modules' outputs can be compared with
the oracle at fp16 tolerances.  It is NOT a CPU fallback: nothing under mqdet_b200/ imports it, the product ops still raise without the
shared library or a CUDA device, and GPU parity is established by the ``-m gpu`` tests through the real kernels.

Importing this module monkey-patches ``mqdet_b200.ops`` and makes every tensor report ``is_cuda`` (the modules refuse CPU tensors), which
is why it must only ever be imported in a throw-away process.
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
import torch.nn.functional as F
torch.Tensor.is_cuda = property(lambda self: True)
from mqdet_b200 import ops, _lib
from oracle import restate

def _need_cuda(*a): pass
ops._need_cuda = _need_cuda

def gemm(a, b, out=None, *, out_dtype=torch.float16, alpha=1.0, bias=None, bias_mode=_lib.VEC_PER_COL, scale_after_bias=False,
         act=0, clamp=0.0, gate=None, gate_mode=0, gate_tanh=False, residual=None, impl=None):
    assert a.dtype == torch.float16 and b.dtype == torch.float16
    acc = torch.matmul(a.float(), b.float().transpose(-1, -2))
    M, N = acc.shape[-2:]
    if bias is not None:
        assert bias.dtype == torch.float32
        bv = bias.view(*bias.shape[:-1], 1, N) if bias_mode == _lib.VEC_PER_COL else bias.view(*bias.shape[:-1], M, 1)
        assert bias.shape[-1] == (N if bias_mode == _lib.VEC_PER_COL else M), (bias.shape, M, N, bias_mode)
    if bias is None: v = alpha * acc
    elif scale_after_bias: v = alpha * (acc + bv)
    else: v = alpha * acc + bv
    if act == _lib.ACT_GELU: v = F.gelu(v)
    elif act == _lib.ACT_RELU: v = F.relu(v)
    if clamp > 0: v = v.clamp(-clamp, clamp)
    if gate is not None:
        g = torch.tanh(gate) if gate_tanh else gate
        if gate_mode == _lib.VEC_SCALAR: v = v * g
        elif gate_mode == _lib.VEC_PER_COL: assert g.numel() == N; v = v * g.view(1, N)
        elif gate_mode == _lib.VEC_PER_ROW: assert g.numel() == v.numel() // N, (g.shape, v.shape); v = v * g.view(*v.shape[:-1], 1) if g.numel()==v.numel()//N else None
    if residual is not None:
        assert residual.shape[-2:] == (M, N), (residual.shape, M, N)
        v = v + residual.float().view(v.shape)
    if out is None:
        return v.to(out_dtype)
    assert out.shape[-2:] == (M, N), (out.shape, M, N)
    out.copy_(v.view(out.shape).to(out.dtype))
    return out
ops.gemm = gemm

def layernorm(x, gamma, beta, eps=1e-5, *, out16=True, out32=False, zero_row_period=0):
    y = F.layer_norm(x.float(), (x.shape[-1],), gamma, beta, eps)
    if out16 and out32: return y.half(), y
    return y.half() if out16 else y
ops.layernorm = layernorm
def add_layernorm(a, b, gamma, beta, eps, *, out16=True, out32=True, clamp=0.0):
    assert a.dtype == torch.float32 and b.dtype == torch.float32 and a.numel() == b.numel()
    y = F.layer_norm(a + b.view(a.shape), (a.shape[-1],), gamma, beta, eps)
    if clamp > 0: y = y.clamp(-clamp, clamp)
    return y.half(), y
ops.add_layernorm = add_layernorm
def softmax_rows(x, *, n=None, scale=1.0, colmask=None, rows_per_batch=0, mask_value=0.0, keep_add=0.0, out=None):
    assert x.is_contiguous() and x.dtype == torch.float32
    n_pad = x.shape[-1]; n = n_pad if n is None else n
    rows = x.numel() // n_pad
    v = x.float().reshape(rows, n_pad)[:, :n] * scale
    if colmask is not None:
        rpb = rows_per_batch if rows_per_batch > 0 else rows
        cm = colmask.reshape(-1, n)
        assert cm.shape[0] * rpb == rows, (cm.shape, rpb, rows)
        idx = torch.arange(rows) // rpb
        m = cm[idx]
        v = v + torch.where(m == 0, torch.full_like(v, mask_value), torch.full_like(v, keep_add))
    p = v.softmax(-1)
    o = torch.zeros(rows, n_pad)
    o[:, :n] = p
    o = o.view(x.shape).half()
    if out is not None: out.copy_(o); return out
    return o
ops.softmax_rows = softmax_rows
ops.cast_f16 = lambda x: (_ for _ in ()).throw(TypeError("cast_f16 needs fp32 contiguous")) if (x.dtype != torch.float32 or not x.is_contiguous()) else x.half()
ops.cast_f32 = lambda x: x.float()
def global_max(x): return x.max().view(1)
ops.global_max = global_max
def shift_clamp_(x, s, lo, hi): x.copy_((x - s).clamp(lo, hi)); return x
ops.shift_clamp_ = shift_clamp_
ops.row_max = lambda x: x.max(-1)[0]
def topk_desc(keys, k):
    # value desc, index asc
    idx = torch.argsort(-keys, dim=1, stable=True)[:, :k]
    return idx.contiguous()
ops.topk_desc = topk_desc
def gather_rows(src, idx, sigmoid=False):
    o = torch.gather(src, 1, idx.unsqueeze(-1).expand(-1, -1, src.shape[-1]))
    return o.sigmoid() if sigmoid else o
ops.gather_rows = gather_rows
def contrastive_embed(x16, y16, mask, L):
    return restate.contrastive_embed(x16.float(), y16.float(), mask, L)
ops.contrastive_embed = contrastive_embed
class Lv:
    def __init__(self, sizes): 
        self.sizes = [(int(h), int(w)) for h, w in sizes]; self.n = len(self.sizes); self.N = sum(h*w for h,w in self.sizes)
        off=[0]
        for h,w in self.sizes: off.append(off[-1]+h*w)
        self.off=off
ops.get_levels = lambda sizes, dev: Lv(sizes)
def ms_deform_attn(value16, proj32, aw_col0, ref, levels, heads, points, out_dtype=torch.float16):
    B, Nv, E = value16.shape; Q = ref.shape[1]; L = levels.n; d = E // heads
    proj = proj32.view(B, Q, -1)
    off = proj[..., :aw_col0].view(B, Q, heads, L, points, 2)
    aw = proj[..., aw_col0:aw_col0 + heads*L*points].view(B, Q, heads, L*points).softmax(-1).view(B, Q, heads, L, points)
    ss = torch.tensor(levels.sizes, dtype=torch.float32)
    if ref.shape[-1] == 2:
        norm = torch.stack([ss[:, 1], ss[:, 0]], -1)
        loc = ref[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    else:
        loc = ref[:, :, None, :, None, :2] + off / points * ref[:, :, None, :, None, 2:] * 0.5
    v = value16.float().view(B, Nv, heads, d)
    vals = v.split([h*w for h,w in levels.sizes], dim=1)
    grids = 2*loc - 1
    sampled = []
    for l,(h,w) in enumerate(levels.sizes):
        vl = vals[l].flatten(2).transpose(1,2).reshape(B*heads, d, h, w)
        g = grids[:, :, :, l].transpose(1,2).flatten(0,1)
        sampled.append(F.grid_sample(vl, g, mode="bilinear", padding_mode="zeros", align_corners=False))
    a = aw.transpose(1,2).reshape(B*heads, 1, Q, L*points)
    out = (torch.stack(sampled, dim=-2).flatten(-2) * a).sum(-1).view(B, heads*d, Q).transpose(1,2)
    return out.to(out_dtype).contiguous()
ops.ms_deform_attn = ms_deform_attn
def add_cast(a32, b32=None, rowgate=None, *, out16=True, out32=False):
    assert a32.dtype == torch.float32
    v = a32 if b32 is None else a32 + b32
    if rowgate is not None:
        assert rowgate.numel() == a32.numel() // a32.shape[-1]
        g = rowgate.view(*a32.shape[:-1], 1)
        v = torch.where(g == 0, torch.zeros_like(v), v * g)
    if out16 and out32: return v.half(), v
    return v.half() if out16 else v
ops.add_cast = add_cast
def groupnorm_rows(x, groups, gamma, beta, eps=1e-5, *, out16=True, out32=False):
    B, HW, C = x.shape
    y = F.group_norm(x.float().transpose(1,2), groups, gamma, beta, eps).transpose(1,2).contiguous()
    if out16 and out32: return y.half(), y
    return y.half() if out16 else y
ops.groupnorm_rows = groupnorm_rows
def box_refine_sine(ref_in, vr, *, delta=None, ref_is_logit=False, want_sine=True):
    if delta is not None:
        base = ref_in if ref_is_logit else restate.inverse_sigmoid(ref_in)
        r = (delta[..., :4] + base).sigmoid()
    else:
        r = ref_in.sigmoid() if ref_is_logit else ref_in
    vr4 = torch.cat([vr, vr], -1)
    ri = r[:, :, None] * vr4[:, None]
    s = restate.sineembed_for_position(ri[:, :, 0]).half() if want_sine else None
    return r, ri.contiguous(), s
ops.box_refine_sine = box_refine_sine
def gdino_detections(logits, boxes, tokmap, img_wh, thr, max_out=None):
    B, nq, T = logits.shape
    pmap = {c+1: [int(t) for t in tokmap[c] if t >= 0] for c in range(tokmap.shape[0]) if (tokmap[c] >= 0).any()}
    sizes = [(int(h), int(w)) for w, h in img_wh.tolist()]
    det = restate.gdino_detections(logits, boxes, pmap, tokmap.shape[0], sizes, thr)
    max_out = nq if max_out is None else max_out
    out = torch.zeros(B, max_out+1, 6)
    for b,(bx,sc,lb) in enumerate(det):
        k = bx.shape[0]
        out[b,:k,:4]=bx; out[b,:k,4]=sc; out[b,:k,5]=lb.float(); out[b,max_out,0]=k
    return out
ops.gdino_detections = gdino_detections
ops.make_tokmap = lambda pm, C, dev: ops.__dict__['make_tokmap_orig'](pm, C, 'cpu')


# ---- training side -------------------------------------------------------------------------------------------------
def transpose_cast(x, scale=1.0):
    R, C = x.shape; Rp = (R+7)//8*8
    o = torch.zeros(C, Rp); o[:, :R] = (x.float()*scale).t(); return o.half()
ops.transpose_cast = transpose_cast
def layernorm_bwd(dy, x, gamma, eps, dx=None, want_param_grads=True):
    D = x.shape[-1]; x2 = x.reshape(-1, D); d2 = dy.reshape(-1, D)
    mean = x2.mean(-1, keepdim=True); var = ((x2-mean)**2).mean(-1, keepdim=True); rstd = (var+eps).rsqrt()
    xh = (x2-mean)*rstd; g = d2*gamma
    o = rstd*(g - g.mean(-1, keepdim=True) - xh*(g*xh).mean(-1, keepdim=True))
    if dx is None: dx = o.view(x.shape)
    else: dx.view(-1, D).add_(o)
    return dx, (d2*xh).sum(0), d2.sum(0)
ops.layernorm_bwd = layernorm_bwd
def gelu_bwd(z16, dh):
    x = z16.float(); cdf = 0.5*(1+torch.erf(x*0.7071067811865476)); pdf = 0.3989422804014327*torch.exp(-0.5*x*x)
    return (dh.float()*(cdf + x*pdf)).half()
ops.gelu_bwd = gelu_bwd
def gcp_gate_bwd(dx1, s, g, w2):
    ds = dx1*g[:, None]; dgpre = (dx1*s).sum(-1)*(1-g*g); dh1 = (dgpre[:, None]*w2[None]).half(); return ds, dgpre, dh1
ops.gcp_gate_bwd = gcp_gate_bwd
ops.colsum_weighted = lambda h16, w: (w[:, None]*h16.float()).sum(0)
def gcp_sparse_attn(q, kv, idx, heads, dim_head):
    B, T, inner = q.shape; V1 = kv.shape[1]; S = idx.shape[-1]
    qf = q.float().view(B, T, heads, dim_head)
    out = torch.zeros(B, T, heads, dim_head)
    for b in range(B):
        k = kv[b, :, :inner].float().view(V1, heads, dim_head)[idx[b].long()]  # [T,S,H,d]
        v = kv[b, :, inner:].float().view(V1, heads, dim_head)[idx[b].long()]
        sim = torch.einsum('thd,tshd->ths', qf[b], k) + (idx[b] == V1-1).float()[:, None, :]*-1e4
        p = sim.softmax(-1)*(idx[b] != V1-1).float()[:, None, :]
        out[b] = torch.einsum('ths,tshd->thd', p, v)
    return out.view(B, T, inner).half()
ops.gcp_sparse_attn = gcp_sparse_attn
def gcp_sparse_attn_bwd(q, kv, idx, dout, heads, dim_head):
    B, T, inner = q.shape; V1 = kv.shape[1]
    dq = torch.zeros(B, T, inner); dkv = torch.zeros(B, V1, 2*inner)
    for b in range(B):
        qf = q[b].float().view(T, heads, dim_head); go = dout[b].float().view(T, heads, dim_head)
        id_ = idx[b].long(); pad = (id_ == V1-1)
        K = kv[b, :, :inner].float().view(V1, heads, dim_head); Vv = kv[b, :, inner:].float().view(V1, heads, dim_head)
        k = K[id_]; v = Vv[id_]
        sim = torch.einsum('thd,tshd->ths', qf, k) + pad.float()[:, None, :]*-1e4
        ps = sim.softmax(-1)
        dp = torch.einsum('thd,tshd->ths', go, v)*(~pad).float()[:, None, :]
        dsim = ps*(dp - (ps*dp).sum(-1, keepdim=True))
        p = ps*(~pad).float()[:, None, :]
        dq[b] = torch.einsum('ths,tshd->thd', dsim, k).reshape(T, inner)
        dk_c = torch.einsum('ths,thd->tshd', dsim, qf).reshape(-1, inner)
        dv_c = torch.einsum('ths,thd->tshd', p, go).reshape(-1, inner)
        dkv[b, :, :inner].index_add_(0, id_.reshape(-1), dk_c)
        dkv[b, :, inner:].index_add_(0, id_.reshape(-1), dv_c)
    return dq.half(), dkv
ops.gcp_sparse_attn_bwd = gcp_sparse_attn_bwd
def dot_sum(a, b=None, one_minus_tanh2_of=None, mul=1.0):
    s = (a*(a if b is None else b)).sum()*mul
    if one_minus_tanh2_of is not None: s = s*(1-torch.tanh(one_minus_tanh2_of)**2)
    return s.view(1)
ops.dot_sum = dot_sum
def scale_cast(x, scalar=None, tanh_scalar=False, alpha=1.0, out16=True, out32=False):
    a = alpha
    if scalar is not None: a = a*(torch.tanh(scalar) if tanh_scalar else scalar)
    v = x*a
    if out16 and out32: return v.half(), v
    return v.half() if out16 else v
ops.scale_cast = scale_cast
def gcp_build_index(mask, S):
    B, V, T = mask.shape
    idx = torch.full((B, T, S), V, dtype=torch.int32); counts = torch.zeros(B, T, dtype=torch.int32)
    for b in range(B):
        for t in range(T):
            vs = torch.nonzero(mask[b, :, t]).flatten()
            counts[b, t] = len(vs); n = min(S, len(vs)); idx[b, t, :n] = vs[:n].int()
    return idx, counts
ops.gcp_build_index = gcp_build_index
def gcp_gate_residual_ln(h1, w2, s, x, gamma, beta, eps=1e-5, want_gate=False):
    g = torch.tanh(h1.float() @ w2); x1 = s*g[:, None] + x.view(s.shape)
    ln = F.layer_norm(x1, (x1.shape[-1],), gamma, beta, eps).half()
    return (x1, ln, g) if want_gate else (x1, ln)
ops.gcp_gate_residual_ln = gcp_gate_residual_ln
def transpose_cast_batched(x):
    nb2, nb1, R, C = x.shape; Rp=(R+7)//8*8
    o = torch.zeros(nb2, nb1, C, Rp); o[..., :R] = x.float().transpose(-1, -2); return o.half()
ops.transpose_cast_batched = transpose_cast_batched
def softmax_bwd_rows(p16, dp32, scale=1.0):
    p = p16.float(); return (scale*p*(dp32 - (p*dp32).sum(-1, keepdim=True))).half()
ops.softmax_bwd_rows = softmax_bwd_rows
_lnb = ops.layernorm_bwd
def layernorm_bwd2(dy, x, gamma, eps, dx=None, want_param_grads=True, x2=None):
    return _lnb(dy, x if x2 is None else x + x2.view(x.shape), gamma, eps, dx=dx, want_param_grads=want_param_grads)
ops.layernorm_bwd = layernorm_bwd2


# ---- remaining entry points used by the modules exercised in tests/hostlogic/run.py ---------------------------------------------
def sum_splits_cast(part, out16):
    out16.copy_(part.sum(2).half())
    return out16
ops.sum_splits_cast = sum_splits_cast


def softmax_rows_shifted(x32, shift, lo, hi, *, n=None, colmask=None, rows_per_batch=0, mask_value=0.0, keep_add=0.0):
    ops.shift_clamp_(x32, shift, lo, hi)
    return ops.softmax_rows(x32, n=n, colmask=colmask, rows_per_batch=rows_per_batch, mask_value=mask_value, keep_add=keep_add)
ops.softmax_rows_shifted = softmax_rows_shifted


def im2col3x3(x16, B, H, W, stride=1, relu_in=False):
    C = x16.shape[-1]
    x = x16.float().view(B, H, W, C).permute(0, 3, 1, 2)
    if relu_in:
        x = F.relu(x)
    cols = F.unfold(x, 3, padding=1, stride=stride)                      # [B, C*9, L], row index c*9 + tap
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    cols = cols.view(B, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 9 * C)   # k = tap*C + c
    return cols.half().contiguous(), Ho, Wo
ops.im2col3x3 = im2col3x3


def avgpool2_levels(x16, levels):
    B, N, C = x16.shape
    outs = []
    for l, (h, w) in enumerate(levels.sizes):
        f = x16[:, levels.off[l]:levels.off[l + 1]].float().transpose(1, 2).reshape(B, C, h, w)
        outs.append(F.avg_pool2d(f, 2).flatten(2).transpose(1, 2))
    return torch.cat(outs, 1).contiguous()
ops.avgpool2_levels = avgpool2_levels


def make_tokmap(positive_map, num_classes, device):
    max_tok = max([len(v) for v in positive_map.values()] + [1])
    tm = torch.full((num_classes, max_tok), -1, dtype=torch.int32)
    for label, toks in positive_map.items():
        tm[label - 1, :len(toks)] = torch.tensor(list(toks), dtype=torch.int32)
    return tm
ops.make_tokmap = make_tokmap


def dense_cross_attn(q, kv, heads, d):
    B, Tq, inner = q.shape
    I = kv.shape[1]
    qf = q.float().view(B, Tq, heads, d).transpose(1, 2)
    k = kv[..., :inner].float().view(B, I, heads, d).transpose(1, 2)
    v = kv[..., inner:].float().view(B, I, heads, d).transpose(1, 2)
    return ((qf @ k.transpose(-1, -2)).softmax(-1) @ v).transpose(1, 2).reshape(B, Tq, inner).half()
ops.dense_cross_attn = dense_cross_attn


def roi_align_levels(pyr16, levels, scales, rois, pooled=7, sampling_ratio=0, mean_only=True):
    B = pyr16.shape[0]
    pyr = [pyr16[:, levels.off[l]:levels.off[l + 1]].float().transpose(1, 2).reshape(B, -1, h, w) for l, (h, w) in enumerate(levels.sizes)]
    per = [rois[rois[:, 0] == b][:, 1:] for b in range(B)]
    f, lv = restate.pool_query_features(pyr, per, scales=tuple(scales), resolution=pooled, sampling_ratio=sampling_ratio)
    return f, lv.int()
ops.roi_align_levels = roi_align_levels


def token_focal_loss(logits, targets, text_mask=None, alpha=0.25, gamma=2.0, want_grad=True, grad_scale=1.0):
    lr = logits.clone().requires_grad_(True)
    loss = restate.token_focal_loss(lr, targets, alpha, gamma, text_mask)
    loss.backward()
    return loss.detach().view(1), lr.grad * grad_scale
ops.token_focal_loss = token_focal_loss


def clip_coef(grads, max_norm):
    n = torch.sqrt(sum((g.float() ** 2).sum() for g in grads))
    return torch.stack([torch.clamp(max_norm / (n + 1e-6), max=1.0) if max_norm > 0 else torch.ones(()), n])
ops.clip_coef = clip_coef


def adamw_step_(p, g, m, v, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, grad_scale=None):
    gr = g * (1.0 if grad_scale is None else grad_scale)
    p.mul_(1 - lr * weight_decay)
    m.mul_(betas[0]).add_(gr, alpha=1 - betas[0])
    v.mul_(betas[1]).addcmul_(gr, gr, value=1 - betas[1])
    bc1, bc2 = 1 - betas[0] ** step, 1 - betas[1] ** step
    p.addcdiv_(m, (v.sqrt() / bc2 ** 0.5).add_(eps), value=-lr / bc1)
    return p
ops.adamw_step_ = adamw_step_
