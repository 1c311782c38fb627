"""Tensor-level wrappers over the C ABI (device pointers + sizes + current CUDA stream).

PyTorch is used for memory, streams and views only; every arithmetic op below is a kernel of
libmqdet_b200.so.  All wrappers launch on ``torch.cuda.current_stream()`` and never synchronise.
"""
import ctypes

import torch

from . import _lib
from ._lib import (ACT_GELU, ACT_NONE, ACT_RELU, F16, F32, IMPL_SIMT, IMPL_TC, IMPL_TC_ONESHOT, VEC_NONE, VEC_PER_COL,
                   VEC_PER_ROW, VEC_SCALAR, GemmArgs, check, load)

# tests flip this to IMPL_SIMT to cross-check the tensor-core kernel against the plain FMA kernel
DEFAULT_GEMM_IMPL = IMPL_TC

# number of kernels launched through this module since the last reset (bench.py's gpu_launches)
launch_count = 0

# bench.py sets this to a list to time every GEMM launch with CUDA events on the launching stream (roofline.achieved)
GEMM_PROFILE = None
# ... and this one to time every launch of the tensor-core kernels (GEMM, dcn_conv, biattn_image, biattn_text_vn):
# entries (start event, end event, kernel name, algorithmic flops, algorithmic bytes, executed flops)
KERNEL_PROFILE = None


class _Timed:
    """Brackets one launch with CUDA events on the launching stream when KERNEL_PROFILE is a list."""

    def __init__(self, name, flops, nbytes, executed=None):
        self.rec = KERNEL_PROFILE is not None
        if self.rec:
            # ``flops`` = the ALGORITHMIC count (what the reference computes for this piece of work); ``executed`` = what the kernel
            # issues to the tensor cores when algebraic folding makes that smaller (defaults to the algorithmic count)
            self.name, self.flops, self.nbytes = name, float(flops), float(nbytes)
            self.executed = float(flops if executed is None else executed)
            self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def __enter__(self):
        if self.rec:
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if self.rec:
            self.e1.record()
            KERNEL_PROFILE.append((self.e0, self.e1, self.name, self.flops, self.nbytes, self.executed))
        return False


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _dt(t):
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.float32:
        return F32
    raise TypeError(f"unsupported dtype {t.dtype}")


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.MqdetError("mqdet_b200 ops require CUDA tensors (no CPU fallback)")


def _as4(t):
    """View a [..., rows, cols] tensor as (nb2, nb1, rows, cols) without copying."""
    if t.dim() < 2 or t.dim() > 4:
        raise ValueError(f"expected 2-4 dims, got {tuple(t.shape)}")
    while t.dim() < 4:
        t = t.unsqueeze(0)
    if t.stride(-1) != 1 and t.shape[-1] != 1:
        raise ValueError("last dimension must be contiguous")
    return t


def gemm(a, b, out=None, *, out_dtype=torch.float16, alpha=1.0, bias=None, bias_mode=VEC_PER_COL,
         scale_after_bias=False, act=ACT_NONE, clamp=0.0, gate=None, gate_mode=VEC_NONE, gate_tanh=False,
         residual=None, impl=None):
    """out[..., m, n] = epilogue(sum_k a[..., m, k] * b[..., n, k]); fp16 operands, fp32 accumulation.

    ``a``: [(nb2, (nb1,)) M, K] fp16, ``b``: [(nb2, (nb1,)) N, K] fp16 (an nn.Linear weight as is); arbitrary
    strides on all but the last dim; size-1 batch dims of ``b``/``a`` broadcast.  See mqdet_gemm_f16 in
    include/mqdet_b200.h for the epilogue order.
    """
    global launch_count
    _need_cuda(a, b, out, bias, gate, residual)
    if a.dtype != torch.float16 or b.dtype != torch.float16:
        raise TypeError("gemm operands must be fp16")
    a4, b4 = _as4(a), _as4(b)
    nb2 = max(a4.shape[0], b4.shape[0])
    nb1 = max(a4.shape[1], b4.shape[1])
    M, K = a4.shape[2], a4.shape[3]
    N = b4.shape[2]
    if b4.shape[3] != K:
        raise ValueError(f"K mismatch: a {tuple(a.shape)} vs b {tuple(b.shape)}")
    if out is None:
        out = torch.empty(torch.broadcast_shapes(a.shape[:-2], b.shape[:-2]) + (M, N), dtype=out_dtype, device=a.device)
    o4 = _as4(out)
    if o4.shape[2] != M or o4.shape[3] != N:
        raise ValueError(f"out shape {tuple(out.shape)} does not match M={M} N={N}")

    def bstride(t4, dim, n):
        return 0 if (t4.shape[dim] == 1 and n > 1) else (t4.stride(dim) if t4.shape[dim] > 1 else 0)

    g = GemmArgs()
    g.A, g.B = a4.data_ptr(), b4.data_ptr()
    g.M, g.N, g.K = M, N, K
    g.lda, g.ldb = a4.stride(2), b4.stride(2)
    g.nb1, g.nb2 = nb1, nb2
    g.a_b1, g.a_b2 = bstride(a4, 1, nb1), bstride(a4, 0, nb2)
    g.b_b1, g.b_b2 = bstride(b4, 1, nb1), bstride(b4, 0, nb2)
    g.C, g.c_dtype = o4.data_ptr(), _dt(out)
    g.ldc, g.c_b1, g.c_b2 = o4.stride(2), bstride(o4, 1, nb1), bstride(o4, 0, nb2)
    g.alpha, g.scale_after_bias = float(alpha), int(bool(scale_after_bias))
    if bias is not None:
        if bias.dtype != torch.float32:
            raise TypeError("bias must be fp32")
        g.bias, g.bias_mode = bias.data_ptr(), bias_mode
        if bias.dim() == 3:  # [nb2, nb1, n]
            g.bias_b1, g.bias_b2 = bstride(bias, 1, nb1), bstride(bias, 0, nb2)
        elif bias.dim() == 2:  # [nb1, n] (the innermost batch dim, like 3-D operands)
            g.bias_b1, g.bias_b2 = bstride(bias, 0, nb1), 0
    g.act, g.clamp = act, float(clamp)
    if gate is not None:
        if gate.dtype != torch.float32:
            raise TypeError("gate must be fp32")
        g.gate, g.gate_mode, g.gate_tanh = gate.data_ptr(), gate_mode, int(bool(gate_tanh))
    if residual is not None:
        r4 = _as4(residual)
        g.R, g.r_dtype = r4.data_ptr(), _dt(residual)
        g.ldr, g.r_b1, g.r_b2 = r4.stride(2), bstride(r4, 1, nb1), bstride(r4, 0, nb2)
    if GEMM_PROFILE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    # algorithmic bytes: every operand once (a broadcast operand once for the whole batch), the output, the residual
    nb = nb1 * nb2
    es_o = 2 if out.dtype == torch.float16 else 4
    gbytes = 2.0 * M * K * (a4.shape[0] * a4.shape[1]) + 2.0 * N * K * (b4.shape[0] * b4.shape[1]) + float(es_o) * M * N * nb
    if residual is not None:
        gbytes += (2.0 if residual.dtype == torch.float16 else 4.0) * M * N * nb
    with _Timed("gemm_wg_kernel", 2.0 * M * N * K * nb, gbytes):
        check(load().mqdet_gemm_f16(ctypes.byref(g), DEFAULT_GEMM_IMPL if impl is None else impl, _stream()), "gemm")
    if GEMM_PROFILE is not None:
        e1.record()
        GEMM_PROFILE.append((e0, e1, 2.0 * M * N * K * nb1 * nb2, (M, N, K, nb1 * nb2)))
    launch_count += 1
    return out


def layernorm(x, gamma, beta, eps=1e-5, *, out16=True, out32=False, zero_row_period=0):
    """nn.LayerNorm over the last dim of a contiguous [..., D] fp16/fp32 tensor -> (fp16, fp32) outputs."""
    global launch_count
    _need_cuda(x, gamma, beta)
    D = x.shape[-1]
    x2 = x.reshape(-1, D)
    rows = x2.shape[0]
    o16 = torch.empty(x.shape, dtype=torch.float16, device=x.device) if out16 else None
    o32 = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out32 else None
    check(load().mqdet_layernorm(_ptr(x2), _dt(x2), x2.stride(0), _ptr(gamma), _ptr(beta), float(eps), rows, D,
                                 _ptr(o16), _ptr(o32), D, int(zero_row_period), _stream()), "layernorm")
    launch_count += 1
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def swin_mlp(x32, ln_w, ln_b, eps, w1, b1, w2, b2):
    """The MLP half of a Swin block in one kernel (mqdet_swin_mlp_f16): x32 + fc2(GELU(fc1(LN(x32)))) for a contiguous fp32
    [rows, C] with C = 96 / 192; w1 fp16 [4C, C], w2 fp16 [C, 4C] (nn.Linear weights), fp32 LN affine and biases -> new fp32
    [rows, C], bit-identical to layernorm -> gemm(bias, GELU) -> gemm(bias, fp32 residual)."""
    global launch_count
    _need_cuda(x32, ln_w, ln_b, w1, b1, w2, b2)
    C = x32.shape[-1]
    rows = x32.numel() // C
    if x32.dtype != torch.float32 or not x32.is_contiguous():
        raise _lib.MqdetError("swin_mlp: contiguous fp32 rows required")
    for w, shape in ((w1, (4 * C, C)), (w2, (C, 4 * C))):
        if w.dtype != torch.float16 or tuple(w.shape) != shape or not w.is_contiguous():
            raise _lib.MqdetError(f"swin_mlp: weights must be contiguous fp16 {shape} (got {w.dtype} {tuple(w.shape)})")
    out = torch.empty_like(x32)
    # algorithmic work: fc1 + fc2 (2 * 2.rows.C.4C); bytes: the fp32 rows in and out, both weights once
    with _Timed("swin_mlp_kernel", 2.0 * 2.0 * rows * C * 4 * C, 2.0 * 4.0 * rows * C + 2.0 * 2.0 * 4 * C * C):
        check(load().mqdet_swin_mlp_f16(_ptr(x32), rows, C, _ptr(ln_w), _ptr(ln_b), float(eps), _ptr(w1), _ptr(b1), _ptr(w2),
                                        _ptr(b2), _ptr(out), _stream()), "swin_mlp")
    launch_count += 1
    return out


def add_layernorm(a, b, gamma, beta, eps, *, out16=True, out32=True, clamp=0.0):
    """LN(a + b) over the last dim; a, b contiguous fp32."""
    global launch_count
    _need_cuda(a, b)
    D = a.shape[-1]
    rows = a.numel() // D
    o16 = torch.empty(a.shape, dtype=torch.float16, device=a.device) if out16 else None
    o32 = torch.empty(a.shape, dtype=torch.float32, device=a.device) if out32 else None
    check(load().mqdet_add_layernorm(_ptr(a), _ptr(b), _ptr(gamma), _ptr(beta), float(eps), rows, D, _ptr(o32),
                                     _ptr(o16), float(clamp), _stream()), "add_layernorm")
    launch_count += 1
    return o16, o32


def softmax_rows(x, *, n=None, scale=1.0, colmask=None, rows_per_batch=0, mask_value=0.0, keep_add=0.0, out=None):
    """Row softmax over the last dim of x [..., n_pad] (fp16/fp32, contiguous) -> fp16; cols >= n are zeroed."""
    global launch_count
    _need_cuda(x, colmask)
    n_pad = x.shape[-1]
    n = n_pad if n is None else n
    rows = x.numel() // n_pad
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    check(load().mqdet_softmax_rows(_ptr(x), _dt(x), n_pad, _ptr(out), n_pad, rows, n, n_pad, float(scale),
                                    _ptr(colmask), int(rows_per_batch), float(mask_value), float(keep_add),
                                    _stream()), "softmax_rows")
    launch_count += 1
    return out


def sum_splits_cast(part32, out16):
    """part32 fp32 [nb2, nb1, S, R, C] contiguous (the fp32 partial products of a K-split GEMM) -> out16 [nb2, nb1, R, C] fp16 (a view with
    arbitrary nb / row strides, contiguous last dim) = the sum over S."""
    global launch_count
    _need_cuda(part32, out16)
    nb2, nb1, S, R, C = part32.shape
    if part32.dtype != torch.float32 or not part32.is_contiguous() or out16.dtype != torch.float16 or tuple(out16.shape) != (nb2, nb1, R, C) \
            or out16.stride(3) != 1:
        raise _lib.MqdetError("sum_splits_cast: part fp32 [nb2,nb1,S,R,C] contiguous, out fp16 [nb2,nb1,R,C] with a contiguous last dim")
    check(load().mqdet_sum_splits_cast(_ptr(part32), nb2, nb1, S, R, C, _ptr(out16), out16.stride(0), out16.stride(1), out16.stride(2),
                                       _stream()), "sum_splits_cast")
    launch_count += 1
    return out16


def softmax_rows_shifted(x32, shift, lo, hi, *, n=None, colmask=None, rows_per_batch=0, mask_value=0.0, keep_add=0.0):
    """softmax over the last dim of clamp(x - shift[0], lo, hi) (+ mask) for contiguous fp32 [..., n_pad] -> fp16; ``shift`` is a device
    scalar.  Fused where the kernel supports the row length, else ``shift_clamp_`` (in place!) followed by ``softmax_rows``."""
    global launch_count
    _need_cuda(x32, shift, colmask)
    n_pad = x32.shape[-1]
    n = n_pad if n is None else n
    if x32.dtype != torch.float32 or not x32.is_contiguous():
        raise _lib.MqdetError("softmax_rows_shifted: contiguous fp32 tensor required")
    if not load().mqdet_softmax_rows_shifted_supported(n, n_pad):
        shift_clamp_(x32, shift, lo, hi)
        return softmax_rows(x32, n=n, colmask=colmask, rows_per_batch=rows_per_batch, mask_value=mask_value, keep_add=keep_add)
    rows = x32.numel() // n_pad
    out = torch.empty(x32.shape, dtype=torch.float16, device=x32.device)
    check(load().mqdet_softmax_rows_shifted(_ptr(x32), n_pad, _ptr(out), n_pad, rows, n, n_pad, _ptr(shift), float(lo), float(hi),
                                            _ptr(colmask), int(rows_per_batch), float(mask_value), float(keep_add), _stream()),
          "softmax_rows_shifted")
    launch_count += 1
    return out


def global_max(x32):
    """max over ALL elements of a contiguous fp32 tensor -> device scalar [1] (no host sync)."""
    global launch_count
    _need_cuda(x32)
    if x32.dtype != torch.float32 or not x32.is_contiguous():
        raise _lib.MqdetError("global_max: contiguous fp32 tensor required")
    out = torch.empty((1,), dtype=torch.float32, device=x32.device)
    ws = torch.empty((int(load().mqdet_global_max_workspace_floats()),), dtype=torch.float32, device=x32.device)
    check(load().mqdet_global_max_f32(_ptr(x32), x32.numel(), _ptr(out), _ptr(ws), _stream()), "global_max")
    launch_count += 2
    return out


def shift_clamp_(x32, shift, lo, hi):
    """x = clamp(x - shift[0], lo, hi) in place over the whole (contiguous fp32) buffer; ``shift`` is a device scalar."""
    global launch_count
    _need_cuda(x32, shift)
    if x32.dtype != torch.float32 or not x32.is_contiguous():
        raise _lib.MqdetError("shift_clamp_: contiguous fp32 tensor required")
    check(load().mqdet_shift_clamp_f32(_ptr(x32), x32.numel(), _ptr(shift), float(lo), float(hi), _stream()), "shift_clamp")
    launch_count += 1
    return x32


def row_max(x32):
    """max over the last dim of a contiguous fp32 [..., D] tensor -> fp32 [...]."""
    global launch_count
    _need_cuda(x32)
    D = x32.shape[-1]
    x2 = x32.reshape(-1, D)
    out = torch.empty(x32.shape[:-1], dtype=torch.float32, device=x32.device)
    check(load().mqdet_row_max_f32(_ptr(x2), x2.shape[0], D, x2.stride(0), _ptr(out), _stream()), "row_max")
    launch_count += 1
    return out


def topk_desc(keys32, k):
    """indices [B, k] (int64) of the k largest entries of each row of fp32 keys [B, n], by (value descending, index ascending)."""
    global launch_count
    _need_cuda(keys32)
    if keys32.dtype != torch.float32 or keys32.dim() != 2 or not keys32.is_contiguous():
        raise _lib.MqdetError("topk_desc: contiguous fp32 [B, n] required")
    B, n = keys32.shape
    idx = torch.empty((B, k), dtype=torch.int64, device=keys32.device)
    check(load().mqdet_topk_desc(_ptr(keys32), B, n, int(k), _ptr(idx), _stream()), "topk_desc")
    launch_count += 1
    return idx


def gather_rows(src32, idx, sigmoid=False):
    """src32 [B, R, D] fp32, idx [B, k] int64 -> [B, k, D] (torch.gather along dim 1 with the index repeated over D), optionally
    through the logistic sigmoid."""
    global launch_count
    _need_cuda(src32, idx)
    if src32.dtype != torch.float32 or src32.dim() != 3 or not src32.is_contiguous() or idx.dtype != torch.int64 or not idx.is_contiguous():
        raise _lib.MqdetError("gather_rows: contiguous fp32 [B, R, D] and int64 [B, k] required")
    B, R, D = src32.shape
    k = idx.shape[1]
    out = torch.empty((B, k, D), dtype=torch.float32, device=src32.device)
    check(load().mqdet_gather_rows_f32(_ptr(src32), _ptr(idx), B, R, k, D, int(bool(sigmoid)), _ptr(out), _stream()), "gather_rows")
    launch_count += 1
    return out


def l2_normalize(x32, w=None, b0=None, eps=1e-12):
    """e = F.normalize(x, p=2, dim=-1) of a contiguous fp32 tensor -> (e fp16, e fp32, dot) with
    dot[r] = e[r, :] . w + b0 when ``w`` is given (the token bias of the dot-product head, vldyhead.py:818)."""
    global launch_count
    _need_cuda(x32, w, b0)
    D = x32.shape[-1]
    rows = x32.numel() // D
    e16 = torch.empty(x32.shape, dtype=torch.float16, device=x32.device)
    e32 = torch.empty_like(x32)
    dot = torch.empty(x32.shape[:-1], dtype=torch.float32, device=x32.device) if w is not None else None
    check(load().mqdet_l2norm_rowdot(_ptr(x32), rows, D, float(eps), _ptr(w), _ptr(b0), _ptr(e16), _ptr(e32), _ptr(dot),
                                     _stream()), "l2norm_rowdot")
    launch_count += 1
    return e16, e32, dot


def colsoftmax_transposed(A16, Np=None):
    """A16 [..., N, T] fp16 -> P [..., T, Np] fp16 with P[t, n] = softmax over n of A[n, t] (zero for n >= N)."""
    global launch_count
    _need_cuda(A16)
    N, T = A16.shape[-2], A16.shape[-1]
    Z = A16.numel() // (N * T)
    Np = (N + 7) // 8 * 8 if Np is None else Np
    P = torch.empty(A16.shape[:-2] + (T, Np), dtype=torch.float16, device=A16.device)
    ws = torch.empty((int(load().mqdet_colsoftmax_workspace_floats(Z, N, T)),), dtype=torch.float32, device=A16.device)
    check(load().mqdet_colsoftmax_transposed(_ptr(A16), Z, N, T, _ptr(P), Np, _ptr(ws), _stream()), "colsoftmax_transposed")
    launch_count += 3
    return P


def colsoftmax_stats(A16):
    """A16 [..., N, T] fp16 -> stat [Z, 2, T] fp32 = (max over n, 1 / sum over n of exp(a - max)) per column."""
    global launch_count
    _need_cuda(A16)
    N, T = A16.shape[-2], A16.shape[-1]
    Z = A16.numel() // (N * T)
    nws = int(load().mqdet_colsoftmax_workspace_floats(Z, N, T))
    ws = torch.empty((nws,), dtype=torch.float32, device=A16.device)
    check(load().mqdet_colsoftmax_stats(_ptr(A16), Z, N, T, _ptr(ws), _stream()), "colsoftmax_stats")
    launch_count += 2
    return ws[nws - Z * 2 * T:].view(Z, 2, T)  # the view keeps the workspace alive


def colstats_rowsoftmax(A16, colmask, z_per_mask, mask_value, keep_add):
    """T == 256.  One pass over A16 [..., N, 256] fp16: returns the column statistics [Z,2,T] of the scores (as
    colsoftmax_stats) and overwrites every row with its masked softmax over the 256 tokens (as softmax_rows)."""
    global launch_count
    _need_cuda(A16, colmask)
    N, T = A16.shape[-2], A16.shape[-1]
    Z = A16.numel() // (N * T)
    nws = int(load().mqdet_colsoftmax_workspace_floats(Z, N, T))
    ws = torch.empty((nws,), dtype=torch.float32, device=A16.device)
    check(load().mqdet_colstats_rowsoftmax(_ptr(A16), Z, N, T, _ptr(colmask), int(z_per_mask), float(mask_value),
                                           float(keep_add), _ptr(ws), _stream()), "colstats_rowsoftmax")
    launch_count += 2
    return ws[nws - Z * 2 * T:].view(Z, 2, T)


def biattn_text(kh, qh, vvT4, stat, clamp, out):
    """Fused text->image attention: kh [B,H,T,d], qh [B,H,N,d], vvT4 [B,H,d,Np] fp16 (strided views), stat [B*H,2,T] fp32
    (colsoftmax_stats of the clamped fp16 scores q.k^T), out [B,H,T,d] fp16 view <- softmax_n(scores)^T . Vv."""
    global launch_count
    _need_cuda(kh, qh, vvT4, stat, out)
    B, H, T, d = kh.shape
    N, Np = qh.shape[2], vvT4.shape[3]
    for t in (kh, qh, vvT4, out):
        if t.stride(3) != 1 or t.dtype != torch.float16:
            raise _lib.MqdetError("biattn_text: fp16 operands with a contiguous last dimension required")
    check(load().mqdet_biattn_text(_ptr(kh), kh.stride(2), kh.stride(1), kh.stride(0), _ptr(qh), qh.stride(2), qh.stride(1),
                                   qh.stride(0), _ptr(vvT4), vvT4.stride(2), vvT4.stride(1), vvT4.stride(0), _ptr(stat),
                                   float(clamp), _ptr(out), out.stride(2), out.stride(1), out.stride(0), H, B, T, N, Np, d,
                                   _stream()), "biattn_text")
    launch_count += 1
    return out


def biattn_image(vn16, gT, gbias, mT, bias, gamma, residual, mask, clamp, heads):
    """Fused image -> text side with the query / value / output projections folded into per-(image, head) operands, layer
    scale and residual (mqdet_biattn_image).  vn16 [B,N,256] fp16 (layer-normed tokens), gT [B,H,T,256] fp16, gbias [B,H,T,ld]
    fp32 (column 0 used) or None, mT [B,H,256,T] fp16; bias/gamma [256] fp32 or None; residual [B,N,256] fp16 or None; mask
    [B,T] fp32 or None -> (out [B,N,256] fp16, colmax [B*H,T] fp32)."""
    global launch_count
    _need_cuda(vn16, gT, gbias, mT, bias, gamma, residual, mask)
    B, N, C = vn16.shape
    T = gT.shape[2]
    for t in (vn16, gT, mT):
        if t.dtype != torch.float16 or t.stride(-1) != 1:
            raise _lib.MqdetError("biattn_image: fp16 operands with a contiguous last dimension required")
    if C != 256 or tuple(gT.shape) != (B, heads, T, 256) or tuple(mT.shape) != (B, heads, 256, T):
        raise _lib.MqdetError(f"biattn_image: need vn [B,N,256], gT [B,H,T,256], mT [B,H,256,T]; got {tuple(vn16.shape)}, "
                              f"{tuple(gT.shape)}, {tuple(mT.shape)}")
    if gbias is not None and (gbias.dtype != torch.float32 or not gbias.is_contiguous() or gbias.shape[:3] != (B, heads, T)):
        raise _lib.MqdetError("biattn_image: gbias must be contiguous fp32 [B, H, T, ld]")
    out = torch.empty((B, N, 256), dtype=torch.float16, device=vn16.device)
    colmax = torch.empty((B * heads, T), dtype=torch.float32, device=vn16.device)
    ws = torch.empty((int(load().mqdet_biattn_image_workspace_floats(B, heads, N, T)),), dtype=torch.float32, device=vn16.device)
    # algorithmic work of the image -> text direction as the reference computes it (fuse_helper.py:218-303): query projection,
    # scores, P.V_l, output projection (4 products of 2.N.T'.E with T' = 256 or T); bytes: tokens in, tokens out, residual
    E = heads * 256
    fl = B * (2.0 * N * 256 * E + 2.0 * 2.0 * N * T * E + 2.0 * N * E * 256)
    # executed: S = vn gT^T and P mT^T per head, 2.N.T.256 each (the query / value / output projections are folded into gT / mT)
    ex = B * heads * 2.0 * (2.0 * N * T * 256)
    with _Timed("biattn_image_kernel", fl, 2.0 * B * N * 256 * (3 if residual is not None else 2) + 2.0 * 2 * B * heads * T * 256, ex):
        check(load().mqdet_biattn_image(_ptr(vn16), vn16.stride(1), vn16.stride(0), _ptr(gT), gT.stride(2), gT.stride(1),
                                        gT.stride(0), _ptr(gbias), gbias.shape[3] if gbias is not None else 0, _ptr(mT),
                                        mT.stride(2), mT.stride(1), mT.stride(0), _ptr(bias), _ptr(gamma), _ptr(residual),
                                        residual.stride(1) if residual is not None else 0,
                                        residual.stride(0) if residual is not None else 0, _ptr(mask), float(clamp), _ptr(out),
                                        out.stride(1), out.stride(0), _ptr(colmax), _ptr(ws), B, heads, N, T, _stream()),
              "biattn_image")
    launch_count += 2
    return out, colmax


def biattn_text_vn(kh, qh, vn16, colmax, clamp, out, rowbias=None):
    """Fused text -> image attention on the image tokens themselves: kh [B,H,T,d], qh [B,H,N,d] (strided views; a head stride of
    0 broadcasts), vn16 [B,N,256] fp16, colmax [B*H,T] fp32 (from biattn_image), rowbias [B,H,T,ld] fp32 (column 0) or None,
    out [B,H,T,256] fp16 view <- softmax_n(scores + rowbias)^T . vn."""
    global launch_count
    _need_cuda(kh, qh, vn16, colmax, out, rowbias)
    B, H, T, d = kh.shape
    N = qh.shape[2]
    for t in (kh, qh, vn16, out):
        if t.stride(-1) != 1 or t.dtype != torch.float16:
            raise _lib.MqdetError("biattn_text_vn: fp16 operands with a contiguous last dimension required")
    # algorithmic work of the text -> image direction (the scores are shared with the other direction in the reference): the
    # image-side value projection and P^T.V_v; bytes: the image tokens once per image, the small text-side operands
    fl = B * (2.0 * N * 256 * H * d + 2.0 * T * N * H * d)
    # executed: S^T recomputed (2.T.N.256 per head) + P^T.vn (2.T.N.256 per head)
    with _Timed("biattn_text_kernel", fl, 2.0 * B * N * 256 + 2.0 * 2 * B * H * T * 256, B * H * 2.0 * (2.0 * T * N * 256)):
        check(load().mqdet_biattn_text_vn(_ptr(kh), kh.stride(2), kh.stride(1), kh.stride(0), _ptr(qh), qh.stride(2), qh.stride(1),
                                          qh.stride(0), _ptr(vn16), vn16.stride(1), 0, vn16.stride(0), _ptr(colmax), _ptr(rowbias),
                                          rowbias.shape[3] if rowbias is not None else 0, float(clamp), _ptr(out), out.stride(2),
                                          out.stride(1), out.stride(0), H, B, T, N, _stream()), "biattn_text_vn")
    launch_count += 1
    return out


def cast_f16(x):
    global launch_count
    _need_cuda(x)
    if x.dtype == torch.float16:
        return x
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    check(load().mqdet_cast_f32_f16(_ptr(x), _ptr(y), x.numel(), _stream()), "cast_f32_f16")
    launch_count += 1
    return y


def cast_f32(x):
    global launch_count
    _need_cuda(x)
    if x.dtype == torch.float32:
        return x
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    check(load().mqdet_cast_f16_f32(_ptr(x), _ptr(y), x.numel(), _stream()), "cast_f16_f32")
    launch_count += 1
    return y


def contrastive_embed(x16, y16, text_token_mask, max_text_len):
    """x16 [B,Q,D] fp16, y16 [B,T,D] fp16, text_token_mask [B,T] bool -> logits [B,Q,max_text_len] fp32:
    x . y^T, -inf on padding tokens and on columns T..max_text_len-1 (GroundingDINO utils.py:242-268)."""
    global launch_count
    _need_cuda(x16, y16, text_token_mask)
    B, Q, _ = x16.shape
    T = y16.shape[1]
    out = torch.empty((B, Q, max_text_len), dtype=torch.float32, device=x16.device)
    gemm(x16, y16, out=out[:, :, :T])
    m8 = text_token_mask.to(torch.uint8).contiguous()
    check(load().mqdet_contrastive_mask(_ptr(out), _ptr(m8), B, Q, T, max_text_len, _stream()), "contrastive_mask")
    launch_count += 1
    return out


def dense_cross_attn(q, kv, heads, dim_head):
    """Flash-style dense cross-attention (PreSelect): q [B,Tq,H*32] fp16 (scaled), kv [B,I,2*H*32] fp16 (K | V halves) ->
    [B,Tq,H*32] fp16 = softmax_i(q.k^T) v per head, without materialising the scores."""
    global launch_count
    _need_cuda(q, kv)
    B, Tq, inner = q.shape
    I = kv.shape[1]
    if q.dtype != torch.float16 or kv.dtype != torch.float16 or q.stride(-1) != 1 or kv.stride(-1) != 1:
        raise _lib.MqdetError("dense_cross_attn: fp16 operands with a contiguous last dimension required")
    out = torch.empty((B, Tq, inner), dtype=torch.float16, device=q.device)
    check(load().mqdet_dense_cross_attn(_ptr(q), q.stride(1), q.stride(0), _ptr(kv), kv.stride(1), kv.stride(0), inner, _ptr(out),
                                        out.stride(1), out.stride(0), B, Tq, I, heads, dim_head, _stream()), "dense_cross_attn")
    launch_count += 1
    return out


def gcp_build_index(mask, S):
    """mask [B, V, T] fp32 0/1 -> (idx int32 [B, T, S] padded with V, counts int32 [B, T])."""
    global launch_count
    _need_cuda(mask)
    B, V, T = mask.shape
    mask = mask.contiguous().float()
    idx = torch.empty((B, T, S), dtype=torch.int32, device=mask.device)
    counts = torch.empty((B, T), dtype=torch.int32, device=mask.device)
    check(load().mqdet_gcp_build_index(_ptr(mask), B, V, T, S, _ptr(idx), _ptr(counts), _stream()), "gcp_build_index")
    launch_count += 1
    return idx, counts


def gcp_sparse_attn(q, kv, idx, heads, dim_head):
    """q [B, T, H*Dh] fp16 (scaled), kv [B, V+1, 2*H*Dh] fp16, idx [B, T, S] int32 -> [B, T, H*Dh] fp16."""
    global launch_count
    _need_cuda(q, kv, idx)
    B, T, inner = q.shape
    V = kv.shape[1] - 1
    S = idx.shape[2]
    out = torch.empty_like(q)
    check(load().mqdet_gcp_sparse_attn(_ptr(q), _ptr(kv), _ptr(idx), _ptr(out), B, T, V, S, heads, dim_head, _stream()),
          "gcp_sparse_attn")
    launch_count += 1
    return out


def gcp_gate_residual_ln(h1, w2, s, x, gamma, beta, eps=1e-5, want_gate=False):
    """g = tanh(h1 . w2); x1 = s*g + x; returns (x1 fp32, LN(x1) fp16[, g])."""
    global launch_count
    _need_cuda(h1, w2, s, x)
    D = s.shape[-1]
    rows = s.numel() // D
    Dg = h1.shape[-1]
    x1 = torch.empty_like(s)
    ln = torch.empty(s.shape, dtype=torch.float16, device=s.device)
    g = torch.empty(s.shape[:-1], dtype=torch.float32, device=s.device) if want_gate else None
    check(load().mqdet_gcp_gate_residual_ln(_ptr(h1), _ptr(w2), Dg, _ptr(s), _ptr(x), _ptr(gamma), _ptr(beta), float(eps),
                                            rows, D, _ptr(x1), _ptr(ln), _ptr(g), _stream()), "gcp_gate_residual_ln")
    launch_count += 1
    return (x1, ln, g) if want_gate else (x1, ln)


def argsort_desc(scores):
    global launch_count
    _need_cuda(scores)
    n = scores.numel()
    order = torch.empty((n,), dtype=torch.int64, device=scores.device)
    if n:
        check(load().mqdet_argsort_desc(_ptr(scores), n, _ptr(order), _stream()), "argsort_desc")
        launch_count += 1
    return order


def ml_nms_device(boxes, scores, labels, thresh, max_det=0):
    """Device-resident multi-label NMS. Returns (keep int64 [n] (first num valid, ascending), num int32 [1])."""
    global launch_count
    _need_cuda(boxes, scores, labels)
    n = boxes.shape[0]
    keep = torch.empty((max(n, 1),), dtype=torch.int64, device=boxes.device)
    num = torch.zeros((1,), dtype=torch.int32, device=boxes.device)
    if n == 0:
        return keep[:0], num
    boxes = boxes.contiguous().float()
    scores = scores.contiguous().float()
    labels = labels.contiguous().float()
    order = argsort_desc(scores)
    ws = torch.empty((int(load().mqdet_ml_nms_workspace_bytes(n)),), dtype=torch.uint8, device=boxes.device)
    check(load().mqdet_ml_nms(_ptr(boxes), _ptr(scores), _ptr(labels), _ptr(order), n, float(thresh), int(max_det),
                              _ptr(keep), _ptr(num), _ptr(ws), _stream()), "ml_nms")
    launch_count += 5
    return keep, num


def ml_nms(boxes, scores, labels, thresh):
    """Drop-in for maskrcnn_benchmark._C.ml_nms (csrc/ml_nms.h:11-27): kept original indices, ascending."""
    if boxes.numel() == 0:
        return torch.empty((0,), dtype=torch.int64, device="cpu")  # reference returns an empty CPU tensor (:19-20)
    keep, num = ml_nms_device(boxes, scores, labels, thresh)
    return keep[: int(num.item())]


# ----------------------------------------------------------------------------------------------------------------------
# DyHead vision path
# ----------------------------------------------------------------------------------------------------------------------
class Levels:
    """FPN level table: sizes [(H, W)], row offsets into the concatenated [B, N, C] tensor, device segment tables."""

    def __init__(self, sizes, device):
        import numpy as np
        self.sizes = [(int(h), int(w)) for h, w in sizes]
        self.n = len(self.sizes)
        hw = np.asarray(self.sizes, dtype=np.int32).reshape(-1, 2)
        self.hw_host = np.ascontiguousarray(hw)
        self.hw_ptr = self.hw_host.ctypes.data_as(ctypes.c_void_p)
        off = [0]
        for h, w in self.sizes:
            off.append(off[-1] + h * w)
        self.off = off
        self.N = off[-1]
        self.N1 = self.N - self.sizes[0][0] * self.sizes[0][1]
        self.seg_all = torch.tensor(off, dtype=torch.int32, device=device)  # levels 0..L-1 over N rows
        self.seg_tail = torch.tensor([o - off[1] for o in off[1:]], dtype=torch.int32, device=device)  # levels 1..L-1
        # GAP weights of the align_corners bilinear upsample (level l+1 -> l), normalised to sum 1 per segment:
        # GAP(up(z)) = sum_q w[q] z[q] with w separable (column sums of the 1-D interpolation matrices)
        ws = []
        for l in range(self.n - 1):
            (H, W), (Hs, Ws) = self.sizes[l], self.sizes[l + 1]
            ws.append((torch.outer(_upsample_colsum(Hs, H), _upsample_colsum(Ws, W)) / float(H * W)).reshape(-1))
        self.up_w = torch.cat(ws).float().to(device) if ws else None


_levels_cache = {}


def get_levels(sizes, device):
    """Cached Levels (building one uploads small tables to the device)."""
    key = (tuple((int(h), int(w)) for h, w in sizes), str(device))
    lv = _levels_cache.get(key)
    if lv is None:
        lv = _levels_cache[key] = Levels(sizes, device)
    return lv


def _upsample_colsum(n_in, n_out):
    """column sums of the [n_out, n_in] align_corners=True linear-interpolation matrix (fp32 like ATen)."""
    import numpy as np
    w = np.zeros(n_in, dtype=np.float64)
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    for i in range(n_out):
        src = np.float32(scale * np.float32(i))
        i0 = int(src)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        lam = float(src - np.float32(i0))
        w[i0] += 1.0 - lam
        w[i1] += lam
    return torch.from_numpy(w)


def dcn_cols(x16, om, levels, branch):
    """x16 [B,N,256] fp16, om [B,N,om_ld] fp32 or None -> fp16 column matrix [B*rows, 2304] for DyConv[branch]."""
    global launch_count
    _need_cuda(x16, om)
    B, N, C = x16.shape
    rows = levels.N if branch == 1 else levels.N1
    cols = torch.empty((B * rows, 9 * C), dtype=torch.float16, device=x16.device)
    check(load().mqdet_dcn_cols(_ptr(x16), _ptr(om), om.shape[-1] if om is not None else 0, levels.hw_ptr, levels.n, B, C,
                                int(branch), _ptr(cols), _stream()), "dcn_cols")
    launch_count += 1
    return cols


def dcn_conv(x16, om, levels, branches, weights, biases):
    """DyConv's DCNv2 convolutions as one implicit GEMM (no column matrix): x16 [B,N,256] fp16, om [B,N,om_ld] fp32 or None,
    branches: list of 0/1/2, weights: fp16 [256, 2304] (k = tap*256 + c) each, biases: fp32 [256] or None each
    -> list of fp16 [B*rows_j, 256]."""
    global launch_count
    _need_cuda(x16, om, *weights)
    B, N, C = x16.shape
    n = len(branches)
    ys = [torch.empty((B * (levels.N if k == 1 else levels.N1), 256), dtype=torch.float16, device=x16.device) for k in branches]
    br = (ctypes.c_int32 * n)(*[int(k) for k in branches])
    wp = (ctypes.c_void_p * n)(*[w.data_ptr() for w in weights])
    bp = (ctypes.c_void_p * n)(*[(b.data_ptr() if b is not None else None) for b in biases])
    yp = (ctypes.c_void_p * n)(*[y.data_ptr() for y in ys])
    for w in weights:
        if w.dtype != torch.float16 or tuple(w.shape) != (256, 9 * C) or not w.is_contiguous():
            raise _lib.MqdetError(f"dcn_conv: weights must be contiguous fp16 [256, {9 * C}] (got {w.dtype} {tuple(w.shape)})")
    rows = sum(y.shape[0] for y in ys)
    with _Timed("dcn_conv_kernel", 2.0 * rows * 256 * 9 * C, 2.0 * (B * N * C + rows * 256 + n * 256 * 9 * C) + (4.0 * B * N * 27 if om is not None else 0.0)):
        check(load().mqdet_dcn_conv(_ptr(x16), _ptr(om), om.shape[-1] if om is not None else 0, levels.hw_ptr, levels.n, B, C, n,
                                    ctypes.cast(br, ctypes.c_void_p), ctypes.cast(wp, ctypes.c_void_p),
                                    ctypes.cast(bp, ctypes.c_void_p), ctypes.cast(yp, ctypes.c_void_p), _stream()), "dcn_conv")
    launch_count += 1
    return ys


def conv3x3_small(x16, w16_, bias, levels, ld=32):
    """Plain 3x3 / pad 1 conv with <= 32 output channels over all levels, no column matrix (the DyConv offset/mask conv):
    x16 [B,N,256] fp16, w16_ [O, 2304] fp16 (k = tap*256 + c), bias [O] fp32 -> [B*N, ld] fp32 (columns >= O untouched)."""
    global launch_count
    _need_cuda(x16, w16_, bias)
    B, N, C = x16.shape
    O = w16_.shape[0]
    out = torch.empty((B * N, ld), dtype=torch.float32, device=x16.device)
    check(load().mqdet_conv3x3_small(_ptr(x16), _ptr(w16_), _ptr(bias), levels.hw_ptr, levels.n, B, C, O, _ptr(out), ld,
                                     _stream()), "conv3x3_small")
    launch_count += 1
    return out


def chan_stats(y16, seg, B, rows_per_img, row_weights=None):
    global launch_count
    nseg = seg.numel() - 1
    C = y16.shape[-1]
    partial = torch.empty((int(load().mqdet_chan_stats_floats(B, nseg, C)),), dtype=torch.float32, device=y16.device)
    check(load().mqdet_chan_stats(_ptr(y16), _ptr(seg), nseg, B, rows_per_img, C, _ptr(row_weights), _ptr(partial),
                                  _stream()), "chan_stats")
    launch_count += 1
    return partial


def gn_attn(partial, seg, B, C, groups, weighted, gn_w, gn_b, eps, attn_w, attn_b):
    global launch_count
    nseg = seg.numel() - 1
    affine = torch.empty((B, nseg, 2, C), dtype=torch.float32, device=partial.device)
    attn = torch.empty((B, nseg), dtype=torch.float32, device=partial.device)
    check(load().mqdet_gn_attn(_ptr(partial), _ptr(seg), nseg, B, C, groups, int(weighted), _ptr(gn_w), _ptr(gn_b),
                               float(eps), _ptr(attn_w), _ptr(attn_b), _ptr(affine), _ptr(attn), _stream()), "gn_attn")
    launch_count += 1
    return affine, attn


def dyconv_combine(y1, y2, y0, aff1, aff2, aff0, at1, at2, at0, levels, B):
    """-> (mid [B,N,C] fp16, mid_sums [B, L, chunks, C] fp32: per-channel sums of `mid` over pixel ranges, for DyReLU's pool)."""
    global launch_count
    C = y1.shape[-1]
    mid = torch.empty((B, levels.N, C), dtype=torch.float16, device=y1.device)
    sums = torch.empty((B, levels.n, int(load().mqdet_dyconv_combine_chunks()), C), dtype=torch.float32, device=y1.device)
    check(load().mqdet_dyconv_combine(_ptr(y1), _ptr(y2), _ptr(y0), _ptr(aff1), _ptr(aff2), _ptr(aff0), _ptr(at1),
                                      _ptr(at2), _ptr(at0), levels.hw_ptr, levels.n, B, C, _ptr(mid), _ptr(sums), _stream()),
          "dyconv_combine")
    launch_count += 1
    return mid, sums


def dyrelu(mid, levels, w1, b1, w2, b2, mid_sums=None):
    """DyReLU over every level of mid [B,N,256] fp16 -> fp16.  ``mid_sums`` = the per-range channel sums dyconv_combine
    produced (else they are taken from `mid` by chan_stats)."""
    global launch_count
    B, N, C = mid.shape
    if mid_sums is None:
        partial, chunks, stats = chan_stats(mid, levels.seg_all, B, N), 32, 3
    else:
        partial, chunks, stats = mid_sums, mid_sums.shape[2], 1
    coef = torch.empty((B, levels.n, 4, C), dtype=torch.float32, device=mid.device)
    check(load().mqdet_dyrelu_coef(_ptr(partial), chunks, stats, _ptr(levels.seg_all), levels.n, B, C, w1.shape[0], _ptr(w1),
                                   _ptr(b1), _ptr(w2), _ptr(b2), _ptr(coef), _stream()), "dyrelu_coef")
    out = torch.empty_like(mid)
    check(load().mqdet_dyrelu_apply(_ptr(mid), _ptr(coef), levels.hw_ptr, levels.n, B, C, _ptr(out), _stream()),
          "dyrelu_apply")
    launch_count += 2
    return out


# ----------------------------------------------------------------------------------------------------------------------
# ATSS post-processing
# ----------------------------------------------------------------------------------------------------------------------
def base_anchor(stride, size):
    """generate_anchors for ONE square anchor (anchor_generator.py:355-425): window [0,0,s-1,s-1] scaled to `size`."""
    import math
    ctr = 0.5 * (stride - 1)
    ws = float(round(math.sqrt(stride * stride)))
    w = ws * (size / stride)
    return [ctr - 0.5 * (w - 1), ctr - 0.5 * (w - 1), ctr + 0.5 * (w - 1), ctr + 0.5 * (w - 1)]


def make_tokmap(positive_map, num_classes, device):
    """{label(1-based): [token positions]} -> int32 [C, max_tok] padded with -1."""
    max_tok = max([len(v) if not isinstance(v, int) else 1 for v in positive_map.values()] + [1])
    tm = torch.full((num_classes, max_tok), -1, dtype=torch.int32)
    for label, toks in positive_map.items():
        toks = [toks] if isinstance(toks, int) else list(toks)
        if 1 <= label <= num_classes:
            tm[label - 1, : len(toks)] = torch.tensor(toks, dtype=torch.int32)
    return tm.to(device)


def atss_postprocess(logits, reg_ctr, tokmap, levels, strides, anchor_sizes, reg_scales, img_w, img_h, *, pre_nms_thresh=0.05,
                     pre_nms_top_n=1000, nms_thresh=0.6, max_det=100, max_out=128, want_keys=False, class_labels=None):
    """logits [B,N,T], reg_ctr [B,N,5] -> dict(det [B,max_out,6], num [B], + the pre-NMS candidates). All on device.
    tokmap int32 [C, max_tok] (shared) or [B, C, max_tok] (one positive map per image: batched prompt chunks);
    class_labels int32 [C] / [B, C] or None (label of score column c = c + 1)."""
    import numpy as np
    global launch_count
    _need_cuda(logits, reg_ctr, tokmap)
    B, N, T = logits.shape
    C, max_tok = tokmap.shape[-2:]
    tm_stride = C * max_tok if tokmap.dim() == 3 else 0
    if tokmap.dim() == 3 and tokmap.shape[0] != B:
        raise ValueError("per-image tokmap must have one table per batch element")
    lab_stride = 0
    if class_labels is not None:
        if class_labels.dtype != torch.int32 or class_labels.shape[-1] != C:
            raise ValueError("class_labels must be int32 [C] or [B, C]")
        lab_stride = C if class_labels.dim() == 2 else 0
    dev = logits.device
    L = levels.n
    stride_h = np.asarray(strides, dtype=np.float32)
    base_h = np.asarray([base_anchor(s, a) for s, a in zip(strides, anchor_sizes)], dtype=np.float32)
    scale_h = np.asarray(reg_scales, dtype=np.float32)
    S = (L * pre_nms_top_n + 255) // 256 * 256
    ws = torch.empty((int(load().mqdet_atss_workspace_bytes(levels.hw_ptr, L, C, B)),), dtype=torch.uint8, device=dev)
    lvl_counts = torch.empty((B, L), dtype=torch.int32, device=dev)
    ob = torch.empty((B, S, 4), dtype=torch.float32, device=dev)
    osc = torch.empty((B, S), dtype=torch.float32, device=dev)
    ol = torch.empty((B, S), dtype=torch.float32, device=dev)
    okey = torch.empty((B, S), dtype=torch.int64, device=dev) if want_keys else None
    cb, csc, cl = torch.empty_like(ob), torch.empty_like(osc), torch.empty_like(ol)
    totals = torch.empty((B,), dtype=torch.int32, device=dev)
    check(load().mqdet_atss_candidates(_ptr(logits), _dt(logits), _ptr(reg_ctr), _ptr(tokmap), tm_stride, _ptr(class_labels),
                                       lab_stride, C, max_tok, T, levels.hw_ptr, L,
                                       stride_h.ctypes.data_as(ctypes.c_void_p), base_h.ctypes.data_as(ctypes.c_void_p),
                                       scale_h.ctypes.data_as(ctypes.c_void_p), B, float(pre_nms_thresh), int(pre_nms_top_n),
                                       S, float(img_w), float(img_h), _ptr(ws), _ptr(lvl_counts), _ptr(ob), _ptr(osc),
                                       _ptr(ol), _ptr(okey), _ptr(cb), _ptr(csc), _ptr(cl), _ptr(totals), _stream()),
          "atss_candidates")
    nws = torch.empty((int(load().mqdet_ml_nms_batched_workspace_bytes(B, S)),), dtype=torch.uint8, device=dev)
    keep = torch.empty((B, S), dtype=torch.int64, device=dev)
    num = torch.empty((B,), dtype=torch.int32, device=dev)
    check(load().mqdet_ml_nms_batched(_ptr(cb), _ptr(csc), _ptr(cl), _ptr(totals), B, S, float(nms_thresh), int(max_det),
                                      _ptr(keep), _ptr(num), _ptr(nws), _stream()), "ml_nms_batched")
    # packed fixed-shape result [B, max_out + 1, 6]: rows 0..max_out-1 = detections, row max_out = (count, 0, ...)
    packed = torch.empty((B, max_out + 1, 6), dtype=torch.float32, device=dev)
    check(load().mqdet_gather_detections(_ptr(cb), _ptr(csc), _ptr(cl), _ptr(keep), _ptr(num), B, S, max_out, max_out + 1,
                                         _ptr(packed), _stream()), "gather_detections")
    launch_count += 10
    return {"det": packed[:, :max_out], "num": num, "det_packed": packed, "cand_boxes": cb, "cand_scores": csc,
            "cand_labels": cl, "cand_totals": totals, "level_counts": lvl_counts, "level_keys": okey, "keep": keep}


def _level_anchor_tables(strides, anchor_sizes, reg_scales=None):
    import numpy as np
    stride_h = np.ascontiguousarray(np.asarray(strides, dtype=np.float32))
    base_h = np.ascontiguousarray(np.asarray([base_anchor(s, a) for s, a in zip(strides, anchor_sizes)], dtype=np.float32))
    scale_h = None if reg_scales is None else np.ascontiguousarray(np.asarray(reg_scales, dtype=np.float32))
    return stride_h, base_h, scale_h


def _gt_pack(gt_boxes, gt_labels, gt_count, B):
    _need_cuda(gt_boxes, gt_labels, gt_count)
    if gt_boxes.dim() != 3 or gt_boxes.shape[0] != B or gt_boxes.shape[2] != 4:
        raise ValueError(f"gt_boxes must be [B={B}, Gmax, 4]; got {tuple(gt_boxes.shape)}")
    G = gt_boxes.shape[1]
    if tuple(gt_labels.shape) != (B, G) or tuple(gt_count.shape) != (B,):
        raise ValueError(f"gt_labels must be [B, Gmax] = {(B, G)} and gt_count [B]; got {tuple(gt_labels.shape)}, "
                         f"{tuple(gt_count.shape)}")
    return (gt_boxes.float().contiguous(), gt_labels.to(torch.int32).contiguous(), gt_count.to(torch.int32).contiguous(), G)


def atss_targets(gt_boxes, gt_labels, gt_count, levels, strides, anchor_sizes, topk=9):
    """ATSS target assignment (loss.py:655-832) for a fixed-capacity GT pack: gt_boxes [B, Gmax, 4] xyxy, gt_labels [B, Gmax],
    gt_count [B] (device) -> dict(match int32 [B, N] (assigned GT, -1 = unmatched), img_stats fp32 [B, 2] (positives, sum of
    centerness targets per image), norm fp32 [4] (the batch totals; ``norm[:2]`` is what data-parallel ranks all-reduce)).
    All on the device, no host synchronisation."""
    global launch_count
    B = gt_count.shape[0]
    gt_boxes, gt_labels, gt_count, G = _gt_pack(gt_boxes, gt_labels, gt_count, B)
    dev = gt_boxes.device
    stride_h, base_h, _ = _level_anchor_tables(strides, anchor_sizes)
    N = levels.N
    ws = torch.empty((int(load().mqdet_atss_assign_workspace_bytes(B, N)),), dtype=torch.uint8, device=dev)
    match = torch.empty((B, N), dtype=torch.int32, device=dev)
    img_stats = torch.empty((B, 2), dtype=torch.float32, device=dev)
    norm = torch.empty((4,), dtype=torch.float32, device=dev)
    check(load().mqdet_atss_assign(_ptr(gt_boxes), _ptr(gt_labels), _ptr(gt_count), B, G, levels.hw_ptr, levels.n,
                                   stride_h.ctypes.data_as(ctypes.c_void_p), base_h.ctypes.data_as(ctypes.c_void_p), int(topk),
                                   _ptr(ws), _ptr(match), _ptr(img_stats), _ptr(norm), _stream()), "atss_assign")
    launch_count += 4
    return {"match": match, "img_stats": img_stats, "norm": norm}


def atss_loss(logits, reg_ctr, gt_boxes, gt_labels, gt_count, gt_tokens, levels, strides, anchor_sizes, reg_scales, text_mask=None, *,
              targets=None, world=1, topk=9, alpha=0.25, gamma=2.0, reg_weight=2.0, token_weight=1.0):
    """The MQ-GLIP pre-training detection losses (loss.py:850-1201 with the shipped flags) and their gradients at the head outputs.

    logits fp32 [B, N, T] (dot-product token logits), reg_ctr fp32 [B, N, 5] (raw box / centerness GEMM output, before the per-level
    ``reg_scales``), the GT pack of ``atss_targets`` plus gt_tokens [B, Gmax, T] (positive_map rows), text_mask [B, T] or None ->
    (losses fp32 [4] = (loss_reg, loss_centerness, loss_dot_product_token, loss_cls = 0), d_logits fp32 [B, N, T],
    d_reg_ctr fp32 [B, N, 5]).  ``targets``: the result of ``atss_targets`` (its ``norm[:2]`` summed over ``world`` ranks), else
    computed here for one rank.  All on the device, no host synchronisation: capturable in a CUDA graph at a fixed Gmax."""
    global launch_count
    _need_cuda(logits, reg_ctr, gt_tokens, text_mask)
    B, N, T = logits.shape
    if N != levels.N or tuple(reg_ctr.shape) != (B, N, 5):
        raise ValueError(f"logits [B, N={levels.N}, T] and reg_ctr [B, N, 5] required; got {tuple(logits.shape)}, "
                         f"{tuple(reg_ctr.shape)}")
    for t in (logits, reg_ctr):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise _lib.MqdetError("atss_loss: logits / reg_ctr must be contiguous fp32")
    gt_boxes, gt_labels, gt_count, G = _gt_pack(gt_boxes, gt_labels, gt_count, B)
    if tuple(gt_tokens.shape) != (B, G, T):
        raise ValueError(f"gt_tokens must be [B, Gmax, T] = {(B, G, T)}; got {tuple(gt_tokens.shape)}")
    if text_mask is not None and tuple(text_mask.shape) != (B, T):
        raise ValueError(f"text_mask must be [B, T] = {(B, T)}; got {tuple(text_mask.shape)}")
    if targets is None:
        targets = atss_targets(gt_boxes, gt_labels, gt_count, levels, strides, anchor_sizes, topk=topk)
    dev = logits.device
    tok = gt_tokens.float().contiguous()
    tm = None if text_mask is None else text_mask.float().contiguous()
    stride_h, base_h, scale_h = _level_anchor_tables(strides, anchor_sizes, reg_scales)
    ws = torch.empty((int(load().mqdet_atss_loss_workspace_floats(B, N)),), dtype=torch.float32, device=dev)
    losses = torch.empty((4,), dtype=torch.float32, device=dev)
    d_logits = torch.empty_like(logits)
    d_reg_ctr = torch.empty_like(reg_ctr)
    with _Timed("atss_loss", 0.0, 8.0 * B * N * T + 40.0 * B * N):
        check(load().mqdet_atss_loss(_ptr(logits), _ptr(reg_ctr), _ptr(targets["match"]), _ptr(gt_boxes), _ptr(gt_labels), _ptr(tok), B, G,
                                     T, _ptr(tm), levels.hw_ptr, levels.n, stride_h.ctypes.data_as(ctypes.c_void_p),
                                     base_h.ctypes.data_as(ctypes.c_void_p), scale_h.ctypes.data_as(ctypes.c_void_p),
                                     _ptr(targets["norm"]), float(world), float(alpha), float(gamma), float(reg_weight),
                                     float(token_weight), _ptr(ws), _ptr(losses), _ptr(d_logits), _ptr(d_reg_ctr), _stream()),
              "atss_loss")
    launch_count += 3
    return losses, d_logits, d_reg_ctr


def anchors(grid_h, grid_w, stride, size, img_w, img_h, device):
    """Anchors [H*W, 4] + visibility [H*W] of one level (anchor_generator.py:72-109)."""
    import numpy as np
    global launch_count
    out = torch.empty((grid_h * grid_w, 4), dtype=torch.float32, device=device)
    vis = torch.empty((grid_h * grid_w,), dtype=torch.uint8, device=device)
    base = np.asarray(base_anchor(stride, size), dtype=np.float32)
    check(load().mqdet_anchors(_ptr(out), _ptr(vis), grid_h, grid_w, float(stride), base.ctypes.data_as(ctypes.c_void_p),
                               float(img_w), float(img_h), _stream()), "anchors")
    launch_count += 1
    return out, vis.bool()


# ----------------------------------------------------------------------------------------------------------------------
# Swin / FPN glue
# ----------------------------------------------------------------------------------------------------------------------
def patchify4(img):
    """[B,3,H,W] fp32 -> (fp16 [B*Hp*Wp, 48], Hp, Wp)."""
    global launch_count
    _need_cuda(img)
    B, _, H, W = img.shape
    Hp, Wp = (H + 3) // 4, (W + 3) // 4
    img = img.float().contiguous()
    out = torch.empty((B * Hp * Wp, 48), dtype=torch.float16, device=img.device)
    check(load().mqdet_patchify4(_ptr(img), B, H, W, _ptr(out), _stream()), "patchify4")
    launch_count += 1
    return out, Hp, Wp


def swin_window_attn(qkv16, qkv_bias, bias_dense, B, H, W, heads, window, shift, scale):
    global launch_count
    _need_cuda(qkv16, qkv_bias, bias_dense)
    C = qkv16.shape[-1] // 3
    out = torch.empty((B * H * W, C), dtype=torch.float16, device=qkv16.device)
    check(load().mqdet_swin_window_attn(_ptr(qkv16), _ptr(qkv_bias), _ptr(bias_dense), B, H, W, heads, window, shift,
                                        float(scale), _ptr(out), _stream()), "swin_window_attn")
    launch_count += 1
    return out


def patch_merge_ln(x32, B, H, W, gamma, beta, eps):
    global launch_count
    _need_cuda(x32)
    C = x32.shape[-1]
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    out = torch.empty((B * H2 * W2, 4 * C), dtype=torch.float16, device=x32.device)
    check(load().mqdet_patch_merge_ln(_ptr(x32), B, H, W, C, _ptr(gamma), _ptr(beta), float(eps), _ptr(out), _stream()),
          "patch_merge_ln")
    launch_count += 1
    return out, H2, W2


def upsample_add(lateral16, top16, B, H, W, Hs, Ws):
    global launch_count
    _need_cuda(lateral16, top16)
    C = lateral16.shape[-1]
    out = torch.empty_like(lateral16)
    check(load().mqdet_upsample_add(_ptr(lateral16), _ptr(top16), B, H, W, Hs, Ws, C, _ptr(out), _stream()), "upsample_add")
    launch_count += 1
    return out


def im2col3x3(x16, B, H, W, stride=1, relu_in=False):
    """x16: fp16 [B, H*W, C] (may be a batch-strided view with contiguous rows) -> cols [B*Ho*Wo, 9C], Ho, Wo."""
    global launch_count
    _need_cuda(x16)
    C = x16.shape[-1]
    assert x16.stride(-1) == 1 and x16.stride(-2) == C
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    cols = torch.empty((B * Ho * Wo, 9 * C), dtype=torch.float16, device=x16.device)
    check(load().mqdet_im2col3x3(_ptr(x16), x16.stride(0) if x16.dim() == 3 else H * W * C, B, H, W, C, stride,
                                 int(bool(relu_in)), _ptr(cols), _stream()), "im2col3x3")
    launch_count += 1
    return cols, Ho, Wo


def avgpool2_levels(x16, levels):
    """fp16 [B,N,C] pyramid -> fp32 [B, I, C] pooled tokens (AvgPool2d(2) per level, concatenated)."""
    global launch_count
    _need_cuda(x16)
    B, N, C = x16.shape
    I = sum((h // 2) * (w // 2) for h, w in levels.sizes)
    out = torch.empty((B, I, C), dtype=torch.float32, device=x16.device)
    check(load().mqdet_avgpool2_levels(_ptr(x16), levels.hw_ptr, levels.n, B, C, _ptr(out), _stream()), "avgpool2_levels")
    launch_count += 1
    return out


def roi_align_levels(pyr16, levels, scales, rois, pooled=7, sampling_ratio=0, mean_only=True):
    """Pooler (LevelMapper + aligned ROIAlign per level) over the fp16 pyramid [B,N,C]: rois [R,5] fp32 (image index, x1, y1, x2,
    y2) -> ([R,C] fp32 mean over the pooled bins | [R,C,pooled,pooled] fp32, level int32 [R])."""
    import numpy as np
    global launch_count
    _need_cuda(pyr16, rois)
    B, N, C = pyr16.shape
    R = rois.shape[0]
    rois = rois.float().contiguous()
    out = torch.empty((R, C) if mean_only else (R, C, pooled, pooled), dtype=torch.float32, device=pyr16.device)
    lvl = torch.empty((R,), dtype=torch.int32, device=pyr16.device)
    sc = np.asarray(scales, dtype=np.float32)
    check(load().mqdet_roi_align_levels(_ptr(pyr16), levels.hw_ptr, levels.n, sc.ctypes.data_as(ctypes.c_void_p), B, C, _ptr(rois), R,
                                        int(pooled), int(sampling_ratio), int(bool(mean_only)), _ptr(out), _ptr(lvl), _stream()),
          "roi_align_levels")
    launch_count += 1
    return out, lvl


def ms_deform_attn(value16, proj32, aw_col0, ref, levels, heads, points, out_dtype=torch.float16):
    """Fused multi-scale deformable attention core: value16 [B,Nv,heads*32] fp16, proj32 [B*Q, >= heads*L*P*3] fp32 (sampling
    offsets | attention logits from column aw_col0), ref [B,Q,L,2|4] fp32 -> [B,Q,heads*32]."""
    global launch_count
    _need_cuda(value16, proj32, ref)
    B, Nv, E = value16.shape
    Q = ref.shape[1]
    if value16.dtype != torch.float16 or proj32.dtype != torch.float32 or not value16.is_contiguous() or proj32.stride(-1) != 1:
        raise _lib.MqdetError("ms_deform_attn: value fp16 contiguous, proj fp32 with contiguous rows required")
    if Nv != levels.N or ref.shape[2] != levels.n:
        raise _lib.MqdetError("ms_deform_attn: value rows / reference points do not match the level table")
    out = torch.empty((B, Q, E), dtype=out_dtype, device=value16.device)
    check(load().mqdet_ms_deform_attn(_ptr(value16), _ptr(proj32), proj32.stride(0), int(aw_col0), _ptr(ref), ref.shape[-1],
                                      levels.hw_ptr, levels.n, B, Q, heads, E // heads, points, _ptr(out), _dt(out), _stream()),
          "ms_deform_attn")
    launch_count += 1
    return out


# ----------------------------------------------------------------------------------------------------------------------
# GroundingDINO encoder / decoder assembly (csrc/gdino_asm.cu)
# ----------------------------------------------------------------------------------------------------------------------
def add_cast(a32, b32=None, rowgate=None, *, out16=True, out32=False):
    """(a + b) * rowgate[row] over contiguous fp32 [..., D] tensors -> fp16 and / or fp32 (a gated-off row is exactly 0)."""
    global launch_count
    _need_cuda(a32, b32, rowgate)
    if a32.dtype != torch.float32 or (b32 is not None and (b32.dtype != torch.float32 or b32.shape != a32.shape)):
        raise TypeError("add_cast: fp32 tensors of one shape expected")
    a32 = a32.contiguous()
    b32 = None if b32 is None else b32.contiguous()
    D = a32.shape[-1]
    rows = a32.numel() // D
    if rowgate is not None and (rowgate.dtype != torch.float32 or rowgate.numel() != rows):
        raise ValueError("add_cast: rowgate must be fp32 with one entry per row")
    o16 = torch.empty(a32.shape, dtype=torch.float16, device=a32.device) if out16 else None
    o32 = torch.empty(a32.shape, dtype=torch.float32, device=a32.device) if out32 else None
    check(load().mqdet_add_cast(_ptr(a32), _ptr(b32), _ptr(rowgate), rows, D, _ptr(o16), _ptr(o32), _stream()), "add_cast")
    launch_count += 1
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def groupnorm_rows(x, groups, gamma, beta, eps=1e-5, *, out16=True, out32=False):
    """nn.GroupNorm(groups, C) over x [B, HW, C] (fp16 / fp32 rows) -> fp16 and / or fp32 [B, HW, C]."""
    global launch_count
    _need_cuda(x, gamma, beta)
    x = x.contiguous()
    B, HW, C = x.shape
    ws = torch.empty((int(load().mqdet_groupnorm_rows_workspace_floats(B, C)),), dtype=torch.float32, device=x.device)
    o16 = torch.empty(x.shape, dtype=torch.float16, device=x.device) if out16 else None
    o32 = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out32 else None
    check(load().mqdet_groupnorm_rows(_ptr(x), _dt(x), B, HW, C, int(groups), _ptr(gamma), _ptr(beta), float(eps), _ptr(o16),
                                      _ptr(o32), _ptr(ws), _stream()), "groupnorm_rows")
    launch_count += 2
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def box_refine_sine(ref_in, valid_ratios, *, delta=None, ref_is_logit=False, want_sine=True):
    """Decoder box refinement + conditional query embedding.  ref_in fp32 [B, nq, 4]; valid_ratios fp32 [B, L, 2]; delta fp32
    [B, nq, >=4] (row stride = its last-dim size) or None -> (ref [B,nq,4], ref_input [B,nq,L,4], sine fp16 [B,nq,512] | None)."""
    global launch_count
    _need_cuda(ref_in, valid_ratios, delta)
    B, nq, _ = ref_in.shape
    L = valid_ratios.shape[1]
    ref_in = ref_in.float().contiguous()
    vr = valid_ratios.float().contiguous()
    ldd = 0
    if delta is not None:
        if delta.dtype != torch.float32 or delta.stride(-1) != 1:
            raise TypeError("box_refine_sine: delta must be fp32, last dim contiguous")
        d2 = delta.reshape(B * nq, delta.shape[-1])
        ldd = d2.stride(0)
        delta = d2
    ref = torch.empty((B, nq, 4), dtype=torch.float32, device=ref_in.device)
    ref_input = torch.empty((B, nq, L, 4), dtype=torch.float32, device=ref_in.device)
    sine = torch.empty((B, nq, 512), dtype=torch.float16, device=ref_in.device) if want_sine else None
    check(load().mqdet_box_refine_sine(_ptr(delta), ldd, _ptr(ref_in), int(bool(ref_is_logit)), _ptr(vr), B, nq, L, _ptr(ref),
                                       _ptr(ref_input), _ptr(sine), _stream()), "box_refine_sine")
    launch_count += 1
    return ref, ref_input, sine


def gdino_detections(logits, boxes, tokmap, img_wh, box_threshold, max_out=None):
    """Raw class logits fp32 [B, nq, T] + boxes fp32 [B, nq, 4] (cxcywh, normalised) -> packed [B, max_out + 1, 6]
    (x1, y1, x2, y2, score, label; last row = count).  tokmap int32 [C, max_tok]; img_wh fp32 [B, 2] = (W, H)."""
    global launch_count
    _need_cuda(logits, boxes, tokmap, img_wh)
    B, nq, T = logits.shape
    C, max_tok = tokmap.shape
    max_out = nq if max_out is None else int(max_out)
    out = torch.empty((B, max_out + 1, 6), dtype=torch.float32, device=logits.device)
    ws = torch.empty((int(load().mqdet_gdino_detections_workspace_floats(B, nq)),), dtype=torch.float32, device=logits.device)
    check(load().mqdet_gdino_detections(_ptr(logits.float().contiguous()), T, _ptr(boxes.float().contiguous()), _ptr(tokmap), C,
                                        max_tok, _ptr(img_wh.float().contiguous()), float(box_threshold), B, nq, max_out,
                                        _ptr(out), _ptr(ws), _stream()), "gdino_detections")
    launch_count += 2
    return out


# ----------------------------------------------------------------------------------------------------------------------
# Training side (csrc/train.cu): GCP backward pieces, token focal loss, clipping + AdamW
# ----------------------------------------------------------------------------------------------------------------------
def transpose_cast(x, scale=1.0):
    """x [R, C] (fp16 / fp32, contiguous rows) -> fp16 [C, Rp] with Rp = R rounded up to 8, the padding columns zero: the K-major
    operand of a weight-gradient product dW = dY^T X (K = the row dimension)."""
    global launch_count
    _need_cuda(x)
    if x.dim() != 2 or x.stride(1) != 1:
        raise _lib.MqdetError("transpose_cast: 2-D tensor with contiguous rows required")
    R, C = x.shape
    Rp = (R + 7) // 8 * 8
    out = torch.empty((C, Rp), dtype=torch.float16, device=x.device)
    check(load().mqdet_transpose_cast(_ptr(x), _dt(x), R, C, x.stride(0), float(scale), _ptr(out), Rp, _stream()), "transpose_cast")
    launch_count += 1
    return out


def transpose_cast_batched(x):
    """x [nb2, nb1, R, C] (fp16 / fp32, arbitrary batch / row strides, contiguous last dim) -> fp16 [nb2, nb1, C, Rp] contiguous,
    Rp = R rounded up to 8 with zero padding."""
    global launch_count
    _need_cuda(x)
    if x.dim() != 4 or x.stride(3) != 1:
        raise _lib.MqdetError("transpose_cast_batched: 4-D tensor with a contiguous last dimension required")
    nb2, nb1, R, C = x.shape
    Rp = (R + 7) // 8 * 8
    out = torch.empty((nb2, nb1, C, Rp), dtype=torch.float16, device=x.device)
    check(load().mqdet_transpose_cast_batched(_ptr(x), _dt(x), nb1, nb2, x.stride(1), x.stride(0), R, C, x.stride(2), 1.0, _ptr(out), Rp,
                                              _stream()), "transpose_cast_batched")
    launch_count += 1
    return out


def softmax_bwd_rows(p16, dp32, scale=1.0):
    """ds = scale * p * (dp - sum(p * dp)) over the last dim: p16 fp16 / dp32 fp32 [..., n] contiguous -> fp16 [..., n]."""
    global launch_count
    _need_cuda(p16, dp32)
    if p16.dtype != torch.float16 or dp32.dtype != torch.float32 or not p16.is_contiguous() or not dp32.is_contiguous() or \
            p16.shape != dp32.shape:
        raise _lib.MqdetError("softmax_bwd_rows: contiguous p fp16 / dp fp32 of one shape")
    n = p16.shape[-1]
    rows = p16.numel() // n
    out = torch.empty_like(p16)
    check(load().mqdet_softmax_bwd_rows(_ptr(p16), n, _ptr(dp32), n, rows, n, n, float(scale), _ptr(out), n, _stream()), "softmax_bwd_rows")
    launch_count += 1
    return out


def layernorm_bwd(dy32, x32, gamma, eps, dx=None, want_param_grads=True, x2=None):
    """nn.LayerNorm backward from the saved input (``x32 + x2`` when ``x2`` is given): dy32 / x32 fp32 [..., D] -> (dx, dgamma,
    dbeta); ``dx`` given: accumulated into."""
    global launch_count
    _need_cuda(dy32, x32, gamma, dx, x2)
    if x2 is not None and (x2.dtype != torch.float32 or not x2.is_contiguous() or x2.numel() != x32.numel()):
        raise _lib.MqdetError("layernorm_bwd: x2 must be contiguous fp32 of x's size")
    D = x32.shape[-1]
    rows = x32.numel() // D
    if dy32.dtype != torch.float32 or x32.dtype != torch.float32 or not dy32.is_contiguous() or not x32.is_contiguous():
        raise _lib.MqdetError("layernorm_bwd: contiguous fp32 tensors required")
    acc = dx is not None
    if dx is None:
        dx = torch.empty_like(x32)
    dg = torch.empty((D,), dtype=torch.float32, device=x32.device) if want_param_grads else None
    db = torch.empty((D,), dtype=torch.float32, device=x32.device) if want_param_grads else None
    ws = torch.empty((int(load().mqdet_layernorm_bwd_workspace_floats(rows, D)),), dtype=torch.float32, device=x32.device)
    check(load().mqdet_layernorm_bwd(_ptr(dy32), _ptr(x32), _ptr(x2), _ptr(gamma), float(eps), rows, D, _ptr(dx), int(acc), _ptr(dg), _ptr(db),
                                     _ptr(ws), _stream()), "layernorm_bwd")
    launch_count += 3
    return dx, dg, db


def gelu_bwd(z16, dh):
    """dz = dh * gelu'(z) (exact erf GELU): z16 fp16, dh fp16 / fp32 of the same shape -> fp16."""
    global launch_count
    _need_cuda(z16, dh)
    if z16.dtype != torch.float16 or not z16.is_contiguous() or not dh.is_contiguous() or dh.shape != z16.shape:
        raise _lib.MqdetError("gelu_bwd: contiguous tensors of one shape, z fp16")
    out = torch.empty_like(z16)
    check(load().mqdet_gelu_bwd(_ptr(z16), _ptr(dh), _dt(dh), z16.numel(), _ptr(out), _stream()), "gelu_bwd")
    launch_count += 1
    return out


def gcp_gate_bwd(dx1, s32, g, w2):
    """Backward of x1 = s * tanh(h1 . w2) + x: dx1 / s32 fp32 [M, D], g fp32 [M] (the gate values), w2 fp32 [Dg] ->
    (ds fp32 [M, D], dgpre fp32 [M], dh1 fp16 [M, Dg])."""
    global launch_count
    _need_cuda(dx1, s32, g, w2)
    M, D = dx1.shape
    Dg = w2.numel()
    ds = torch.empty_like(dx1)
    dgpre = torch.empty((M,), dtype=torch.float32, device=dx1.device)
    dh1 = torch.empty((M, Dg), dtype=torch.float16, device=dx1.device)
    check(load().mqdet_gcp_gate_bwd(_ptr(dx1), _ptr(s32), _ptr(g), _ptr(w2), M, D, Dg, _ptr(ds), _ptr(dgpre), _ptr(dh1), _stream()),
          "gcp_gate_bwd")
    launch_count += 1
    return ds, dgpre, dh1


def colsum_weighted(h16, w32):
    """out[j] = sum_r w32[r] * h16[r, j] -> fp32 [C]."""
    global launch_count
    _need_cuda(h16, w32)
    R, C = h16.shape
    out = torch.empty((C,), dtype=torch.float32, device=h16.device)
    ws = torch.empty((int(load().mqdet_colsum_weighted_workspace_floats(C)),), dtype=torch.float32, device=h16.device)
    check(load().mqdet_colsum_weighted(_ptr(h16.contiguous()), _ptr(w32), R, C, _ptr(out), _ptr(ws), _stream()), "colsum_weighted")
    launch_count += 2
    return out


def gcp_sparse_attn_bwd(q, kv, idx, dout16, heads, dim_head):
    """Backward of gcp_sparse_attn: q [B,T,512] fp16, kv [B,V+1,1024] fp16, idx int32 [B,T,S], dout16 [B,T,512] fp16 ->
    (dq fp16 [B,T,512], dkv fp32 [B,V+1,1024])."""
    global launch_count
    _need_cuda(q, kv, idx, dout16)
    B, T, inner = q.shape
    V1 = kv.shape[1]
    S = idx.shape[-1]
    dq = torch.empty_like(q)
    dkv = torch.zeros((B, V1, 2 * inner), dtype=torch.float32, device=q.device)
    check(load().mqdet_gcp_sparse_attn_bwd(_ptr(q.contiguous()), _ptr(kv.contiguous()), _ptr(idx), _ptr(dout16.contiguous()), B, T, V1 - 1,
                                           S, heads, dim_head, _ptr(dq), _ptr(dkv), _stream()), "gcp_sparse_attn_bwd")
    launch_count += 1
    return dq, dkv


def dot_sum(a32, b32=None, one_minus_tanh2_of=None, mul=1.0):
    """mul * sum(a * b) (b None: sum a^2), times 1 - tanh(s)^2 for a device scalar ``one_minus_tanh2_of`` -> device scalar [1]."""
    global launch_count
    _need_cuda(a32, b32, one_minus_tanh2_of)
    out = torch.empty((1,), dtype=torch.float32, device=a32.device)
    ws = torch.empty((int(load().mqdet_reduce_workspace_floats()),), dtype=torch.float32, device=a32.device)
    check(load().mqdet_dot_sum(_ptr(a32.contiguous()), _ptr(None if b32 is None else b32.contiguous()), a32.numel(),
                               _ptr(one_minus_tanh2_of), float(mul), _ptr(out), _ptr(ws), _stream()), "dot_sum")
    launch_count += 2
    return out


def scale_cast(x32, scalar=None, tanh_scalar=False, alpha=1.0, out16=True, out32=False):
    """x * alpha * (tanh)(scalar[0]) -> fp16 and / or fp32 (``scalar``: a device scalar, read on the device)."""
    global launch_count
    _need_cuda(x32, scalar)
    x32 = x32.contiguous()
    o16 = torch.empty(x32.shape, dtype=torch.float16, device=x32.device) if out16 else None
    o32 = torch.empty(x32.shape, dtype=torch.float32, device=x32.device) if out32 else None
    check(load().mqdet_scale_cast(_ptr(x32), _ptr(scalar), int(bool(tanh_scalar)), float(alpha), x32.numel(), _ptr(o16), _ptr(o32),
                                  _stream()), "scale_cast")
    launch_count += 1
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def token_focal_loss(logits, targets, text_mask=None, alpha=0.25, gamma=2.0, want_grad=True, grad_scale=1.0):
    """token_sigmoid_binary_focal_loss(...).sum() over logits / targets fp32 [B, N, T] with the text mask [B, T] ->
    (loss device scalar [1], dlogits fp32 [B, N, T] | None)."""
    global launch_count
    _need_cuda(logits, targets, text_mask)
    B, N, T = logits.shape
    loss = torch.empty((1,), dtype=torch.float32, device=logits.device)
    dl = torch.empty_like(logits, dtype=torch.float32) if want_grad else None
    ws = torch.empty((int(load().mqdet_reduce_workspace_floats()),), dtype=torch.float32, device=logits.device)
    tm = None if text_mask is None else text_mask.float().contiguous()
    check(load().mqdet_token_focal_loss(_ptr(logits.float().contiguous()), _ptr(targets.float().contiguous()), _ptr(tm), float(alpha),
                                        float(gamma), B, N, T, float(grad_scale), _ptr(loss), _ptr(dl), _ptr(ws), _stream()),
          "token_focal_loss")
    launch_count += 2
    return loss, dl


def clip_coef(grads, max_norm):
    """Global L2 norm over a list of fp32 gradient tensors and the clip_grad_norm_ coefficient, all on the device ->
    fp32 [2] = (coefficient, norm)."""
    global launch_count
    _need_cuda(*grads)
    dev = grads[0].device
    partials = torch.zeros((64 * len(grads),), dtype=torch.float32, device=dev)
    n_written = ctypes.c_int64(0)
    off = 0
    for g in grads:
        g = g if g.is_contiguous() else g.contiguous()
        check(load().mqdet_sqnorm_partials(_ptr(g), g.numel(), ctypes.c_void_p(partials.data_ptr() + 4 * off), 64,
                                           ctypes.byref(n_written), _stream()), "sqnorm_partials")
        off += int(n_written.value)
    coef = torch.empty((2,), dtype=torch.float32, device=dev)
    check(load().mqdet_clip_coef(_ptr(partials), off, float(max_norm), _ptr(coef), _stream()), "clip_coef")
    launch_count += len(grads) + 1
    return coef


def adamw_step_(param, grad, exp_avg, exp_avg_sq, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, grad_scale=None):
    """torch.optim.AdamW update of one fp32 tensor in place; ``grad_scale`` = a device scalar (the clip coefficient) or None."""
    global launch_count
    _need_cuda(param, grad, exp_avg, exp_avg_sq, grad_scale)
    for t in (param, grad, exp_avg, exp_avg_sq):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise _lib.MqdetError("adamw_step_: contiguous fp32 tensors required")
    check(load().mqdet_adamw_step(_ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), param.numel(), float(lr), float(betas[0]),
                                  float(betas[1]), float(eps), float(weight_decay), int(step), _ptr(grad_scale), _stream()), "adamw_step")
    launch_count += 1
    return param
