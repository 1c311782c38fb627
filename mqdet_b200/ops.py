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


def _launch(symbol, *args, what, kernels=1, timed=None, gemm_shape=None):
    """Call the C entry point ``symbol`` with ``args`` and the current stream (read per call, so that a graph capture sees the
    capturing stream), raise MqdetError naming ``what`` on a failure code, and add ``kernels`` (what the call launches) to
    launch_count.  One pair of CUDA events brackets the call when it is profiled: always by _lib.CALL_PROFILE, by KERNEL_PROFILE
    when ``timed`` = (kernel name, algorithmic flops, algorithmic bytes[, executed flops]), by GEMM_PROFILE when ``gemm_shape``
    is given (the flops then come from ``timed``)."""
    global launch_count
    fn = getattr(load(), symbol)
    calls = _lib.CALL_PROFILE
    kprof = KERNEL_PROFILE if timed is not None else None
    gprof = GEMM_PROFILE if gemm_shape is not None else None
    if calls is None and kprof is None and gprof is None:
        check(fn(*args, _stream()), what)
    else:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*args, _stream())
        e1.record()
        if calls is not None:
            calls.append((symbol, e0, e1))
        if kprof is not None:
            # ``flops`` = the ALGORITHMIC count (what the reference computes for this piece of work); ``executed`` = what the kernel
            # issues to the tensor cores when algebraic folding makes that smaller (defaults to the algorithmic count)
            name, flops, nbytes, *executed = timed
            kprof.append((e0, e1, name, float(flops), float(nbytes), float(executed[0] if executed else flops)))
        if gprof is not None:
            gprof.append((e0, e1, float(timed[1]), gemm_shape))
        check(rc, what)
    launch_count += kernels


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
    # algorithmic bytes: every operand once (a broadcast operand once for the whole batch), the output, the residual
    nb = nb1 * nb2
    es_o = 2 if out.dtype == torch.float16 else 4
    gbytes = 2.0 * M * K * (a4.shape[0] * a4.shape[1]) + 2.0 * N * K * (b4.shape[0] * b4.shape[1]) + float(es_o) * M * N * nb
    if residual is not None:
        gbytes += (2.0 if residual.dtype == torch.float16 else 4.0) * M * N * nb
    _launch("mqdet_gemm_f16", ctypes.byref(g), DEFAULT_GEMM_IMPL if impl is None else impl, what="gemm",
            timed=("gemm_wg_kernel", 2.0 * M * N * K * nb, gbytes), gemm_shape=(M, N, K, nb))
    return out


def layernorm(x, gamma, beta, eps=1e-5, *, out16=True, out32=False, zero_row_period=0):
    """nn.LayerNorm over the last dim of a contiguous [..., D] fp16/fp32 tensor -> (fp16, fp32) outputs."""
    _need_cuda(x, gamma, beta)
    D = x.shape[-1]
    x2 = x.reshape(-1, D)
    rows = x2.shape[0]
    o16 = torch.empty(x.shape, dtype=torch.float16, device=x.device) if out16 else None
    o32 = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out32 else None
    _launch("mqdet_layernorm", _ptr(x2), _dt(x2), x2.stride(0), _ptr(gamma), _ptr(beta), float(eps), rows, D,
            _ptr(o16), _ptr(o32), D, int(zero_row_period), what="layernorm")
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def swin_mlp(x32, ln_w, ln_b, eps, w1, b1, w2, b2):
    """The MLP half of a Swin block in one kernel (mqdet_swin_mlp_f16): x32 + fc2(GELU(fc1(LN(x32)))) for a contiguous fp32
    [rows, C] with C = 96 / 192; w1 fp16 [4C, C], w2 fp16 [C, 4C] (nn.Linear weights), fp32 LN affine and biases -> new fp32
    [rows, C], bit-identical to layernorm -> gemm(bias, GELU) -> gemm(bias, fp32 residual)."""
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
    _launch("mqdet_swin_mlp_f16", _ptr(x32), rows, C, _ptr(ln_w), _ptr(ln_b), float(eps), _ptr(w1), _ptr(b1), _ptr(w2),
            _ptr(b2), _ptr(out), what="swin_mlp",
            timed=("swin_mlp_kernel", 2.0 * 2.0 * rows * C * 4 * C, 2.0 * 4.0 * rows * C + 2.0 * 2.0 * 4 * C * C))
    return out


def add_layernorm(a, b, gamma, beta, eps, *, out16=True, out32=True, clamp=0.0):
    """LN(a + b) over the last dim; a, b contiguous fp32."""
    _need_cuda(a, b)
    D = a.shape[-1]
    rows = a.numel() // D
    o16 = torch.empty(a.shape, dtype=torch.float16, device=a.device) if out16 else None
    o32 = torch.empty(a.shape, dtype=torch.float32, device=a.device) if out32 else None
    _launch("mqdet_add_layernorm", _ptr(a), _ptr(b), _ptr(gamma), _ptr(beta), float(eps), rows, D, _ptr(o32),
            _ptr(o16), float(clamp), what="add_layernorm")
    return o16, o32


def softmax_rows(x, *, n=None, scale=1.0, colmask=None, rows_per_batch=0, mask_value=0.0, keep_add=0.0, out=None):
    """Row softmax of fp32 scores over the last dim of x [..., n_pad] (contiguous) -> fp16; cols >= n are zeroed.  Other
    dtypes raise MqdetError (mqdet_softmax_rows rejects them)."""
    _need_cuda(x, colmask)
    n_pad = x.shape[-1]
    n = n_pad if n is None else n
    rows = x.numel() // n_pad
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _launch("mqdet_softmax_rows", _ptr(x), _dt(x), n_pad, _ptr(out), n_pad, rows, n, n_pad, float(scale),
            _ptr(colmask), int(rows_per_batch), float(mask_value), float(keep_add), what="softmax_rows")
    return out


def sum_splits_cast(part32, out16):
    """part32 fp32 [nb2, nb1, S, R, C] contiguous (the fp32 partial products of a K-split GEMM) -> out16 [nb2, nb1, R, C] fp16 (a view with
    arbitrary nb / row strides, contiguous last dim) = the sum over S."""
    _need_cuda(part32, out16)
    nb2, nb1, S, R, C = part32.shape
    if part32.dtype != torch.float32 or not part32.is_contiguous() or out16.dtype != torch.float16 or tuple(out16.shape) != (nb2, nb1, R, C) \
            or out16.stride(3) != 1:
        raise _lib.MqdetError("sum_splits_cast: part fp32 [nb2,nb1,S,R,C] contiguous, out fp16 [nb2,nb1,R,C] with a contiguous last dim")
    _launch("mqdet_sum_splits_cast", _ptr(part32), nb2, nb1, S, R, C, _ptr(out16), out16.stride(0), out16.stride(1), out16.stride(2),
            what="sum_splits_cast")
    return out16


def softmax_rows_shifted(x32, shift, lo, hi, *, n=None, colmask=None, rows_per_batch=0, mask_value=0.0, keep_add=0.0,
                         rows_per_shift=0):
    """softmax over the last dim of clamp(x - shift[r // rows_per_shift], lo, hi) (+ mask) for contiguous fp32 [..., n_pad] -> fp16;
    ``shift`` is on the device: one value per ``rows_per_shift`` rows (one per batch element), or ``rows_per_shift = 0`` = shift[0]
    for every row.  Fused where the kernel supports the row length, else ``shift_clamp_`` (in place!) followed by ``softmax_rows``."""
    _need_cuda(x32, shift, colmask)
    n_pad = x32.shape[-1]
    n = n_pad if n is None else n
    if x32.dtype != torch.float32 or not x32.is_contiguous():
        raise _lib.MqdetError("softmax_rows_shifted: contiguous fp32 tensor required")
    rows = x32.numel() // n_pad
    _check_shift(shift, rows, rows_per_shift, "softmax_rows_shifted")
    if not load().mqdet_softmax_rows_shifted_supported(n, n_pad):
        shift_clamp_(x32, shift, lo, hi, rows_per_shift=rows_per_shift)
        return softmax_rows(x32, n=n, colmask=colmask, rows_per_batch=rows_per_batch, mask_value=mask_value, keep_add=keep_add)
    out = torch.empty(x32.shape, dtype=torch.float16, device=x32.device)
    _launch("mqdet_softmax_rows_shifted", _ptr(x32), n_pad, _ptr(out), n_pad, rows, n, n_pad, _ptr(shift), int(rows_per_shift),
            float(lo), float(hi), _ptr(colmask), int(rows_per_batch), float(mask_value),
            float(keep_add), what="softmax_rows_shifted")
    return out


def _check_shift(shift, rows, rows_per_shift, what):
    """The shift vector must cover every row group: rows_per_shift divides rows and shift holds rows // rows_per_shift values."""
    if rows_per_shift < 0 or (rows_per_shift and (rows % rows_per_shift or shift.numel() < rows // rows_per_shift)):
        raise ValueError(f"{what}: rows_per_shift={rows_per_shift} does not split {rows} rows over {shift.numel()} shifts")
    if shift.dtype != torch.float32 or not shift.is_contiguous():
        raise _lib.MqdetError(f"{what}: contiguous fp32 shift required")


def global_max(x32, *, segments=1):
    """Maximum of each of ``segments`` equal contiguous segments of a contiguous fp32 tensor -> device fp32 [segments] (no host
    sync); ``segments = 1`` is the maximum over all elements.  One pass over x, deterministic."""
    _need_cuda(x32)
    if x32.dtype != torch.float32 or not x32.is_contiguous():
        raise _lib.MqdetError("global_max: contiguous fp32 tensor required")
    segments = int(segments)
    if segments < 1 or x32.numel() % segments:
        raise ValueError(f"global_max: {x32.numel()} elements do not split into {segments} equal segments")
    out = torch.empty((segments,), dtype=torch.float32, device=x32.device)
    ws = torch.empty((int(load().mqdet_global_max_workspace_floats(segments)),), dtype=torch.float32, device=x32.device)
    _launch("mqdet_global_max_f32", _ptr(x32), x32.numel(), segments, _ptr(out), _ptr(ws), what="global_max", kernels=2)
    return out


def shift_clamp_(x32, shift, lo, hi, *, rows_per_shift=0):
    """x = clamp(x - shift[r // rows_per_shift], lo, hi) in place over the whole (contiguous fp32) buffer, r = the row of the last
    dim; ``shift`` is on the device (``rows_per_shift = 0``: shift[0] for every element)."""
    _need_cuda(x32, shift)
    if x32.dtype != torch.float32 or not x32.is_contiguous():
        raise _lib.MqdetError("shift_clamp_: contiguous fp32 tensor required")
    n_row = x32.shape[-1] if x32.dim() else 1
    _check_shift(shift, x32.numel() // n_row, rows_per_shift, "shift_clamp_")
    _launch("mqdet_shift_clamp_f32", _ptr(x32), x32.numel(), _ptr(shift), int(rows_per_shift) * n_row, float(lo), float(hi),
            what="shift_clamp")
    return x32


def row_max(x32):
    """max over the last dim of a contiguous fp32 [..., D] tensor -> fp32 [...]."""
    _need_cuda(x32)
    D = x32.shape[-1]
    x2 = x32.reshape(-1, D)
    out = torch.empty(x32.shape[:-1], dtype=torch.float32, device=x32.device)
    _launch("mqdet_row_max_f32", _ptr(x2), x2.shape[0], D, x2.stride(0), _ptr(out), what="row_max")
    return out


def topk_desc(keys32, k):
    """indices [B, k] (int64) of the k largest entries of each row of fp32 keys [B, n], by (value descending, index ascending)."""
    _need_cuda(keys32)
    if keys32.dtype != torch.float32 or keys32.dim() != 2 or not keys32.is_contiguous():
        raise _lib.MqdetError("topk_desc: contiguous fp32 [B, n] required")
    B, n = keys32.shape
    idx = torch.empty((B, k), dtype=torch.int64, device=keys32.device)
    _launch("mqdet_topk_desc", _ptr(keys32), B, n, int(k), _ptr(idx), what="topk_desc")
    return idx


def gather_rows(src32, idx, sigmoid=False):
    """src32 [B, R, D] fp32, idx [B, k] int64 -> [B, k, D] (torch.gather along dim 1 with the index repeated over D), optionally
    through the logistic sigmoid."""
    _need_cuda(src32, idx)
    if src32.dtype != torch.float32 or src32.dim() != 3 or not src32.is_contiguous() or idx.dtype != torch.int64 or not idx.is_contiguous():
        raise _lib.MqdetError("gather_rows: contiguous fp32 [B, R, D] and int64 [B, k] required")
    B, R, D = src32.shape
    k = idx.shape[1]
    out = torch.empty((B, k, D), dtype=torch.float32, device=src32.device)
    _launch("mqdet_gather_rows_f32", _ptr(src32), _ptr(idx), B, R, k, D, int(bool(sigmoid)), _ptr(out), what="gather_rows")
    return out


def l2_normalize(x32, w=None, b0=None, eps=1e-12):
    """e = F.normalize(x, p=2, dim=-1) of a contiguous fp32 tensor -> (e fp16, e fp32, dot) with
    dot[r] = e[r, :] . w + b0 when ``w`` is given (the token bias of the dot-product head, vldyhead.py:818)."""
    _need_cuda(x32, w, b0)
    D = x32.shape[-1]
    rows = x32.numel() // D
    e16 = torch.empty(x32.shape, dtype=torch.float16, device=x32.device)
    e32 = torch.empty_like(x32)
    dot = torch.empty(x32.shape[:-1], dtype=torch.float32, device=x32.device) if w is not None else None
    _launch("mqdet_l2norm_rowdot", _ptr(x32), rows, D, float(eps), _ptr(w), _ptr(b0), _ptr(e16), _ptr(e32), _ptr(dot),
            what="l2norm_rowdot")
    return e16, e32, dot


def biattn_image(vn16, gT, gbias, mT, bias, gamma, residual, mask, clamp, heads):
    """Fused image -> text side with the query / value / output projections folded into per-(image, head) operands, layer
    scale and residual (mqdet_biattn_image).  vn16 [B,N,256] fp16 (layer-normed tokens), gT [B,H,T,256] fp16, gbias [B,H,T,ld]
    fp32 (column 0 used) or None, mT [B,H,256,T] fp16; bias/gamma [256] fp32 or None; residual [B,N,256] fp16 or None; mask
    [B,T] fp32 or None -> (out [B,N,256] fp16, colmax [B*H,T] fp32)."""
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
    _launch("mqdet_biattn_image", _ptr(vn16), vn16.stride(1), vn16.stride(0), _ptr(gT), gT.stride(2), gT.stride(1),
            gT.stride(0), _ptr(gbias), gbias.shape[3] if gbias is not None else 0, _ptr(mT),
            mT.stride(2), mT.stride(1), mT.stride(0), _ptr(bias), _ptr(gamma), _ptr(residual),
            residual.stride(1) if residual is not None else 0,
            residual.stride(0) if residual is not None else 0, _ptr(mask), float(clamp), _ptr(out),
            out.stride(1), out.stride(0), _ptr(colmax), _ptr(ws), B, heads, N, T, what="biattn_image", kernels=2,
            timed=("biattn_image_kernel", fl, 2.0 * B * N * 256 * (3 if residual is not None else 2) + 2.0 * 2 * B * heads * T * 256, ex))
    return out, colmax


def biattn_text_vn(kh, qh, vn16, colmax, clamp, out, rowbias=None):
    """Fused text -> image attention on the image tokens themselves: kh [B,H,T,d], qh [B,H,N,d] (strided views; a head stride of
    0 broadcasts), vn16 [B,N,256] fp16, colmax [B*H,T] fp32 (from biattn_image), rowbias [B,H,T,ld] fp32 (column 0) or None,
    out [B,H,T,256] fp16 view <- softmax_n(scores + rowbias)^T . vn."""
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
    _launch("mqdet_biattn_text_vn", _ptr(kh), kh.stride(2), kh.stride(1), kh.stride(0), _ptr(qh), qh.stride(2), qh.stride(1),
            qh.stride(0), _ptr(vn16), vn16.stride(1), 0, vn16.stride(0), _ptr(colmax), _ptr(rowbias),
            rowbias.shape[3] if rowbias is not None else 0, float(clamp), _ptr(out), out.stride(2),
            out.stride(1), out.stride(0), H, B, T, N, what="biattn_text_vn",
            timed=("biattn_text_kernel", fl, 2.0 * B * N * 256 + 2.0 * 2 * B * H * T * 256, B * H * 2.0 * (2.0 * T * N * 256)))
    return out


def cast_f16(x):
    _need_cuda(x)
    if x.dtype == torch.float16:
        return x
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _launch("mqdet_cast_f32_f16", _ptr(x), _ptr(y), x.numel(), what="cast_f32_f16")
    return y


def cast_f32(x):
    _need_cuda(x)
    if x.dtype == torch.float32:
        return x
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    _launch("mqdet_cast_f16_f32", _ptr(x), _ptr(y), x.numel(), what="cast_f16_f32")
    return y


def contrastive_embed(x16, y16, text_token_mask, max_text_len):
    """x16 [B,Q,D] fp16, y16 [B,T,D] fp16, text_token_mask [B,T] bool -> logits [B,Q,max_text_len] fp32:
    x . y^T, -inf on padding tokens and on columns T..max_text_len-1 (GroundingDINO utils.py:242-268)."""
    _need_cuda(x16, y16, text_token_mask)
    B, Q, _ = x16.shape
    T = y16.shape[1]
    out = torch.empty((B, Q, max_text_len), dtype=torch.float32, device=x16.device)
    gemm(x16, y16, out=out[:, :, :T])
    m8 = text_token_mask.to(torch.uint8).contiguous()
    _launch("mqdet_contrastive_mask", _ptr(out), _ptr(m8), B, Q, T, max_text_len, what="contrastive_mask")
    return out


def dense_cross_attn(q, kv, heads, dim_head):
    """Flash-style dense cross-attention (PreSelect): q [B,Tq,H*32] fp16 (scaled), kv [B,I,2*H*32] fp16 (K | V halves) ->
    [B,Tq,H*32] fp16 = softmax_i(q.k^T) v per head, without materialising the scores."""
    _need_cuda(q, kv)
    B, Tq, inner = q.shape
    I = kv.shape[1]
    if q.dtype != torch.float16 or kv.dtype != torch.float16 or q.stride(-1) != 1 or kv.stride(-1) != 1:
        raise _lib.MqdetError("dense_cross_attn: fp16 operands with a contiguous last dimension required")
    out = torch.empty((B, Tq, inner), dtype=torch.float16, device=q.device)
    _launch("mqdet_dense_cross_attn", _ptr(q), q.stride(1), q.stride(0), _ptr(kv), kv.stride(1), kv.stride(0), inner, _ptr(out),
            out.stride(1), out.stride(0), B, Tq, I, heads, dim_head, what="dense_cross_attn")
    return out


def gcp_build_index(mask, S):
    """mask [B, V, T] fp32 0/1 -> (idx int32 [B, T, S] padded with V, counts int32 [B, T])."""
    _need_cuda(mask)
    B, V, T = mask.shape
    mask = mask.contiguous().float()
    idx = torch.empty((B, T, S), dtype=torch.int32, device=mask.device)
    counts = torch.empty((B, T), dtype=torch.int32, device=mask.device)
    _launch("mqdet_gcp_build_index", _ptr(mask), B, V, T, S, _ptr(idx), _ptr(counts), what="gcp_build_index")
    return idx, counts


# Most vision queries one text token can attend to in gcp_sparse_attn (GCP_MAX_S in csrc/gcp.cu: the largest S whose per-warp
# shared-memory slice of indices and per-head scores fits a CTA at 32 heads).
GCP_MAX_S = 1760


def gcp_sparse_attn(q, kv, idx, heads, dim_head):
    """q [B, T, H*Dh] fp16 (scaled), kv [B, V+1, 2*H*Dh] fp16, idx [B, T, S] int32 -> [B, T, H*Dh] fp16.
    Any S in [1, GCP_MAX_S]."""
    _need_cuda(q, kv, idx)
    B, T, inner = q.shape
    V = kv.shape[1] - 1
    S = idx.shape[2]
    if not 1 <= S <= GCP_MAX_S:
        raise _lib.MqdetError(f"gcp_sparse_attn: {S} vision queries per text token; the kernel takes 1 to GCP_MAX_S = {GCP_MAX_S}")
    out = torch.empty_like(q)
    _launch("mqdet_gcp_sparse_attn", _ptr(q), _ptr(kv), _ptr(idx), _ptr(out), B, T, V, S, heads, dim_head, what="gcp_sparse_attn")
    return out


def gcp_gate_residual_ln(h1, w2, s, x, gamma, beta, eps=1e-5, want_gate=False):
    """g = tanh(h1 . w2); x1 = s*g + x; returns (x1 fp32, LN(x1) fp16[, g])."""
    _need_cuda(h1, w2, s, x)
    D = s.shape[-1]
    rows = s.numel() // D
    Dg = h1.shape[-1]
    x1 = torch.empty_like(s)
    ln = torch.empty(s.shape, dtype=torch.float16, device=s.device)
    g = torch.empty(s.shape[:-1], dtype=torch.float32, device=s.device) if want_gate else None
    _launch("mqdet_gcp_gate_residual_ln", _ptr(h1), _ptr(w2), Dg, _ptr(s), _ptr(x), _ptr(gamma), _ptr(beta), float(eps),
            rows, D, _ptr(x1), _ptr(ln), _ptr(g), what="gcp_gate_residual_ln")
    return (x1, ln, g) if want_gate else (x1, ln)


def argsort_desc(scores):
    _need_cuda(scores)
    n = scores.numel()
    order = torch.empty((n,), dtype=torch.int64, device=scores.device)
    if n:
        _launch("mqdet_argsort_desc", _ptr(scores), n, _ptr(order), what="argsort_desc")
    return order


def ml_nms_device(boxes, scores, labels, thresh, max_det=0):
    """Device-resident multi-label NMS. Returns (keep int64 [n] (first num valid, ascending), num int32 [1])."""
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
    _launch("mqdet_ml_nms", _ptr(boxes), _ptr(scores), _ptr(labels), _ptr(order), n, float(thresh), int(max_det),
            _ptr(keep), _ptr(num), _ptr(ws), what="ml_nms", kernels=5)
    return keep, num


def ml_nms(boxes, scores, labels, thresh):
    """Drop-in for maskrcnn_benchmark._C.ml_nms (csrc/ml_nms.h:11-27): kept original indices, ascending."""
    if boxes.numel() == 0:
        return torch.empty((0,), dtype=torch.int64, device="cpu")  # reference returns an empty CPU tensor (:19-20)
    keep, num = ml_nms_device(boxes, scores, labels, thresh)
    return keep[: int(num.item())]


def upload_async(t, device):
    """Small host tensor -> ``device`` without waiting for the stream: staged in pinned memory and copied asynchronously (a
    copy from pageable memory synchronises the stream first).  Other devices get a plain copy."""
    if torch.device(device).type != "cuda":
        return t.to(device)
    return t.pin_memory().to(device, non_blocking=True)


# ----------------------------------------------------------------------------------------------------------------------
# Multi-scale / flip test-time augmentation: the cross-pass merge (csrc/bbox_aug.cu)
# ----------------------------------------------------------------------------------------------------------------------
BBOX_AUG_MAX_CAP = 1 << 17
BBOX_AUG_BAD_COUNT = 1 << 30   # set in MergedBoxes.overflow by a packed pass whose count row is not an integer in [0, rows]


def hflip_pad(images, out_hw):
    """fp32 [B, C, h, w] -> [B, C, H, W]: every row reversed within the width w, zeros to the right and below (the
    horizontally flipped batch after SIZE_DIVISIBILITY padding; flipping the normalised tensor equals flipping the image before
    ToTensor / Normalize, both being per-pixel)."""
    _need_cuda(images)
    if images.dim() != 4 or images.dtype != torch.float32 or not images.is_contiguous():
        raise _lib.MqdetError("hflip_pad: contiguous fp32 [B, C, h, w] required")
    B, C, h, w = images.shape
    H, W = int(out_hw[0]), int(out_hw[1])
    out = torch.empty((B, C, H, W), dtype=torch.float32, device=images.device)
    _launch("mqdet_hflip_pad", _ptr(images), B * C, h, w, H, W, _ptr(out), what="hflip_pad")
    return out


class MergedBoxes:
    """The per-image union of the candidates of every augmentation pass, device-resident: boxes fp32 [B, cap, 4] (original
    image coordinates), scores fp32 [B, cap], labels int32 [B, cap], count int32 [B] (rows in use), overflow int32 [B]
    (candidates that did not fit)."""

    def __init__(self, B, cap, device):
        if not 0 < cap <= BBOX_AUG_MAX_CAP:
            raise _lib.MqdetError(f"bbox_aug: 1 <= cap <= {BBOX_AUG_MAX_CAP} merged boxes per image (got {cap})")
        self.B, self.cap = int(B), int(cap)
        self.boxes = torch.zeros((B, cap, 4), dtype=torch.float32, device=device)
        self.scores = torch.zeros((B, cap), dtype=torch.float32, device=device)
        self.labels = torch.zeros((B, cap), dtype=torch.int32, device=device)
        self.count = torch.zeros((B,), dtype=torch.int32, device=device)
        self.overflow = torch.zeros((B,), dtype=torch.int32, device=device)


def bbox_aug_collect(merged, cand_boxes, cand_scores, cand_labels, cand_totals, pass_size, orig_size, *, flip=False,
                     keep_range=None):
    """Append one pass's candidates (``cand_*`` of ``atss_postprocess``) to ``merged``: un-flip about the pass's image width
    (BoxList.transpose), drop boxes whose area is outside ``keep_range`` = (lo, hi), both bounds strict (remove_boxes), scale
    from ``pass_size`` to ``orig_size`` (both (width, height); BoxList.resize), in that order.  Candidate order is kept and
    the running count stays on the device."""
    _need_cuda(cand_boxes, cand_scores, cand_labels, cand_totals)
    B, S = cand_scores.shape
    for t, dt in ((cand_boxes, torch.float32), (cand_scores, torch.float32), (cand_labels, torch.float32), (cand_totals, torch.int32)):
        if t.dtype != dt or not t.is_contiguous():
            raise _lib.MqdetError("bbox_aug_collect: contiguous fp32 boxes / scores / labels and int32 totals required")
    if B != merged.B or tuple(cand_boxes.shape) != (B, S, 4):
        raise _lib.MqdetError(f"bbox_aug_collect: candidates {tuple(cand_boxes.shape)} do not match a merged buffer of {merged.B} images")
    _launch("mqdet_bbox_aug_collect", _ptr(cand_boxes), _ptr(cand_scores), _ptr(cand_labels), _ptr(cand_totals), B, S,
            *_aug_pass_args(pass_size, orig_size, flip, keep_range), _ptr(merged.boxes),
            _ptr(merged.scores), _ptr(merged.labels), merged.cap, _ptr(merged.count),
            _ptr(merged.overflow), what="bbox_aug_collect")
    return merged


def _aug_pass_args(pass_size, orig_size, flip, keep_range):
    """(flip, pass_w, has_range, lo2, hi2, ratio_x, ratio_y) of a collect, rounded to fp32 as the reference's tensors are."""
    import numpy as np
    rx, ry = float(orig_size[0]) / float(pass_size[0]), float(orig_size[1]) / float(pass_size[1])
    rx32, ry32 = float(np.float32(rx)), float(np.float32(ry))      # tensor * python_float multiplies by the fp32 ratio
    lo2 = hi2 = 0.0
    if keep_range is not None:
        lo2, hi2 = float(np.float32(keep_range[0] * keep_range[0])), float(np.float32(keep_range[1] * keep_range[1]))
    return int(bool(flip)), float(pass_size[0]), int(keep_range is not None), lo2, hi2, rx32, ry32


def bbox_aug_collect_packed(merged, packed, pass_size, orig_size, *, flip=False, keep_range=None):
    """``bbox_aug_collect`` for one pass's packed detector rows fp32 [B, M + 1, 6] (x1, y1, x2, y2, score, label; row M =
    (count, ...)), the output of ``gdino_detections``: the same steps in the same order, rows kept in order.  The count is read on
    the device; one that is not an integer in [0, M] reads no row and flags the image in ``merged.overflow``
    (``BBOX_AUG_BAD_COUNT``)."""
    _need_cuda(packed)
    if packed.dtype != torch.float32 or not packed.is_contiguous() or packed.dim() != 3 or packed.shape[2] != 6 or packed.shape[1] < 2:
        raise _lib.MqdetError(f"bbox_aug_collect_packed: contiguous fp32 [B, M + 1, 6] rows required (got {packed.dtype} "
                              f"{tuple(packed.shape)})")
    B, M = packed.shape[0], packed.shape[1] - 1
    if B != merged.B:
        raise _lib.MqdetError(f"bbox_aug_collect_packed: {B} images do not match a merged buffer of {merged.B} images")
    _launch("mqdet_bbox_aug_collect_packed", _ptr(packed), B, M, *_aug_pass_args(pass_size, orig_size, flip, keep_range),
            _ptr(merged.boxes), _ptr(merged.scores), _ptr(merged.labels), merged.cap,
            _ptr(merged.count), _ptr(merged.overflow), what="bbox_aug_collect_packed")
    return merged


def nms_by_class(boxes, scores, labels, count, classes, thresh, *, mode="nms", top_n=0, max_out, overflow=None):
    """merge_result_from_multi_scales for a batch: boxes fp32 [B, cap, 4], scores fp32 [B, cap], labels int32 [B, cap], count
    int32 [B]; classes = sorted int32 table of the labels considered.  mode "nms" | "vote".  -> packed fp32 [B, max_out + 1, 6]
    rows (x1, y1, x2, y2, score, label), last row = (count, overflow, 0...).  See include/mqdet_b200.h for the exact rules."""
    _need_cuda(boxes, scores, labels, count, classes, overflow)
    if mode not in ("nms", "vote"):
        raise NotImplementedError(f"nms_by_class: mode {mode!r} (only 'nms' and 'vote' are implemented)")
    B, cap = scores.shape
    for t, dt in ((boxes, torch.float32), (scores, torch.float32), (labels, torch.int32), (count, torch.int32), (classes, torch.int32)):
        if t.dtype != dt or not t.is_contiguous():
            raise _lib.MqdetError("nms_by_class: contiguous fp32 boxes / scores and int32 labels / count / classes required")
    if tuple(boxes.shape) != (B, cap, 4) or tuple(labels.shape) != (B, cap) or count.numel() != B or classes.dim() != 1:
        raise _lib.MqdetError("nms_by_class: boxes [B, cap, 4], scores / labels [B, cap], count [B], classes [C] required")
    C = classes.numel()
    out = torch.zeros((B, max_out + 1, 6), dtype=torch.float32, device=boxes.device)
    ws = torch.empty((int(load().mqdet_nms_by_class_workspace_bytes(B, cap, C)),), dtype=torch.uint8, device=boxes.device)
    passes = max(0, (max(cap - 1, 1) // 2048).bit_length())
    _launch("mqdet_nms_by_class", _ptr(boxes), _ptr(scores), _ptr(labels), _ptr(count), _ptr(overflow), B, cap, _ptr(classes), C,
            float(thresh), int(mode == "vote"), int(top_n), int(max_out), _ptr(out), _ptr(ws), what="nms_by_class",
            kernels=6 + 2 * passes)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# The test transform: PIL-exact resize, ToTensor, Normalize, padding (csrc/transform.cu)
# ----------------------------------------------------------------------------------------------------------------------
def resize_coeffs(n_in, n_out, device):
    """Coefficient table of PIL's bilinear resampler for one length pair: int32 [n_out, 2 + ksize] rows of (first input
    index, taps, 22-bit fixed-point weights), built on the device."""
    n_in, n_out = int(n_in), int(n_out)
    K = int(load().mqdet_resize_coeffs_ksize(n_in, n_out))
    if K <= 0:
        raise _lib.MqdetError(f"resize_coeffs: bad lengths {n_in} -> {n_out}")
    table = torch.empty((n_out, 2 + K), dtype=torch.int32, device=device)
    _launch("mqdet_resize_coeffs", n_in, n_out, _ptr(table), what="resize_coeffs")
    return table


def test_transform(images, xtabs, ytabs, out_hw, pad_hw, mean, std, *, bgr=False, times255=False, want_resized=False, out=None):
    """uint8 [h_i, w_i, 3] CUDA images (RGB) -> fp32 [B, 3, Hp, Wp]: each image resized to ``out_hw`` = (oh, ow) with
    ``xtabs[i]`` = resize_coeffs(w_i, ow) and ``ytabs[i]`` = resize_coeffs(h_i, oh), then / 255, channels reversed (``bgr``),
    x 255 (``times255``), (x - mean) / std, zero beyond (oh, ow) up to ``pad_hw``.  With ``want_resized`` also returns the
    resized uint8 images [B, oh, ow, 3].  ``out_hw`` may also be B per-image sizes [(oh_i, ow_i)] (a padded batch of differently
    sized images, the tables built for each image's own size); ``want_resized`` then needs them all equal.  ``out``: a contiguous
    fp32 [B, 3, Hp, Wp] tensor on the images' device to write instead of a new one (every element is written)."""
    B = len(images)
    if B == 0 or len(xtabs) != B or len(ytabs) != B:
        raise _lib.MqdetError("test_transform: one x and one y coefficient table per image required")
    _need_cuda(*images, *xtabs, *ytabs)
    per_image = isinstance(out_hw[0], (tuple, list))
    sizes = [(int(h), int(w)) for h, w in out_hw] if per_image else [(int(out_hw[0]), int(out_hw[1]))] * B
    if len(sizes) != B:
        raise _lib.MqdetError(f"test_transform: {len(sizes)} output sizes for {B} images")
    Hp, Wp = (int(v) for v in pad_hw)
    for im, xt, yt, (oh, ow) in zip(images, xtabs, ytabs, sizes):
        if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3 or not im.is_contiguous():
            raise _lib.MqdetError(f"test_transform: contiguous uint8 [h, w, 3] images required (got {im.dtype} {tuple(im.shape)})")
        h, w = im.shape[:2]
        for t, n_in, n_out in ((xt, w, ow), (yt, h, oh)):
            K = int(load().mqdet_resize_coeffs_ksize(n_in, n_out))
            if t.dtype != torch.int32 or not t.is_contiguous() or tuple(t.shape) != (n_out, 2 + K):
                raise _lib.MqdetError(f"test_transform: the coefficient table of {n_in} -> {n_out} must be int32 [{n_out}, {2 + K}]")
    if want_resized and len(set(sizes)) != 1:
        raise _lib.MqdetError("test_transform: want_resized needs one output size for every image")
    dev = images[0].device
    if out is None:
        out = torch.empty((B, 3, Hp, Wp), dtype=torch.float32, device=dev)
    elif out.dtype != torch.float32 or tuple(out.shape) != (B, 3, Hp, Wp) or not out.is_contiguous() or out.device != dev:
        raise _lib.MqdetError(f"test_transform: out must be a contiguous fp32 [{B}, 3, {Hp}, {Wp}] tensor on {dev}")
    oh, ow = sizes[0]
    resized = torch.empty((B, oh, ow, 3), dtype=torch.uint8, device=dev) if want_resized else None
    src = (ctypes.c_void_p * B)(*[im.data_ptr() for im in images])
    hw = (ctypes.c_int64 * (2 * B))(*[int(v) for im in images for v in im.shape[:2]])
    xp = (ctypes.c_void_p * B)(*[t.data_ptr() for t in xtabs])
    yp = (ctypes.c_void_p * B)(*[t.data_ptr() for t in ytabs])
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s = (ctypes.c_float * 3)(*[float(v) for v in std])
    if per_image:
        ohw = (ctypes.c_int64 * (2 * B))(*[v for p in sizes for v in p])
        _launch("mqdet_test_transform_sizes", src, hw, ohw, xp, yp, B, Hp, Wp, int(bool(bgr)), int(bool(times255)), m, s, _ptr(out),
                _ptr(resized), what="test_transform", kernels=-(-B // 64))
    else:
        _launch("mqdet_test_transform", src, hw, xp, yp, B, oh, ow, Hp, Wp, int(bool(bgr)), int(bool(times255)), m, s, _ptr(out),
                _ptr(resized), what="test_transform", kernels=-(-B // 64))
    return (out, resized) if want_resized else out


# ----------------------------------------------------------------------------------------------------------------------
# Vision-only evaluation: [MASK] over the tokens of the categories drawn for masking (csrc/prompt_mask.cu)
# ----------------------------------------------------------------------------------------------------------------------
def mask_prompt_tokens(ids, tok_cat, flags, mask_id, out=None):
    """int64 token ids [E, T] -> a new int64 [E, T] (or ``out``): ``mask_id`` where the token's category ``tok_cat[e, t]``
    (int32 [E, T], -1 = none) has ``flags[e, category]`` set (uint8 [E, C]), the id otherwise.  One launch, no host read."""
    _need_cuda(ids, tok_cat, flags)
    if ids.dtype != torch.int64 or ids.dim() != 2 or not ids.is_contiguous():
        raise _lib.MqdetError("mask_prompt_tokens: contiguous int64 [E, T] token ids required")
    E, T = ids.shape
    if tok_cat.dtype != torch.int32 or tuple(tok_cat.shape) != (E, T) or not tok_cat.is_contiguous():
        raise _lib.MqdetError(f"mask_prompt_tokens: contiguous int32 [{E}, {T}] category table required")
    if flags.dtype != torch.uint8 or flags.dim() != 2 or flags.shape[0] != E or not flags.is_contiguous():
        raise _lib.MqdetError(f"mask_prompt_tokens: contiguous uint8 [{E}, C] flags required")
    if out is None:
        out = torch.empty_like(ids)
    elif out.dtype != torch.int64 or out.shape != ids.shape or not out.is_contiguous():
        raise _lib.MqdetError(f"mask_prompt_tokens: out must be contiguous int64 [{E}, {T}]")
    _launch("mqdet_mask_prompt_tokens", _ptr(ids), _ptr(tok_cat), _ptr(flags) if flags.numel() else None, E, T, flags.shape[1],
            int(mask_id), _ptr(out), what="mask_prompt_tokens")
    return out


# ----------------------------------------------------------------------------------------------------------------------
# The test-time vision-query update: candidates, the counted pooling, the bank update (csrc/query_bank.cu)
# ----------------------------------------------------------------------------------------------------------------------
class QueryBank:
    """Device-resident vision-query bank with one pooled scale per query: rows fp32 [L, cap, C] (row j of label l), count int32
    [L] (rows in use), norm fp32 [L, cap] (the L2 norm of every row in use).  Labels index the first axis directly."""

    def __init__(self, L, cap, C, device):
        if L < 1 or cap < 1 or C < 1:
            raise _lib.MqdetError(f"QueryBank: bad sizes L={L} cap={cap} C={C}")
        self.L, self.cap, self.C = int(L), int(cap), int(C)
        self.rows = torch.zeros((L, cap, C), dtype=torch.float32, device=device)
        self.count = torch.zeros((L,), dtype=torch.int32, device=device)
        self.norm = torch.zeros((L, cap), dtype=torch.float32, device=device)

    @classmethod
    def from_dict(cls, bank, L, min_cap, C, device):
        """{label: tensor [n, 1, C]} (the reference's format; missing labels and ``[]`` entries are empty) -> a bank whose capacity
        per label is max(min_cap, the most rows any label brings).  Uploaded without waiting for the stream."""
        items = {int(k): v for k, v in (bank or {}).items() if torch.is_tensor(v) and v.shape[0] > 0}
        for k, v in items.items():
            if v.dim() != 3 or v.shape[1] != 1 or v.shape[2] != C:
                raise _lib.MqdetError(f"QueryBank: label {k} has rows {tuple(v.shape)}; [n, 1, {C}] required (one pooled scale)")
            if not 0 <= k < L:
                raise _lib.MqdetError(f"QueryBank: label {k} outside [0, {L})")
        cap = max([int(min_cap)] + [v.shape[0] for v in items.values()])
        qb = cls(L, cap, C, device)
        if items:
            rows = torch.zeros((L, cap, C), dtype=torch.float32)
            cnt = torch.zeros((L,), dtype=torch.int32)
            for k, v in items.items():
                rows[k, :v.shape[0]] = v[:, 0].detach().to("cpu", torch.float32)
                cnt[k] = v.shape[0]
            qb.rows.copy_(upload_async(rows, device))
            qb.count.copy_(upload_async(cnt, device))
            _launch("mqdet_query_bank_norms", _ptr(qb.rows), _ptr(qb.count), L, cap, C, _ptr(qb.norm), what="query_bank_norms")
        return qb

    def as_dict(self, count_host):
        """The reference's format {label: [n, 1, C]} as views of the device rows (rows below a label's count never change), given
        the counts read on the host: a ``defaultdict(list)``, so that a label without rows reads as ``[]``."""
        from collections import defaultdict
        out = defaultdict(list)
        for k, n in enumerate(count_host.tolist()):
            if n > 0:
                out[k] = self.rows[k, :n, None, :]
        return out


def query_candidates(packed, img_wh, score_thr, expand_ratio, bad):
    """Packed detector rows fp32 [B, M + 1, 6] of images of one size ``img_wh`` = (w, h), or of B sizes ``img_wh`` = [(w_b, h_b)]
    (a padded batch of differently sized images; each image's boxes are clipped to its own size) -> (rois fp32 [B * M, 5], labels int32
    [B * M], count int32 [1]): the rows with score > ``score_thr``, grown by ``expand_ratio`` about their centre, clipped to the image,
    the empty ones removed, in image-then-row order; only the first ``count`` rows are written.  A count row that is not an integer in
    [0, M] adds 1 to ``bad`` (int32 [1], device).  Nothing is read on the host."""
    _need_cuda(packed, bad)
    if packed.dtype != torch.float32 or not packed.is_contiguous() or packed.dim() != 3 or packed.shape[2] != 6 or packed.shape[1] < 2:
        raise _lib.MqdetError(f"query_candidates: contiguous fp32 [B, M + 1, 6] rows required (got {packed.dtype} {tuple(packed.shape)})")
    if bad.dtype != torch.int32 or bad.numel() != 1:
        raise _lib.MqdetError("query_candidates: bad must be an int32 counter [1]")
    B, M = packed.shape[0], packed.shape[1] - 1
    dev = packed.device
    rois = torch.empty((B * M, 5), dtype=torch.float32, device=dev)
    labels = torch.empty((B * M,), dtype=torch.int32, device=dev)
    count = torch.empty((1,), dtype=torch.int32, device=dev)
    wh = [(int(w), int(h)) for w, h in img_wh] if isinstance(img_wh[0], (tuple, list)) else [(int(img_wh[0]), int(img_wh[1]))]
    wh_h = (ctypes.c_int64 * (2 * len(wh)))(*[v for p in wh for v in p])
    _launch("mqdet_query_candidates", _ptr(packed), B, M, float(score_thr), float(expand_ratio), wh_h, len(wh),
            _ptr(rois), _ptr(labels), B * M, _ptr(count), _ptr(bad), what="query_candidates")
    return rois, labels, count


def roi_align_levels_counted(pyr16, levels, scales, rois, count, pooled=7, sampling_ratio=0):
    """``roi_align_levels(mean_only=True)`` over the first ``count`` (int32 [1], device) of the rows of ``rois`` [cap, 5] -> fp32
    [cap, C]; the rows past the count are left unwritten."""
    import numpy as np
    _need_cuda(pyr16, rois, count)
    if rois.dtype != torch.float32 or not rois.is_contiguous() or rois.dim() != 2 or rois.shape[1] != 5:
        raise _lib.MqdetError("roi_align_levels_counted: contiguous fp32 rois [cap, 5] required")
    if pyr16.dtype != torch.float16 or not pyr16.is_contiguous() or count.dtype != torch.int32:
        raise _lib.MqdetError("roi_align_levels_counted: contiguous fp16 pyramid and int32 count required")
    B, N, C = pyr16.shape
    cap = rois.shape[0]
    out = torch.empty((cap, C), dtype=torch.float32, device=pyr16.device)
    sc = np.asarray(scales, dtype=np.float32)
    _launch("mqdet_roi_align_levels_counted", _ptr(pyr16), levels.hw_ptr, levels.n, sc.ctypes.data_as(ctypes.c_void_p), B, C,
            _ptr(rois), _ptr(count), cap, int(pooled), int(sampling_ratio), 1, _ptr(out), None, what="roi_align_levels_counted")
    return out


def query_bank_update(bank, feats, labels, count, max_query, sim_thr):
    """Append the first ``count`` (int32 [1], device) pooled features fp32 [cap, C] with labels int32 [cap] to ``bank`` (a
    ``QueryBank``) in order, as extract_query(exclude_similar=True) does: a feature is skipped when its label has ``max_query``
    rows, or when its normalised dot product with some row of that label exceeds ``sim_thr``.  One launch, no host read."""
    _need_cuda(feats, labels, count)
    if feats.dtype != torch.float32 or not feats.is_contiguous() or feats.dim() != 2 or feats.shape[1] != bank.C:
        raise _lib.MqdetError(f"query_bank_update: contiguous fp32 features [cap, {bank.C}] required")
    if labels.dtype != torch.int32 or labels.numel() != feats.shape[0] or count.dtype != torch.int32:
        raise _lib.MqdetError("query_bank_update: int32 labels (one per feature) and int32 count required")
    if not 0 <= int(max_query) <= bank.cap:
        raise _lib.MqdetError(f"query_bank_update: max_query {max_query} outside [0, {bank.cap}]")
    _launch("mqdet_query_bank_update", _ptr(feats), _ptr(labels), _ptr(count), bank.C, _ptr(bank.rows), _ptr(bank.count),
            _ptr(bank.norm), bank.L, bank.cap, int(max_query), float(sim_thr), what="query_bank_update")
    return bank


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
    _need_cuda(x16, om)
    B, N, C = x16.shape
    rows = levels.N if branch == 1 else levels.N1
    cols = torch.empty((B * rows, 9 * C), dtype=torch.float16, device=x16.device)
    _launch("mqdet_dcn_cols", _ptr(x16), _ptr(om), om.shape[-1] if om is not None else 0, levels.hw_ptr, levels.n, B, C,
            int(branch), _ptr(cols), what="dcn_cols")
    return cols


def dcn_conv(x16, om, levels, branches, weights, biases):
    """DyConv's DCNv2 convolutions as one implicit GEMM (no column matrix): x16 [B,N,256] fp16, om [B,N,om_ld] fp32 or None,
    branches: list of 0/1/2, weights: fp16 [256, 2304] (k = tap*256 + c) each, biases: fp32 [256] or None each
    -> list of fp16 [B*rows_j, 256]."""
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
    _launch("mqdet_dcn_conv", _ptr(x16), _ptr(om), om.shape[-1] if om is not None else 0, levels.hw_ptr, levels.n, B, C, n,
            ctypes.cast(br, ctypes.c_void_p), ctypes.cast(wp, ctypes.c_void_p),
            ctypes.cast(bp, ctypes.c_void_p), ctypes.cast(yp, ctypes.c_void_p), what="dcn_conv",
            timed=("dcn_conv_kernel", 2.0 * rows * 256 * 9 * C, 2.0 * (B * N * C + rows * 256 + n * 256 * 9 * C) + (4.0 * B * N * 27 if om is not None else 0.0)))
    return ys


def conv3x3_small(x16, w16_, bias, levels, ld=32):
    """Plain 3x3 / pad 1 conv with <= 32 output channels over all levels, no column matrix (the DyConv offset/mask conv):
    x16 [B,N,256] fp16, w16_ [O, 2304] fp16 (k = tap*256 + c), bias [O] fp32 -> [B*N, ld] fp32 (columns >= O untouched)."""
    _need_cuda(x16, w16_, bias)
    B, N, C = x16.shape
    O = w16_.shape[0]
    out = torch.empty((B * N, ld), dtype=torch.float32, device=x16.device)
    _launch("mqdet_conv3x3_small", _ptr(x16), _ptr(w16_), _ptr(bias), levels.hw_ptr, levels.n, B, C, O, _ptr(out), ld,
            what="conv3x3_small")
    return out


def chan_stats(y16, seg, B, rows_per_img, row_weights=None):
    nseg = seg.numel() - 1
    C = y16.shape[-1]
    partial = torch.empty((int(load().mqdet_chan_stats_floats(B, nseg, C)),), dtype=torch.float32, device=y16.device)
    _launch("mqdet_chan_stats", _ptr(y16), _ptr(seg), nseg, B, rows_per_img, C, _ptr(row_weights), _ptr(partial), what="chan_stats")
    return partial


def gn_attn(partial, seg, B, C, groups, weighted, gn_w, gn_b, eps, attn_w, attn_b):
    nseg = seg.numel() - 1
    affine = torch.empty((B, nseg, 2, C), dtype=torch.float32, device=partial.device)
    attn = torch.empty((B, nseg), dtype=torch.float32, device=partial.device)
    _launch("mqdet_gn_attn", _ptr(partial), _ptr(seg), nseg, B, C, groups, int(weighted), _ptr(gn_w), _ptr(gn_b),
            float(eps), _ptr(attn_w), _ptr(attn_b), _ptr(affine), _ptr(attn), what="gn_attn")
    return affine, attn


def dyconv_combine(y1, y2, y0, aff1, aff2, aff0, at1, at2, at0, levels, B):
    """-> (mid [B,N,C] fp16, mid_sums [B, L, chunks, C] fp32: per-channel sums of `mid` over pixel ranges, for DyReLU's pool)."""
    C = y1.shape[-1]
    mid = torch.empty((B, levels.N, C), dtype=torch.float16, device=y1.device)
    sums = torch.empty((B, levels.n, int(load().mqdet_dyconv_combine_chunks()), C), dtype=torch.float32, device=y1.device)
    _launch("mqdet_dyconv_combine", _ptr(y1), _ptr(y2), _ptr(y0), _ptr(aff1), _ptr(aff2), _ptr(aff0), _ptr(at1),
            _ptr(at2), _ptr(at0), levels.hw_ptr, levels.n, B, C, _ptr(mid), _ptr(sums), what="dyconv_combine")
    return mid, sums


def dyrelu(mid, levels, w1, b1, w2, b2, mid_sums=None):
    """DyReLU over every level of mid [B,N,256] fp16 -> fp16.  ``mid_sums`` = the per-range channel sums dyconv_combine
    produced (else they are taken from `mid` by chan_stats)."""
    B, N, C = mid.shape
    if mid_sums is None:
        partial, chunks, stats = chan_stats(mid, levels.seg_all, B, N), 32, 3
    else:
        partial, chunks, stats = mid_sums, mid_sums.shape[2], 1
    coef = torch.empty((B, levels.n, 4, C), dtype=torch.float32, device=mid.device)
    _launch("mqdet_dyrelu_coef", _ptr(partial), chunks, stats, _ptr(levels.seg_all), levels.n, B, C, w1.shape[0], _ptr(w1),
            _ptr(b1), _ptr(w2), _ptr(b2), _ptr(coef), what="dyrelu_coef")
    out = torch.empty_like(mid)
    _launch("mqdet_dyrelu_apply", _ptr(mid), _ptr(coef), levels.hw_ptr, levels.n, B, C, _ptr(out), what="dyrelu_apply")
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
    class_labels int32 [C] / [B, C] or None (label of score column c = c + 1).
    ``img_w`` / ``img_h``: the clip size of every element, or sequences of n per-image sizes (a padded batch of differently sized
    images); element e clips to size e % n, so a chunked pass (e = chunk * B + image) passes its B image sizes.  ``img_w`` may
    also be a CUDA fp32 tensor [n, 2] of (w, h) rows, with ``img_h`` None: the kernel reads the sizes from device memory, so a
    captured graph clips each replay to what the table holds then."""
    import numpy as np
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
    wh_dev = img_w if torch.is_tensor(img_w) and img_w.is_cuda else None
    if wh_dev is not None:
        if img_h is not None or wh_dev.dtype != torch.float32 or wh_dev.dim() != 2 or wh_dev.shape[1] != 2 or \
                not wh_dev.is_contiguous() or wh_dev.device != dev:
            raise _lib.MqdetError("atss_postprocess: a device size table must be a contiguous fp32 [n, 2] (w, h) tensor on the "
                                  "logits' device, with img_h None")
        n_sizes = wh_dev.shape[0]
    else:
        wh_h = np.ascontiguousarray(np.stack(np.broadcast_arrays(np.asarray(img_w, dtype=np.float32).reshape(-1),
                                                                 np.asarray(img_h, dtype=np.float32).reshape(-1)), 1))
        n_sizes = wh_h.shape[0]
    S = (L * pre_nms_top_n + 255) // 256 * 256
    ws = torch.empty((int(load().mqdet_atss_workspace_bytes(levels.hw_ptr, L, C, B)),), dtype=torch.uint8, device=dev)
    lvl_counts = torch.empty((B, L), dtype=torch.int32, device=dev)
    ob = torch.empty((B, S, 4), dtype=torch.float32, device=dev)
    osc = torch.empty((B, S), dtype=torch.float32, device=dev)
    ol = torch.empty((B, S), dtype=torch.float32, device=dev)
    okey = torch.empty((B, S), dtype=torch.int64, device=dev) if want_keys else None
    cb, csc, cl = torch.empty_like(ob), torch.empty_like(osc), torch.empty_like(ol)
    totals = torch.empty((B,), dtype=torch.int32, device=dev)
    entry = "mqdet_atss_candidates" if wh_dev is None else "mqdet_atss_candidates_sizes_dev"
    wh_ptr = wh_h.ctypes.data_as(ctypes.c_void_p) if wh_dev is None else _ptr(wh_dev)
    _launch(entry, _ptr(logits), _dt(logits), _ptr(reg_ctr), _ptr(tokmap), tm_stride, _ptr(class_labels), lab_stride, C, max_tok, T,
            levels.hw_ptr, L, stride_h.ctypes.data_as(ctypes.c_void_p), base_h.ctypes.data_as(ctypes.c_void_p),
            scale_h.ctypes.data_as(ctypes.c_void_p), B, float(pre_nms_thresh), int(pre_nms_top_n), S, wh_ptr, n_sizes, _ptr(ws),
            _ptr(lvl_counts), _ptr(ob), _ptr(osc), _ptr(ol), _ptr(okey), _ptr(cb), _ptr(csc), _ptr(cl), _ptr(totals),
            what="atss_candidates", kernels=3)
    nws = torch.empty((int(load().mqdet_ml_nms_batched_workspace_bytes(B, S)),), dtype=torch.uint8, device=dev)
    keep = torch.empty((B, S), dtype=torch.int64, device=dev)
    num = torch.empty((B,), dtype=torch.int32, device=dev)
    _launch("mqdet_ml_nms_batched", _ptr(cb), _ptr(csc), _ptr(cl), _ptr(totals), B, S, float(nms_thresh), int(max_det),
            _ptr(keep), _ptr(num), _ptr(nws), what="ml_nms_batched", kernels=6)
    # packed fixed-shape result [B, max_out + 1, 6]: rows 0..max_out-1 = detections, row max_out = (count, 0, ...)
    packed = torch.empty((B, max_out + 1, 6), dtype=torch.float32, device=dev)
    _launch("mqdet_gather_detections", _ptr(cb), _ptr(csc), _ptr(cl), _ptr(keep), _ptr(num), B, S, max_out, max_out + 1,
            _ptr(packed), what="gather_detections")
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
    B = gt_count.shape[0]
    gt_boxes, gt_labels, gt_count, G = _gt_pack(gt_boxes, gt_labels, gt_count, B)
    dev = gt_boxes.device
    stride_h, base_h, _ = _level_anchor_tables(strides, anchor_sizes)
    N = levels.N
    ws = torch.empty((int(load().mqdet_atss_assign_workspace_bytes(B, N)),), dtype=torch.uint8, device=dev)
    match = torch.empty((B, N), dtype=torch.int32, device=dev)
    img_stats = torch.empty((B, 2), dtype=torch.float32, device=dev)
    norm = torch.empty((4,), dtype=torch.float32, device=dev)
    _launch("mqdet_atss_assign", _ptr(gt_boxes), _ptr(gt_labels), _ptr(gt_count), B, G, levels.hw_ptr, levels.n,
            stride_h.ctypes.data_as(ctypes.c_void_p), base_h.ctypes.data_as(ctypes.c_void_p), int(topk),
            _ptr(ws), _ptr(match), _ptr(img_stats), _ptr(norm), what="atss_assign", kernels=4)
    return {"match": match, "img_stats": img_stats, "norm": norm}


def atss_loss(logits, reg_ctr, gt_boxes, gt_labels, gt_count, gt_tokens, levels, strides, anchor_sizes, reg_scales, text_mask=None, *,
              targets=None, world=1, topk=9, alpha=0.25, gamma=2.0, reg_weight=2.0, token_weight=1.0):
    """The MQ-GLIP pre-training detection losses (loss.py:850-1201 with the shipped flags) and their gradients at the head outputs.

    logits fp32 [B, N, T] (dot-product token logits), reg_ctr fp32 [B, N, 5] (raw box / centerness GEMM output, before the per-level
    ``reg_scales``), the GT pack of ``atss_targets`` plus gt_tokens [B, Gmax, T] (positive_map rows), text_mask [B, T] or None ->
    (losses fp32 [4] = (loss_reg, loss_centerness, loss_dot_product_token, loss_cls = 0), d_logits fp32 [B, N, T],
    d_reg_ctr fp32 [B, N, 5]).  ``targets``: the result of ``atss_targets`` (its ``norm[:2]`` summed over ``world`` ranks), else
    computed here for one rank.  All on the device, no host synchronisation: capturable in a CUDA graph at a fixed Gmax."""
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
    _launch("mqdet_atss_loss", _ptr(logits), _ptr(reg_ctr), _ptr(targets["match"]), _ptr(gt_boxes), _ptr(gt_labels), _ptr(tok), B, G,
            T, _ptr(tm), levels.hw_ptr, levels.n, stride_h.ctypes.data_as(ctypes.c_void_p),
            base_h.ctypes.data_as(ctypes.c_void_p), scale_h.ctypes.data_as(ctypes.c_void_p),
            _ptr(targets["norm"]), float(world), float(alpha), float(gamma), float(reg_weight),
            float(token_weight), _ptr(ws), _ptr(losses), _ptr(d_logits), _ptr(d_reg_ctr), what="atss_loss", kernels=3,
            timed=("atss_loss", 0.0, 8.0 * B * N * T + 40.0 * B * N))
    return losses, d_logits, d_reg_ctr


def _gdino_gt_pack(gt_boxes, gt_count, gt_tokens, B, Q, T):
    """Validates the GroundingDINO GT pack (``atss_targets`` convention, boxes normalised cxcywh) -> contiguous tensors + Gmax."""
    _need_cuda(gt_boxes, gt_count, gt_tokens)
    if gt_boxes.dim() != 3 or gt_boxes.shape[0] != B or gt_boxes.shape[2] != 4:
        raise ValueError(f"gt_boxes must be [B={B}, Gmax, 4]; got {tuple(gt_boxes.shape)}")
    G = gt_boxes.shape[1]
    if tuple(gt_count.shape) != (B,) or tuple(gt_tokens.shape) != (B, G, T):
        raise ValueError(f"gt_count must be [B] = ({B},) and gt_tokens [B, Gmax, T] = {(B, G, T)}; got {tuple(gt_count.shape)}, "
                         f"{tuple(gt_tokens.shape)}")
    if G < 1 or G > Q:
        raise ValueError(f"GT capacity Gmax={G} must be in 1..Q={Q}")
    return gt_boxes.float().contiguous(), gt_count.to(torch.int32).contiguous(), gt_tokens.float().contiguous(), G


def _decoder_outputs(pred_logits, pred_boxes):
    _need_cuda(pred_logits, pred_boxes)
    if pred_logits.dim() != 4 or pred_boxes.dim() != 4 or pred_boxes.shape[:3] != pred_logits.shape[:3] or pred_boxes.shape[3] != 4:
        raise ValueError(f"pred_logits [L, B, Q, T] and pred_boxes [L, B, Q, 4] required; got {tuple(pred_logits.shape)}, "
                         f"{tuple(pred_boxes.shape)}")
    for t in (pred_logits, pred_boxes):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise _lib.MqdetError("gdino: pred_logits / pred_boxes must be contiguous fp32")
    return pred_logits.shape


def linear_sum_assignment(cost, counts):
    """``scipy.optimize.linear_sum_assignment`` of a batch of cost matrices on the device, index for index scipy's result (ties
    included): cost fp32 [P, Q, Gmax], counts [P] (device) -> match int32 [P, Q] = the column (GT) assigned to row (query) q of
    ``cost[p, :, :counts[p]]``, -1 for unassigned rows.  Requires counts[p] <= Gmax <= Q (rows >= columns) and finite costs."""
    _need_cuda(cost, counts)
    if cost.dim() != 3 or cost.dtype != torch.float32:
        raise ValueError(f"cost must be fp32 [P, Q, Gmax]; got {cost.dtype} {tuple(cost.shape)}")
    P, Q, G = cost.shape
    if tuple(counts.shape) != (P,):
        raise ValueError(f"counts must be [P] = ({P},); got {tuple(counts.shape)}")
    if G < 1 or G > Q:
        raise ValueError(f"Gmax={G} must be in 1..Q={Q}")
    return _lsa(cost.contiguous(), counts.to(torch.int32).contiguous(), P, Q, G)


def _lsa(cost, counts, P, Q, G):
    ws = torch.empty((int(load().mqdet_linear_sum_assignment_workspace_bytes(P, Q, G)),), dtype=torch.uint8, device=cost.device)
    match = torch.empty((P, Q), dtype=torch.int32, device=cost.device)
    _launch("mqdet_linear_sum_assignment", _ptr(cost), _ptr(counts), counts.shape[0], P, Q, G, _ptr(ws), _ptr(match),
            what="linear_sum_assignment", kernels=2)
    return match


def gdino_match(pred_logits, pred_boxes, gt_boxes, gt_count, gt_tokens, *, cost_class=1.0, cost_bbox=5.0, cost_giou=2.0,
                focal_alpha=0.25):
    """HungarianMatcher (matcher.py:49-86) of every decoder layer on the device: pred_logits fp32 [L, B, Q, T] (raw), pred_boxes fp32
    [L, B, Q, 4] (sigmoid cxcywh), GT pack gt_boxes [B, Gmax, 4] (normalised cxcywh), gt_count [B], gt_tokens [B, Gmax, T] ->
    dict(cost fp32 [L, B, Q, Gmax] (0 beyond gt_count), match int32 [L, B, Q] (matched GT or -1), norm fp32 [1] = sum of gt_count,
    the normaliser data-parallel ranks all-reduce).  No host synchronisation: capturable in a CUDA graph at a fixed Gmax."""
    L, B, Q, T = _decoder_outputs(pred_logits, pred_boxes)
    gt_boxes, gt_count, gt_tokens, G = _gdino_gt_pack(gt_boxes, gt_count, gt_tokens, B, Q, T)
    dev = pred_logits.device
    cost = torch.empty((L, B, Q, G), dtype=torch.float32, device=dev)
    norm = torch.empty((1,), dtype=torch.float32, device=dev)
    _launch("mqdet_gdino_match_cost", _ptr(pred_logits), _ptr(pred_boxes), _ptr(gt_boxes), _ptr(gt_count), _ptr(gt_tokens), L, B, Q,
            T, G, float(focal_alpha), float(cost_class), float(cost_bbox), float(cost_giou),
            _ptr(cost), _ptr(norm), what="gdino_match_cost",
            timed=("gdino_match_cost", 2.0 * L * B * Q * T * G, 4.0 * L * B * Q * (T + G)))
    match = _lsa(cost.view(L * B, Q, G), gt_count, L * B, Q, G).view(L, B, Q)
    return {"cost": cost, "match": match, "norm": norm}


def gdino_set_loss(pred_logits, pred_boxes, gt_boxes, gt_count, gt_tokens, text_mask=None, *, targets=None, world=1, alpha=0.25,
                   gamma=2.0, ce_coef=2.0, bbox_coef=5.0, giou_coef=2.0, cost_class=1.0, cost_bbox=5.0, cost_giou=2.0, focal_alpha=0.25):
    """SetCriterion (loss.py:42-178) of every decoder layer on the device, with its gradients at the decoder outputs.

    Inputs as ``gdino_match``, plus text_mask [B, T] (> 0 = token in use) or None.  ``targets``: the result of ``gdino_match``
    (its ``norm`` summed over ``world`` ranks), else computed here for one rank.  -> (losses fp32 [L, 3] = (loss_ce, loss_bbox,
    loss_giou) per layer, already weighted; d_logits fp32 [L, B, Q, T], d_boxes fp32 [L, B, Q, 4] = the gradient of their sum;
    norm fp32 [1], the device-resident normaliser).  Row L-1 is the reference's un-suffixed keys, row k < L-1 its ``_k`` keys."""
    L, B, Q, T = _decoder_outputs(pred_logits, pred_boxes)
    gt_boxes, gt_count, gt_tokens, G = _gdino_gt_pack(gt_boxes, gt_count, gt_tokens, B, Q, T)
    _need_cuda(text_mask)
    if text_mask is not None and tuple(text_mask.shape) != (B, T):
        raise ValueError(f"text_mask must be [B, T] = {(B, T)}; got {tuple(text_mask.shape)}")
    if targets is None:
        targets = gdino_match(pred_logits, pred_boxes, gt_boxes, gt_count, gt_tokens, cost_class=cost_class, cost_bbox=cost_bbox,
                              cost_giou=cost_giou, focal_alpha=focal_alpha)
    if tuple(targets["match"].shape) != (L, B, Q):
        raise ValueError(f"targets['match'] must be [L, B, Q] = {(L, B, Q)}; got {tuple(targets['match'].shape)}")
    dev = pred_logits.device
    tm = None if text_mask is None else text_mask.float().contiguous()
    ws = torch.empty((int(load().mqdet_gdino_set_loss_workspace_floats(L, B, Q)),), dtype=torch.float32, device=dev)
    losses = torch.empty((L, 3), dtype=torch.float32, device=dev)
    d_logits = torch.empty_like(pred_logits)
    d_boxes = torch.empty_like(pred_boxes)
    _launch("mqdet_gdino_set_loss", _ptr(pred_logits), _ptr(pred_boxes), _ptr(targets["match"]), _ptr(gt_boxes), _ptr(gt_tokens),
            L, B, Q, T, G, _ptr(tm), _ptr(targets["norm"]), float(world), float(alpha), float(gamma),
            float(ce_coef), float(bbox_coef), float(giou_coef), _ptr(ws), _ptr(losses), _ptr(d_logits),
            _ptr(d_boxes), what="gdino_set_loss", kernels=3, timed=("gdino_set_loss", 0.0, 8.0 * L * B * Q * T + 32.0 * L * B * Q))
    return losses, d_logits, d_boxes, targets["norm"]


def anchors(grid_h, grid_w, stride, size, img_w, img_h, device):
    """Anchors [H*W, 4] + visibility [H*W] of one level (anchor_generator.py:72-109)."""
    import numpy as np
    out = torch.empty((grid_h * grid_w, 4), dtype=torch.float32, device=device)
    vis = torch.empty((grid_h * grid_w,), dtype=torch.uint8, device=device)
    base = np.asarray(base_anchor(stride, size), dtype=np.float32)
    _launch("mqdet_anchors", _ptr(out), _ptr(vis), grid_h, grid_w, float(stride), base.ctypes.data_as(ctypes.c_void_p),
            float(img_w), float(img_h), what="anchors")
    return out, vis.bool()


# ----------------------------------------------------------------------------------------------------------------------
# Swin / FPN glue
# ----------------------------------------------------------------------------------------------------------------------
def patchify4(img):
    """[B,3,H,W] fp32 -> (fp16 [B*Hp*Wp, 48], Hp, Wp)."""
    _need_cuda(img)
    B, _, H, W = img.shape
    Hp, Wp = (H + 3) // 4, (W + 3) // 4
    img = img.float().contiguous()
    out = torch.empty((B * Hp * Wp, 48), dtype=torch.float16, device=img.device)
    _launch("mqdet_patchify4", _ptr(img), B, H, W, _ptr(out), what="patchify4")
    return out, Hp, Wp


def swin_window_attn(qkv16, qkv_bias, bias_dense, B, H, W, heads, window, shift, scale):
    _need_cuda(qkv16, qkv_bias, bias_dense)
    C = qkv16.shape[-1] // 3
    out = torch.empty((B * H * W, C), dtype=torch.float16, device=qkv16.device)
    _launch("mqdet_swin_window_attn", _ptr(qkv16), _ptr(qkv_bias), _ptr(bias_dense), B, H, W, heads, window, shift,
            float(scale), _ptr(out), what="swin_window_attn")
    return out


def patch_merge_ln(x32, B, H, W, gamma, beta, eps):
    _need_cuda(x32)
    C = x32.shape[-1]
    H2, W2 = (H + 1) // 2, (W + 1) // 2
    out = torch.empty((B * H2 * W2, 4 * C), dtype=torch.float16, device=x32.device)
    _launch("mqdet_patch_merge_ln", _ptr(x32), B, H, W, C, _ptr(gamma), _ptr(beta), float(eps), _ptr(out), what="patch_merge_ln")
    return out, H2, W2


def upsample_add(lateral16, top16, B, H, W, Hs, Ws):
    _need_cuda(lateral16, top16)
    C = lateral16.shape[-1]
    out = torch.empty_like(lateral16)
    _launch("mqdet_upsample_add", _ptr(lateral16), _ptr(top16), B, H, W, Hs, Ws, C, _ptr(out), what="upsample_add")
    return out


def im2col3x3(x16, B, H, W, stride=1, relu_in=False):
    """x16: fp16 [B, H*W, C] (may be a batch-strided view with contiguous rows) -> cols [B*Ho*Wo, 9C], Ho, Wo."""
    _need_cuda(x16)
    C = x16.shape[-1]
    assert x16.stride(-1) == 1 and x16.stride(-2) == C
    Ho, Wo = (H + 2 - 3) // stride + 1, (W + 2 - 3) // stride + 1
    cols = torch.empty((B * Ho * Wo, 9 * C), dtype=torch.float16, device=x16.device)
    _launch("mqdet_im2col3x3", _ptr(x16), x16.stride(0) if x16.dim() == 3 else H * W * C, B, H, W, C, stride,
            int(bool(relu_in)), _ptr(cols), what="im2col3x3")
    return cols, Ho, Wo


def avgpool2_levels(x16, levels):
    """fp16 [B,N,C] pyramid -> fp32 [B, I, C] pooled tokens (AvgPool2d(2) per level, concatenated)."""
    _need_cuda(x16)
    B, N, C = x16.shape
    I = sum((h // 2) * (w // 2) for h, w in levels.sizes)
    out = torch.empty((B, I, C), dtype=torch.float32, device=x16.device)
    _launch("mqdet_avgpool2_levels", _ptr(x16), levels.hw_ptr, levels.n, B, C, _ptr(out), what="avgpool2_levels")
    return out


def roi_align_levels(pyr16, levels, scales, rois, pooled=7, sampling_ratio=0, mean_only=True):
    """Pooler (LevelMapper + aligned ROIAlign per level) over the fp16 pyramid [B,N,C]: rois [R,5] fp32 (image index, x1, y1, x2,
    y2) -> ([R,C] fp32 mean over the pooled bins | [R,C,pooled,pooled] fp32, level int32 [R])."""
    import numpy as np
    _need_cuda(pyr16, rois)
    B, N, C = pyr16.shape
    R = rois.shape[0]
    rois = rois.float().contiguous()
    out = torch.empty((R, C) if mean_only else (R, C, pooled, pooled), dtype=torch.float32, device=pyr16.device)
    lvl = torch.empty((R,), dtype=torch.int32, device=pyr16.device)
    sc = np.asarray(scales, dtype=np.float32)
    _launch("mqdet_roi_align_levels", _ptr(pyr16), levels.hw_ptr, levels.n, sc.ctypes.data_as(ctypes.c_void_p), B, C, _ptr(rois), R,
            int(pooled), int(sampling_ratio), int(bool(mean_only)), _ptr(out), _ptr(lvl), what="roi_align_levels")
    return out, lvl


def ms_deform_attn(value16, proj32, aw_col0, ref, levels, heads, points, out_dtype=torch.float16):
    """Fused multi-scale deformable attention core: value16 [B,Nv,heads*32] fp16, proj32 [B*Q, >= heads*L*P*3] fp32 (sampling
    offsets | attention logits from column aw_col0), ref [B,Q,L,2|4] fp32 -> [B,Q,heads*32]."""
    _need_cuda(value16, proj32, ref)
    B, Nv, E = value16.shape
    Q = ref.shape[1]
    if value16.dtype != torch.float16 or proj32.dtype != torch.float32 or not value16.is_contiguous() or proj32.stride(-1) != 1:
        raise _lib.MqdetError("ms_deform_attn: value fp16 contiguous, proj fp32 with contiguous rows required")
    if Nv != levels.N or ref.shape[2] != levels.n:
        raise _lib.MqdetError("ms_deform_attn: value rows / reference points do not match the level table")
    out = torch.empty((B, Q, E), dtype=out_dtype, device=value16.device)
    _launch("mqdet_ms_deform_attn", _ptr(value16), _ptr(proj32), proj32.stride(0), int(aw_col0), _ptr(ref), ref.shape[-1],
            levels.hw_ptr, levels.n, B, Q, heads, E // heads, points, _ptr(out), _dt(out), what="ms_deform_attn")
    return out


# ----------------------------------------------------------------------------------------------------------------------
# GroundingDINO encoder / decoder assembly (csrc/gdino_asm.cu)
# ----------------------------------------------------------------------------------------------------------------------
def add_cast(a32, b32=None, rowgate=None, *, out16=True, out32=False):
    """(a + b) * rowgate[row] over contiguous fp32 [..., D] tensors -> fp16 and / or fp32 (a gated-off row is exactly 0)."""
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
    _launch("mqdet_add_cast", _ptr(a32), _ptr(b32), _ptr(rowgate), rows, D, _ptr(o16), _ptr(o32), what="add_cast")
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def groupnorm_rows(x, groups, gamma, beta, eps=1e-5, *, out16=True, out32=False):
    """nn.GroupNorm(groups, C) over x [B, HW, C] (fp16 / fp32 rows) -> fp16 and / or fp32 [B, HW, C]."""
    _need_cuda(x, gamma, beta)
    x = x.contiguous()
    B, HW, C = x.shape
    ws = torch.empty((int(load().mqdet_groupnorm_rows_workspace_floats(B, C)),), dtype=torch.float32, device=x.device)
    o16 = torch.empty(x.shape, dtype=torch.float16, device=x.device) if out16 else None
    o32 = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out32 else None
    _launch("mqdet_groupnorm_rows", _ptr(x), _dt(x), B, HW, C, int(groups), _ptr(gamma), _ptr(beta), float(eps), _ptr(o16),
            _ptr(o32), _ptr(ws), what="groupnorm_rows", kernels=2)
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def box_refine_sine(ref_in, valid_ratios, *, delta=None, ref_is_logit=False, want_sine=True):
    """Decoder box refinement + conditional query embedding.  ref_in fp32 [B, nq, 4]; valid_ratios fp32 [B, L, 2]; delta fp32
    [B, nq, >=4] (row stride = its last-dim size) or None -> (ref [B,nq,4], ref_input [B,nq,L,4], sine fp16 [B,nq,512] | None)."""
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
    _launch("mqdet_box_refine_sine", _ptr(delta), ldd, _ptr(ref_in), int(bool(ref_is_logit)), _ptr(vr), B, nq, L, _ptr(ref),
            _ptr(ref_input), _ptr(sine), what="box_refine_sine")
    return ref, ref_input, sine


def gdino_detections(logits, boxes, tokmap, img_wh, box_threshold, max_out=None, *, class_labels=None):
    """Raw class logits fp32 [B, nq, T] + boxes fp32 [B, nq, 4] (cxcywh, normalised) -> packed [B, max_out + 1, 6]
    (x1, y1, x2, y2, score, label; last row = count).  tokmap int32 [C, max_tok] (shared; column c = label c + 1) or
    [B, C, max_tok] (one table per element: batched prompt chunks); class_labels int32 [C] / [B, C] = the label of each column,
    columns in ascending label order (ties go to the lowest label), or None (label c + 1); img_wh fp32 [B, 2] = (W, H)."""
    _need_cuda(logits, boxes, tokmap, img_wh, class_labels)
    B, nq, T = logits.shape
    C, max_tok = tokmap.shape[-2:]
    if tokmap.dtype != torch.int32 or not tokmap.is_contiguous() or tokmap.dim() not in (2, 3) or \
            (tokmap.dim() == 3 and tokmap.shape[0] != B):
        raise ValueError("gdino_detections: tokmap must be contiguous int32 [C, max_tok] or [B, C, max_tok]")
    tm_stride = C * max_tok if tokmap.dim() == 3 else 0
    lab_stride = 0
    if class_labels is not None:
        if class_labels.dtype != torch.int32 or not class_labels.is_contiguous() or class_labels.shape[-1] != C or \
                class_labels.dim() not in (1, 2) or (class_labels.dim() == 2 and class_labels.shape[0] != B):
            raise ValueError("gdino_detections: class_labels must be contiguous int32 [C] or [B, C]")
        lab_stride = C if class_labels.dim() == 2 else 0
    max_out = nq if max_out is None else int(max_out)
    out = torch.empty((B, max_out + 1, 6), dtype=torch.float32, device=logits.device)
    ws = torch.empty((int(load().mqdet_gdino_detections_workspace_floats(B, nq)),), dtype=torch.float32, device=logits.device)
    _launch("mqdet_gdino_detections", _ptr(logits.float().contiguous()), T, _ptr(boxes.float().contiguous()), _ptr(tokmap),
            tm_stride, _ptr(class_labels), lab_stride, C, max_tok, _ptr(img_wh.float().contiguous()),
            float(box_threshold), B, nq, max_out, _ptr(out), _ptr(ws), what="gdino_detections", kernels=2)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# Training side (csrc/train.cu): GCP backward pieces, token focal loss, clipping + AdamW
# ----------------------------------------------------------------------------------------------------------------------
def transpose_cast(x, scale=1.0):
    """x [R, C] (fp16 / fp32, contiguous rows) -> fp16 [C, Rp] with Rp = R rounded up to 8, the padding columns zero: the K-major
    operand of a weight-gradient product dW = dY^T X (K = the row dimension)."""
    _need_cuda(x)
    if x.dim() != 2 or x.stride(1) != 1:
        raise _lib.MqdetError("transpose_cast: 2-D tensor with contiguous rows required")
    R, C = x.shape
    Rp = (R + 7) // 8 * 8
    out = torch.empty((C, Rp), dtype=torch.float16, device=x.device)
    _launch("mqdet_transpose_cast", _ptr(x), _dt(x), R, C, x.stride(0), float(scale), _ptr(out), Rp, what="transpose_cast")
    return out


def transpose_cast_batched(x):
    """x [nb2, nb1, R, C] (fp16 / fp32, arbitrary batch / row strides, contiguous last dim) -> fp16 [nb2, nb1, C, Rp] contiguous,
    Rp = R rounded up to 8 with zero padding."""
    _need_cuda(x)
    if x.dim() != 4 or x.stride(3) != 1:
        raise _lib.MqdetError("transpose_cast_batched: 4-D tensor with a contiguous last dimension required")
    nb2, nb1, R, C = x.shape
    Rp = (R + 7) // 8 * 8
    out = torch.empty((nb2, nb1, C, Rp), dtype=torch.float16, device=x.device)
    _launch("mqdet_transpose_cast_batched", _ptr(x), _dt(x), nb1, nb2, x.stride(1), x.stride(0), R, C, x.stride(2), 1.0, _ptr(out), Rp,
            what="transpose_cast_batched")
    return out


def softmax_bwd_rows(p16, dp32, scale=1.0):
    """ds = scale * p * (dp - sum(p * dp)) over the last dim: p16 fp16 / dp32 fp32 [..., n] contiguous -> fp16 [..., n]."""
    _need_cuda(p16, dp32)
    if p16.dtype != torch.float16 or dp32.dtype != torch.float32 or not p16.is_contiguous() or not dp32.is_contiguous() or \
            p16.shape != dp32.shape:
        raise _lib.MqdetError("softmax_bwd_rows: contiguous p fp16 / dp fp32 of one shape")
    n = p16.shape[-1]
    rows = p16.numel() // n
    out = torch.empty_like(p16)
    _launch("mqdet_softmax_bwd_rows", _ptr(p16), n, _ptr(dp32), n, rows, n, n, float(scale), _ptr(out), n, what="softmax_bwd_rows")
    return out


def layernorm_bwd(dy32, x32, gamma, eps, dx=None, want_param_grads=True, x2=None):
    """nn.LayerNorm backward from the saved input (``x32 + x2`` when ``x2`` is given): dy32 / x32 fp32 [..., D] -> (dx, dgamma,
    dbeta); ``dx`` given: accumulated into."""
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
    _launch("mqdet_layernorm_bwd", _ptr(dy32), _ptr(x32), _ptr(x2), _ptr(gamma), float(eps), rows, D, _ptr(dx), int(acc), _ptr(dg), _ptr(db),
            _ptr(ws), what="layernorm_bwd", kernels=3)
    return dx, dg, db


def gelu_bwd(z16, dh):
    """dz = dh * gelu'(z) (exact erf GELU): z16 fp16, dh fp16 / fp32 of the same shape -> fp16."""
    _need_cuda(z16, dh)
    if z16.dtype != torch.float16 or not z16.is_contiguous() or not dh.is_contiguous() or dh.shape != z16.shape:
        raise _lib.MqdetError("gelu_bwd: contiguous tensors of one shape, z fp16")
    out = torch.empty_like(z16)
    _launch("mqdet_gelu_bwd", _ptr(z16), _ptr(dh), _dt(dh), z16.numel(), _ptr(out), what="gelu_bwd")
    return out


def gcp_gate_bwd(dx1, s32, g, w2):
    """Backward of x1 = s * tanh(h1 . w2) + x: dx1 / s32 fp32 [M, D], g fp32 [M] (the gate values), w2 fp32 [Dg] ->
    (ds fp32 [M, D], dgpre fp32 [M], dh1 fp16 [M, Dg])."""
    _need_cuda(dx1, s32, g, w2)
    M, D = dx1.shape
    Dg = w2.numel()
    ds = torch.empty_like(dx1)
    dgpre = torch.empty((M,), dtype=torch.float32, device=dx1.device)
    dh1 = torch.empty((M, Dg), dtype=torch.float16, device=dx1.device)
    _launch("mqdet_gcp_gate_bwd", _ptr(dx1), _ptr(s32), _ptr(g), _ptr(w2), M, D, Dg, _ptr(ds), _ptr(dgpre), _ptr(dh1),
            what="gcp_gate_bwd")
    return ds, dgpre, dh1


def colsum_weighted(h16, w32):
    """out[j] = sum_r w32[r] * h16[r, j] -> fp32 [C]."""
    _need_cuda(h16, w32)
    R, C = h16.shape
    out = torch.empty((C,), dtype=torch.float32, device=h16.device)
    ws = torch.empty((int(load().mqdet_colsum_weighted_workspace_floats(C)),), dtype=torch.float32, device=h16.device)
    _launch("mqdet_colsum_weighted", _ptr(h16.contiguous()), _ptr(w32), R, C, _ptr(out), _ptr(ws), what="colsum_weighted", kernels=2)
    return out


def gcp_sparse_attn_bwd(q, kv, idx, dout16, heads, dim_head):
    """Backward of gcp_sparse_attn: q [B,T,512] fp16, kv [B,V+1,1024] fp16, idx int32 [B,T,S], dout16 [B,T,512] fp16 ->
    (dq fp16 [B,T,512], dkv fp32 [B,V+1,1024])."""
    _need_cuda(q, kv, idx, dout16)
    B, T, inner = q.shape
    V1 = kv.shape[1]
    S = idx.shape[-1]
    dq = torch.empty_like(q)
    dkv = torch.zeros((B, V1, 2 * inner), dtype=torch.float32, device=q.device)
    _launch("mqdet_gcp_sparse_attn_bwd", _ptr(q.contiguous()), _ptr(kv.contiguous()), _ptr(idx), _ptr(dout16.contiguous()), B, T, V1 - 1,
            S, heads, dim_head, _ptr(dq), _ptr(dkv), what="gcp_sparse_attn_bwd")
    return dq, dkv


def dot_sum(a32, b32=None, one_minus_tanh2_of=None, mul=1.0):
    """mul * sum(a * b) (b None: sum a^2), times 1 - tanh(s)^2 for a device scalar ``one_minus_tanh2_of`` -> device scalar [1]."""
    _need_cuda(a32, b32, one_minus_tanh2_of)
    out = torch.empty((1,), dtype=torch.float32, device=a32.device)
    ws = torch.empty((int(load().mqdet_reduce_workspace_floats()),), dtype=torch.float32, device=a32.device)
    _launch("mqdet_dot_sum", _ptr(a32.contiguous()), _ptr(None if b32 is None else b32.contiguous()), a32.numel(),
            _ptr(one_minus_tanh2_of), float(mul), _ptr(out), _ptr(ws), what="dot_sum", kernels=2)
    return out


def scale_cast(x32, scalar=None, tanh_scalar=False, alpha=1.0, out16=True, out32=False):
    """x * alpha * (tanh)(scalar[0]) -> fp16 and / or fp32 (``scalar``: a device scalar, read on the device)."""
    _need_cuda(x32, scalar)
    x32 = x32.contiguous()
    o16 = torch.empty(x32.shape, dtype=torch.float16, device=x32.device) if out16 else None
    o32 = torch.empty(x32.shape, dtype=torch.float32, device=x32.device) if out32 else None
    _launch("mqdet_scale_cast", _ptr(x32), _ptr(scalar), int(bool(tanh_scalar)), float(alpha), x32.numel(), _ptr(o16), _ptr(o32),
            what="scale_cast")
    if out16 and out32:
        return o16, o32
    return o16 if out16 else o32


def token_focal_loss(logits, targets, text_mask=None, alpha=0.25, gamma=2.0, want_grad=True, grad_scale=1.0):
    """token_sigmoid_binary_focal_loss(...).sum() over logits / targets fp32 [B, N, T] with the text mask [B, T] ->
    (loss device scalar [1], dlogits fp32 [B, N, T] | None)."""
    _need_cuda(logits, targets, text_mask)
    B, N, T = logits.shape
    loss = torch.empty((1,), dtype=torch.float32, device=logits.device)
    dl = torch.empty_like(logits, dtype=torch.float32) if want_grad else None
    ws = torch.empty((int(load().mqdet_reduce_workspace_floats()),), dtype=torch.float32, device=logits.device)
    tm = None if text_mask is None else text_mask.float().contiguous()
    _launch("mqdet_token_focal_loss", _ptr(logits.float().contiguous()), _ptr(targets.float().contiguous()), _ptr(tm), float(alpha),
            float(gamma), B, N, T, float(grad_scale), _ptr(loss), _ptr(dl), _ptr(ws), what="token_focal_loss", kernels=2)
    return loss, dl


def clip_coef(grads, max_norm):
    """Global L2 norm over a list of fp32 gradient tensors and the clip_grad_norm_ coefficient, all on the device ->
    fp32 [2] = (coefficient, norm)."""
    _need_cuda(*grads)
    dev = grads[0].device
    partials = torch.zeros((64 * len(grads),), dtype=torch.float32, device=dev)
    n_written = ctypes.c_int64(0)
    off = 0
    for g in grads:
        g = g if g.is_contiguous() else g.contiguous()
        _launch("mqdet_sqnorm_partials", _ptr(g), g.numel(), ctypes.c_void_p(partials.data_ptr() + 4 * off), 64,
                ctypes.byref(n_written), what="sqnorm_partials")
        off += int(n_written.value)
    coef = torch.empty((2,), dtype=torch.float32, device=dev)
    _launch("mqdet_clip_coef", _ptr(partials), off, float(max_norm), _ptr(coef), what="clip_coef")
    return coef


def adamw_step_(param, grad, exp_avg, exp_avg_sq, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, grad_scale=None):
    """torch.optim.AdamW update of one fp32 tensor in place; ``grad_scale`` = a device scalar (the clip coefficient) or None."""
    _need_cuda(param, grad, exp_avg, exp_avg_sq, grad_scale)
    for t in (param, grad, exp_avg, exp_avg_sq):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise _lib.MqdetError("adamw_step_: contiguous fp32 tensors required")
    _launch("mqdet_adamw_step", _ptr(param), _ptr(grad), _ptr(exp_avg), _ptr(exp_avg_sq), param.numel(), float(lr), float(betas[0]),
            float(betas[1]), float(eps), float(weight_decay), int(step), _ptr(grad_scale), what="adamw_step")
    return param


# ----------------------------------------------------------------------------------------------------------------------
# Box AP, LVIS and COCO (csrc/lvis_eval.cu)
# ----------------------------------------------------------------------------------------------------------------------
class LvisPool:
    """Device-resident detection pool of the box AP evaluators: score fp32 [cap], box fp32 xywh [cap, 4], img / cat int32 [cap]
    (indices into the sorted GT image / category ids; cat -1 = empty slot), seq int64 [cap] (arrival number)."""

    def __init__(self, cap, device):
        self.cap = int(cap)
        self.score = torch.zeros((cap,), dtype=torch.float32, device=device)
        self.box = torch.zeros((cap, 4), dtype=torch.float32, device=device)
        self.img = torch.full((cap,), -1, dtype=torch.int32, device=device)
        self.cat = torch.full((cap,), -1, dtype=torch.int32, device=device)
        self.seq = torch.zeros((cap,), dtype=torch.int64, device=device)

    def fields(self):
        return self.score, self.box, self.img, self.cat, self.seq


def lvis_collect(pool, base, seq_base, packed, img_idx, ratios, cat_ids, *, label_map=None, need_img, bad, need_cat=None,
                 wh_plus_one=False, bad_img=None):
    """Append packed detector rows fp32 [G, B, M + 1, 6] to ``pool`` at slots base + (b * G + g) * M + r (rule 1 conversion with
    ratios fp32 [B, 2], widths and heights + 1 when ``wh_plus_one``; img_idx int32 [B]; cat_ids = sorted int32 GT category ids;
    label_map int32 [L] label -> category id).  Rows never counted are marked empty: those of images outside the GT file when
    ``need_img``, those of categories outside it when ``need_cat`` (default: not ``need_img``).  ``bad_img`` (int32 [1]) counts
    detections on images outside the GT file."""
    _need_cuda(packed, img_idx, ratios, cat_ids, label_map, bad, bad_img)
    G, B, M1, six = packed.shape
    if six != 6 or packed.dtype != torch.float32 or not packed.is_contiguous():
        raise _lib.MqdetError("lvis_collect: contiguous fp32 [G, B, max_out + 1, 6] required")
    if base + G * B * (M1 - 1) > pool.cap:
        raise _lib.MqdetError("lvis_collect: pool full")
    need_cat = not need_img if need_cat is None else need_cat
    drop = int(bool(need_cat)) | (int(bool(need_img)) << 1)
    _launch("mqdet_lvis_collect", _ptr(packed), G, B, M1 - 1, _ptr(img_idx), _ptr(ratios), _ptr(label_map),
            0 if label_map is None else label_map.numel(), _ptr(cat_ids), cat_ids.numel(), drop,
            int(bool(wh_plus_one)), *[_ptr(t) for t in pool.fields()], int(base), int(seq_base), _ptr(bad),
            _ptr(bad_img), what="lvis_collect")


CUT_BY_CATEGORY, CUT_BY_IMAGE, CUT_BY_PAIR = 0, 1, 2   # the ``group`` argument of mqdet_lvis_cut


def lvis_cut(src, n, dst, *, n_groups, k, by_image=False, group=None, n_cat=0):
    """The first k rows per group, by score descending then arrival, from src[:n] to dst.  ``group``: CUT_BY_CATEGORY,
    CUT_BY_IMAGE or CUT_BY_PAIR ((image, category) pairs: n_groups = images * n_cat); without it, ``by_image`` picks between
    the first two (the LVIS protocols).  -> int32 [1] device count of rows written."""
    if group is None:
        group = CUT_BY_IMAGE if by_image else CUT_BY_CATEGORY
    if group not in (CUT_BY_CATEGORY, CUT_BY_IMAGE, CUT_BY_PAIR):
        raise _lib.MqdetError(f"lvis_cut: unknown grouping {group!r}")
    count = torch.zeros((1,), dtype=torch.int32, device=src.score.device)
    ws = torch.empty((load().mqdet_lvis_cut_workspace_bytes(n, n_groups),), dtype=torch.uint8, device=src.score.device)
    _launch("mqdet_lvis_cut", *[_ptr(t) for t in src.fields()], int(n), group, int(n_groups), int(n_cat), int(k),
            *[_ptr(t) for t in dst.fields()], _ptr(count), _ptr(ws), what="lvis_cut")
    return count


def lvis_evaluate(pool, n, gt, *, want_match=False):
    """Pairing, greedy matching and accumulation of pool[:n] against a ground truth's device tables ``gt.dev``: the federated
    filter when they hold ``pos_pairs``, crowd GTs when they hold ``gt_crowd``, a maxDets axis when they hold ``max_dets``; the
    0 < area < inf filter on detections when ``gt.det_area_filter``.  -> dict(precision fp64 [10, 101, K, 4] (LVIS) or [10, 101, K, 4, M], recall fp64 [10, K, 4] or [10, K, 4, M],
    n_paired int32 [1], order int32 [n], tp_bits / ig_bits int64 [n], match_gt int32 [n, 40] when want_match)."""
    dev = pool.score.device
    K = len(gt.cat_ids)
    t = gt.dev
    max_dets = t.get("max_dets")
    M = 1 if max_dets is None else max_dets.numel()
    tail = () if max_dets is None else (M,)
    federated = "pos_pairs" in t
    out = {"precision": torch.full((10, 101, K, 4) + tail, -1.0, dtype=torch.float64, device=dev),
           "recall": torch.full((10, K, 4) + tail, -1.0, dtype=torch.float64, device=dev),
           "n_paired": torch.zeros((1,), dtype=torch.int32, device=dev),
           "order": torch.empty((max(n, 1),), dtype=torch.int32, device=dev),
           "tp_bits": torch.empty((max(n, 1),), dtype=torch.int64, device=dev),
           "ig_bits": torch.empty((max(n, 1),), dtype=torch.int64, device=dev),
           "match_gt": torch.zeros((max(n, 1), 40), dtype=torch.int32, device=dev) if want_match else None}

    def table(name):
        x = t.get(name)
        return (None, 0) if x is None else (_ptr(x), x.numel())

    ws = torch.empty((load().mqdet_lvis_evaluate_workspace_bytes(n, t["gt_pair"].numel()),), dtype=torch.uint8, device=dev)
    _launch("mqdet_lvis_evaluate", *[_ptr(x) for x in pool.fields()], int(n), K, int(federated), *table("pos_pairs"),
            *table("neg_pairs"), *table("nel_pairs"), int(gt.det_area_filter), _ptr(t["gt_pair"]), _ptr(t["gt_box"]),
            _ptr(t["gt_area"]), _ptr(t["gt_ignore"]), _ptr(t.get("gt_crowd")), _ptr(t["gt_id"]),
            t["gt_pair"].numel(), _ptr(t["num_gt"]), _ptr(t["iou_thrs"]), _ptr(t["rec_thrs"]),
            _ptr(t["area_rng"]), _ptr(max_dets), M, _ptr(out["precision"]), _ptr(out["recall"]),
            _ptr(out["n_paired"]), _ptr(out["order"]), _ptr(out["tp_bits"]), _ptr(out["ig_bits"]),
            _ptr(out["match_gt"]), _ptr(ws), what="lvis_evaluate")
    return out
