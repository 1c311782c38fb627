"""The text -> image half of the BiAttention fusion restated in float64, its per-element error bound, and seeded inputs that
each expose one class of mistake in ``ops.biattn_text_vn`` (biattn_text_kernel):

    u[b,h,t,:] = sum_n softmax_n(clamp(k[b,h,t] . q[b,h,n] + rowbias[b,h,t])) * vn[b,n,:]

The kernel shifts the exponent by colmax[b*H+h, t] (the max over n of the clamped scores, from biattn_image), so that
e = exp(a - colmax) <= 1, rounds e to fp16 for the P . vn product, sums e in fp32 and divides at the end.  Its roundings
give the bound below.  tests/test_biattn_text_cpu.py checks this file without a GPU; tests/test_biattn_text_gpu.py uses it.
"""
import math

import torch

EPS16 = 2.0 ** -11          # unit roundoff of fp16
F16_SUBNORMAL_HALF = 2.0 ** -25   # half the spacing of fp16 subnormals: the absolute rounding error of a P below 2^-14
CLAMP = 5.0e4               # the +-5e4 score clamp of fuse_helper.py (CLAMP_MIN_FOR_UNDERFLOW / CLAMP_MAX_FOR_OVERFLOW)
TAIL_EVERY = 3              # tail-dominant pattern: text tokens t with t % TAIL_EVERY == 0 have only negative real scores
PATTERNS = ("diffuse", "spread", "tail", "clamp", "clamp0", "peaked")


def _clamp(a, clamp):
    return a.clamp(-clamp, clamp) if clamp > 0 else a


def scores(kh, qh, rowbias, clamp, b, h):
    """clamp(k . q^T + rowbias) of one (image, head) in float64, [T, N]; clamp = 0 means no clamp."""
    a = kh[b, h].double() @ qh[b, h].double().t()
    if rowbias is not None:
        a = a + rowbias[b, h, :, 0].double()[:, None]
    return _clamp(a, clamp)


def colmax_of(kh, qh, rowbias, clamp):
    """[B*H, T] fp32: the max over the image tokens of the clamped scores, as biattn_image hands it to the text side."""
    B, H, T, _ = kh.shape
    out = torch.empty(B * H, T, dtype=torch.float32, device=kh.device)
    for b in range(B):
        for h in range(H):
            out[b * H + h] = scores(kh, qh, rowbias, clamp, b, h).max(1).values.float()
    return out


def restate_text(kh, qh, vn16, colmax, rowbias, clamp):
    """u [B, H, T, 256] float64 from the same fp16 / fp32 operands, with the per-element bound of the kernel's error and the
    column sums sum_n e_n (e = exp(a - colmax)) the bound divides by:

        bound = 2^-11 |u|                                  fp16 output
              + 2^-10 sum_n p_n |vn[n, c]|                 P rounded to fp16 (2^-11), ex2.approx and the fp32 sums
              + N 2^-25 max_n |vn[n, c]| / sum_n e_n       fp16 subnormal rounding of the unnormalised P

    There is no absolute floor: without a channel offset |u| is a mean of ~N unit rows and far below any fixed floor."""
    B, H, T, _ = kh.shape
    N = vn16.shape[1]
    dev = kh.device
    u = torch.empty(B, H, T, 256, dtype=torch.float64, device=dev)
    bound = torch.empty_like(u)
    colsum = torch.empty(B, H, T, dtype=torch.float64, device=dev)
    for b in range(B):
        vn = vn16[b].double()
        avn = vn.abs()
        vmax = avn.max(0).values
        for h in range(H):
            e = torch.exp(scores(kh, qh, rowbias, clamp, b, h) - colmax[b * H + h].double()[:, None])
            s = e.sum(1, keepdim=True)
            p = e / s
            u[b, h] = p @ vn
            bound[b, h] = EPS16 * u[b, h].abs() + 2 * EPS16 * (p @ avn) + N * F16_SUBNORMAL_HALF * vmax[None, :] / s
            colsum[b, h] = s[:, 0]
    return u, bound, colsum


def make_inputs(pattern, B, H, T, N, seed, q="broadcast", rb_ld=8, device="cpu"):
    """Seeded operands of ops.biattn_text_vn -> dict(kh, qh, vn16, rowbias, clamp).  kh [B,H,T,256] fp16; qh [B,H,N,256] fp16,
    either vn16 broadcast over the heads (head stride 0, as the module passes it) or distinct per head (q="distinct");
    rowbias [B,H,T,rb_ld] fp32 (column 0 is the bias; the other columns hold values that overflow any exponent if read) or
    None (rb_ld=None).  Patterns:
      diffuse:  vn = per-(image, channel) mean in [-2, 2] + N(0, 1), so |u| = O(1); k rows std 1/16 (scores std ~1, like
                the model); rowbias N(0, 1).
      spread:   k rows scaled log-uniformly over [1e-2, 30] per (b, h, t); rowbias = +-U(150, 200) with the sign flipping
                between rows t and t + 8 (the two rows one thread holds) and between neighbouring images and heads, so
                their colmax values lie more than 100 apart: a shift taken from the wrong row or (b, h), or a dropped
                rowbias, overflows or underflows the exponent.
      tail:     every TAIL_EVERY-th text token has only negative real scores and rowbias 0, so a zero-filled image token
                beyond N (score = rowbias = 0) would dominate its softmax.
      clamp:    integer operands, vn / q / k in [-100, 100], rowbias in +-2000: scores are exact fp32 sums, over 20 % of them
                beyond the +-5e4 clamp, many tied at it; clamp(S + rowbias) and clamp(S) + rowbias differ by e^2000.
      clamp0:   the same operands without the clamp.
      peaked:   one image token per (b, h, t) scores 17-18 above the others' mean, so their unnormalised P falls into the
                fp16 subnormal range."""
    assert pattern in PATTERNS, pattern
    g = torch.Generator().manual_seed(seed)
    ints = pattern in ("clamp", "clamp0")

    def rnd(*shape):
        return torch.randn(*shape, generator=g, dtype=torch.float64)

    def tokens(*lead):  # [*lead, N, 256]
        if ints:
            return torch.randint(-100, 101, (*lead, N, 256), generator=g).double()
        if pattern == "peaked":
            return rnd(*lead, N, 256)
        return (4 * torch.rand(*lead, 1, 256, generator=g, dtype=torch.float64) - 2) + rnd(*lead, N, 256)

    vn = tokens(B).half()
    qd = tokens(B, H).half() if q == "distinct" else None
    qsrc = qd if qd is not None else vn[:, None]   # [B, H or 1, N, 256]: the q operand as the kernel sees it
    rb = rnd(B, H, T, 1)
    if ints:
        k = torch.randint(-100, 101, (B, H, T, 256), generator=g).double()
        rb = torch.randint(-2000, 2001, (B, H, T, 1), generator=g).double()
    elif pattern == "spread":
        scale = torch.empty(B, H, T, 1, dtype=torch.float64).uniform_(math.log(1e-2), math.log(30.0), generator=g).exp()
        k = rnd(B, H, T, 256) / 16 * scale
        t = torch.arange(T).view(1, 1, T, 1)
        sign = 1 - 2 * ((t // 8 + torch.arange(B).view(B, 1, 1, 1) + torch.arange(H).view(1, H, 1, 1)) % 2)
        rb = sign * torch.empty(B, H, T, 1, dtype=torch.float64).uniform_(150, 200, generator=g)
    elif pattern == "tail":
        k = rnd(B, H, T, 256) / 16
        m = qsrc.double().mean(2, keepdim=True)                               # channel means of q, [B, H or 1, 1, 256]
        alpha = torch.empty(B, H, T, 1, dtype=torch.float64).uniform_(6, 10, generator=g)
        tail = (torch.arange(T) % TAIL_EVERY == 0).view(1, 1, T, 1)
        k = torch.where(tail, -alpha * m / (m * m).sum(-1, keepdim=True), k)  # k . q_n = -alpha (1 + O(1/|m|)) < 0
        rb = torch.where(tail, torch.zeros_like(rb), rb)
    elif pattern == "peaked":
        k = rnd(B, H, T, 256) / 32
        n_pk = torch.randint(0, N, (B, H, T), generator=g)
        hi = torch.arange(H).view(1, H, 1) if qd is not None else torch.zeros(1, H, 1, dtype=torch.long)
        qp = qsrc[torch.arange(B).view(B, 1, 1), hi, n_pk].double()          # q of each token's peak image token
        gap = torch.empty(B, H, T, 1, dtype=torch.float64).uniform_(17, 18, generator=g)
        k = k + (gap - (k * qp).sum(-1, keepdim=True)) * qp / (qp * qp).sum(-1, keepdim=True)
    else:
        k = rnd(B, H, T, 256) / 16
    kh = k.half()
    rowbias = None
    if rb_ld is not None:
        rowbias = torch.cat([rb, 1e4 * rnd(B, H, T, rb_ld - 1)], -1).float() if rb_ld > 1 else rb.float().contiguous()
    vn16 = vn.to(device)
    qh = qd.to(device) if qd is not None else vn16.view(B, 1, N, 256).expand(B, H, N, 256)
    # every pattern but clamp0 runs with the module's clamp; only the clamp pattern's scores reach it
    return dict(kh=kh.to(device), qh=qh, vn16=vn16, rowbias=rowbias.to(device) if rowbias is not None else None,
                clamp=0.0 if pattern == "clamp0" else CLAMP)


# ---- the fusion layer's attention from its layer-normed inputs (BiMultiHeadAttention without residual or layer scale) -------
def _proj(w, name, x):
    return x @ w[name + ".weight"].t() + w[name + ".bias"]


def attention_restate(vn, ln, w, heads, clamp, mask=None):
    """dv [B,N,Cv], dl [B,T,Cl] in float64 from the layer-normed tokens vn [B,N,Cv] and ln [B,T,Cl], the unfolded reference
    formula (fuse_helper.py:218-303): q = (vn Wq^T + bq) d^-1/2, k = ln Wl^T + bl, A_h = clamp(q_h k_h^T);
    dl = (softmax_n(A_h^T) (vn Wvv^T + bvv)_h) Wol^T + bol,  dv = (softmax_t(A_h + mask) (ln Wvl^T + bvl)_h) Wov^T + bov.
    ``w``: the module's parameters by name (v_proj.weight, ...), ``mask`` [B,T] 1 keep / 0 padding or None."""
    B, N, _ = vn.shape
    T = ln.shape[1]
    E = w["v_proj.weight"].shape[0]
    d = E // heads
    q = (_proj(w, "v_proj", vn) * d ** -0.5).view(B, N, heads, d)
    k = _proj(w, "l_proj", ln).view(B, T, heads, d)
    vv = _proj(w, "values_v_proj", vn).view(B, N, heads, d)
    vl = _proj(w, "values_l_proj", ln).view(B, T, heads, d)
    ov = vn.new_empty(B, N, heads, d)
    ol = vn.new_empty(B, T, heads, d)
    for b in range(B):
        for h in range(heads):
            A = _clamp(q[b, :, h] @ k[b, :, h].t(), clamp)   # [N, T]
            ol[b, :, h] = torch.softmax(A.t(), dim=1) @ vv[b, :, h]
            if mask is not None:
                A = A.masked_fill(mask[b][None, :] == 0, float("-inf"))
            ov[b, :, h] = torch.softmax(A, dim=1) @ vl[b, :, h]
    return _proj(w, "out_v_proj", ov.reshape(B, N, E)), _proj(w, "out_l_proj", ol.reshape(B, T, E))


def text_folded(vn, ln, w, heads, clamp):
    """dl as the product path computes it, in float64: the query projection folded into the keys (gT_h = k_h d^-1/2 Wq_h,
    gbias_h = d^-1/2 bq_h . k_h), u = softmax_n(clamp(vn gT_h^T + gbias_h)) vn on the image tokens themselves, and the value
    projection applied after the token reduction (sum_n p_n = 1): ol_h = u Wvv_h^T + bvv_h."""
    B, N, Cv = vn.shape
    T = ln.shape[1]
    E = w["v_proj.weight"].shape[0]
    d = E // heads
    s = d ** -0.5
    k = _proj(w, "l_proj", ln).view(B, T, heads, d)
    wq, bq = w["v_proj.weight"].view(heads, d, Cv), w["v_proj.bias"].view(heads, d)
    wv, bv = w["values_v_proj.weight"].view(heads, d, Cv), w["values_v_proj.bias"].view(heads, d)
    ol = vn.new_empty(B, T, heads, d)
    for b in range(B):
        for h in range(heads):
            gT = k[b, :, h] @ (s * wq[h])                      # [T, Cv]
            gb = k[b, :, h] @ (s * bq[h])                      # [T]
            a = _clamp(gT @ vn[b].t() + gb[:, None], clamp)    # [T, N]
            e = torch.exp(a - a.max(1, keepdim=True).values)
            u = (e @ vn[b]) / e.sum(1, keepdim=True)
            ol[b, :, h] = u @ wv[h].t() + bv[h]
    return _proj(w, "out_l_proj", ol.reshape(B, T, E))
