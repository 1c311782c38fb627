"""DyConv's stages after the three DCNv2 convolutions restated in float64 (GroupNorm -> scale attention -> mean over the
branches -> DyReLU), the pyramids the DyHead kernels are checked at, and seeded branch features with per-image statistics.

Layout as in mqdet_b200/ops.py: a branch output is [B, rows, C] with every level's (h, w) pixels concatenated row-major;
branch 1 covers levels 0..L-1, branches 2 and 0 cover levels 1..L-1 (branch 0 at the coarser level's size, upsampled to
level l - 1 after the norm).  tests/test_dyconv_kernels_cpu.py pins this restatement to ``oracle.restate.dyconv``.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import restate  # noqa: E402

C, G, EPS = 256, 16, 1e-5

PYRAMIDS = {
    "bench": [(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)],   # 800x1344 padded MQ-GLIP-T input
    "portrait": [(168, 100), (84, 50), (42, 25), (21, 13), (11, 7)],
    "small": [(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)],            # the composed DyConv test's pyramid
    "tiny": [(9, 13), (5, 7), (3, 4), (2, 2), (1, 1)],                # every level < 128 pixels, a 1x1 level
    "rows": [(2, 9), (1, 5), (1, 3)],                                 # single-row levels: source row scale 0
    "cols": [(9, 2), (5, 1), (3, 1)],                                 # single-column levels: source column scale 0
    "single": [(9, 11)],                                              # one level: no cross-level branches
}
# (pyramid, batch): B = 8 on the portrait shape is the graph engines' largest batch (B * L = 40 segments)
CASES = [("bench", 1), ("bench", 2), ("portrait", 8), ("small", 3), ("tiny", 2), ("rows", 2), ("cols", 2), ("single", 2)]


def case_id(case):
    return f"{case[0]}-B{case[1]}"


def seg_offsets(sizes):
    off = [0]
    for h, w in sizes:
        off.append(off[-1] + h * w)
    return off


def features(sizes, B, seed, pattern="pad", integer=False):
    """fp16 [B, rows, C] branch output over the levels ``sizes`` with a distinct mean and scale per (image, channel group)
    and a distinct per-channel offset per (image, level), so a wrong image or segment index changes every statistic.
      pattern "pad":    the right / bottom ~40% of every level of image 0 is a per-channel constant (what a convolution
                        returns over the zero padding of a mixed-size batch);
      pattern "offset": |mean| / std = 16 within each group (cancellation in E[x^2] - mu^2).
    integer: values rounded to integers in [-8, 8], for which every fp32 partial sum of chan_stats is exact."""
    g = torch.Generator().manual_seed(seed)
    cpg = C // G
    scale = (0.5 + 1.5 * torch.rand(B, G, generator=g)).repeat_interleave(cpg, 1)
    if pattern == "offset":
        sign = torch.where(torch.rand(B, G, generator=g) < 0.5, -1.0, 1.0).repeat_interleave(cpg, 1)
        # the channel offsets below make the within-group spread ~sqrt(2) * scale
        mean = 16.0 * 2.0 ** 0.5 * scale * sign
    else:
        mean = (2.0 * torch.randn(B, G, generator=g)).repeat_interleave(cpg, 1)
    const = torch.randn(C, generator=g) * 2.0
    out = []
    for h, w in sizes:
        dev = torch.randn(B, C, generator=g) * scale
        x = (mean + dev)[:, None, :] + scale[:, None, :] * torch.randn(B, h * w, C, generator=g)
        if pattern == "pad":
            hh = torch.arange(h).view(-1, 1).expand(h, w).reshape(-1)
            ww = torch.arange(w).view(1, -1).expand(h, w).reshape(-1)
            pad = (hh >= -(-3 * h // 5)) | (ww >= -(-3 * w // 5))
            x[0, pad] = const
        out.append(x)
    y = torch.cat(out, 1)
    if integer:
        y = y.round().clamp(-8, 8)
    return y.half()


def branch_outputs(sizes, B, pattern="pad", integer=False):
    """(y1 [B, N, C], y2 [B, N1, C], y0 [B, N1, C]) fp16 stand-ins for the three convolution outputs; y2 = y0 = None on
    a single level."""
    y1 = features(sizes, B, 101, pattern, integer)
    if len(sizes) == 1:
        return y1, None, None
    return y1, features(sizes[1:], B, 102, pattern, integer), features(sizes[1:], B, 100, pattern, integer)


def dyconv_params(seed=11):
    """GroupNorm / attention / DyReLU parameters of one DyConv (fp32, CPU).  The attention weights are large enough that
    w.GAP + b spans ReLU's zero, the linear part of h_sigmoid and its saturation across segments; the DyReLU weights
    (synth.dyconv_sd's scales) zero some hidden units and saturate some coefficients."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for k in range(3):
        p[f"DyConv.{k}.bn.weight"] = 1.0 + 0.3 * torch.randn(C, generator=g)
        p[f"DyConv.{k}.bn.bias"] = 0.3 * torch.randn(C, generator=g)
    p["AttnConv.1.weight"] = 0.3 * torch.randn(1, C, 1, 1, generator=g)
    p["AttnConv.1.bias"] = 0.5 * torch.randn(1, generator=g)
    p["relu.fc.0.weight"] = 0.2 * torch.randn(C // 4, C, generator=g)
    p["relu.fc.0.bias"] = 0.1 * torch.randn(C // 4, generator=g)
    p["relu.fc.2.weight"] = 0.3 * torch.randn(4 * C, C // 4, generator=g)
    p["relu.fc.2.bias"] = 0.3 * torch.randn(4 * C, generator=g)
    return p


def levels_of(y, sizes):
    """[B, rows, C] -> [B, C, h, w] per level, float64."""
    B = y.shape[0]
    off = seg_offsets(sizes)
    return [y[:, off[i]:off[i + 1]].double().transpose(1, 2).reshape(B, C, h, w) for i, (h, w) in enumerate(sizes)]


def flat(levels):
    return torch.cat([t.flatten(2).transpose(1, 2) for t in levels], 1)


def upsample(t, size):
    return F.interpolate(t, size=tuple(size), mode="bilinear", align_corners=True)


def interp_matrix(n_in, n_out):
    """[n_out, n_in] float64 align_corners=True linear interpolation taken at ATen's fp32 source positions: for fp32 maps
    ATen (and dyconv_combine_kernel) computes scale = (n_in - 1) / (n_out - 1) and scale * i in fp32, where a float64 map
    gets float64 positions; at 100 x 168 the two differ by up to ~1e-5 of a pixel, more than an fp16 ulp of a value near 0."""
    scale = torch.tensor(float(n_in - 1) if n_out > 1 else 0.0, dtype=torch.float32) / float(max(n_out - 1, 1))
    src = scale * torch.arange(n_out, dtype=torch.float32)
    i0 = src.long()
    i1 = i0 + (i0 < n_in - 1).long()
    lam = (src - i0.float()).double()
    m = torch.zeros(n_out, n_in, dtype=torch.float64)
    o = torch.arange(n_out)
    m.index_put_((o, i0), 1.0 - lam, accumulate=True)
    m.index_put_((o, i1), lam, accumulate=True)
    return m


def upsample_fp32_index(t, size):
    """F.interpolate(t, size, bilinear, align_corners=True) of a float64 map at the source positions of an fp32 one."""
    return torch.einsum("oh,bchw,pw->bcop", interp_matrix(t.shape[2], size[0]), t, interp_matrix(t.shape[3], size[1]))


def gn_affine(y, sizes, gn_w, gn_b):
    """GroupNorm of each level segment as a per-channel affine: GN(y)[c] = ga[c] * y + gb[c] -> [B, nseg, 2, C] float64."""
    gn_w, gn_b = gn_w.double(), gn_b.double()
    out = []
    for t in levels_of(y, sizes):
        B = t.shape[0]
        grp = t.reshape(B, G, -1)
        mu = grp.mean(2)
        rstd = (grp.var(2, unbiased=False) + EPS).rsqrt()
        ga = rstd.repeat_interleave(C // G, 1) * gn_w
        gb = gn_b - (mu * rstd).repeat_interleave(C // G, 1) * gn_w
        out.append(torch.stack([ga, gb], 1))
    return torch.stack(out, 1)


def apply_affine(t, aff):
    """t [B, C, h, w], aff [B, 2, C] -> ga * t + gb."""
    return t * aff[:, 0, :, None, None].double() + aff[:, 1, :, None, None].double()


def attention(y, sizes, aff, attn_w, attn_b, up_to=None):
    """h_sigmoid(relu(w . GAP(GN(y)) + b)) per segment -> [B, nseg] float64; ``up_to``: the sizes each normalised segment
    is bilinearly upsampled to (align_corners=True) before the pool (DyConv's branch 0)."""
    gaps = []
    for i, t in enumerate(levels_of(y, sizes)):
        n = apply_affine(t, aff[:, i])
        if up_to is not None:
            n = upsample(n, up_to[i])
        gaps.append(n.mean((2, 3)))
    z = torch.stack(gaps, 1) @ attn_w.double().view(-1) + attn_b.double().view(())
    return F.relu6(F.relu(z) + 3.0) / 6.0


def combine(y1, y2, y0, aff1, aff2, aff0, at1, at2, at0, sizes):
    """Mean over the branches of attn_k * GN_k(y_k), branch 0 upsampled (at fp32 source positions, like the fp32 model)
    -> (mid [B, N, C], the same mean of
    |attn_k| * (|ga_k * y_k| + |gb_k|): the scale of the fp32 rounding errors of a kernel computing mid), float64."""
    L = len(sizes)
    s1 = levels_of(y1, sizes)
    s2 = levels_of(y2, sizes[1:]) if L > 1 else []
    s0 = levels_of(y0, sizes[1:]) if L > 1 else []

    def term(at, t, aff, size=None):
        a = at[:, None, None, None].double()
        v, m = apply_affine(t, aff), t.abs() * aff[:, 0, :, None, None].double().abs()
        if size is not None:
            v, m = upsample_fp32_index(v, size), upsample_fp32_index(m, size)
        return a * v, a.abs() * (m + aff[:, 1, :, None, None].double().abs())

    mids, mags = [], []
    for l in range(L):
        terms = [term(at1[:, l], s1[l], aff1[:, l])]
        if l > 0:
            terms.append(term(at2[:, l - 1], s2[l - 1], aff2[:, l - 1]))
        if l < L - 1:
            terms.append(term(at0[:, l], s0[l], aff0[:, l], sizes[l]))
        mids.append(torch.stack([v for v, _ in terms]).mean(0))
        mags.append(torch.stack([m for _, m in terms]).mean(0))
    return flat(mids), flat(mags)


def dyrelu(mid, sizes, p):
    """DYReLU per level (``oracle.restate.dyrelu``) on mid [B, N, C] -> [B, N, C] float64."""
    sd = {k: v.double() for k, v in p.items() if k.startswith("relu.")}
    return flat([restate.dyrelu(t, sd, "relu.") for t in levels_of(mid, sizes)])


def dyrelu_hidden(mid, sizes, p):
    """(hidden units after the ReLU [B, L, C/4], h_sigmoid outputs [B, L, 4C]) of DYReLU, float64."""
    gap = torch.stack([t.mean((2, 3)) for t in levels_of(mid, sizes)], 1)
    hid = F.relu(F.linear(gap, p["relu.fc.0.weight"].double(), p["relu.fc.0.bias"].double()))
    return hid, F.relu6(F.linear(hid, p["relu.fc.2.weight"].double(), p["relu.fc.2.bias"].double()) + 3.0) / 6.0


def post_dcn(y1, y2, y0, sizes, p):
    """Everything DyConv does after its three convolutions, from their outputs y1 [B, N, C], y2 / y0 [B, N1, C]."""
    L = len(sizes)
    aw, ab = p["AttnConv.1.weight"], p["AttnConv.1.bias"]

    def branch(k, y, segs, up_to=None):
        aff = gn_affine(y, segs, p[f"DyConv.{k}.bn.weight"], p[f"DyConv.{k}.bn.bias"])
        return aff, attention(y, segs, aff, aw, ab, up_to)

    aff1, at1 = branch(1, y1, sizes)
    aff2 = at2 = aff0 = at0 = None
    if L > 1:
        aff2, at2 = branch(2, y2, sizes[1:])
        aff0, at0 = branch(0, y0, sizes[1:], sizes[:-1])
    mid, _ = combine(y1, y2, y0, aff1, aff2, aff0, at1, at2, at0, sizes)
    return dyrelu(mid, sizes, p)


def gap_weights(sizes):
    """The GAP weights of DyConv's branch 0 obtained directly: each unit vector on level l + 1 pushed through the float64
    align_corners upsample to level l and averaged -> [N1] (level 1..L-1 order), float64."""
    out = []
    for (H, W), (Hs, Ws) in zip(sizes[:-1], sizes[1:]):
        n = Hs * Ws
        w = torch.empty(n, dtype=torch.float64)
        for q0 in range(0, n, 256):   # a few unit vectors at a time: level 0 -> 1 of the portrait pyramid is 4,200 x 16,800
            q1 = min(n, q0 + 256)
            e = torch.zeros(q1 - q0, Hs * Ws, dtype=torch.float64)
            e[torch.arange(q1 - q0), torch.arange(q0, q1)] = 1.0
            w[q0:q1] = upsample(e.view(-1, 1, Hs, Ws), (H, W)).mean((1, 2, 3))
        out.append(w)
    return torch.cat(out)


def fp16_ulp(v):
    """Spacing of fp16 at |v| (float64 in, float64 out): 2^(e - 11) for |v| in [2^(e-1), 2^e), 2^-24 below 2^-14."""
    _, e = torch.frexp(v.abs().to(torch.float64))
    return torch.where(v.abs() < 2.0 ** -14, torch.full_like(v, 2.0 ** -24, dtype=torch.float64),
                       torch.ldexp(torch.ones_like(v, dtype=torch.float64), (e - 11)))
