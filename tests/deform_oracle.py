"""The two bilinear-gather kernels restated in float64: DyConv's DCNv2 convolutions (``ops.dcn_conv`` / ``ops.dcn_cols``,
dcn_conv_kernel / dcn_cols_kernel) and the multi-scale deformable attention core (``ops.ms_deform_attn``, ms_deform_attn_kernel
/ ms_deform_attn_v2_kernel), with per-element error bounds for realistic inputs and generators of exact inputs.

Exact inputs.  Both kernels are sums of four-corner bilinear blends.  On dyadic inputs small enough that every intermediate is
representable, each rounding the kernel does is exact, so its output must equal the float64 reference rounded once to the
output type, bit for bit.  The generators below say in their docstrings why their values have that property.

Realistic inputs are held to a per-element bound built from the kernel's own roundings, with no global-max scaling and no
absolute floor.  tests/test_deform_cpu.py checks this file without a GPU; tests/test_dcn_kernels_gpu.py and
tests/test_msda_gpu.py use it.

Edge rules of the bilinear sample (deform_conv_kernel_cuda.cu dmcn_im2col_bilinear, restated by both DCN kernels): a sample at
(h, w) is zero unless -1 < h < H and -1 < w < W; inside, a corner contributes only if it lies in the map.  The lower rule is
unobservable: at exactly h = -1 the only corner it would admit is row 0 with weight h - floor(h) = 0.  The upper one is not:
at exactly h = H a "<=" would give the clamped row H - 1 the weight 1.  So the exact cases target both, but only the upper
rule's strictness can move an output.
"""
import torch
import torch.nn.functional as F

EPS16 = 2.0 ** -11       # unit roundoff of fp16
TAPS = 9

# ----------------------------------------------------------------------------------------------------------------------
# DCNv2 (DyConv's three 3x3 modulated deformable convolutions, vldyhead.py DyConv.forward; dcnconv.cu)
# ----------------------------------------------------------------------------------------------------------------------
# mutations a kernel rewrite could make, emulated in the reference (tests/test_deform_cpu.py checks each one is caught)
DCN_MUTATIONS = ("lower_ge", "no_lower", "upper_le", "swap23", "no_mask", "quirk_out_strides", "stride2_base")


def level_offsets(sizes):
    off = [0]
    for h, w in sizes:
        off.append(off[-1] + h * w)
    return off


def branch_levels(sizes, branch):
    """[(lo, li, Ho, Wo, stride)] in dcn_conv's row order within one image: the level whose offset / mask record is read (lo),
    the input level sampled (li), the output grid and the stride.  Branch 1 is every level at stride 1; branch 2 samples level
    l-1 at stride 2 onto level l's grid; branch 0 samples level l at stride 1 with the record of the finer level l-1, re-read
    through level l's strides (the reference computes DyConv[0] of level l-1 at level l's size before upsampling it)."""
    L = len(sizes)
    if branch == 1:
        return [(l, l, *sizes[l], 1) for l in range(L)]
    if branch == 2:
        return [(l, l - 1, *sizes[l], 2) for l in range(1, L)]
    return [(l - 1, l, *sizes[l], 1) for l in range(1, L)]


def rows_per_image(sizes, branch):
    return sum(h * w for _, _, h, w, _ in branch_levels(sizes, branch))


def om_records(om_b):
    """[N, >= 27] offset / mask-logit records of one image -> float64 [N, 27] with the mask channels as fp32 values, as the
    kernel uses them: the sigmoid of the fp32 logit rounded to fp32 (logits of +-200 / 0 give exactly 1, 0 and 1/2).  It is
    evaluated in float64 and rounded once, so that it does not depend on the layout the way torch's vectorised fp32 sigmoid
    does; the kernel's 1 / (1 + expf(-z)) is within a few fp32 ulps of it."""
    rec = om_b[:, :27].double().clone()
    rec[:, 18:] = torch.sigmoid(om_b[:, 18:27].float().double()).float().double()
    return rec


def _read(rec_lo, HWl, P, c0, nch, pix, quirk):
    """[nch, P] values of channels c0 .. c0+nch-1 for output pixels pix.  The reference holds each level's record as an
    NCHW-flat buffer [channels][HWl] and indexes it with the OUTPUT grid's strides (deform_conv_kernel_cuda.cu:605-618):
    flat index c * P + pix, which is channel c0 + f / HWl at pixel f % HWl of the level it was produced at."""
    c = torch.arange(nch, device=pix.device)[:, None]
    if quirk:
        f = c * P + pix[None]
        return rec_lo[f % HWl, c0 + f // HWl]
    return rec_lo[pix[None].expand(nch, P), c0 + c]


def sample_level(x_in, Hi, Wi, rec_lo, HWl, Ho, Wo, stride, mut=()):
    """Column block [Ho*Wo, 9*C] (k = tap*C + c) of one output grid in float64, and the sample coordinates (h, w), each [9, P].
    x_in [Hi*Wi, C] float64 is the input level; rec_lo [HWl, 27] the records of level lo (None: no offsets, mask 1)."""
    P = Ho * Wo
    dev = x_in.device
    C = x_in.shape[1]
    pix = torch.arange(P, device=dev)
    ho, wo = pix // Wo, pix % Wo
    quirk = "quirk_out_strides" not in mut
    if rec_lo is not None:
        offs = _read(rec_lo, HWl, P, 0, 18, pix, quirk)
        mask = _read(rec_lo, HWl, P, 18, 9, pix, quirk)
    pad = 0 if (stride == 2 and "stride2_base" in mut) else 1
    cols = x_in.new_empty(P, TAPS, C)
    hs, ws = [], []
    for t in range(TAPS):
        h = (ho * stride - pad + t // 3).double()
        w = (wo * stride - pad + t % 3).double()
        m = 1.0
        if rec_lo is not None:
            h = h + offs[2 * t]
            w = w + offs[2 * t + 1]
            m = mask[t]
        hs.append(h)
        ws.append(w)
        if "no_lower" in mut:
            valid = torch.ones_like(h, dtype=torch.bool)
        elif "lower_ge" in mut:
            valid = (h >= -1) & (w >= -1)
        else:
            valid = (h > -1) & (w > -1)
        valid &= (h <= Hi) & (w <= Wi) if "upper_le" in mut else (h < Hi) & (w < Wi)
        hl, wl = torch.floor(h), torch.floor(w)
        lh, lw = h - hl, w - wl
        hh, hw = 1 - lh, 1 - lw
        hl, wl = hl.long(), wl.long()
        hu, wu = hl + 1, wl + 1

        def corner(hc, wc, ok):
            v = x_in[hc.clamp(0, Hi - 1) * Wi + wc.clamp(0, Wi - 1)]
            return v * (ok & valid).double()[:, None]

        c1 = corner(hl, wl, (hl >= 0) & (wl >= 0))
        c2 = corner(hl, wu, (hl >= 0) & (wu <= Wi - 1))
        c3 = corner(hu, wl, (hu <= Hi - 1) & (wl >= 0))
        c4 = corner(hu, wu, (hu <= Hi - 1) & (wu <= Wi - 1))
        if "swap23" in mut:
            c2, c3 = c3, c2
        val = (hh * hw)[:, None] * c1 + (hh * lw)[:, None] * c2 + (lh * hw)[:, None] * c3 + (lh * lw)[:, None] * c4
        if "no_mask" not in mut:
            val = val * (m[:, None] if torch.is_tensor(m) else m)
        cols[:, t] = val
    return cols.reshape(P, TAPS * C), torch.stack(hs), torch.stack(ws)


def dcn_image(x16, om, sizes, branch, b, mut=(), coords=False):
    """Column matrix [rows_per_image, 9*C] float64 of image b for DyConv[branch], in dcn_conv's row order, on x16's device.
    x16 [B, N, C]; om [B, N, ld >= 27] offsets (dh, dw per tap) in channels 0-17 and mask logits in 18-26, or None.
    With coords=True also returns [(lo, li, Hi, Wi, h [9, P], w [9, P])] per output level."""
    off = level_offsets(sizes)
    xb = x16[b].double()
    rec = om_records(om[b]) if om is not None else None
    cols, where = [], []
    for lo, li, Ho, Wo, stride in branch_levels(sizes, branch):
        Hi, Wi = sizes[li]
        HWl = sizes[lo][0] * sizes[lo][1]
        assert Ho * Wo <= HWl, "the record of level lo must cover the output grid"
        rec_lo = rec[off[lo]:off[lo] + HWl] if rec is not None else None
        c, h, w = sample_level(xb[off[li]:off[li] + Hi * Wi], Hi, Wi, rec_lo, HWl, Ho, Wo, stride, mut)
        cols.append(c)
        where.append((lo, li, Hi, Wi, h, w))
    cols = torch.cat(cols)
    return (cols, where) if coords else cols


def dcn_y(cols, weight, bias):
    """y64 = cols . W^T + bias in float64: weight [O, 9*C] (k = tap*C + c), bias [O] or None."""
    y = cols @ weight.double().t()
    return y + bias.double() if bias is not None else y


def dcn_bound(cols, y, weight):
    """Per-element bound of |dcn_conv - y64| (and of the dcn_cols + GEMM pair):

        2^-11 |y64|                        the one fp16 rounding of the output
      + 2^-10 sum_k |W_k| |col64_k|        each column rounded to fp16 (2^-11 |col|) and the fp32 sums

    The fp32 sums are the four-corner blend (about 2^-22 of sum |w_i v_i|, with the mask folded into the corner weights), the
    rounding of the sample position base + offset to fp32 (at most 2^-24 |h| <= 2^-16 for maps up to 168 wide, times the
    difference of two corner values) and the 2304-term tensor-core accumulation (at most 2304 * 2^-23 < 2^-11.8 of
    sum |W_k col_k| with truncating adds).  Together they stay below the 2^-11 left over by the factor 2^-10 wherever sum_k
    |W_k| |col64_k| is made of O(1) columns, as it is for every realistic input here; fp16 subnormals (2^-25 absolute) are
    negligible next to it.  There is no absolute floor."""
    return EPS16 * y.abs() + 2 * EPS16 * (cols.abs() @ weight.double().abs().t())


# ---- exact inputs ---------------------------------------------------------------------------------------------------------
def _targets(S):
    """Sample coordinates the targeted offsets aim at on an axis of length S: exactly -1, inside (-1, 0), 0, S-1, inside
    (S-1, S), S, and far outside / inside at -50 and +50."""
    return torch.tensor([-1.0, -0.75, -0.5, -0.25, 0.0, S - 1.0, S - 0.75, S - 0.5, S - 0.25, float(S), -50.0, 50.0],
                        dtype=torch.float64)


EDGE_CLASSES = ("-1", "(-1,0)", "0", "S-1", "(S-1,S)", "S", "far")


def edge_classes(c, S):
    """The edge classes that occur among coordinates c on an axis of length S."""
    found = set()
    for name, hit in (("-1", c == -1), ("(-1,0)", (c > -1) & (c < 0)), ("0", c == 0), ("S-1", c == S - 1),
                      ("(S-1,S)", (c > S - 1) & (c < S)), ("S", c == S), ("far", c.abs() >= 50)):
        if bool(hit.any()):
            found.add(name)
    return found


def _uses(sizes, lo, ch, branch):
    """For the record of level lo, offset channel ch (0-17), at every pixel p: (used, base, S) of the sample that reads it in
    DyConv[branch]: whether it is read, the integer base coordinate the offset is added to, and the input axis length."""
    L = len(sizes)
    H, W = sizes[lo]
    HW = H * W
    p = torch.arange(HW)
    if branch == 1 or branch == 2:
        if branch == 2 and lo == 0:
            return None
        ho, wo = p // W, p % W
        tap, comp = ch // 2, ch % 2
        st = 1 if branch == 1 else 2
        Hi, Wi = sizes[lo] if branch == 1 else sizes[lo - 1]
        base = (ho * st - 1 + tap // 3) if comp == 0 else (wo * st - 1 + tap % 3)
        return torch.ones(HW, dtype=torch.bool), base, (Hi if comp == 0 else Wi)
    if lo >= L - 1:
        return None
    Ho, Wo = sizes[lo + 1]
    f = ch * HW + p                     # flat index of (channel ch, pixel p) in level lo's NCHW buffer
    c2, pix = f // (Ho * Wo), f % (Ho * Wo)
    used = c2 < 18
    tap, comp = c2 // 2, c2 % 2
    ho, wo = pix // Wo, pix % Wo
    base = torch.where(comp == 0, ho - 1 + tap // 3, wo - 1 + tap % 3)
    S = torch.where(comp == 0, torch.full_like(p, Ho), torch.full_like(p, Wo))
    return used, base, S


def dcn_exact_inputs(sizes, B, seed, om_ld=32, device="cpu", nweights=3):
    """Seeded exact operands of ops.dcn_conv -> dict(x16, om, weights, biases).

      x        integers in [-4, 4] (fp16, exact);
      weights  integers in [-2, 2] (fp16, exact), one [256, 2304] per job;
      biases   multiples of 1/32 in [-4, 4] (fp32, exact);
      offsets  multiples of 1/4: each record entry is given to one of the branches that read it (1, 2 or the re-reading
               branch 0) or to none; for its branch the offset is target - base, where the target is drawn from _targets
               (or a random interior point on the 1/4 grid), and otherwise it is uniform on the 1/4 grid in [-3, 3];
      masks    logits in {-200, 0, 200}, i.e. masks of exactly 0, 1/2 and 1 in fp32;
      om       channels 27 .. om_ld-1 NaN (never read).

    Why every rounding is then exact: a sample coordinate base + offset is a multiple of 1/4 below 2^9 in magnitude, so its
    fractional parts lh, lw are multiples of 1/4, each corner weight (with the mask) a multiple of 1/32 in [0, 1] and the fp32
    blend of four corners in [-4, 4] a multiple of 1/32: exact in fp32 and in fp16 (7 significant bits).  Each product of the
    GEMM is a multiple of 1/32 below 8 in magnitude and every partial sum of 2304 of them a multiple of 1/32 below 2^15, i.e.
    below 2^20 units of 1/32: exact in fp32 in any order and under any alignment the tensor cores use.  The output with bias
    is below 2^15 + 4 on the 1/32 grid, so the kernel's one fp16 rounding equals y64.half()."""
    g = torch.Generator().manual_seed(seed)
    L = len(sizes)
    off = level_offsets(sizes)
    N = off[-1]
    x16 = torch.randint(-4, 5, (B, N, 256), generator=g).half()
    om = torch.full((B, N, om_ld), float("nan"), dtype=torch.float64)
    om[..., :18] = torch.randint(-12, 13, (B, N, 18), generator=g) / 4.0
    for lo in range(L):
        HW = sizes[lo][0] * sizes[lo][1]
        rows = slice(off[lo], off[lo] + HW)
        for ch in range(18):
            owner = torch.randint(0, 4, (B, HW), generator=g)   # 0, 1, 2: that branch; 3: nobody
            for br in (0, 1, 2):
                u = _uses(sizes, lo, ch, br)
                if u is None:
                    continue
                used, base, S = u
                S = torch.as_tensor(S).expand(HW)
                pick = torch.randint(0, 14, (B, HW), generator=g)
                tgt = torch.empty(B, HW, dtype=torch.float64)
                for s in S.unique().tolist():
                    t = _targets(int(s))
                    interior = torch.randint(0, 4 * int(s) - 3, (B, HW), generator=g) / 4.0
                    tgt_s = torch.where(pick < len(t), t[pick.clamp(max=len(t) - 1)], interior)
                    sel = (S == s)[None].expand(B, HW)
                    tgt[sel] = tgt_s[sel]
                take = (owner == br) & used[None]
                om[:, rows, ch] = torch.where(take, tgt - base[None].double(), om[:, rows, ch])
    om[..., 18:27] = (torch.randint(-1, 2, (B, N, 9), generator=g) * 200).double()
    ws = [torch.randint(-2, 3, (256, 2304), generator=g).half() for _ in range(nweights)]
    bs = [(torch.randint(-128, 129, (256,), generator=g) / 32.0).float() for _ in range(nweights)]
    return dict(x16=x16.to(device), om=om.float().to(device), weights=[w.to(device) for w in ws],
                biases=[b.to(device) for b in bs])


def dcn_realistic_inputs(sizes, B, seed, om_ld=32, device="cpu", nweights=3):
    """x ~ N(0, 1), offsets ~ N(0, 2.5^2), mask logits ~ N(0, 1), W ~ N(0, 0.03^2), bias ~ N(0, 1), as the comparison tests
    of dcn_conv against dcn_cols + GEMM use."""
    g = torch.Generator().manual_seed(seed)
    N = level_offsets(sizes)[-1]
    x16 = torch.randn(B, N, 256, generator=g).half()
    om = torch.randn(B, N, om_ld, generator=g)
    om[..., :18] *= 2.5
    ws = [(torch.randn(256, 2304, generator=g) * 0.03).half() for _ in range(nweights)]
    bs = [torch.randn(256, generator=g) for _ in range(nweights)]
    return dict(x16=x16.to(device), om=om.to(device), weights=[w.to(device) for w in ws], biases=[b.to(device) for b in bs])


# ----------------------------------------------------------------------------------------------------------------------
# Multi-scale deformable attention core (GroundingDINO ms_deform_attn.py multi_scale_deformable_attn_pytorch; msda.cu)
# ----------------------------------------------------------------------------------------------------------------------
MSDA_MUTATIONS = ("align_corners", "no_half_pixel", "last_level_shift")
MSDA_CLASSES = ("-1", "-0.5", "0", "S-1", "S-0.5", "S", "outside")


def msda_locations(proj, ref, sizes, heads, P):
    """Sampling locations [B, Q, heads, L, P, 2] (x, y in [0, 1] units) in float64 from the kernel's operands: offsets at
    column h*L*P*2 + (l*P + p)*2 of proj [B*Q, ld]; ref [B, Q, L, 2] points (ref + off / (W, H)) or [B, Q, L, 4] boxes
    (ref[:2] + off / P * ref[2:] * 0.5)."""
    B, Q, L, rd = ref.shape
    off = proj.double()[:, :heads * L * P * 2].reshape(B, Q, heads, L, P, 2)
    r = ref.double()[:, :, None, :, None, :]
    if rd == 2:
        norm = torch.tensor([[w, h] for h, w in sizes], dtype=torch.float64, device=proj.device)
        return r + off / norm[None, None, None, :, None, :]
    return r[..., :2] + off / P * r[..., 2:] * 0.5


def msda_reference(value, proj, aw_col0, ref, sizes, heads, P, mut=(), bound=False):
    """out64 [B, Q, heads*32] of the core, out[b, q, h*32 + c] = sum_{l,p} softmax(logits)_lp *
    bilinear_zero_pad(value_l[h], loc_lp * (W_l, H_l) - 0.5), sampled by F.grid_sample(bilinear, zeros, align_corners=False)
    in float64 as multi_scale_deformable_attn_pytorch does.  value [B, Nv, heads*32]; logits at columns aw_col0 + h*L*P + lp.
    With bound=True also returns the per-element bound of the kernel's error:

        2^-11 |out|                                       the fp16 output (fp32 output: this term is slack)
      + sum_i a_i S_i (2^-17 + 2^-22 |z_i - max z|)      the softmax (__expf, its argument, the fp32 sum of <= 32 terms and
                                                          the division) and the fp32 blend and sums of <= 4 * 32 terms, with
                                                          S_i the bilinear sample of |value|
      + sum_i a_i 2 M_i (dx_i + dy_i)                     the fp32 sample position: dx = 2^-22 (W |loc_x| + W |o_x| + |x| + 1)
                                                          with o_x the offset term added to the reference, and M_i the
                                                          largest |value| of the 4x4 pixels around the sample (the sample is
                                                          continuous in the position, with slope below 2 M_i there)."""
    B, Nv, E = value.shape
    Q, L = ref.shape[1], ref.shape[2]
    d = E // heads
    dev = value.device
    v = value.double()
    pr = proj.double().reshape(B, Q, -1)
    z = pr[..., aw_col0:aw_col0 + heads * L * P].reshape(B, Q, heads, L * P)
    aw = torch.softmax(z, -1).view(B, Q, heads, L, P)
    loc = msda_locations(proj, ref, sizes, heads, P)
    norm = torch.tensor([[w, h] for h, w in sizes], dtype=torch.float64, device=dev)[None, None, None, :, None, :]
    if "no_half_pixel" in mut:      # pixel = loc * size instead of loc * size - 0.5
        loc = loc + 0.5 / norm
    start = level_offsets(sizes)
    out = torch.zeros(B * heads, d, Q, dtype=torch.float64, device=dev)
    if bound:
        extra = torch.zeros_like(out)
        zspread = (z.max(-1, keepdim=True).values - z).nan_to_num(posinf=0.0).view(B, Q, heads, L, P)
        rd = ref.shape[-1]
        offv = proj.double()[:, :heads * L * P * 2].reshape(B, Q, heads, L, P, 2)
        if rd == 2:
            oterm = (offv / norm).abs()
        else:
            oterm = (offv / P * ref.double()[:, :, None, :, None, 2:] * 0.5).abs()
    for l, (h, w) in enumerate(sizes):
        s0 = start[l] + (1 if ("last_level_shift" in mut and l == L - 1) else 0)
        rows = v[:, s0:s0 + h * w]
        if rows.shape[1] < h * w:
            rows = torch.cat([rows, rows.new_zeros(B, h * w - rows.shape[1], E)], 1)
        vl = rows.reshape(B, h * w, heads, d).permute(0, 2, 3, 1).reshape(B * heads, d, h, w)
        g = (2 * loc[:, :, :, l] - 1).transpose(1, 2).reshape(B * heads, Q, P, 2)
        smp = F.grid_sample(vl, g, mode="bilinear", padding_mode="zeros", align_corners="align_corners" in mut)
        a = aw[:, :, :, l].permute(0, 2, 1, 3).reshape(B * heads, 1, Q, P)
        out += (smp * a).sum(-1)
        if bound:
            absS = F.grid_sample(vl.abs(), g, mode="bilinear", padding_mode="zeros", align_corners=False)
            zs = zspread[:, :, :, l].permute(0, 2, 1, 3).reshape(B * heads, 1, Q, P)
            extra += (a * absS * (2.0 ** -17 + 2.0 ** -22 * zs)).sum(-1)
            # largest |value| of the 4x4 pixels around each sample: rows y0-1 .. y0+2, columns x0-1 .. x0+2
            nm = F.max_pool2d(F.pad(vl.abs(), (3, 3, 3, 3)), 4, stride=1)         # [BH, d, h+3, w+3]; index i <-> i-2
            lx = loc[:, :, :, l, :, 0].transpose(1, 2).reshape(B * heads, Q * P)
            ly = loc[:, :, :, l, :, 1].transpose(1, 2).reshape(B * heads, Q * P)
            px, py = lx * w - 0.5, ly * h - 0.5
            ix, iy = torch.floor(px).long() + 2, torch.floor(py).long() + 2
            ok = (ix >= 0) & (ix <= w + 2) & (iy >= 0) & (iy <= h + 2)
            idx = (iy.clamp(0, h + 2) * (w + 3) + ix.clamp(0, w + 2))[:, None, :].expand(B * heads, d, Q * P)
            M = torch.gather(nm.flatten(2), 2, idx) * ok[:, None, :].double()
            ox = oterm[:, :, :, l, :, 0].transpose(1, 2).reshape(B * heads, Q * P)
            oy = oterm[:, :, :, l, :, 1].transpose(1, 2).reshape(B * heads, Q * P)
            dx = 2.0 ** -22 * (w * lx.abs() + w * ox + px.abs() + 1)
            dy = 2.0 ** -22 * (h * ly.abs() + h * oy + py.abs() + 1)
            extra += (a * (2 * M * (dx + dy)[:, None, :]).view(B * heads, d, Q, P)).sum(-1)
    out = out.view(B, heads, d, Q).permute(0, 3, 1, 2).reshape(B, Q, E)
    if not bound:
        return out
    extra = extra.view(B, heads, d, Q).permute(0, 3, 1, 2).reshape(B, Q, E)
    return out, EPS16 * out.abs() + extra


def msda_pixel_coords(proj, ref, sizes, heads, P):
    """Pixel coordinates (x, y) = loc * (W, H) - 0.5 of every sample, [B, Q, heads, L, P, 2] float64."""
    loc = msda_locations(proj, ref, sizes, heads, P)
    norm = torch.tensor([[w, h] for h, w in sizes], dtype=torch.float64, device=proj.device)
    return loc * norm[None, None, None, :, None, :] - 0.5


def msda_classes(c, S):
    """The border classes of grid_sample(align_corners=False) that occur among pixel coordinates c on an axis of length S."""
    found = set()
    for name, hit in (("-1", c == -1), ("-0.5", c == -0.5), ("0", c == 0), ("S-1", c == S - 1), ("S-0.5", c == S - 0.5),
                      ("S", c == S), ("outside", (c < -1) | (c > S))):
        if bool(hit.any()):
            found.add(name)
    return found


def msda_exact_inputs(sizes, B, Q, heads, P, ref_dim, seed, device="cpu", proj_pad=3):
    """Seeded exact operands of ops.ms_deform_attn -> dict(value16, proj, aw_col0, ref).  Level sizes must be powers of two.

      value    integers in [-8, 8] (fp16, exact);
      ref      2-d: points on the 1/64 grid in [-0.25, 1.25]; 4-d: centres likewise, sizes in {1/4, 1/2, 1};
      offsets  per coordinate, a pixel target t (loc * S - 0.5 = t) drawn from {-1, -0.5, 0, S-1, S-0.5, S, -2.25, S+1.5} or
               a random point on the 1/4 grid in [0, S-1], with probability 1/2; otherwise random.  2-d: off = t + 0.5 -
               ref * S, or uniform on the 1/4 grid in [-4, 4].  4-d: off = P k with k = 2 (t + 0.5 - ref * S) / (S size),
               or k uniform on the 1/4 grid in [-4, 4];
      logits   per (query, head) 1, 2 or 4 (at most L*P) equal finite logits (an integer in [-4, 4]) and -inf elsewhere;
      proj     proj_pad NaN columns after the logits (never read).

    Why every rounding is then exact: S is a power of two, so off / S (2-d) is exact; in 4-d off / P = k exactly and
    k * size * 0.5 = (t + 0.5 - ref S) / S exactly.  loc is a multiple of 2^-6 / S below 2^7, and loc * S - 0.5 a multiple
    of 2^-6: exact in fp32.  The bilinear weights are then multiples of 2^-12, the softmax weights exactly 1, 1/2 or 1/4
    (__expf(0) = 1, __expf(-inf) = 0, and the sum is 1, 2 or 4), so every product and partial sum is a multiple of 2^-14
    below 2^7 in magnitude (at most 2^21 units): exact in fp32 in any order.  The fp32 output therefore equals the float64
    reference and the fp16 output equals its one rounding."""
    g = torch.Generator().manual_seed(seed)
    L = len(sizes)
    for h, w in sizes:
        assert h & (h - 1) == 0 and w & (w - 1) == 0, "exact MSDA inputs need power-of-two level sizes"
    Nv = sum(h * w for h, w in sizes)
    E = heads * 32
    LP = L * P
    value16 = torch.randint(-8, 9, (B, Nv, E), generator=g).half()
    ref = torch.randint(-16, 81, (B, Q, L, ref_dim), generator=g).double() / 64
    if ref_dim == 4:
        ref[..., 2:] = 2.0 ** -torch.randint(0, 3, (B, Q, L, 2), generator=g).double()
    S = torch.tensor([[w, h] for h, w in sizes], dtype=torch.float64)[None, None, None, :, None, :]   # (x: W, y: H)
    S = S.expand(B, Q, heads, L, P, 2)
    cls = torch.randint(0, 9, (B, Q, heads, L, P, 2), generator=g)
    fixed = torch.stack([torch.full_like(S, -1.0), torch.full_like(S, -0.5), torch.zeros_like(S), S - 1, S - 0.5, S,
                         torch.full_like(S, -2.25), S + 1.5], 0)
    interior = torch.floor(torch.rand(S.shape, generator=g, dtype=torch.float64) * (4 * S - 3)) / 4
    t = torch.where(cls < 8, fixed.gather(0, cls.clamp(max=7)[None]).squeeze(0), interior)
    targeted = torch.rand(S.shape, generator=g) < 0.5
    rnd = torch.randint(-16, 17, S.shape, generator=g).double() / 4
    r = ref[:, :, None, :, None, :]
    if ref_dim == 2:
        off = torch.where(targeted, t + 0.5 - r * S, rnd)
    else:
        k = torch.where(targeted, 2 * (t + 0.5 - r[..., :2] * S) / (S * r[..., 2:]), rnd)
        off = P * k
    logits = torch.full((B, Q, heads, LP), float("-inf"), dtype=torch.float64)
    counts = torch.tensor([n for n in (1, 2, 4) if n <= LP])
    nhot = counts[torch.randint(0, len(counts), (B, Q, heads), generator=g)]
    order = torch.rand(B, Q, heads, LP, generator=g).argsort(-1)
    hot = torch.arange(LP)[None, None, None, :] < nhot[..., None]
    val = torch.randint(-4, 5, (B, Q, heads, 1), generator=g).double().expand(B, Q, heads, LP)
    logits.scatter_(-1, order, torch.where(hot, val, logits))
    aw_col0 = heads * LP * 2
    proj = torch.cat([off.reshape(B * Q, -1), logits.reshape(B * Q, -1),
                      torch.full((B * Q, proj_pad), float("nan"), dtype=torch.float64)], 1)
    return dict(value16=value16.to(device), proj=proj.float().to(device), aw_col0=aw_col0, ref=ref.float().to(device))


def msda_realistic_inputs(sizes, B, Q, heads, P, ref_dim, seed, device="cpu"):
    """value ~ N(0, 1); 2-d reference points uniform in [0, 1] with offsets ~ N(0, 2^2) pixels, or 4-d boxes with centres
    uniform in [0, 1], sizes uniform in [0.05, 0.35] and offsets ~ N(0, P^2 / 4); logits ~ N(0, 1.5^2)."""
    g = torch.Generator().manual_seed(seed)
    L = len(sizes)
    Nv = sum(h * w for h, w in sizes)
    value16 = torch.randn(B, Nv, heads * 32, generator=g).half()
    ref = torch.rand(B, Q, L, ref_dim, generator=g)
    if ref_dim == 4:
        ref[..., 2:] = ref[..., 2:] * 0.3 + 0.05
    off = torch.randn(B * Q, heads * L * P * 2, generator=g) * (2.0 if ref_dim == 2 else P / 2)
    logits = torch.randn(B * Q, heads * L * P, generator=g) * 1.5
    proj = torch.cat([off, logits], 1)
    return dict(value16=value16.to(device), proj=proj.to(device), aw_col0=heads * L * P * 2, ref=ref.to(device))
