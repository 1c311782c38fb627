"""ops.biattn_text_vn (biattn_text_kernel, the text -> image side of the BiAttention fusion) against the float64 restatement of
tests/biattn_text_oracle.py on the same fp16 / fp32 operands, each element held to the bound that follows from the kernel's
own roundings (no absolute floor).  Inputs are built so that each class of mistake moves the output: ragged image-token
counts with zero-filled tails that would dominate a softmax, text lengths that leave a partial or single-row last tile,
colmax values far apart between a thread's two rows and between heads and images, an active clamp, and probabilities in the
fp16 subnormal range.  Also checked: q broadcast or distinct per head, rowbias absent or strided, strided and permuted output
views, bit-identical reruns and graph replays, and the kernel inside BiMultiHeadAttention._attend_fused."""
import pytest
import torch

import biattn_text_oracle as bo

pytestmark = pytest.mark.gpu


def run(c, out=None):
    from mqdet_b200 import ops
    B, H, T, _ = c["kh"].shape
    if out is None:
        out = torch.empty(B, H, T, 256, dtype=torch.float16, device=c["kh"].device)
    ops.biattn_text_vn(c["kh"], c["qh"], c["vn16"], c["colmax"], c["clamp"], out, rowbias=c["rowbias"])
    return out


def check(c, what, out=None):
    """Launch, compare with the float64 restatement, return (out, largest error / bound)."""
    c["colmax"] = bo.colmax_of(c["kh"], c["qh"], c["rowbias"], c["clamp"])
    out = run(c, out)
    u, bound, _ = bo.restate_text(c["kh"], c["qh"], c["vn16"], c["colmax"], c["rowbias"], c["clamp"])
    got = out.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    ratio = ((got - u).abs() / bound).max().item()
    print(f"{what}: max err/bound {ratio:.3f}")
    assert ratio <= 1.0, f"{what}: max |err| / bound = {ratio:.3f}"
    return out, ratio


def case(dev, pattern, B, H, T, N, seed, **kw):
    return bo.make_inputs(pattern, B, H, T, N, seed, device=dev, **kw)


@pytest.mark.parametrize("pattern", ["diffuse", "peaked"])
def test_bench_shape(dev, pattern):
    """B = 8, H = 8, T = 256, N = 22400: every fusion layer of the benchmark."""
    check(case(dev, pattern, 8, 8, 256, 22400, seed=100), f"bench {pattern}")


@pytest.mark.parametrize("pattern", ["diffuse", "tail"])
@pytest.mark.parametrize("N", [1, 63, 64, 65, 128, 129, 193, 1000])
def test_ragged_image_tokens(dev, N, pattern):
    """1 to 16 steps of 64 image tokens with every kind of partial last step."""
    check(case(dev, pattern, 2, 3, 256, N, seed=200 + N), f"N={N} {pattern}")


@pytest.mark.parametrize("T", [1, 8, 63, 64, 65, 200, 256])
def test_text_lengths(dev, T):
    """A partial or single-row last tile of 64 text tokens."""
    check(case(dev, "diffuse", 2, 3, T, 333, seed=300 + T), f"T={T}")


@pytest.mark.parametrize("q", ["broadcast", "distinct"])
@pytest.mark.parametrize("rb_ld", [None, 1, 8])
def test_operands(dev, q, rb_ld):
    """q broadcast over the heads (head stride 0, as _fused_text passes it) or distinct per head; rowbias absent, [B,H,T,1],
    or the module's [B,H,T,8] gbias with column 0 used (the other columns would overflow the exponent if read)."""
    check(case(dev, "diffuse", 2, 3, 200, 333, seed=400, q=q, rb_ld=rb_ld), f"q={q} rb_ld={rb_ld}")


@pytest.mark.parametrize("layout", ["row_stride_264", "permuted"])
def test_output_layout(dev, layout):
    """The output as a view into a larger NaN-filled buffer: rows 264 apart, or [B, T, H, 256] permuted to [B, H, T, 256].
    Nothing outside the [T, 256] rows of each (image, head) may be written."""
    B, H, T = 2, 3, 65
    c = case(dev, "diffuse", B, H, T, 333, seed=500)
    if layout == "row_stride_264":
        buf = torch.full((B, H, T + 5, 264), float("nan"), dtype=torch.float16, device=dev)
        out = buf[:, :, :T, :256]
    else:
        buf = torch.full((B, T + 3, H, 256), float("nan"), dtype=torch.float16, device=dev)
        out = buf[:, :T].permute(0, 2, 1, 3)
    check(c, layout, out=out)
    written = torch.zeros_like(buf, dtype=torch.bool)
    if layout == "row_stride_264":
        written[:, :, :T, :256] = True
    else:
        written[:, :T] = True
    assert torch.isnan(buf[~written]).all(), f"{layout}: elements outside the output view were written"


SHAPES = [(2, 3, 256, 1000), (2, 3, 65, 129), (2, 3, 200, 333)]


@pytest.mark.parametrize("pattern", ["clamp", "clamp0"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "B{}H{}T{}N{}".format(*s))
def test_clamp(dev, pattern, shape):
    """Integer operands: exact fp32 scores, over 20 % beyond +-5e4 and many tied at the clamp; clamp(S + rowbias) differs
    from clamp(S) + rowbias by thousands of nats.  The same operands without a clamp."""
    B, H, T, N = shape
    check(case(dev, pattern, B, H, T, N, seed=600 + T), f"{pattern} {shape}")


@pytest.mark.parametrize("shape", SHAPES[:2] + [(8, 8, 256, 22400)], ids=lambda s: "B{}H{}T{}N{}".format(*s))
@pytest.mark.parametrize("q", ["broadcast", "distinct"])
def test_spread(dev, shape, q):
    """colmax of a thread's two rows (t, t + 8) and of neighbouring heads / images more than 100 apart: a shift taken from
    the wrong row or (image, head), or a dropped rowbias, overflows or underflows the exponent."""
    B, H, T, N = shape
    if q == "distinct" and N > 1000:
        pytest.skip("distinct q at the benchmark shape adds nothing the smaller shapes do not cover")
    check(case(dev, "spread", B, H, T, N, seed=700 + T, q=q), f"spread {shape} q={q}")


def test_reruns_and_graph_replay_bit_identical(dev):
    """No float atomics: two launches, and a CUDA-graph replay, give the same bits."""
    c = case(dev, "diffuse", 4, 8, 256, 3000, seed=800)
    c["colmax"] = bo.colmax_of(c["kh"], c["qh"], c["rowbias"], c["clamp"])
    a = run(c).clone()
    b = run(c)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(c)   # warm-up on a side stream before capture
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    out = torch.empty_like(a)
    with torch.cuda.graph(gr):
        run(c, out)
    for _ in range(2):
        out.fill_(float("nan"))
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, a)


# ---- the kernel as BiMultiHeadAttention._attend_fused runs it --------------------------------------------------------------
LAMBDA = 8.0   # sum of independent zero-mean errors |x_i| <= s_i: P(|sum| > 8 sqrt(sum s_i^2)) <= 2 exp(-32) (Hoeffding)


def attend_reference(mod, vn16, ln16, mask, clamp):
    """dv [B,N,256], dl [B,T,768] of _attend_fused (no residual, no layer scale) in float64 from vn16 / ln16 and the module's
    fp32 parameters, and a per-element bound LAMBDA * sqrt(v) built from the path's fp16 intermediates.  Every rounding is an
    independent error of half-width eps |x| (eps = 2^-11) - the fp16 weight copies, kh, gT, u, ol and the other stored
    intermediates - and v sums their squares through the path (a product C = A B turns v_A into v_A B^2):
        kh  = fp16(ln Wl^T + bl)                  v_k  = eps^2 (ln^2 Wl^2^T + k^2)
        gT  = fp16(kh (d^-1/2 Wq_h))              v_g  = v_k (sWq_h)^2 + eps^2 (k^2 (sWq_h)^2 + gT^2)
        gbias = kh . (d^-1/2 bq_h), fp32          v_gb = v_k (s bq_h)^2 + eps^2 k^2 (s bq_h)^2
        S   = vn gT^T + gbias, fp32               v_S  = vn^2 v_g^T + v_gb
        u   = softmax_n(S^T) vn (the kernel)      v_u  = (sum_n P_n v_S,n) (sum_n P_n (vn_n - u)^2) + b_u^2
            the first term bounds the variance of du = sum_n P_n dS_n (vn_n - u) (first order in the scores) by Cauchy-Schwarz
            whatever the correlation of the dS_n, which all share the errors of gT_h[t]; b_u is the kernel's own bound
            (biattn_text_oracle.restate_text)
        ol  = fp16(u Wvv_h^T + bvv_h)             v_ol = v_u Wvv_h^2^T + eps^2 (u^2 Wvv_h^2^T + ol^2)
        dl  = ol Wol^T + bol, fp32                v_dl = v_ol Wol^2^T + eps^2 ol^2 Wol^2^T
    and on the image side, with vl = fp16(ln Wvl^T + bvl), M_h = fp16(vl_h Wov_h^T) (the kernel's mT) and the normalised
    P_v = softmax_t(S + mask) rounded to fp16 in the kernel (2^-10 with its exp and sums):
        dv  = fp16(sum_h P_v,h M_h + bov)         v_dv = sum_h [(sum_t P_v v_S) (sum_t P_v (M_t - D_h)^2) + P_v^2 v_M + 4 eps^2 P_v^2 M^2]
                                                       + eps^2 dv^2
    The fp32 sums (relative 2^-24 per term) are far below these and left out."""
    w = {k: v.detach().double() for k, v in mod.state_dict().items()}
    H = mod.num_heads
    E = w["v_proj.weight"].shape[0]
    d = E // H
    s = d ** -0.5
    e2 = bo.EPS16 ** 2
    B, N, Cv = vn16.shape
    T = ln16.shape[1]
    dev = vn16.device
    dv = torch.empty(B, N, Cv, dtype=torch.float64, device=dev)
    dv_bound = torch.empty_like(dv)
    dl = torch.empty(B, T, w["out_l_proj.weight"].shape[0], dtype=torch.float64, device=dev)
    dl_bound = torch.empty_like(dl)
    Wol2 = w["out_l_proj.weight"] ** 2

    def spread(pv, x, y):
        """sum_n pv[r, n] (x[n, c] - y[r, c])^2 for pv [R, n] >= 0, x [n, C], y [R, C]."""
        return pv @ (x * x) - 2 * y * (pv @ x) + y * y * pv.sum(1, keepdim=True)

    for b in range(B):
        vn, ln = vn16[b].double(), ln16[b].double()
        vn2, ln2 = vn * vn, ln * ln
        k = ln @ w["l_proj.weight"].t() + w["l_proj.bias"]
        v_k = e2 * (ln2 @ (w["l_proj.weight"] ** 2).t() + k * k)
        vl = ln @ w["values_l_proj.weight"].t() + w["values_l_proj.bias"]
        v_vl = e2 * (ln2 @ (w["values_l_proj.weight"] ** 2).t() + vl * vl)
        kept = torch.ones(T, dtype=torch.bool, device=dev) if mask is None else mask[b] != 0
        ol = torch.empty(T, E, dtype=torch.float64, device=dev)
        v_ol = torch.empty_like(ol)
        D_sum = torch.zeros(N, Cv, dtype=torch.float64, device=dev)
        v_D = torch.zeros_like(D_sum)
        for h in range(H):
            sl = slice(h * d, (h + 1) * d)
            kh, vk, kh2 = k[:, sl], v_k[:, sl], k[:, sl] ** 2
            wq = s * w["v_proj.weight"][sl]                  # [d, Cv]
            bq = s * w["v_proj.bias"][sl]
            gT = kh @ wq
            v_g = vk @ wq ** 2 + e2 * (kh2 @ wq ** 2 + gT * gT)
            gb = kh @ bq
            v_gb = vk @ bq ** 2 + e2 * (kh2 @ bq ** 2)
            A = bo._clamp(vn @ gT.t() + gb[None, :], clamp)  # [N, T]
            v_S = vn2 @ v_g.t() + v_gb[None, :]
            # text side: u, then the value projection after the reduction
            At = A.t()
            e = torch.exp(At - At.max(1, keepdim=True).values)
            colsum = e.sum(1, keepdim=True)
            P = e / colsum
            u = P @ vn
            b_u = (bo.EPS16 * u.abs() + 2 * bo.EPS16 * (P @ vn.abs())
                   + N * bo.F16_SUBNORMAL_HALF * vn.abs().max(0).values[None, :] / colsum)
            v_u = (P * v_S.t()).sum(1, keepdim=True) * spread(P, vn, u) + b_u * b_u
            wv = w["values_v_proj.weight"][sl]               # [d, Cv]
            ol[:, sl] = u @ wv.t() + w["values_v_proj.bias"][sl]
            v_ol[:, sl] = v_u @ (wv ** 2).t() + e2 * ((u * u) @ (wv ** 2).t() + ol[:, sl] ** 2)
            # image side: P_v . M_h summed over the heads
            wo = w["out_v_proj.weight"][:, sl]               # [Cv, d]
            M = vl[:, sl] @ wo.t()                           # [T, Cv]
            v_M = v_vl[:, sl] @ (wo ** 2).t() + e2 * ((vl[:, sl] ** 2) @ (wo ** 2).t() + M * M)
            Pv = torch.softmax(A.masked_fill(~kept[None, :], float("-inf")), dim=1)
            D = Pv @ M
            Pv2 = Pv * Pv
            D_sum += D
            v_D += (Pv * v_S).sum(1, keepdim=True) * spread(Pv, M, D) + Pv2 @ v_M + 4 * e2 * (Pv2 @ (M * M))
        dv[b] = D_sum + w["out_v_proj.bias"]
        dv_bound[b] = LAMBDA * (v_D + e2 * dv[b] ** 2).sqrt()
        dl[b] = ol @ w["out_l_proj.weight"].t() + w["out_l_proj.bias"]
        dl_bound[b] = LAMBDA * (v_ol @ Wol2.t() + e2 * ((ol * ol) @ Wol2.t())).sqrt()
    return dv, dv_bound, dl, dl_bound


@pytest.mark.parametrize("B,N,T", [(8, 22400, 256), (2, 333, 200), (3, 65, 64)])
def test_attend_fused_text_and_image(dev, B, N, T):
    """_attend_fused with no epilogues returns dv and dl without residual or layer scale: compared, element by element, with
    the float64 reference formula from the same fp16 layer-normed tokens.  This checks the query fold on the text side (gT,
    gbias), the value projection after the token reduction, and the pairing with the colmax biattn_image produces.  The image
    tokens carry a per-channel offset, so the text side's u is O(1) rather than a mean of ~N unit rows."""
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.utils.fuse_helper import BiMultiHeadAttention
    from oracle import synth
    from util import load_sd
    sd = synth.bi_attention_sd(synth.Gen(900))
    mod = BiMultiHeadAttention(v_dim=256, l_dim=768, embed_dim=2048, num_heads=8, cfg=mq_glip_t_cfg())
    mod = load_sd(mod, sd, prefix="attn.").to(dev).eval()
    g = torch.Generator().manual_seed(901 + N)
    vn16 = ((4 * torch.rand(B, 1, 256, generator=g) - 2) + torch.randn(B, N, 256, generator=g)).half().to(dev)
    ln16 = torch.randn(B, T, 768, generator=g).half().to(dev)
    mask = torch.ones(B, T)
    mask[0, T // 3:] = 0
    mask = mask.to(dev)
    clamp = mod._score_clamp()
    with torch.no_grad():
        dv, dl = mod._attend_fused(vn16, ln16, mask, None, None)
    dv_ref, dv_bound, dl_ref, dl_bound = attend_reference(mod, vn16, ln16, mask, clamp)
    for what, got, ref, bound in (("dl", dl, dl_ref, dl_bound), ("dv", dv, dv_ref, dv_bound)):
        got = got.double()
        assert got.shape == ref.shape and torch.isfinite(got).all(), what
        ratio = ((got - ref).abs() / bound).max().item()
        print(f"_attend_fused {what} {B, N, T}: max err/bound {ratio:.3f}")
        assert ratio <= 1.0, f"_attend_fused {what} {B, N, T}: max |err| / bound = {ratio:.3f}"
