"""The DyConv kernels after the DCNv2 convolutions (mqdet_b200/csrc/dyhead.cu: chan_stats, gn_attn, dyconv_combine,
dyrelu_coef + dyrelu_apply), each through its ops wrapper against a float64 CPU reference computed from the same rounded
inputs (tests/dyconv_oracle.py), at the pyramids inference runs: the 800x1344 benchmark input, the portrait padded batch
of the graph engines (B * L = 40), B > 2, levels under 128 pixels and of size 1x1, single-row / single-column levels and a
single level.  Every check records its worst error / bound ratio (tests/util.py)."""
import pytest
import torch
import torch.nn.functional as F

import dyconv_oracle as do
from util import _records, assert_close, load_sd

pytestmark = pytest.mark.gpu

C = do.C


@pytest.fixture(scope="module")
def params(dev):
    p = do.dyconv_params()
    return p, {k: v.reshape(-1).contiguous().to(dev) if k.startswith("AttnConv") else v.contiguous().to(dev)
               for k, v in p.items()}


def _levels(sizes, dev):
    from mqdet_b200 import ops
    return ops.Levels(sizes, dev)


def _check(what, err, bound):
    """err <= bound elementwise (float64 tensors of one shape); records the worst ratio."""
    ratio = (err / bound).flatten()
    i = int(ratio.argmax())
    r = ratio[i].item()
    _records.append(dict(what=what, max_abs_err=err.flatten()[i].item(), bound=bound.flatten()[i].item(), ratio=r))
    assert r <= 1.0, f"{what}: err {err.flatten()[i].item():.3e} > bound {bound.flatten()[i].item():.3e} (x{r:.2f})"


def _branches(sizes, lv):
    """(branch k, level sizes of its rows, segment table, GAP row weights, sizes its segments are upsampled to)."""
    out = [(1, sizes, lv.seg_all, None, None)]
    if len(sizes) > 1:
        out += [(2, sizes[1:], lv.seg_tail, None, None), (0, sizes[1:], lv.seg_tail, lv.up_w, sizes[:-1])]
    return out


@pytest.mark.parametrize("case", do.CASES, ids=do.case_id)
def test_chan_stats(dev, case):
    """Integer fp16 inputs in [-8, 8]: every fp32 partial is exact, so the chunk-folded sum and sum of squares equal the
    float64 sums bit for bit — a dropped or repeated row anywhere shows.  The weighted sum (Levels.up_w) to 1e-6 of
    sum |w * y|; without weights it equals the plain sum."""
    from mqdet_b200 import ops
    name, B = case
    sizes = do.PYRAMIDS[name]
    lv = _levels(sizes, dev)
    ys = dict(zip((1, 2, 0), do.branch_outputs(sizes, B, "pad", integer=True)))
    for k, segs, seg, rw, _ in _branches(sizes, lv):
        y = ys[k]
        rows, nseg = y.shape[1], len(segs)
        part = ops.chan_stats(y.to(dev), seg, B, rows, rw).view(B, nseg, 32, 3, C).double().sum(2).cpu()
        off = do.seg_offsets(segs)
        yd = y.double()
        w = rw.double().cpu() if rw is not None else torch.ones(rows, dtype=torch.float64)
        tag = f"chan_stats {do.case_id(case)} branch {k}"
        for i in range(nseg):
            t = yd[:, off[i]:off[i + 1]]
            s, q = t.sum(1), (t * t).sum(1)
            assert torch.equal(part[:, i, 0], s), f"{tag} segment {i}: sum differs by {(part[:, i, 0] - s).abs().max()}"
            assert torch.equal(part[:, i, 1], q), f"{tag} segment {i}: sum of squares differs"
            if rw is None:
                assert torch.equal(part[:, i, 2], s), f"{tag} segment {i}: unweighted third statistic != sum"
            else:
                wy = w[None, off[i]:off[i + 1], None] * t
                _check(f"{tag} weighted sum segment {i}", (part[:, i, 2] - wy.sum(1)).abs(), 1e-6 * wy.abs().sum(1) + 1e-30)
        _records.append(dict(what=f"{tag}: sum / sum of squares", max_abs_err=0.0, bound=0.0, ratio=0.0))


@pytest.mark.parametrize("pattern", ["pad", "offset"])
@pytest.mark.parametrize("case", do.CASES, ids=do.case_id)
def test_gn_attn(dev, params, case, pattern):
    """GroupNorm affine and scale attention from chan_stats' partials: ga * y + gb against F.group_norm in float64 per
    segment (1e-4 * max + 1e-4), attn against h_sigmoid(relu(w . GAP + b)) (1e-5, 1e-4 at |mean| / std = 16).  Branch 0 pools
    with Levels.up_w; its reference pools F.interpolate(GN(y0), fine size, align_corners=True) itself."""
    from mqdet_b200 import ops
    name, B = case
    sizes = do.PYRAMIDS[name]
    p, pd = params
    lv = _levels(sizes, dev)
    ys = dict(zip((1, 2, 0), do.branch_outputs(sizes, B, pattern)))
    at_tol = 1e-4 if pattern == "offset" else 1e-5
    for k, segs, seg, rw, up_to in _branches(sizes, lv):
        y = ys[k]
        gw, gb = p[f"DyConv.{k}.bn.weight"], p[f"DyConv.{k}.bn.bias"]
        part = ops.chan_stats(y.to(dev), seg, B, y.shape[1], rw)
        aff, at = ops.gn_attn(part, seg, B, C, 16, rw is not None, pd[f"DyConv.{k}.bn.weight"], pd[f"DyConv.{k}.bn.bias"],
                              do.EPS, pd["AttnConv.1.weight"], pd["AttnConv.1.bias"])
        aff, at = aff.cpu(), at.cpu()
        tag = f"gn_attn {do.case_id(case)} {pattern} branch {k}"
        for i, t in enumerate(do.levels_of(y, segs)):
            ref = F.group_norm(t, 16, gw.double(), gb.double(), do.EPS)
            err = (do.apply_affine(t, aff[:, i]) - ref).abs()
            _check(f"{tag} GN segment {i}", err, torch.full_like(err, 1e-4 * ref.abs().max().item() + 1e-4))
        ref_at = do.attention(y, segs, do.gn_affine(y, segs, gw, gb), p["AttnConv.1.weight"], p["AttnConv.1.bias"], up_to)
        err = (at.double() - ref_at).abs()
        _check(f"{tag} attn", err, torch.full_like(err, at_tol))


def _reference_affines(sizes, p, ys):
    """float64 GN affines / attentions of the three branches -> fp32 (the kernel's inputs) on the CPU."""
    aw, ab = p["AttnConv.1.weight"], p["AttnConv.1.bias"]
    aff, at = {}, {}
    for k, segs, up_to in ((1, sizes, None), (2, sizes[1:], None), (0, sizes[1:], sizes[:-1])):
        if ys[k] is None:
            aff[k] = at[k] = None
            continue
        a = do.gn_affine(ys[k], segs, p[f"DyConv.{k}.bn.weight"], p[f"DyConv.{k}.bn.bias"])
        aff[k], at[k] = a.float(), do.attention(ys[k], segs, a, aw, ab, up_to).float()
    return aff, at


def _combine(dev, lv, B, ys, aff, at):
    from mqdet_b200 import ops
    d = lambda t: None if t is None else t.contiguous().to(dev)  # noqa: E731
    return ops.dyconv_combine(d(ys[1]), d(ys[2]), d(ys[0]), d(aff[1]), d(aff[2]), d(aff[0]), d(at[1]), d(at[2]), d(at[0]),
                              lv, B)


@pytest.mark.parametrize("case", do.CASES, ids=do.case_id)
def test_dyconv_combine(dev, params, case):
    """mean_k attn_k * GN_k(y_k), branch 0 bilinearly upsampled (align_corners), from float64 affines / attentions cast to
    fp32: mid within one fp16 ulp of the float64 value plus the fp32 accumulation error (1e-6 of sum_k |attn_k|
    (|ga_k y_k| + |gb_k|) / branches); the chunk-folded mid_sums equal the float64 per-(image, level, channel) sums of the
    returned mid to 1e-5 of sum |mid|."""
    name, B = case
    sizes = do.PYRAMIDS[name]
    p, _ = params
    lv = _levels(sizes, dev)
    ys = dict(zip((1, 2, 0), do.branch_outputs(sizes, B, "pad")))
    aff, at = _reference_affines(sizes, p, ys)
    mid, sums = _combine(dev, lv, B, ys, aff, at)
    mid, sums = mid.cpu().double(), sums.cpu()
    ref, mag = do.combine(ys[1], ys[2], ys[0], aff[1], aff[2], aff[0], at[1], at[2], at[0], sizes)
    tag = f"dyconv_combine {do.case_id(case)}"
    _check(f"{tag} mid", (mid - ref).abs(), do.fp16_ulp(ref) + 1e-6 * mag)
    folded = sums.view(B, len(sizes), -1, C).double().sum(2)
    for l, t in enumerate(do.levels_of(mid, sizes)):
        err = (folded[:, l] - t.sum((2, 3))).abs()
        _check(f"{tag} mid_sums level {l}", err, 1e-5 * t.abs().sum((2, 3)) + 1e-30)


@pytest.mark.parametrize("case", do.CASES, ids=do.case_id)
def test_dyrelu(dev, params, case):
    """DyReLU on dyconv_combine's output, its coefficients pooled from mid_sums (128 x 1 partials) and from chan_stats
    (mid_sums=None, 32 x 3 partials): within one fp16 ulp of restate.dyrelu in float64 plus 1e-5 * max|mid| each, and
    within one ulp (plus 2e-6 * max|mid| for the different summation order of the pool) of each other."""
    from mqdet_b200 import ops
    name, B = case
    sizes = do.PYRAMIDS[name]
    p, pd = params
    lv = _levels(sizes, dev)
    ys = dict(zip((1, 2, 0), do.branch_outputs(sizes, B, "pad")))
    aff, at = _reference_affines(sizes, p, ys)
    mid, sums = _combine(dev, lv, B, ys, aff, at)
    w = [pd["relu.fc.0.weight"], pd["relu.fc.0.bias"], pd["relu.fc.2.weight"], pd["relu.fc.2.bias"]]
    out_s = ops.dyrelu(mid, lv, *w, mid_sums=sums).cpu().double()
    out_c = ops.dyrelu(mid, lv, *w).cpu().double()
    mid = mid.cpu()
    ref = do.dyrelu(mid, sizes, p)
    mmax = mid.abs().max().double().item()
    tag = f"dyrelu {do.case_id(case)}"
    _check(f"{tag} (mid_sums)", (out_s - ref).abs(), do.fp16_ulp(ref) + 1e-5 * mmax)
    _check(f"{tag} (chan_stats)", (out_c - ref).abs(), do.fp16_ulp(ref) + 1e-5 * mmax)
    _check(f"{tag} paths agree", (out_s - out_c).abs(), do.fp16_ulp(torch.maximum(out_s.abs(), out_c.abs())) + 2e-6 * mmax)


def test_dyconv_bench_pyramid(dev):
    """DyConv.forward_flat at the benchmark pyramid (800x1344 input, B = 1) against restate.dyconv, at the bound of
    test_fusion_gpu.py::test_dyconv."""
    from mqdet_b200.modeling.rpn.vldyhead import Conv3x3Norm, DyConv
    from oracle import restate, synth
    sizes = do.PYRAMIDS["bench"]
    gen = synth.Gen(81)
    sd = synth.dyconv_sd(gen)
    feats = [gen.randn(1, 256, h, w) for h, w in sizes]
    ref = restate.flatten_levels(restate.dyconv(feats, sd))
    conv_func = lambda i, o, s: Conv3x3Norm(i, o, s, deformable=True, bn_type=["gn", 16])  # noqa: E731
    mod = load_sd(DyConv(256, 256, conv_func=conv_func, use_dyrelu=True, use_dyfuse=True, use_deform=True), sd).to(dev).eval()
    out = mod.forward_flat(restate.flatten_levels(feats).half().to(dev).contiguous(), _levels(sizes, dev))
    assert_close(out, ref, 3e-3, "DyConv at the benchmark pyramid (fp16 activations)")
