"""The float64 references of tests/test_dyconv_kernels_gpu.py, checked without a GPU: the post-convolution restatement in
tests/dyconv_oracle.py reproduces ``oracle.restate.dyconv`` (pinned to the reference's own DyConv.forward by
test_oracle_pinning.py), ``Levels.up_w`` equals the pooled align_corners upsample, and the seeded inputs reach every clamp
of the attention and of DyReLU."""
import pytest
import torch
import torch.nn.functional as F

import dyconv_oracle as do
from oracle import restate, synth


@pytest.mark.parametrize("name", ["small", "tiny", "rows", "cols", "single"])
def test_post_dcn_reference_matches_restate(name):
    """restate.dyconv's three DCNv2 outputs per level, fed through dyconv_oracle.post_dcn, give restate.dyconv's result."""
    sizes = do.PYRAMIDS[name]
    L = len(sizes)
    gen = synth.Gen(90)
    sd = {k: v.double() for k, v in synth.dyconv_sd(gen).items()}
    feats = [gen.randn(2, 256, h, w).double() for h, w in sizes]
    y1, y2, y0 = [], [], []
    for l, f in enumerate(feats):
        om = F.conv2d(f, sd["offset.weight"], sd["offset.bias"], padding=1)
        off, mask = om[:, :18].reshape(2, -1), om[:, 18:].sigmoid().reshape(2, -1)

        def conv(k, x, stride):
            return restate.dcn_v2(x, off, mask, sd[f"DyConv.{k}.conv.weight"], sd[f"DyConv.{k}.conv.bias"], stride)

        y1.append(conv(1, f, 1))
        if l > 0:
            y2.append(conv(2, feats[l - 1], 2))
        if l < L - 1:
            y0.append(conv(0, feats[l + 1], 1))
    got = do.post_dcn(do.flat(y1), do.flat(y2) if y2 else None, do.flat(y0) if y0 else None, sizes, sd)
    ref = restate.flatten_levels(restate.dyconv(feats, sd))
    err = (got - ref).abs().max().item()
    assert err <= 1e-5 * ref.abs().max().item() + 1e-5, (name, err)


@pytest.mark.parametrize("name", list(do.PYRAMIDS))
def test_gn_affine_is_group_norm(name):
    sizes = do.PYRAMIDS[name]
    y = do.features(sizes, 2, 5, "offset")
    p = do.dyconv_params(6)
    aff = do.gn_affine(y, sizes, p["DyConv.1.bn.weight"], p["DyConv.1.bn.bias"])
    for i, t in enumerate(do.levels_of(y, sizes)):
        ref = F.group_norm(t, 16, p["DyConv.1.bn.weight"].double(), p["DyConv.1.bn.bias"].double(), do.EPS)
        assert (do.apply_affine(t, aff[:, i]) - ref).abs().max().item() <= 1e-9 * ref.abs().max().item()


@pytest.mark.parametrize("name", list(do.PYRAMIDS))
def test_up_w_is_the_pooled_upsample(name):
    """Levels.up_w (closed-form column sums in mqdet_b200/ops.py) against unit vectors pushed through F.interpolate.
    up_w takes the source index from an fp32 scale as ATen does for fp32 maps, the float64 upsample from a float64 scale:
    the weights agree to ~4e-6 relative; a wrong index or edge clamp moves a weight by a few percent."""
    from mqdet_b200 import ops
    sizes = do.PYRAMIDS[name]
    lv = ops.Levels(sizes, "cpu")
    if len(sizes) == 1:
        assert lv.up_w is None
        return
    ref = do.gap_weights(sizes)
    got = lv.up_w.double()
    assert got.shape == ref.shape
    assert (ref > 0).all()
    assert ((got - ref).abs() <= 1e-5 * ref).all(), ((got - ref).abs() / ref).max().item()
    off = do.seg_offsets(sizes[1:])
    for i in range(len(sizes) - 1):
        assert abs(got[off[i]:off[i + 1]].sum().item() - 1.0) <= 1e-6


@pytest.mark.parametrize("name", [n for n in do.PYRAMIDS if len(do.PYRAMIDS[n]) > 1])
def test_fp32_index_upsample_is_atens_fp32_upsample(name):
    """The upsample of the scale-fusion reference (float64 values at fp32 source positions) against ATen's bilinear
    align_corners upsample of the same map in fp32, for every level pair of the pyramid."""
    sizes = do.PYRAMIDS[name]
    g = torch.Generator().manual_seed(3)
    for (H, W), (Hs, Ws) in zip(sizes[:-1], sizes[1:]):
        t = torch.randn(1, 8, Hs, Ws, generator=g).float()
        ref = F.interpolate(t, size=(H, W), mode="bilinear", align_corners=True).double()
        got = do.upsample_fp32_index(t.double(), (H, W))
        assert (got - ref).abs().max().item() <= 1e-6 * t.abs().max().item(), (H, W)


@pytest.mark.parametrize("case", do.CASES, ids=do.case_id)
def test_inputs_reach_every_clamp(case):
    """The GPU tests' inputs and parameters put segments on both sides of the attention's ReLU and into h_sigmoid's
    saturation, and zero some DyReLU hidden units while saturating some coefficients, at every pyramid with enough
    segments for it."""
    name, B = case
    sizes = do.PYRAMIDS[name]
    p = do.dyconv_params()
    aw, ab = p["AttnConv.1.weight"], p["AttnConv.1.bias"]
    for pattern in ("offset", "pad"):
        ys = do.branch_outputs(sizes, B, pattern)
        affs, ats = [None] * 3, [None] * 3
        for k, y, segs, up_to in ((1, ys[0], sizes, None), (2, ys[1], sizes[1:], None), (0, ys[2], sizes[1:], sizes[:-1])):
            if y is not None:
                affs[k] = do.gn_affine(y, segs, p[f"DyConv.{k}.bn.weight"], p[f"DyConv.{k}.bn.bias"])
                ats[k] = do.attention(y, segs, affs[k], aw, ab, up_to)
        at = torch.cat([a.flatten() for a in ats if a is not None])
        regimes = {"relu0": bool((at == 0.5).any()), "sat": bool((at == 1.0).any()),
                   "linear": bool(((at > 0.5) & (at < 1.0)).any())}
        if at.numel() >= 6:
            assert all(regimes.values()), (pattern, regimes, at)
        else:
            assert sum(regimes.values()) >= 2, (pattern, regimes, at)
    # DyReLU runs on the scale-fused output of the "pad" inputs in the GPU tests (the loop's last pattern)
    mid, _ = do.combine(*ys, affs[1], affs[2], affs[0], ats[1], ats[2], ats[0], sizes)
    hid, ys = do.dyrelu_hidden(mid, sizes, p)
    assert (hid == 0).any() and (hid > 0).any()
    assert (ys == 0).any() and (ys == 1).any() and ((ys > 0) & (ys < 1)).any()
