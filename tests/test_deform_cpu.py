"""The float64 references of tests/test_dcn_kernels_gpu.py and tests/test_msda_gpu.py, checked without a GPU.

DCNv2: the restatement in dcn_conv's row layout equals torchvision.ops.deform_conv2d (branches 1 and 2) and
``oracle.restate.dcn_v2`` (all three branches, including DyConv[0]'s re-read offsets), exactly on exact inputs.  MSDA: the core,
wrapped in the module's value / output projections, reproduces ``oracle.restate.ms_deform_attn``.  The exact-input generators
put samples on every edge class of every branch and level, and each emulated kernel mistake moves an output."""
import pytest
import torch

import deform_oracle as do
from oracle import restate

PYRAMID = [(13, 17), (7, 9), (4, 5), (2, 3), (1, 2)]   # odd sizes; each level is the stride-2 grid of the one before
SMALL = [(9, 11), (5, 6), (3, 3)]


def _nchw(t, sizes, l, B):
    """Level l of a [B, N, ch] tensor as float64 [B, ch, H, W]."""
    off = do.level_offsets(sizes)
    h, w = sizes[l]
    return t[:, off[l]:off[l] + h * w].double().transpose(1, 2).reshape(B, -1, h, w)


def _w4(weight):
    """[O, 9*C] (k = tap*C + c) -> [O, C, 3, 3] float64."""
    O = weight.shape[0]
    return weight.double().view(O, 9, -1).permute(0, 2, 1).reshape(O, -1, 3, 3)


def _oracle_y(case, sizes, branch, j=0, mut=()):
    """[B, rows_per_image, 256] float64."""
    B = case["x16"].shape[0]
    return torch.stack([do.dcn_y(do.dcn_image(case["x16"], case["om"], sizes, branch, b, mut), case["weights"][j],
                                 case["biases"][j]) for b in range(B)])


def _per_level(y, sizes, branch):
    o = 0
    for lo, li, Ho, Wo, stride in do.branch_levels(sizes, branch):
        yield lo, li, stride, y[:, o:o + Ho * Wo].transpose(1, 2).reshape(y.shape[0], -1, Ho, Wo)
        o += Ho * Wo


def _masks(om, sizes, l, B):
    """Level l's masks as float64 [B, 9, H, W], the fp32 values of deform_oracle.om_records."""
    rec = torch.stack([do.om_records(om[b]) for b in range(B)])
    return _nchw(rec[..., 18:27], sizes, l, B)


@pytest.mark.parametrize("om_ld", [27, 32])
@pytest.mark.parametrize("branch", [1, 2])
def test_dcn_oracle_equals_torchvision(branch, om_ld):
    """Branches 1 and 2 read each level's own records, so torchvision's deform_conv2d computes the same thing; on exact inputs
    (targeted edges, stride 1 and 2, odd sizes) the two agree to the last bit."""
    import torchvision
    sizes, B = PYRAMID, 2
    c = do.dcn_exact_inputs(sizes, B, seed=10 + branch, om_ld=om_ld, nweights=1)
    y = _oracle_y(c, sizes, branch)
    for lo, li, stride, got in _per_level(y, sizes, branch):
        x = _nchw(c["x16"], sizes, li, B)
        want = torchvision.ops.deform_conv2d(x, _nchw(c["om"][..., :18], sizes, lo, B), _w4(c["weights"][0]),
                                             c["biases"][0].double(), stride=stride, padding=1, mask=_masks(c["om"], sizes, lo, B))
        assert want.shape == got.shape
        assert torch.equal(got, want), f"branch {branch} level {lo}: max |diff| {(got - want).abs().max().item()}"


@pytest.mark.parametrize("kind", ["exact", "realistic"])
@pytest.mark.parametrize("branch", [0, 1, 2])
def test_dcn_oracle_equals_restate_dcn_v2(branch, kind):
    """All three branches against oracle.restate.dcn_v2 (pinned to the reference's CUDA kernel), which takes the NCHW-flat
    record of level lo and indexes it with the output's strides: DyConv[0] re-reads the finer level's buffer."""
    sizes, B = PYRAMID, 2
    make = do.dcn_exact_inputs if kind == "exact" else do.dcn_realistic_inputs
    c = make(sizes, B, seed=20 + branch, nweights=1)
    y = _oracle_y(c, sizes, branch)
    for lo, li, stride, got in _per_level(y, sizes, branch):
        x = _nchw(c["x16"], sizes, li, B)
        want = restate.dcn_v2(x, _nchw(c["om"][..., :18], sizes, lo, B).reshape(B, -1),
                              _masks(c["om"], sizes, lo, B).reshape(B, -1), _w4(c["weights"][0]), c["biases"][0].double(),
                              stride)
        assert want.shape == got.shape
        if kind == "exact":
            assert torch.equal(got, want), f"branch {branch} level {lo}"
        else:
            torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("sizes,B", [(PYRAMID, 2), (SMALL, 1), ([(13, 17), (7, 9), (4, 5), (2, 3), (1, 1)], 3),
                                     ([(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)], 8)])
def test_dcn_exact_inputs_reach_every_edge(sizes, B):
    """Every branch, including branch 0 whose offsets are re-read, samples exactly at -1, inside (-1, 0), at 0, at S-1,
    inside (S-1, S), at S and far away, on both axes."""
    c = do.dcn_exact_inputs(sizes, B, seed=7, nweights=0)
    x1 = c["x16"][..., :1]      # the coordinates do not depend on the channels
    for branch in (1, 2, 0):
        found_h, found_w = set(), set()
        for b in range(B):
            _, where = do.dcn_image(x1, c["om"], sizes, branch, b, coords=True)
            for lo, li, Hi, Wi, h, w in where:
                found_h |= do.edge_classes(h, Hi)
                found_w |= do.edge_classes(w, Wi)
        assert found_h >= set(do.EDGE_CLASSES), (branch, set(do.EDGE_CLASSES) - found_h)
        assert found_w >= set(do.EDGE_CLASSES), (branch, set(do.EDGE_CLASSES) - found_w)


def test_dcn_exact_inputs_are_exact_in_fp16():
    """Columns are multiples of 1/32 in [-4, 4] and outputs multiples of 1/32: their fp16 roundings are exact."""
    sizes, B = PYRAMID, 2
    c = do.dcn_exact_inputs(sizes, B, seed=30, nweights=1)
    for branch in (0, 1, 2):
        cols = do.dcn_image(c["x16"], c["om"], sizes, branch, 0)
        assert torch.equal(cols.half().double(), cols) and cols.abs().max() <= 4
        assert torch.equal(torch.round(cols * 32), cols * 32)
        y = do.dcn_y(cols, c["weights"][0], c["biases"][0])
        assert torch.equal(torch.round(y * 32), y * 32) and y.abs().max() < 2 ** 15


# which branch shows each mistake: the re-read only exists in branch 0, the stride-2 base only in branch 2
_DCN_MUT_BRANCHES = {"quirk_out_strides": (0,), "stride2_base": (2,)}
# a sample exactly at H or W only occurs in the exact inputs
_DCN_EXACT_ONLY = ("upper_le",)


@pytest.mark.parametrize("mut", [m for m in do.DCN_MUTATIONS if m != "lower_ge"])
def test_dcn_mutations_are_caught(mut):
    """Each emulated kernel mistake changes at least one fp16 output of the exact case, in a branch that has the code it
    breaks, and (unless it only acts exactly on the upper edge) exceeds the bound on the realistic one."""
    sizes, B = PYRAMID, 2
    for branch in _DCN_MUT_BRANCHES.get(mut, (0, 1, 2)):
        c = do.dcn_exact_inputs(sizes, B, seed=40, nweights=1)
        good, bad = _oracle_y(c, sizes, branch), _oracle_y(c, sizes, branch, mut=(mut,))
        assert not torch.equal(good.half(), bad.half()), (mut, branch, "exact")
        if mut in _DCN_EXACT_ONLY:
            continue
        c = do.dcn_realistic_inputs(sizes, B, seed=41, nweights=1)
        worst = 0.0
        for b in range(B):
            cols = do.dcn_image(c["x16"], c["om"], sizes, branch, b)
            y = do.dcn_y(cols, c["weights"][0], c["biases"][0])
            ybad = do.dcn_y(do.dcn_image(c["x16"], c["om"], sizes, branch, b, (mut,)), c["weights"][0], c["biases"][0])
            worst = max(worst, ((ybad - y).abs() / do.dcn_bound(cols, y, c["weights"][0])).max().item())
        assert worst > 1, (mut, branch, "realistic", worst)


def test_dcn_lower_edge_strictness_is_unobservable():
    """'> -1' and '>= -1' give the same samples: at exactly -1 the one corner the wider rule admits (row or column 0) has
    weight h - floor(h) = 0.  The exact inputs do sample at exactly -1, so this is not a gap in the inputs."""
    sizes, B = PYRAMID, 2
    c = do.dcn_exact_inputs(sizes, B, seed=40, nweights=1)
    for branch in (0, 1, 2):
        assert torch.equal(_oracle_y(c, sizes, branch), _oracle_y(c, sizes, branch, mut=("lower_ge",)))


def test_dcn_bound_holds_for_fp16_columns():
    """An ideal kernel on realistic inputs, columns rounded to fp16, summed in fp32 and rounded to fp16, stays inside the
    bound; the output rounding alone may use most of its first term."""
    sizes, B = PYRAMID, 2
    c = do.dcn_realistic_inputs(sizes, B, seed=50, nweights=1)
    w = c["weights"][0]
    for branch in (0, 1, 2):
        cols = do.dcn_image(c["x16"], c["om"], sizes, branch, 0)
        y = do.dcn_y(cols, w, c["biases"][0])
        y16 = ((cols.half().float() @ w.float().t()) + c["biases"][0]).half().double()
        ratio = ((y16 - y).abs() / do.dcn_bound(cols, y, w)).max().item()
        assert ratio <= 1, (branch, ratio)


# ---- multi-scale deformable attention -------------------------------------------------------------------------------------
def _msda_sd(seed, E, heads, L, P):
    g = torch.Generator().manual_seed(seed)

    def lin(o, i, scale, bscale):
        return (torch.randn(o, i, generator=g, dtype=torch.float64) * scale,
                torch.randn(o, generator=g, dtype=torch.float64) * bscale)

    sd = {}
    for name, o, s, bs in (("sampling_offsets", heads * L * P * 2, 0.05, 2.0), ("attention_weights", heads * L * P, 0.1, 1.0),
                           ("value_proj", E, E ** -0.5, 0.1), ("output_proj", E, E ** -0.5, 0.1)):
        sd[name + ".weight"], sd[name + ".bias"] = lin(o, E, s, bs)
    return sd


@pytest.mark.parametrize("ref_dim", [2, 4])
def test_msda_core_matches_restate(ref_dim):
    """value_proj -> the restated core on proj = [sampling_offsets | attention_weights](query) -> output_proj equals
    oracle.restate.ms_deform_attn (pinned to the reference module)."""
    sizes, B, Q, E, heads, P = [(12, 17), (6, 9), (3, 5), (2, 3)], 2, 37, 256, 8, 4
    L = len(sizes)
    sd = _msda_sd(60 + ref_dim, E, heads, L, P)
    g = torch.Generator().manual_seed(61)
    Nv = sum(h * w for h, w in sizes)
    query = torch.randn(B, Q, E, generator=g, dtype=torch.float64)
    value = torch.randn(B, Nv, E, generator=g, dtype=torch.float64)
    ref = torch.rand(B, Q, L, ref_dim, generator=g, dtype=torch.float64) * 1.2 - 0.1
    if ref_dim == 4:
        ref[..., 2:] = ref[..., 2:] * 0.3 + 0.05
    want = restate.ms_deform_attn(query, value, ref, sizes, sd, heads=heads, points=P)
    lin = torch.nn.functional.linear
    proj = lin(query, torch.cat([sd["sampling_offsets.weight"], sd["attention_weights.weight"]]),
               torch.cat([sd["sampling_offsets.bias"], sd["attention_weights.bias"]])).reshape(B * Q, -1)
    v = lin(value, sd["value_proj.weight"], sd["value_proj.bias"])
    core = do.msda_reference(v, proj, heads * L * P * 2, ref, sizes, heads, P)
    got = lin(core, sd["output_proj.weight"], sd["output_proj.bias"])
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


MSDA_EXACT = [([(8, 16), (4, 8), (2, 4), (1, 2)], 4), ([(16, 8), (8, 4), (1, 1)], 8), ([(4, 1), (1, 4)], 4)]


@pytest.mark.parametrize("ref_dim", [2, 4])
@pytest.mark.parametrize("sizes,P", MSDA_EXACT)
def test_msda_exact_inputs_reach_every_border(sizes, P, ref_dim):
    """Every level, both axes: samples exactly at -1, -0.5, 0, S-1, S-0.5, S and outside."""
    c = do.msda_exact_inputs(sizes, 2, 64, 8, P, ref_dim, seed=70)
    pc = do.msda_pixel_coords(c["proj"], c["ref"], sizes, 8, P)
    for l, (h, w) in enumerate(sizes):
        for axis, S in ((0, w), (1, h)):
            found = do.msda_classes(pc[:, :, :, l, :, axis], S)
            assert found >= set(do.MSDA_CLASSES), (l, axis, set(do.MSDA_CLASSES) - found)


@pytest.mark.parametrize("ref_dim", [2, 4])
def test_msda_exact_inputs_are_exact(ref_dim):
    """Pixel coordinates on the 1/64 grid, softmax weights 1, 1/2 or 1/4, outputs on the 2^-14 grid."""
    sizes, P, heads = MSDA_EXACT[0][0], 4, 8
    c = do.msda_exact_inputs(sizes, 2, 64, heads, P, ref_dim, seed=71)
    pc = do.msda_pixel_coords(c["proj"], c["ref"], sizes, heads, P)
    assert torch.equal(torch.round(pc * 64), pc * 64)
    L = len(sizes)
    a = torch.softmax(c["proj"].double()[:, c["aw_col0"]:c["aw_col0"] + heads * L * P].view(-1, heads, L * P), -1)
    assert set(a.unique().tolist()) <= {0.0, 0.25, 0.5, 1.0}
    out = do.msda_reference(c["value16"], c["proj"], c["aw_col0"], c["ref"], sizes, heads, P)
    assert torch.equal(torch.round(out * 2 ** 14), out * 2 ** 14)
    assert torch.equal(out.float().double(), out)


@pytest.mark.parametrize("mut", do.MSDA_MUTATIONS)
@pytest.mark.parametrize("ref_dim", [2, 4])
def test_msda_mutations_are_caught(mut, ref_dim):
    """align_corners=True, the pixel position without the -0.5, and the last level's rows shifted by one each change an fp16
    output of the exact case and exceed the bound on a realistic one."""
    sizes, P, heads = MSDA_EXACT[0][0], 4, 8
    c = do.msda_exact_inputs(sizes, 2, 64, heads, P, ref_dim, seed=72)
    args = (c["value16"], c["proj"], c["aw_col0"], c["ref"], sizes, heads, P)
    assert not torch.equal(do.msda_reference(*args).half(), do.msda_reference(*args, mut=(mut,)).half())
    c = do.msda_realistic_inputs(sizes, 2, 64, heads, P, ref_dim, seed=73)
    args = (c["value16"], c["proj"], c["aw_col0"], c["ref"], sizes, heads, P)
    ref, bound = do.msda_reference(*args, bound=True)
    assert ((do.msda_reference(*args, mut=(mut,)) - ref).abs() > bound).any()


@pytest.mark.parametrize("ref_dim", [2, 4])
def test_msda_bound_covers_fp16_output(ref_dim):
    """The reference rounded to fp16 is inside the bound (its first term is that rounding); a 1 % error in the values of part
    of one level is not."""
    sizes, P, heads = [(20, 28), (10, 14), (5, 7), (3, 4)], 4, 8
    c = do.msda_realistic_inputs(sizes, 2, 300, heads, P, ref_dim, seed=74)
    args = (c["value16"], c["proj"], c["aw_col0"], c["ref"], sizes, heads, P)
    ref, bound = do.msda_reference(*args, bound=True)
    assert ((ref.half().double() - ref).abs() / bound).max() <= 1
    v = c["value16"].double()
    v[:, 560:700] *= 1.01
    assert ((do.msda_reference(v, *args[1:]) - ref).abs() > bound).any()
