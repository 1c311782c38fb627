"""dcn_conv_kernel (``ops.dcn_conv``) and dcn_cols_kernel (``ops.dcn_cols``) against the float64 restatement of
tests/deform_oracle.py.  On exact inputs (samples placed exactly on every edge of every branch, masks of 0, 1/2 and 1) each
output must equal the reference rounded once to fp16: dcn_conv's y == y64.half() and dcn_cols' columns == col64.half(), on
every row.  Realistic inputs are held to the per-element bound of deform_oracle.dcn_bound.  Shapes: ragged pyramids, single
levels, levels one pixel high or wide, every job list, om_ld 27 and 32, bias absent, no offsets at all (checked against
F.conv2d), and the benchmark's B = 8 pyramid, where each CTA walks about 32 tiles across all three jobs."""
import pytest
import torch
import torch.nn.functional as F

import deform_oracle as do

pytestmark = pytest.mark.gpu

BENCH = [(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)]
RAGGED = [(13, 17), (7, 9), (4, 5), (2, 3), (1, 1)]
SMALL = [(9, 11), (5, 6), (3, 3)]


def _run(c, sizes, jobs, no_bias=False):
    from mqdet_b200 import ops
    lv = ops.Levels(sizes, c["x16"].device)
    biases = [None] * len(jobs) if no_bias else c["biases"][:len(jobs)]
    return ops.dcn_conv(c["x16"], c["om"], lv, jobs, c["weights"][:len(jobs)], biases), biases


def _check_exact(c, sizes, jobs, no_bias=False, cols_too=True):
    from mqdet_b200 import ops
    ys, biases = _run(c, sizes, jobs, no_bias)
    x16, om = c["x16"], c["om"]
    B = x16.shape[0]
    lv = ops.Levels(sizes, x16.device)
    for j, (k, y) in enumerate(zip(jobs, ys)):
        rows = do.rows_per_image(sizes, k)
        assert y.shape == (B * rows, 256)
        y = y.view(B, rows, 256)
        gc = ops.dcn_cols(x16, om, lv, k).view(B, rows, -1) if cols_too else None
        for b in range(B):
            cols = do.dcn_image(x16, om, sizes, k, b)
            if gc is not None:
                bad = (gc[b] != cols.half()).any(1).nonzero()
                assert bad.numel() == 0, f"dcn_cols branch {k} image {b}: {bad.numel()} rows differ, first {bad[:4].view(-1).tolist()}"
            want = do.dcn_y(cols, c["weights"][j], biases[j]).half()
            bad = (y[b] != want).any(1).nonzero()
            assert bad.numel() == 0, f"dcn_conv job {j} (branch {k}) image {b}: {bad.numel()} rows differ, first {bad[:4].view(-1).tolist()}"


def _check_bound(c, sizes, jobs):
    ys, biases = _run(c, sizes, jobs)
    B = c["x16"].shape[0]
    worst = 0.0
    for j, (k, y) in enumerate(zip(jobs, ys)):
        y = y.view(B, -1, 256).double()
        for b in range(B):
            cols = do.dcn_image(c["x16"], c["om"], sizes, k, b)
            y64 = do.dcn_y(cols, c["weights"][j], biases[j])
            ratio = ((y[b] - y64).abs() / do.dcn_bound(cols, y64, c["weights"][j])).max().item()
            assert ratio <= 1, f"branch {k} image {b}: max |err| / bound = {ratio:.3f}"
            worst = max(worst, ratio)
    print(f"max err/bound {worst:.3f}")


@pytest.mark.parametrize("sizes,B,jobs,om_ld,no_bias", [
    (RAGGED, 3, [1, 2, 0], 32, False),          # ragged last tiles, tiles across levels and images
    (RAGGED, 3, [2], 27, True),
    (SMALL, 1, [1, 2, 0], 27, True),            # B = 1, every job shorter than two tiles
    (SMALL, 2, [2, 0], 32, False),
    ([(16, 24)], 1, [1], 32, False),            # one level: exactly six 64-row tiles
    ([(1, 1)], 2, [1], 27, False),              # one pixel: every tap but the centre outside
    ([(1, 9), (1, 5), (1, 3)], 2, [1, 2, 0], 32, True),     # one pixel high
    ([(8, 1), (4, 1), (2, 1), (1, 1)], 2, [0], 27, False),   # one pixel wide
])
def test_exact_pyramids(dev, sizes, B, jobs, om_ld, no_bias):
    c = do.dcn_exact_inputs(sizes, B, seed=100 + B + len(jobs), om_ld=om_ld, device=dev)
    _check_exact(c, sizes, jobs, no_bias)


@pytest.mark.parametrize("sizes,B", [(RAGGED, 3), (SMALL, 1), ([(1, 9), (1, 5), (1, 3)], 2)])
def test_no_offsets_is_a_plain_convolution(dev, sizes, B):
    """om = None: each branch is a 3x3, pad 1 convolution (stride 2 for branch 2), equal to F.conv2d in float64 rounded to
    fp16, on exact inputs."""
    c = do.dcn_exact_inputs(sizes, B, seed=150, device=dev)
    c["om"] = None
    jobs = [1, 2, 0]
    ys, biases = _run(c, sizes, jobs)
    off = do.level_offsets(sizes)
    for j, (k, y) in enumerate(zip(jobs, ys)):
        y = y.view(B, -1, 256)
        w4 = c["weights"][j].double().view(256, 9, 256).permute(0, 2, 1).reshape(256, 256, 3, 3)
        o = 0
        for lo, li, Ho, Wo, stride in do.branch_levels(sizes, k):
            Hi, Wi = sizes[li]
            x = c["x16"][:, off[li]:off[li] + Hi * Wi].double().transpose(1, 2).reshape(B, 256, Hi, Wi)
            want = F.conv2d(x, w4, biases[j].double(), stride=stride, padding=1)[:, :, :Ho, :Wo]
            got = y[:, o:o + Ho * Wo].transpose(1, 2).reshape(B, 256, Ho, Wo)
            assert torch.equal(got, want.half()), f"branch {k} level {lo}"
            o += Ho * Wo


def test_bench_shape_exact(dev):
    """B = 8, levels 100x168 ... 7x11, jobs [1, 2, 0]: 4200 tiles, so every CTA carries its ring phases, its weight prefetch
    and its bias across about 32 tiles and both job boundaries.  Every row of all three outputs, and of dcn_cols, bit for
    bit."""
    c = do.dcn_exact_inputs(BENCH, 8, seed=200, device=dev)
    _check_exact(c, BENCH, [1, 2, 0])


def test_bench_shape_realistic(dev):
    """The benchmark shape on realistic inputs, every element within the bound."""
    c = do.dcn_realistic_inputs(BENCH, 8, seed=201, device=dev)
    _check_bound(c, BENCH, [1, 2, 0])


@pytest.mark.parametrize("sizes,B,jobs", [(RAGGED, 3, [1, 2, 0]), (SMALL, 1, [1, 2, 0]), ([(16, 24)], 1, [1]),
                                          (RAGGED, 3, [0])])
def test_realistic_pyramids(dev, sizes, B, jobs):
    c = do.dcn_realistic_inputs(sizes, B, seed=300 + B, device=dev)
    _check_bound(c, sizes, jobs)
