"""``ops.ms_deform_attn`` (ms_deform_attn_v2_kernel and the lane-per-channel ms_deform_attn_kernel) against the float64
restatement of tests/deform_oracle.py, called directly rather than through the module's projections.  On exact inputs (samples
exactly at -1, -0.5, 0, S-1, S-0.5 and S on both axes of every level, softmax weights 1, 1/2 or 1/4) the fp32 output must
equal the reference and the fp16 output its one rounding.  Covered: both kernels (L*P a multiple of 8 or not, and a value
tensor that is not 16-byte aligned), 1 and 8 heads, B = 1 and 2, Q = 1, 7 and 901 (the last CTA with idle warps), 2-d
reference points and 4-d boxes, and the GroundingDINO-T encoder and decoder shapes on realistic inputs against the per-element
bound of deform_oracle.msda_reference."""
import pytest
import torch

import deform_oracle as do

pytestmark = pytest.mark.gpu

# power-of-two level sizes, with levels one pixel high or wide
SIZES = {1: [(8, 16)], 2: [(16, 8), (4, 4)], 3: [(8, 16), (4, 8), (1, 2)], 4: [(16, 32), (8, 16), (4, 8), (2, 4)],
         5: [(8, 8), (4, 4), (2, 2), (1, 1), (2, 1)]}
GDINO = [(100, 168), (50, 84), (25, 42), (13, 21)]


def _run(c, sizes, heads, P, out_dtype, value16=None):
    from mqdet_b200 import ops
    lv = ops.Levels(sizes, c["proj"].device)
    v = c["value16"] if value16 is None else value16
    return ops.ms_deform_attn(v, c["proj"], c["aw_col0"], c["ref"], lv, heads, P, out_dtype=out_dtype)


def _check_exact(c, sizes, heads, P, out_dtype, value16=None):
    out = _run(c, sizes, heads, P, out_dtype, value16)
    want = do.msda_reference(c["value16"], c["proj"], c["aw_col0"], c["ref"], sizes, heads, P)
    want = want.float() if out_dtype == torch.float32 else want.half()
    assert out.dtype == out_dtype and out.shape == want.shape
    bad = (out != want).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} elements differ, first (b, q, channel) {bad[:4].tolist()}"


def _case(dev, L, P, B, Q, heads, ref_dim, seed):
    return do.msda_exact_inputs(SIZES[L], B, Q, heads, P, ref_dim, seed=seed, device=dev)


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("ref_dim", [2, 4])
@pytest.mark.parametrize("L,P", [(2, 4), (4, 4), (3, 8), (4, 8)])
def test_fast_kernel_exact(dev, L, P, ref_dim, out_dtype):
    """L*P = 8, 16, 24, 32: the 8-group x 4-quad kernel."""
    c = _case(dev, L, P, 2, 901, 8, ref_dim, seed=10 * L + P)
    _check_exact(c, SIZES[L], 8, P, out_dtype)


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("ref_dim", [2, 4])
@pytest.mark.parametrize("L,P", [(1, 1), (1, 3), (3, 4), (5, 3)])
def test_lane_kernel_exact(dev, L, P, ref_dim, out_dtype):
    """L*P = 1, 3, 12, 15: one lane per channel."""
    c = _case(dev, L, P, 2, 901, 8, ref_dim, seed=100 + 10 * L + P)
    _check_exact(c, SIZES[L], 8, P, out_dtype)


@pytest.mark.parametrize("ref_dim", [2, 4])
def test_misaligned_value_takes_lane_kernel(dev, ref_dim):
    """L*P = 16 with value a contiguous view 2 bytes past a 16-byte boundary: the lane-per-channel fallback."""
    c = _case(dev, 4, 4, 2, 901, 8, ref_dim, seed=200)
    v = c["value16"]
    buf = torch.empty(v.numel() + 8, dtype=torch.float16, device=dev)
    vm = buf[1:1 + v.numel()].view(v.shape)
    vm.copy_(v)
    assert vm.is_contiguous() and vm.data_ptr() % 16 == 2
    _check_exact(c, SIZES[4], 8, 4, torch.float16, value16=vm)
    _check_exact(c, SIZES[4], 8, 4, torch.float32, value16=vm)


@pytest.mark.parametrize("ref_dim", [2, 4])
@pytest.mark.parametrize("heads,B,Q", [(1, 1, 1), (8, 1, 7), (1, 2, 901), (8, 2, 7), (1, 1, 7)])
@pytest.mark.parametrize("L,P", [(4, 4), (3, 4)])
def test_heads_batch_queries(dev, L, P, heads, B, Q, ref_dim):
    """Both kernels at 1 and 8 heads, B = 1 and 2, and query counts whose last CTA of 8 warps is partly idle."""
    c = _case(dev, L, P, B, Q, heads, ref_dim, seed=300 + heads + B + Q)
    _check_exact(c, SIZES[L], heads, P, torch.float16)
    _check_exact(c, SIZES[L], heads, P, torch.float32)


def _check_bound(c, sizes, heads, P):
    out = _run(c, sizes, heads, P, torch.float16).double()
    ref, bound = do.msda_reference(c["value16"], c["proj"], c["aw_col0"], c["ref"], sizes, heads, P, bound=True)
    assert torch.isfinite(out).all()
    ratio = ((out - ref).abs() / bound).max().item()
    print(f"max err/bound {ratio:.3f}")
    assert ratio <= 1, f"max |err| / bound = {ratio:.3f}"


def test_gdino_encoder_shape(dev):
    """GroundingDINO-T encoder: B = 2, every one of the 22323 pyramid positions a query, 2-d reference points."""
    c = do.msda_realistic_inputs(GDINO, 2, sum(h * w for h, w in GDINO), 8, 4, 2, seed=400, device=dev)
    _check_bound(c, GDINO, 8, 4)


def test_gdino_decoder_shape(dev):
    """GroundingDINO-T decoder: 900 queries with 4-d reference boxes."""
    c = do.msda_realistic_inputs(GDINO, 2, 900, 8, 4, 4, seed=401, device=dev)
    _check_bound(c, GDINO, 8, 4)
