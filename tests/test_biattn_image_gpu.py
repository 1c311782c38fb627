"""ops.biattn_image (the fused image -> text side of the BiAttention fusion) against a float64 torch restatement on the same fp16
operands: the output v' = res + gamma * (sum_h softmax_t(clamp(vn gT_h^T + gbias_h) + mask) mT_h^T + bias) and the column
maxima of the clamped scores.  Covers the benchmark shape, ragged image-token counts, text lengths on both sides of the split of
the T tokens between the kernel's two MMA warpgroups, 1 / 3 / 8 heads, padded and fully masked prompts, an active +-5e4 clamp,
each optional operand present or absent, and bit-identical reruns and CUDA-graph replays."""
import pytest
import torch

from util import assert_close

pytestmark = pytest.mark.gpu

CLAMP = 5.0e4


def make_case(dev, B, N, T, H, seed, mask="pad", gbias=True, gamma=True, res=True, clamp_active=False):
    g = torch.Generator().manual_seed(seed)

    def rnd(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    if clamp_active:
        # small integers: every score is an exact fp32 sum (|S| < 2^24), most rows reach the clamp, many tie at it
        vn = torch.randint(-100, 101, (B, N, 256), generator=g).half()
        gT = torch.randint(-100, 101, (B, H, T, 256), generator=g).half()
        gb = torch.randint(-2000, 2001, (B, H, T, 8), generator=g).float()
    else:
        vn = rnd(B, N, 256).half()
        gT = rnd(B, H, T, 256, std=0.2).half()
        gb = rnd(B, H, T, 8)
    mT = rnd(B, H, 256, T, std=0.25).half()
    m = None
    if mask != "none":
        m = torch.ones(B, T)
        m[0, max(1, T // 3):] = 0  # padded tokens
        if mask == "allmasked":
            m[B - 1] = 0  # an image whose prompt tokens are all masked
    c = dict(vn16=vn, gT=gT, gbias=gb if gbias else None, mT=mT, bias=rnd(256, std=0.1), gamma=0.5 + torch.rand(256, generator=g)
             if gamma else None, residual=rnd(B, N, 256).half() if res else None, mask=m, clamp=CLAMP, heads=H)
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in c.items()}


def restate(vn16, gT, gbias, mT, bias, gamma, residual, mask, clamp, heads):
    B, N, _ = vn16.shape
    T = gT.shape[2]
    dev = vn16.device
    lim = clamp if clamp > 0 else float("inf")
    out = torch.empty(B, N, 256, dtype=torch.float64, device=dev)
    colmax = torch.empty(B, heads, T, dtype=torch.float64, device=dev)
    for b in range(B):
        kept = torch.ones(T, dtype=torch.bool, device=dev) if mask is None else mask[b] != 0
        acc = torch.zeros(N, 256, dtype=torch.float64, device=dev)
        for h in range(heads):
            s = vn16[b].double() @ gT[b, h].double().t()
            gb = gbias[b, h, :, 0].double() if gbias is not None else torch.zeros(T, dtype=torch.float64, device=dev)
            colmax[b, h] = (s.max(0).values + gb).clamp(-lim, lim)  # over every image token, no mask
            a = (s + gb).clamp(-lim, lim)
            if kept.any():
                p = torch.softmax(a.masked_fill(~kept, float("-inf")), dim=1)
            else:  # the reference's fp32 A + (-9e15) swallows A: uniform over the T tokens
                p = torch.full_like(a, 1.0 / T)
            acc += p @ mT[b, h].double().t()
        o = acc + bias.double()
        if gamma is not None:
            o = o * gamma.double()
        if residual is not None:
            o = o + residual[b].double()
        out[b] = o
    return out, colmax.view(B * heads, T)


def check(case, what, colmax_tol=1e-5):
    from mqdet_b200 import ops
    out, colmax = ops.biattn_image(**case)
    ref_out, ref_cm = restate(**case)
    assert_close(out, ref_out, 1e-3, f"biattn_image output {what}")
    assert_close(colmax, ref_cm, colmax_tol, f"biattn_image colmax {what}")
    return out, colmax


def test_bench_shape(dev):
    """B = 8, N = 22400, T = 256, H = 8: the shape of every fusion layer in the benchmark."""
    check(make_case(dev, 8, 22400, 256, 8, seed=1), "bench shape")


@pytest.mark.parametrize("N", [37, 64, 333, 1000])
def test_ragged_image_tokens(dev, N):
    check(make_case(dev, 2, N, 256, 8, seed=N), f"N={N}")


@pytest.mark.parametrize("T", [8, 120, 128, 136, 256])
def test_text_lengths(dev, T):
    """T <= 128 leaves the second half of the text tokens, whose scores the second MMA warpgroup computes, fully masked."""
    check(make_case(dev, 2, 200, T, 3, seed=T), f"T={T}")


@pytest.mark.parametrize("H", [1, 3, 8])
def test_heads(dev, H):
    check(make_case(dev, 2, 150, 256, H, seed=10 + H), f"H={H}")


@pytest.mark.parametrize("mask", ["none", "pad", "allmasked"])
@pytest.mark.parametrize("T", [120, 256])
def test_masks(dev, mask, T):
    check(make_case(dev, 3, 130, T, 3, seed=20 + T, mask=mask), f"mask={mask} T={T}")


@pytest.mark.parametrize("T", [64, 256])
def test_active_clamp(dev, T):
    """Scores far beyond +-5e4: the clamp decides the row maxima, ties at the clamp share the row's probability, and the column
    maxima are exact (integer operands make every score an exact fp32 sum in any order)."""
    case = make_case(dev, 2, 190, T, 3, seed=30 + T, clamp_active=True, mask="pad")
    _, colmax = check(case, f"active clamp T={T}", colmax_tol=0.0)
    assert (colmax.abs() == CLAMP).float().mean().item() > 0.2


@pytest.mark.parametrize("gbias,gamma,res", [(False, False, False), (True, False, False), (False, True, False),
                                             (False, False, True), (True, True, True)])
def test_optional_operands(dev, gbias, gamma, res):
    check(make_case(dev, 2, 100, 136, 2, seed=40, gbias=gbias, gamma=gamma, res=res), f"gbias={gbias} gamma={gamma} res={res}")


def test_reruns_and_graph_replay_bit_identical(dev):
    """No float atomics: two launches, and a CUDA-graph replay, give the same bits as an eager launch."""
    from mqdet_b200 import ops
    case = make_case(dev, 4, 3000, 256, 8, seed=50, mask="allmasked")
    a_out, a_cm = ops.biattn_image(**case)
    b_out, b_cm = ops.biattn_image(**case)
    torch.cuda.synchronize()
    assert torch.equal(a_out, b_out) and torch.equal(a_cm, b_cm)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.biattn_image(**case)  # warm-up on a side stream before capture
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        g_out, g_cm = ops.biattn_image(**case)
    for _ in range(2):
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(g_out, a_out) and torch.equal(g_cm, a_cm)
