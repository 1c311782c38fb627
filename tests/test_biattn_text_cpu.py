"""The float64 references of tests/test_biattn_text_gpu.py, checked without a GPU: the attention restated from the layer-normed
inputs reproduces ``oracle.restate.bi_attention`` (pinned to the reference by the golden tests), the product path's folded
text side equals the unfolded q . k^T form with and without an active clamp, and the seeded inputs have the properties each
pattern of tests/biattn_text_oracle.py is built for."""
import pytest
import torch

import biattn_text_oracle as bo
from oracle import restate, synth


def _weights(sd):
    return {k[len("attn."):]: v for k, v in sd.items() if k.startswith("attn.")}


def _sd(seed):
    return {k: v.double() for k, v in synth.bi_attention_sd(synth.Gen(seed)).items()}


def test_attention_restate_matches_restate_bi_attention():
    """ln + gamma_l * dl and vn + gamma_v * dv from the layer-normed inputs == restate.bi_attention's two streams."""
    sd = _sd(60)
    gen = synth.Gen(61)
    B, N, T = 2, 150, 40
    v, l = gen.randn(B, N, 256).double(), gen.randn(B, T, 768).double()
    mask = torch.ones(B, T, dtype=torch.long)
    mask[0, 13:] = 0
    v_ref, l_ref = restate.bi_attention(v, l, mask, sd)
    vn, ln = restate._ln(v, sd, "layer_norm_v"), restate._ln(l, sd, "layer_norm_l")
    dv, dl = bo.attention_restate(vn, ln, _weights(sd), 8, bo.CLAMP, mask)
    for got, ref in ((ln + sd["gamma_l"] * dl, l_ref), (vn + sd["gamma_v"] * dv, v_ref)):
        err = (got - ref).abs().max().item()
        assert err <= 1e-12 * ref.abs().max().item(), err


@pytest.mark.parametrize("clamp_active", [False, True])
def test_folded_text_side_equals_unfolded(clamp_active):
    """gT / gbias, the softmax on the image tokens themselves and the value projection after the reduction == the unfolded
    softmax_n(clamp(q k^T)) (vn Wvv^T + bvv).  With the key projection scaled up, over 20 % of the scores sit at the clamp."""
    sd = _sd(62)
    w = _weights(sd)
    gen = synth.Gen(63)
    B, N, T = 2, 130, 24
    vn = (gen.randn(B, N, 256) + 2 * gen.randn(1, 1, 256)).double()
    ln = gen.randn(B, T, 768).double()
    if clamp_active:
        w["l_proj.weight"] = w["l_proj.weight"] * 3e5
        w["l_proj.bias"] = w["l_proj.bias"] * 3e5
        E, d = 2048, 256
        q = (bo._proj(w, "v_proj", vn) * d ** -0.5).view(B, N, 8, d)
        k = bo._proj(w, "l_proj", ln).view(B, T, 8, d)
        frac = (torch.einsum("bnhd,bthd->bhnt", q, k).abs() >= bo.CLAMP).double().mean().item()
        assert frac > 0.2, frac
    _, dl = bo.attention_restate(vn, ln, w, 8, bo.CLAMP)
    got = bo.text_folded(vn, ln, w, 8, bo.CLAMP)
    err = (got - dl).abs().max().item()
    assert err <= 1e-9 * dl.abs().max().item(), err


def _colmax64(c):
    """[B, H, T] float64 max over n of the clamped scores."""
    B, H, T, _ = c["kh"].shape
    return torch.stack([torch.stack([bo.scores(c["kh"], c["qh"], c["rowbias"], c["clamp"], b, h).max(1).values
                                     for h in range(H)]) for b in range(B)])


@pytest.mark.parametrize("B,H,T,N,q", [(2, 3, 256, 1000, "broadcast"), (2, 3, 65, 129, "distinct"), (2, 8, 256, 333, "broadcast")])
def test_spread_separates_rows_and_heads(B, H, T, N, q):
    """colmax of rows t and t + 8 (one thread's two rows), and of neighbouring heads and images, lie more than 100 apart."""
    cm = _colmax64(bo.make_inputs("spread", B, H, T, N, seed=1, q=q))
    t = torch.arange(T)
    lo = t[(t % 16 < 8) & (t + 8 < T)]
    assert (cm[:, :, lo] - cm[:, :, lo + 8]).abs().min().item() > 100
    assert (cm[:, 1:] - cm[:, :-1]).abs().min().item() > 100
    assert (cm[1:] - cm[:-1]).abs().min().item() > 100


@pytest.mark.parametrize("q", ["broadcast", "distinct"])
@pytest.mark.parametrize("N", [1, 63, 65, 1000])
def test_tail_tokens_have_only_negative_scores(N, q):
    """On the tail-dominant tokens every real score is below rowbias = 0, the score of a zero-filled image token."""
    c = bo.make_inputs("tail", 2, 3, 256, N, seed=2, q=q)
    tail = torch.arange(256) % bo.TAIL_EVERY == 0
    assert (c["rowbias"][:, :, tail, 0] == 0).all()
    assert _colmax64(c)[:, :, tail].max().item() < 0


def test_clamp_pattern_reaches_the_clamp():
    c = bo.make_inputs("clamp", 2, 3, 256, 333, seed=3)
    B, H = 2, 3
    a = torch.stack([bo.scores(c["kh"], c["qh"], c["rowbias"], 0.0, b, h) for b in range(B) for h in range(H)])
    assert (a.abs() >= bo.CLAMP).double().mean().item() > 0.2
    assert a.abs().max().item() < 2 ** 24   # every score an exact fp32 sum
    # clamp(S) + rowbias would exceed the row's maximum by thousands of nats somewhere
    s = torch.stack([bo.scores(c["kh"], c["qh"], None, bo.CLAMP, b, h) for b in range(B) for h in range(H)])
    rb = c["rowbias"][..., 0].reshape(B * H, -1, 1).double()
    assert ((s + rb) - a.clamp(-bo.CLAMP, bo.CLAMP)).max().item() > 1000


def test_peaked_pattern_is_subnormal():
    """At N = 22400 at least 99 % of the non-dominant unnormalised P lie below 2^-14, the smallest normal fp16."""
    B, H, N = 2, 2, 22400
    c = bo.make_inputs("peaked", B, H, 256, N, seed=4)
    cm = _colmax64(c)
    for b in range(B):
        for h in range(H):
            e = torch.exp(bo.scores(c["kh"], c["qh"], c["rowbias"], c["clamp"], b, h) - cm[b, h][:, None])
            top = e.max(1).values
            assert (top == 1).all()
            rest = e.sort(1, descending=True).values[:, 1:]
            assert (rest < 2.0 ** -14).double().mean().item() >= 0.99
            assert (rest.max(1).values < 2.0 ** -14).double().mean().item() > 0.5


def test_restate_text_is_the_softmax():
    """restate_text's u equals torch.softmax over the clamped scores times vn, and its colsum counts the shift by colmax."""
    c = bo.make_inputs("diffuse", 2, 2, 40, 77, seed=5, q="distinct")
    cm = bo.colmax_of(c["kh"], c["qh"], c["rowbias"], c["clamp"])
    u, bound, colsum = bo.restate_text(c["kh"], c["qh"], c["vn16"], cm, c["rowbias"], c["clamp"])
    for b in range(2):
        for h in range(2):
            a = bo.scores(c["kh"], c["qh"], c["rowbias"], c["clamp"], b, h)
            assert torch.allclose(u[b, h], torch.softmax(a, 1) @ c["vn16"][b].double(), rtol=1e-12, atol=1e-12)
            assert torch.allclose(colsum[b, h], torch.exp(a - cm[b * 2 + h].double()[:, None]).sum(1), rtol=1e-12)
    assert (bound > 0).all() and (colsum >= 1 - 1e-6).all()
