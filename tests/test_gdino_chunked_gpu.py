"""Chunked many-category evaluation of MQ-GroundingDINO-T (LVIS: 1203 classes as 31 prompts of 40): the per-element stable-softmax
maximum (segmented ``global_max``, per-element shifts of ``softmax_rows_shifted`` / ``shift_clamp_``), the per-element class
tables of ``gdino_detections`` and ``GroundingDINO.forward_chunked(_device)`` against one ``forward_device`` per (image, chunk),
which is what the reference runs (engine/inference.py:600-660)."""
import pytest
import torch

from util import FP16_TOL, assert_close, load_sd

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# device ops
# ---------------------------------------------------------------------------------------------------------------------
def test_segment_max(dev):
    """out[s] = max of segment s, exactly, with -inf entries, a segment that is all -inf, and segment lengths off the float4 width;
    one segment is the existing op."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(41)
    for S, L in ((1, 1024 * 1024 + 3), (2, 4 * 256 * 300), (3, 1001), (8, 22223 * 4), (5, 7)):
        x = torch.randn(S, L, generator=g) * 1000
        x[:, ::7] = float("-inf")
        if S > 2:
            x[1] = float("-inf")
        xd = x.to(dev).contiguous()
        got = ops.global_max(xd, segments=S).cpu()
        assert torch.equal(got, x.max(1)[0]), (S, L)
        if S == 1:
            assert torch.equal(got, ops.global_max(xd).cpu())
    with pytest.raises(ValueError):
        ops.global_max(torch.zeros(10, device=dev), segments=3)


def _scores(g, B, R, n, scale0, lo):
    """[B, R, n] scores: element 0 scaled so that (x - its max) falls below ``lo`` (clamp active), element 1 not."""
    x = torch.randn(B, R, n, generator=g) * 3.0
    x[0] *= scale0
    shift = x.view(B, -1).max(1)[0]
    assert ((x[0] - shift[0]) < lo).any() and not ((x[1:] - shift[1:].view(-1, 1, 1)) < lo).any()
    return x, shift


@pytest.mark.parametrize("n", [256, 5003, 120])
def test_softmax_rows_shifted_per_element(dev, n):
    """Per-element shifts (shift[row // rows_per_shift]) at the warp-per-row length 256, the CTA-per-row length >= 4096 and a length
    that falls back to ``shift_clamp_`` + ``softmax_rows``, against the unfused formula, with the clamp active in element 0 only."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(42 + n)
    B, R, lo, hi = 2, 96, -60.0, 60.0
    x, shift = _scores(g, B, R, n, 40.0, lo)
    keep = (torch.rand(B, n, generator=g) > 0.2).float()
    ref = ((x - shift.view(B, 1, 1)).clamp(lo, hi) + torch.where(keep == 0, float("-inf"), 0.0)[:, None, :]).softmax(-1)
    out = ops.softmax_rows_shifted(x.to(dev).contiguous(), shift.to(dev), lo, hi, colmask=keep.to(dev).contiguous(), rows_per_batch=R,
                                   mask_value=float("-inf"), rows_per_shift=R).cpu()
    assert_close(out, ref, FP16_TOL, f"softmax_rows_shifted per element n={n}")
    # the batch-wide shift is a different result wherever the clamp engages
    one = ops.softmax_rows_shifted(x.to(dev).contiguous(), shift.max().view(1).to(dev), lo, hi, colmask=keep.to(dev).contiguous(),
                                   rows_per_batch=R, mask_value=float("-inf")).cpu()
    assert (one[1].float() - ref[1]).abs().max() > 0.1
    y = x.to(dev).contiguous()
    ops.shift_clamp_(y, shift.to(dev), lo, hi, rows_per_shift=R)
    assert torch.equal(y.cpu(), (x - shift.view(B, 1, 1)).clamp(lo, hi))
    with pytest.raises(ValueError):
        ops.shift_clamp_(y, shift.to(dev), lo, hi, rows_per_shift=R - 1)


# ---------------------------------------------------------------------------------------------------------------------
# fusion layer
# ---------------------------------------------------------------------------------------------------------------------
def test_bi_attention_per_element_max(dev):
    """GroundingDINO's BiMultiHeadAttention at B = 2 with element 0 scaled so that its scores exceed the 5e4 clamp: with per-element
    maxima, element 1 equals its own B = 1 run; with the batch-wide maximum element 0's maximum shifts element 1's scores into the
    clamp, and element 1 is visibly different."""
    from mqdet_b200 import ops
    from mqdet_b200.modeling.groundingdino.fuse_modules import BiMultiHeadAttention
    torch.manual_seed(43)
    a = BiMultiHeadAttention(256, 256, 1024, 4).to(dev).eval()
    g = torch.Generator().manual_seed(44)
    B, N, T = 2, 1500, 256
    v, l = torch.randn(B, N, 256, generator=g), torch.randn(B, T, 256, generator=g)
    # scale element 0 so that its largest score is about 2e5 (scores grow with the square of the input scale)
    with torch.no_grad():
        H, d = a.num_heads, a.head_dim
        q = ((v[0] @ a.v_proj.weight.cpu().t() + a.v_proj.bias.cpu()) * a.scale).view(N, H, d).transpose(0, 1)
        k = (l[0] @ a.l_proj.weight.cpu().t() + a.l_proj.bias.cpu()).view(T, H, d).transpose(0, 1)
        s = float((q @ k.transpose(1, 2)).abs().max())
    f = (2e5 / s) ** 0.5
    v[0] *= f
    l[0] *= f
    keep_l = torch.ones(B, T)
    keep_l[:, 200:] = 0
    keep_v = torch.ones(B, N)
    keep_v[1, 1400:] = 0
    v16, l16 = ops.cast_f16(v.to(dev).contiguous()), ops.cast_f16(l.to(dev).contiguous())
    kl, kv = keep_l.to(dev).contiguous(), keep_v.to(dev).contiguous()
    dv, dl = a._attend(v16, l16, kl, mask_v=kv, per_element_max=True)
    dv1, dl1 = a._attend(v16[1:].contiguous(), l16[1:].contiguous(), kl[1:].contiguous(), mask_v=kv[1:].contiguous())
    e_v = assert_close(dv[1:], dv1, FP16_TOL, "per-element max: image side of element 1 vs its B=1 run")
    e_l = assert_close(dl[1:], dl1, FP16_TOL, "per-element max: text side of element 1 vs its B=1 run")
    dvb, dlb = a._attend(v16, l16, kl, mask_v=kv)
    ref_v, ref_l = dv1.float().abs().max().item(), dl1.float().abs().max().item()
    bad_v = (dvb[1:].float() - dv1.float()).abs().max().item()
    bad_l = (dlb[1:].float() - dl1.float()).abs().max().item()
    assert bad_v > 10 * (FP16_TOL * ref_v + FP16_TOL) or bad_l > 10 * (FP16_TOL * ref_l + FP16_TOL), (bad_v, bad_l, e_v, e_l)


# ---------------------------------------------------------------------------------------------------------------------
# detections with per-element class tables
# ---------------------------------------------------------------------------------------------------------------------
def _tables(pmaps, dev):
    """Per-element tables as forward_chunked_device builds them: columns = classes in ascending label order."""
    Cmax = max(len(pm) for pm in pmaps)
    mt = max(len(t) for pm in pmaps for t in pm.values())
    tok = torch.full((len(pmaps), Cmax, mt), -1, dtype=torch.int32)
    lab = torch.zeros((len(pmaps), Cmax), dtype=torch.int32)
    for e, pm in enumerate(pmaps):
        for j, c in enumerate(sorted(pm)):
            tok[e, j, :len(pm[c])] = torch.tensor(pm[c], dtype=torch.int32)
            lab[e, j] = c
    return tok.to(dev), lab.to(dev)


def test_gdino_detections_per_element_tables(dev):
    """Per-element token tables + label tables (chunks of different length, global labels) against the oracle element by element,
    with exact score ties resolved to the lowest label; shared tables given per element equal the shared-table output bitwise."""
    from mqdet_b200 import ops
    from oracle import restate
    g = torch.Generator().manual_seed(45)
    B, nq, T, C = 3, 300, 256, 40
    logits = torch.randn(B, nq, T, generator=g) * 2.0 - 1.0
    logits[:, :, 120:] = float("-inf")
    boxes = torch.rand(B, nq, 4, generator=g) * 0.6 + 0.2
    sizes = [(480, 640), (400, 600), (512, 512)]
    wh = torch.tensor([[w, h] for h, w in sizes], dtype=torch.float32)
    # element e holds chunk e: labels 10e+1 .. 10e+k (k = 10, 10, 7), inserted in DESCENDING label order
    pmaps = []
    for e, k in enumerate((10, 10, 7)):
        pm, pos = {}, 1
        for c in range(10 * e + 1, 10 * e + k + 1):
            n = 2 + (c % 2)
            pm[c] = list(range(pos, pos + n))
            pos += n + 1
        pmaps.append(dict(sorted(pm.items(), reverse=True)))
    # exact ties: the second class of each chunk copies the token logits of the first (both two-token classes)
    for e, pm in enumerate(pmaps):
        c0, c1 = 10 * e + 2, 10 * e + 4
        logits[e][:, pm[c1]] = logits[e][:, pm[c0]]
        logits[e][:, pm[c0] + pm[c1]] += 4.0   # make the tied pair win often
    tok, lab = _tables(pmaps, dev)
    out = ops.gdino_detections(logits.to(dev), boxes.to(dev), tok, wh.to(dev), 0.05, class_labels=lab).cpu()
    ties = 0
    for e, pm in enumerate(pmaps):
        rb, rs, rl = restate.gdino_detections(logits[e:e + 1], boxes[e:e + 1], pm, C, sizes[e:e + 1], 0.05)[0]
        k = int(out[e, nq, 0])
        assert k == rb.shape[0] and k > 50
        assert torch.equal(out[e, :k, 5].long(), rl), e
        assert_close(out[e, :k, :4], rb, 1e-5, f"per-element tables: boxes of element {e}")
        assert_close(out[e, :k, 4], rs, 1e-5, f"per-element tables: scores of element {e}")
        ties += int((rl == 10 * e + 2).sum())
    assert ties > 10
    # one shared table, given once per element with labels c + 1, is today's output bit for bit
    pm = {c: [1 + (c % 50) * 2, 2 + (c % 50) * 2] for c in range(1, C + 1)}
    shared = ops.make_tokmap(pm, C, dev)
    base = ops.gdino_detections(logits.to(dev), boxes.to(dev), shared, wh.to(dev), 0.05)
    per = ops.gdino_detections(logits.to(dev), boxes.to(dev), shared.expand(B, -1, -1).contiguous(), wh.to(dev), 0.05,
                               class_labels=torch.arange(1, C + 1, dtype=torch.int32, device=dev).expand(B, -1).contiguous())
    assert torch.equal(per, base)
    with pytest.raises(ValueError):
        ops.gdino_detections(logits.to(dev), boxes.to(dev), tok[:2].contiguous(), wh.to(dev), 0.05)


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
def _model(sd, el, dl, nq, dev, num_classes):
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO
    cfg = mq_groundingdino_t_cfg(**{"GROUNDINGDINO.enc_layers": el, "GROUNDINGDINO.dec_layers": dl, "GROUNDINGDINO.num_queries": nq,
                                    "MODEL.DYHEAD.NUM_CLASSES": num_classes})
    model = GroundingDINO(cfg)
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    return load_sd(model, full).to(dev).eval()


def test_forward_chunked_equals_per_chunk_forwards(dev):
    """2 + 2 layers, 100 queries, two images of different size, 27 classes in chunks of 10 (the last one shorter; token positions
    differ per chunk), K = 5: ``forward_chunked`` packs, image by image and chunk by chunk, exactly the rows of ``forward_device``
    on that image alone (B = 1, same padded geometry) with that chunk's prompt; 1, 2 or 3 chunks per pass give the same result;
    a ``chunk_ids`` subset is the matching slice; a second call builds no new chunk state."""
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    el, dl, nq = 2, 2, 100
    gen = synth.Gen(2041)
    sd = synth.gdino_sd(gen, el, dl, nq)
    chunks = synth.chunked_prompts(27, 10, 256, gen)
    bank = {}
    for _, _, pm in chunks:
        bank.update(synth.query_bank(pm, 5, gen))
    B, h, w = 2, 150, 203
    img = synth.rgb_images(gen, B, h, w)
    sizes = [(h, w), (h - 22, w - 37)]
    img[1, :, sizes[1][0]:, :] = 0
    img[1, :, :, sizes[1][1]:] = 0
    model = _model(sd, el, dl, nq, dev, 28)
    model.query_selector.set_query_bank(bank)
    il = ImageList(img.to(dev), sizes)
    caps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    pmaps = [pm for _, _, pm in chunks]
    out = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)
    pk = out["det_packed"]
    assert tuple(pk.shape) == (3, B, nq + 1, 6) and out["chunks"] == [0, 1, 2]
    total = 0
    for b in range(B):
        one = ImageList(img[b:b + 1].to(dev), sizes[b:b + 1])
        for c, (cap, pm) in enumerate(zip(caps, pmaps)):
            ref = model.forward_device(one, cap, pm)["det_packed"][0]
            n = int(ref[nq, 0])
            assert torch.equal(pk[c, b], ref), f"image {b}, chunk {c}: {int(pk[c, b, nq, 0])} vs {n} detections"
            assert set(ref[:n, 5].long().tolist()) <= set(pm)
            total += n
    assert total > 20
    for cpp in (1, 3):
        assert torch.equal(model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=cpp)["det_packed"], pk), cpp
    sub = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2, chunk_ids=[2, 0])
    assert sub["chunks"] == [2, 0] and torch.equal(sub["det_packed"], pk[[2, 0]])
    # public form: per image the chunks' detections concatenated in chunk order, global labels
    res = model.forward_chunked(il, caps, pmaps, chunks_per_pass=2)
    for b in range(B):
        rows = torch.cat([pk[c, b, :int(pk[c, b, nq, 0])] for c in range(3)]).cpu()
        assert len(res[b]) == rows.shape[0] and res[b].mode == "xyxy"
        assert torch.equal(res[b].bbox, rows[:, :4]) and torch.equal(res[b].get_field("labels"), rows[:, 5].long())
    # a second call reuses every chunk state
    calls = []
    tok = model._tokenize
    model._tokenize = lambda c: (calls.append(1), tok(c))[1]
    n_state = len(model._chunk_cache)
    model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)
    assert not calls and len(model._chunk_cache) == n_state
    model.train()
    with pytest.raises(NotImplementedError):
        model.forward_chunked_device(il, caps, pmaps)


def test_forward_chunked_full_depth(dev):
    """6 + 6 layers, 900 queries, 800x1333, B = 1, eight of the 31 LVIS-shaped chunks (1203 classes in chunks of 40) at four chunks
    per pass: finite outputs with labels of the evaluated chunks, within memory."""
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    gen = synth.Gen(2042)
    sd = synth.gdino_sd(gen, 6, 6, 900)
    chunks = synth.chunked_prompts(1203, 40, 256, gen)
    assert len(chunks) == 31
    ids = [0, 3, 7, 12, 18, 22, 29, 30]
    bank = {}
    for c in ids:
        bank.update(synth.query_bank(chunks[c][2], 5, gen))
    h, w = 800, 1333
    img = synth.rgb_images(gen, 1, h, w)
    model = _model(sd, 6, 6, 900, dev, 1204)
    model.query_selector.set_query_bank(bank)
    caps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    pmaps = [pm for _, _, pm in chunks]
    torch.cuda.reset_peak_memory_stats(dev)
    out = model.forward_chunked_device(ImageList(img.to(dev), [(h, w)]), caps, pmaps, chunks_per_pass=4, chunk_ids=ids)
    pk = out["det_packed"].cpu()
    assert tuple(pk.shape) == (8, 1, 901, 6) and torch.isfinite(pk).all()
    for j, c in enumerate(ids):
        n = int(pk[j, 0, 900, 0])
        assert set(pk[j, 0, :n, 5].long().tolist()) <= set(pmaps[c])
    assert torch.cuda.max_memory_allocated(dev) < 70 * 2 ** 30
