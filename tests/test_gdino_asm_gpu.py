"""GPU parity of the GroundingDINO encoder / decoder assembly (SURVEY.md §8 f1, BASELINE config 4) through the C ABI against the CPU
oracle (oracle/restate.py, pinned to the reference's own Transformer / Swin / BERT loop / post-processing by
tests/test_gdino_pinning.py) and against the golden fixture recorded from the reference's own ``Transformer.forward``."""
import json
import os

import pytest
import torch

from util import FP16_TOL, ROOT, assert_close, load_sd

pytestmark = pytest.mark.gpu


def _record(name, payload):
    d = os.path.join(ROOT, "gpurun_out")
    if os.path.isdir(d):
        p = os.path.join(d, "gdino_parity.json")
        cur = json.load(open(p)) if os.path.exists(p) else {}
        cur[name] = payload
        json.dump(cur, open(p, "w"), indent=1)


# ---------------------------------------------------------------------------------------------------------------------
# the new device ops
# ---------------------------------------------------------------------------------------------------------------------
def test_add_cast(dev):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(1)
    a, b = torch.randn(3, 77, 256, generator=g), torch.randn(3, 77, 256, generator=g)
    gate = (torch.rand(3 * 77, generator=g) > 0.3).float()
    a[0, 5] = float("inf")
    gate[5] = 0.0
    o16, o32 = ops.add_cast(a.to(dev), b.to(dev), gate.to(dev), out16=True, out32=True)
    ref = (a + b) * gate.view(3, 77, 1)
    ref[0, 5] = 0.0
    assert torch.equal(o32.cpu(), ref)
    assert torch.equal(o16.cpu(), ref.half())
    o16 = ops.add_cast(a.to(dev)[1:], None, None)
    assert torch.equal(o16.cpu(), a[1:].half())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_groupnorm_rows(dev, dtype):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(2)
    B, H, W, C = 2, 37, 53, 256
    x = (torch.randn(B, H * W, C, generator=g) * 2.0 + 0.7).to(dtype)
    w, b = torch.randn(C, generator=g), torch.randn(C, generator=g)
    ref = torch.nn.functional.group_norm(x.float().transpose(1, 2).reshape(B, C, H, W), 32, w, b, 1e-5).flatten(2).transpose(1, 2)
    o16, o32 = ops.groupnorm_rows(x.to(dev), 32, w.to(dev), b.to(dev), 1e-5, out16=True, out32=True)
    assert_close(o32, ref, 2e-5, f"groupnorm_rows {dtype}")
    assert_close(o16, ref, FP16_TOL, f"groupnorm_rows {dtype} fp16 out")


def test_box_refine_sine(dev):
    from mqdet_b200 import ops
    from oracle import restate
    g = torch.Generator().manual_seed(3)
    B, nq, L = 2, 900, 4
    logit = torch.randn(B, nq, 4, generator=g) * 2
    logit[0, 0] = float("inf")   # an invalid anchor proposal selected by the two-stage top-k
    vr = torch.rand(B, L, 2, generator=g) * 0.5 + 0.5
    ref0 = logit.sigmoid()
    r, ri, s = ops.box_refine_sine(logit.to(dev), vr.to(dev), ref_is_logit=True)
    vr4 = torch.cat([vr, vr], -1)
    assert_close(r, ref0, 1e-6, "box_refine: sigmoid")
    assert_close(ri, ref0[:, :, None] * vr4[:, None], 1e-6, "box_refine: reference_points_input")
    assert_close(s, restate.sineembed_for_position((ref0[:, :, None] * vr4[:, None])[:, :, 0]), 2e-3, "box_refine: sine embedding")
    delta = torch.randn(B, nq, 4, generator=g) * 0.3
    ref1 = (delta + restate.inverse_sigmoid(ref0)).sigmoid()
    r1, ri1, s1 = ops.box_refine_sine(r, vr.to(dev), delta=delta.to(dev))
    assert_close(r1, ref1, 1e-5, "box_refine: refined")
    assert_close(s1, restate.sineembed_for_position((ref1[:, :, None] * vr4[:, None])[:, :, 0]), 2e-3, "box_refine: refined sine")
    r2, _, s2 = ops.box_refine_sine(r, vr.to(dev), delta=delta.to(dev), want_sine=False)
    assert s2 is None and torch.equal(r2, r1)


def test_gdino_detections_vs_oracle(dev):
    from mqdet_b200 import ops
    from oracle import restate, synth
    gen = synth.Gen(75)
    B, nq, T, C = 2, 900, 256, 80
    _, am, pmap = synth.prompt(13, 2, T, gen)
    logits = gen.randn(B, nq, T, scale=2.0) - 2.0
    logits[:, :, am[0] == 0] = float("-inf")
    boxes = torch.rand(B, nq, 4, generator=gen.g)
    boxes[0, 3] = torch.tensor([0.99, 0.5, 0.3, 0.2])
    boxes[1, 5] = torch.tensor([0.1, 0.98, 0.05, 0.3])
    sizes = [(480, 640), (400, 600)]
    ref = restate.gdino_detections(logits, boxes, pmap, C, sizes, 0.05)
    wh = torch.tensor([[w, h] for h, w in sizes], dtype=torch.float32)
    out = ops.gdino_detections(logits.to(dev), boxes.to(dev), ops.make_tokmap(pmap, C, dev), wh.to(dev), 0.05).cpu()
    for b, (rb, rs, rl) in enumerate(ref):
        k = int(out[b, nq, 0])
        assert k == rb.shape[0] and k > 100
        assert torch.equal(out[b, :k, 5].long(), rl)                      # labels and the kept set: index work, exact
        assert (out[b, :k, 4] - rs).abs().max() <= 2e-6
        assert (out[b, :k, :4] - rb).abs().max() <= 1e-3
        assert (out[b, k:nq] == 0).all()


def test_multihead_attention_vs_oracle(dev):
    from mqdet_b200 import ops
    from mqdet_b200.modeling.groundingdino.transformer import multihead_attention
    from oracle import restate, synth
    gen = synth.Gen(76)
    E = 256
    for heads, Lq, Lk, kind in ((4, 256, 256, "mask2d"), (8, 900, 900, "self"), (8, 900, 256, "keymask")):
        sd = synth.mha_sd(gen, "", E, {})
        m = torch.nn.MultiheadAttention(E, heads).to(dev)
        m.load_state_dict(sd)
        B = 2
        q = gen.randn(B, Lq, E)
        k = q if kind != "keymask" else gen.randn(B, Lk, E)
        v = gen.randn(B, Lk, E)
        mask2d = keypad = None
        if kind == "mask2d":
            mask2d = torch.eye(Lk, dtype=torch.bool)[None].repeat(B, 1, 1)
            for s in range(1, 200, 5):
                mask2d[:, s:s + 5, s:s + 5] = True
        if kind == "keymask":
            keypad = torch.zeros(B, Lk, dtype=torch.bool)
            keypad[:, 200:] = True
        ref = restate.mha(q, k, v, sd, "", heads, attn_mask=None if mask2d is None else ~mask2d, key_padding_mask=keypad)
        q16 = ops.cast_f16(q.to(dev))
        k16 = q16 if kind != "keymask" else ops.cast_f16(k.to(dev))
        out = multihead_attention(m, q16, k16, ops.cast_f16(v.to(dev)),
                                  mask2d=None if mask2d is None else mask2d.float().to(dev).contiguous(),
                                  keymask=None if keypad is None else (~keypad).float().to(dev).contiguous())
        assert_close(out.view(B, Lq, E), ref, FP16_TOL, f"multihead_attention {kind}")


def test_bert_layer_with_category_mask_vs_oracle(dev):
    from mqdet_b200 import ops
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import BertLayer
    from oracle import restate, synth
    gen = synth.Gen(77)
    sd = synth.bert_layer_sd(gen, "")
    layer = load_sd(BertLayer(768, 12, 3072), sd).to(dev)
    ids, am, pmap = synth.prompt(20, 2, 256, gen)
    self_mask, _ = restate.gdino_text_masks(ids.expand(2, -1))
    h = gen.randn(2, 256, 768)
    ref = restate.bert_layer(h, (1.0 - self_mask[:, None].float()) * -10000.0, sd, "", 12)
    o32, o16 = layer(h.to(dev), ops.cast_f16(h.to(dev)), self_mask.float().to(dev).contiguous())
    assert_close(o32, ref, FP16_TOL, "BertLayer with the per-category mask")


# ---------------------------------------------------------------------------------------------------------------------
# transformer and whole model
# ---------------------------------------------------------------------------------------------------------------------
TKW = dict(d_model=256, nhead=8, dim_feedforward=2048, dropout=0.0, activation="relu", return_intermediate_dec=True, query_dim=4,
           num_feature_levels=4, enc_n_points=4, dec_n_points=4, learnable_tgt_init=True, two_stage_type="standard",
           embed_init_tgt=True, use_text_enhancer=True, use_fusion_layer=True, use_text_cross_attention=True, text_dropout=0.0,
           fusion_dropout=0.0, fusion_droppath=0.1)


def _build_transformer(sd, nq, el, dl, dev):
    from mqdet_b200.modeling.groundingdino.transformer import Transformer
    from mqdet_b200.modeling.groundingdino.utils import MLP, ContrastiveEmbed
    T = Transformer(num_queries=nq, num_encoder_layers=el, num_decoder_layers=dl, **TKW)
    be = MLP(256, 256, 4, 3)
    T.decoder.bbox_embed = torch.nn.ModuleList([be for _ in range(dl)])
    T.decoder.class_embed = torch.nn.ModuleList([ContrastiveEmbed() for _ in range(dl)])
    T.enc_out_bbox_embed = MLP(256, 256, 4, 3)
    T.enc_out_class_embed = ContrastiveEmbed()
    return load_sd(T, sd).to(dev).eval()


def _run_transformer(T, srcs, masks, poss, enc_text, tmask, pid, sam, dev, proposals=None):
    geo = T.prepare([m.to(dev) for m in masks], [p.to(dev) for p in poss], tmask.to(dev), pid.to(dev), sam.to(dev))
    src = torch.cat([s.flatten(2).transpose(1, 2) for s in srcs], 1).contiguous().to(dev)
    return T.forward_flat(src, geo, enc_text.to(dev).contiguous(), all_layers=True,
                          proposals=None if proposals is None else proposals.to(dev))


def _selection_equivalent(ours, ref_idx, ref_logits, bound):
    """The two-stage top-k selections agree up to near-ties: every position selected by one side only has an oracle logit within
    `bound` (the class-logit tolerance) of the oracle's k-th largest one, i.e. its rank is decided by fp16 noise."""
    for b in range(ref_idx.shape[0]):
        kth = ref_logits[b].sort(descending=True).values[ref_idx.shape[1] - 1]
        diff = set(ours[b].tolist()) ^ set(ref_idx[b].tolist())
        if any(abs(float(ref_logits[b, i] - kth)) > bound for i in diff):
            return False
    return True


def test_transformer_small_vs_oracle_and_golden(dev):
    """2 encoder + 2 decoder layers, 4 small levels (image 1 padded), 20 queries: every decoder layer's hidden state and box against
    the oracle, and against the fixture recorded from the reference's own Transformer.forward (tests/golden/gdino_transformer.pt)."""
    from oracle import make_golden, restate
    c = make_golden.case_inputs("gdino_transformer")
    sd, nq, el, dl = c["sd"], c["nq"], c["enc_layers"], c["dec_layers"]
    poss = [restate.position_embedding_sine_hw(m) for m in c["masks"]]
    ref = restate.gdino_transformer(c["srcs"], c["masks"], poss, c["enc_text"], c["tmask"], c["pid"], c["sam"], sd, num_queries=nq,
                                    enc_layers=el, dec_layers=dl, return_all=True)
    T = _build_transformer(sd, nq, el, dl, dev)
    out = _run_transformer(T, c["srcs"], c["masks"], poss, c["enc_text"], c["tmask"], c["pid"], c["sam"], dev)
    errs = []
    # padded / invalid memory positions all carry the same class logit (their memory row is zeroed): torch.topk picks any of those
    # ties, mqdet_topk_desc the lowest indices; and two valid positions whose logits differ by less than the fp16 noise of the
    # encoder may swap ranks.  The selection has to agree up to such near-ties; everything downstream of it is then compared on
    # the oracle's selection, so that a swapped rank does not pair up different queries
    fin = torch.isfinite(ref["enc_class"])
    ec = torch.where(fin, ref["enc_class"], torch.full((), -1e30))
    bound = 3e-3 * torch.where(fin, ref["enc_class"], torch.zeros(())).abs().max().item() + 3e-3  # the class-logit tolerance below
    same_sel = torch.equal(out["topk_proposals"].cpu(), ref["topk"])
    assert _selection_equivalent(out["topk_proposals"].cpu(), ref["topk"], ec.max(-1).values, bound), \
        (out["topk_proposals"].cpu(), ref["topk"])
    if not same_sel:
        out = _run_transformer(T, c["srcs"], c["masks"], poss, c["enc_text"], c["tmask"], c["pid"], c["sam"], dev, proposals=ref["topk"])
    hs, refs = out["hs"], out["references"]
    assert_close(refs[0], ref["references"][0], 2e-3, "gdino transformer: two-stage selected boxes", defer=errs)
    assert_close(out["memory"], ref["memory"], 3e-3, "gdino transformer: encoder memory", defer=errs)
    assert_close(out["memory_text"], ref["memory_text"], 3e-3, "gdino transformer: enhanced text", defer=errs)
    assert torch.equal(torch.isfinite(out["enc_class"]).cpu(), fin)
    assert_close(torch.where(fin, out["enc_class"].cpu(), torch.zeros(())), torch.where(fin, ref["enc_class"], torch.zeros(())), 3e-3,
                 "gdino transformer: two-stage class logits", defer=errs)
    for i in range(dl):
        assert_close(hs[i], ref["hs"][i], 5e-3, f"gdino transformer: hs[{i}]", defer=errs)
        assert_close(refs[i + 1], ref["references"][i + 1], 5e-3, f"gdino transformer: reference[{i + 1}]", defer=errs)
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "gdino_transformer.pt"))
    assert_close(hs[-1], fx["hs_last"], 5e-3, "gdino transformer: hs[-1] vs the reference's own forward", defer=errs)
    assert_close(refs[-1], fx["ref_last"], 5e-3, "gdino transformer: boxes vs the reference's own forward", defer=errs)
    assert_close(out["memory_text"], fx["text"], 3e-3, "gdino transformer: text vs the reference's own forward", defer=errs)
    _record("transformer_small", {"errors": errs, "same_selection": bool(same_sel)})
    assert not errs, errs


def _gdino_case(seed, B, h, w, ncls, el, dl, nq):
    from oracle import synth
    gen = synth.Gen(seed)
    sd = synth.gdino_sd(gen, el, dl, nq)
    ids, am, pmap = synth.prompt(ncls, 2, 256, gen)
    bank = synth.query_bank(pmap, 5, gen)
    img = synth.rgb_images(gen, B, h, w)
    return sd, ids, am, pmap, bank, img


def _build_model(sd, el, dl, nq, dev):
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO
    cfg = mq_groundingdino_t_cfg(**{"GROUNDINGDINO.enc_layers": el, "GROUNDINGDINO.dec_layers": dl, "GROUNDINGDINO.num_queries": nq})
    model = GroundingDINO(cfg)
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    return load_sd(model, full).to(dev).eval()


def test_groundingdino_forward_vs_oracle(dev):
    """The whole MQ-GroundingDINO-T forward (Swin-T -> input_proj -> vision-conditioned BERT with category masks -> feat_map ->
    2 + 2 layer transformer -> heads -> detections) on two images of different size, 13-class prompt, K = 5 vision queries."""
    from mqdet_b200.structures.image_list import ImageList
    from oracle import restate
    B, h, w, el, dl, nq = 2, 150, 203, 2, 2, 100
    sd, ids, am, pmap, bank, img = _gdino_case(2031, B, h, w, 13, el, dl, nq)
    sizes = [(h, w), (h - 22, w - 37)]
    img[1, :, sizes[1][0]:, :] = 0
    img[1, :, :, sizes[1][1]:] = 0
    ref = restate.gdino_forward(img, sizes, ids, am, pmap, bank, sd, num_queries=nq, enc_layers=el, dec_layers=dl)
    model = _build_model(sd, el, dl, nq, dev)
    model.query_selector.set_query_bank(bank)
    out = model.forward_device(ImageList(img.to(dev), sizes), {"input_ids": ids, "attention_mask": am}, pmap, all_layers=True)
    errs = []
    N = out["srcs"].shape[1]
    ref_src = torch.cat([s.flatten(2).transpose(1, 2) for s in ref["srcs"]], 1)
    assert_close(out["srcs"], ref_src, 3e-3, "gdino: input_proj pyramid", defer=errs)
    assert_close(out["bert_hidden"], ref["bert_hidden"], 3e-3, "gdino: BERT hidden (category masks + GCP)", defer=errs)
    assert_close(out["encoded_text"], ref["encoded_text"], 3e-3, "gdino: feat_map", defer=errs)
    assert_close(out["transformer"]["memory"], ref["memory"], 5e-3, "gdino: encoder memory", defer=errs)
    assert_close(out["transformer"]["memory_text"], ref["memory_text"], 5e-3, "gdino: enhanced text", defer=errs)
    # two-stage selection: the same SET of proposals (near-tied class logits may rank differently under fp16 operands, and the
    # decoder compares slot by slot) -> the decoder is compared on a second run fed with the oracle's selection
    overlap = [len(set(a.tolist()) & set(b.tolist())) for a, b in zip(out["transformer"]["topk_proposals"].cpu(), ref["topk"])]
    assert min(overlap) >= nq - 3, overlap
    f = model.forward_device(ImageList(img.to(dev), sizes), {"input_ids": ids, "attention_mask": am}, pmap, all_layers=True,
                             proposals=ref["topk"].to(dev))
    assert_close(f["hs"][-1], ref["hs"][-1], 5e-3, "gdino: decoder output (oracle's selection)", defer=errs)
    assert_close(f["pred_boxes"], ref["pred_boxes"], 5e-3, "gdino: boxes (oracle's selection)", defer=errs)
    fin = torch.isfinite(ref["pred_logits"])
    assert torch.equal(torch.isfinite(f["pred_logits"]).cpu(), fin)
    assert_close(torch.where(fin, f["pred_logits"].cpu(), torch.zeros(())), torch.where(fin, ref["pred_logits"], torch.zeros(())), 1e-2,
                 "gdino: class logits (oracle's selection)", defer=errs)
    from mqdet_b200.structures.bounding_box import boxlists_from_packed
    res = boxlists_from_packed(out["det_packed"], out["image_sizes"])
    n, n_ref = [len(r) for r in res], [d[0].shape[0] for d in ref["detections"]]
    _record("forward_small", {"errors": errs, "detections": n, "oracle_detections": n_ref, "selection_overlap": overlap})
    assert not errs, errs
    assert all(abs(a - b) <= max(3, b // 10) for a, b in zip(n, n_ref)), (n, n_ref)
    # public API: forward() -> list[BoxList]
    res2 = model(ImageList(img.to(dev), sizes), captions={"input_ids": ids, "attention_mask": am}, positive_map=pmap)
    assert [len(r) for r in res2] == n and res2[0].mode == "xyxy" and set(res2[0].fields()) == {"labels", "scores"}


def test_groundingdino_full_depth_runs_at_benchmark_shape(dev):
    """6 + 6 layers, 900 queries, 800x1333 (padded 800x1344), 13-class prompt, B = 2 (BASELINE config 4 per GPU): finite outputs,
    image i of the batch equals its B = 1 run (no cross-image leakage through the batched kernels)."""
    from mqdet_b200.structures.image_list import ImageList
    B, h, w = 2, 800, 1333
    sd, ids, am, pmap, bank, img = _gdino_case(2032, B, h, w, 13, 6, 6, 900)
    model = _build_model(sd, 6, 6, 900, dev)
    model.query_selector.set_query_bank(bank)
    caps = {"input_ids": ids, "attention_mask": am}
    out = model.forward_device(ImageList(img.to(dev), [(h, w)] * B), caps, pmap)
    assert torch.isfinite(out["pred_boxes"]).all() and torch.isfinite(out["hs"][-1]).all()
    assert out["srcs"].shape[1] == 100 * 168 + 50 * 84 + 25 * 42 + 13 * 21
    # same selection order in both runs: the global-maximum shift of stable_softmax_2d makes the scores (not the probabilities)
    # batch dependent, so near-tied proposals could otherwise swap slots
    one = model.forward_device(ImageList(img[1:].to(dev), [(h, w)]), caps, pmap, proposals=out["transformer"]["topk_proposals"][1:])
    e = assert_close(out["pred_boxes"][1:], one["pred_boxes"].cpu(), 2e-3, "gdino: image 1 of B=2 vs its B=1 run")
    _record("full_depth", {"batch_vs_single_box_err": e, "detections": [int(v) for v in out["num"].cpu()]})


def test_softmax_long_fp32_rows_with_mask(dev):
    """CTA-per-row softmax (n >= 4096 fp32: the text -> image side of the explicit BiAttention path, PreSelect's training forward)."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(9)
    B, H, T, N = 2, 4, 16, 5003
    Np = (N + 7) // 8 * 8
    x = torch.zeros(B, H, T, Np)
    x[..., :N] = torch.randn(B, H, T, N, generator=g) * 3
    keep = (torch.rand(B, N, generator=g) > 0.2).float()
    ref = (x[..., :N] + torch.where(keep == 0, float("-inf"), 0.0)[:, None, None, :]).softmax(-1)
    out = ops.softmax_rows(x.to(dev), n=N, colmask=keep.to(dev).contiguous(), rows_per_batch=H * T, mask_value=float("-inf")).cpu()
    assert (out[..., N:] == 0).all()
    assert_close(out[..., :N], ref, FP16_TOL, "softmax_rows long fp32 rows, masked")
    out2 = ops.softmax_rows(x.to(dev), n=N, scale=0.5).cpu()
    assert_close(out2[..., :N], (0.5 * x[..., :N]).softmax(-1), FP16_TOL, "softmax_rows long fp32 rows, scaled")


def test_softmax_rows_shifted(dev):
    """STABLE_SOFTMAX_2D's global shift + clamps fused into the softmax kernels (fuse_modules.py:177-187): both supported row lengths,
    with the clamp ACTIVE on part of the scores, against the unfused formula."""
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(10)
    for shape, n in (((2, 4, 300, 256), 256), ((2, 4, 16, 5008), 5003)):
        x = torch.randn(*shape, generator=g) * 4.0
        x[..., 7] += 30.0
        rows_per_batch = shape[1] * shape[2]
        keep = (torch.rand(shape[0], n, generator=g) > 0.2).float()
        shift = x[..., :n].max().view(1)
        lo, hi = -25.0, 25.0
        ref = ((x[..., :n] - shift).clamp(lo, hi) + torch.where(keep == 0, float("-inf"), 0.0)[:, None, None, :]).softmax(-1)
        out = ops.softmax_rows_shifted(x.to(dev).contiguous(), shift.to(dev), lo, hi, n=n, colmask=keep.to(dev).contiguous(),
                                       rows_per_batch=rows_per_batch, mask_value=float("-inf")).cpu()
        assert (out[..., n:] == 0).all()
        assert_close(out[..., :n], ref, FP16_TOL, f"softmax_rows_shifted n={n}")
    # unsupported row length: falls back to shift_clamp_ + softmax_rows
    x = torch.randn(3, 40, 120, generator=g) * 4.0
    shift = x.max().view(1)
    out = ops.softmax_rows_shifted(x.to(dev).contiguous(), shift.to(dev), -5.0, 5.0).cpu()
    assert_close(out, (x - shift).clamp(-5.0, 5.0).softmax(-1), FP16_TOL, "softmax_rows_shifted fallback")


def test_groundingdino_extract_query_vs_oracle(dev):
    """GroundingDINO.extract_query (groundingdino.py:340-430): boxes expanded x1.5, pooled from their level of the 4-level input_proj
    pyramid (POOLER_SCALES 1/8 .. 1/64), bank appended per label — against the oracle's pooling of the oracle's pyramid."""
    from collections import defaultdict
    from mqdet_b200.structures.bounding_box import BoxList
    from mqdet_b200.structures.image_list import ImageList
    from oracle import restate, synth
    sd, ids, am, pmap, bank, _ = _gdino_case(2040, 1, 32, 32, 5, 1, 1, 20)
    model = _build_model(sd, 1, 1, 20, dev)
    gen = synth.Gen(557)
    W_, H_ = 640, 480
    img = synth.rgb_images(gen, 2, H_, W_)
    boxes = [torch.tensor([[10., 12., 40., 50.], [100., 60., 330., 300.], [0., 0., 639., 479.], [300., 200., 620., 460.]]),
             torch.tensor([[30., 30., 190., 200.], [5., 200., 80., 318.]])]
    labels = [torch.tensor([3, 1, 2, 3]), torch.tensor([1, 4])]
    targets = []
    for b, l in zip(boxes, labels):
        t = BoxList(b.clone(), (W_, H_), mode="xyxy")
        t.add_field("labels", l)
        targets.append(t)
    got = model.extract_query(samples=ImageList(img.to(dev), [(H_, W_)] * 2), targets=targets, query_images=defaultdict(list))
    srcs, _ = restate.gdino_visual_features(img, [(H_, W_)] * 2, sd)
    ex, lab = [], []
    for b, l in zip(boxes, labels):
        nb, keep = restate.expand_boxes(b.clone(), (W_, H_), 1.5)
        ex.append(nb)
        lab.append(l[keep])
    feats, lvls = restate.pool_query_features(srcs, ex, scales=(0.125, 0.0625, 0.03125, 0.015625))
    assert len(set(lvls.tolist())) >= 2
    lab = torch.cat(lab)
    assert sorted(got) == sorted(set(lab.tolist()))
    for label in got:
        want = feats[lab == label][:, None, :]
        assert got[label].shape == want.shape
        assert_close(got[label], want, 4e-3, f"gdino extract_query label {label}")


def test_groundingdino_engine_graph_replay_equals_eager(dev):
    """GroundingDINOEngine (CUDA-graph replay over a static input buffer, pinned host batches in, list[BoxList] out) returns exactly
    what the eager forward returns, for two different batches through the same captured graph."""
    from mqdet_b200.engine.inference import GroundingDINOEngine
    from mqdet_b200.structures.bounding_box import boxlists_from_packed
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    B, h, w, el, dl, nq = 2, 150, 203, 1, 1, 50
    sd, ids, am, pmap, bank, img = _gdino_case(2050, B, h, w, 13, el, dl, nq)
    model = _build_model(sd, el, dl, nq, dev)
    model.query_selector.set_query_bank(bank)
    caps = {"input_ids": ids, "attention_mask": am}
    img2 = synth.rgb_images(synth.Gen(2051), B, h, w)
    eng = GroundingDINOEngine(model, caps, pmap, tuple(img.shape), [(h, w)] * B)
    assert eng.graph is not None, eng.note
    got = list(eng.run([img.pin_memory(), img2.pin_memory(), img.pin_memory()]))
    for x, res in zip((img, img2, img), got):
        ref = boxlists_from_packed(model.forward_device(ImageList(x.to(dev), [(h, w)] * B), caps, pmap)["det_packed"], [(h, w)] * B)
        for a, b in zip(res, ref):
            assert len(a) == len(b) and torch.equal(a.bbox, b.bbox) and torch.equal(a.get_field("scores"), b.get_field("scores"))
            assert torch.equal(a.get_field("labels"), b.get_field("labels"))
    assert any(len(a) != len(c) or not torch.equal(a.bbox, c.bbox) for a, c in zip(got[0], got[1]))   # the two batches do differ
