"""GPU: the GCP path with more than 16 vision queries per text token (NUM_QUERY_PER_CLASS up to 100 and beyond): the sparse-attention
kernel up to its ceiling, the GCP block, the whole language backbone and detector against the CPU oracle, the chunked MQ-GroundingDINO
path and the graph-replayed engine, and the training guard that keeps the GCP backward at 16."""
import pytest
import torch

from test_gcp_many_queries_cpu import many_query_case
from util import assert_close, load_sd, vq_cfg

pytestmark = pytest.mark.gpu


def _attn_ref(q, kv, idx, heads, dim_head):
    """float64 restatement of gcp_sparse_attn on the same fp16 operands (MaskedCrossAttention.forward, modeling_bert_new.py:215-233)."""
    q, kv, idx = q.double().cpu(), kv.double().cpu(), idx.long().cpu()
    B, T, inner = q.shape
    V, S = kv.shape[1] - 1, idx.shape[2]
    out = torch.zeros(B, T, inner, dtype=torch.float64)
    for b in range(B):
        kb = kv[b, :, :inner][idx[b]].view(T, S, heads, dim_head)
        vb = kv[b, :, inner:][idx[b]].view(T, S, heads, dim_head)
        pad = idx[b] == V
        sim = torch.einsum("thd,tshd->ths", q[b].view(T, heads, dim_head), kb) + pad[:, None, :] * -1e4
        attn = sim.softmax(-1) * (~pad)[:, None, :]
        out[b] = torch.einsum("ths,tshd->thd", attn, vb).reshape(T, inner)
    return out


def _attn_inputs(B, T, V, S, seed, dev):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B, T, 512, generator=g) * 0.25).half()
    kv = torch.randn(B, V + 1, 1024, generator=g).half()
    idx = torch.randint(0, V + 1, (B, T, S), generator=g, dtype=torch.int32)
    idx[0, 0] = V                     # a token of no class
    idx[0, 1] = torch.arange(S) % V   # no padding slot
    return q.to(dev), kv.to(dev), idx.to(dev)


@pytest.mark.parametrize("S", [17, 31, 32, 33, 100, 257])
def test_gcp_block_many_queries(dev, S):
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import GatedCrossAttentionBlock
    from oracle import restate
    c = many_query_case(S)
    x, vision, mask = c["x"], c["vision"], c["mask"]
    ref = restate.gcp_block(x, vision, mask, c["sd"])
    blk = load_sd(GatedCrossAttentionBlock(dim=768, cfg=vq_cfg()), c["sd"]).to(dev).eval()
    out = blk(x.to(dev), vision.to(dev), mask.to(dev))
    assert_close(out, ref, what=f"GCP block S={S}")
    s_ref = restate.gcp_sparse_attention(x, vision, mask, c["sd"], "attn.")
    s = blk.attn(x.to(dev), vision.to(dev), mask.to(dev))
    assert_close(s, s_ref, what=f"sparse attention S={S}")
    no_cls = mask.sum(1) == 0
    assert no_cls[2].all() and s.cpu()[no_cls].abs().max().item() == 0.0


@pytest.mark.parametrize("S,heads", [(17, 8), (31, 8), (32, 8), (33, 8), (100, 8), (257, 8), (100, 32), (100, 2)])
def test_sparse_attn_op(dev, S, heads):
    from mqdet_b200 import ops
    q, kv, idx = _attn_inputs(2, 24, 3 * S, S, S + heads, dev)
    out = ops.gcp_sparse_attn(q, kv, idx, heads, 512 // heads)
    assert_close(out, _attn_ref(q, kv, idx, heads, 512 // heads), 1e-3, f"gcp_sparse_attn S={S} H={heads}")
    assert out[0, 0].abs().max().item() == 0.0


@pytest.mark.parametrize("heads", [8, 32])
def test_sparse_attn_1024_and_ceiling(dev, heads):
    """S = 1024 and S = GCP_MAX_S (one warp per CTA at 32 heads: the largest shared-memory slice) against the restatement; one
    more raises, in ops and in the C ABI, naming the ceiling."""
    from mqdet_b200 import _lib, ops
    for S in (1024, ops.GCP_MAX_S):
        q, kv, idx = _attn_inputs(2, 6, 2000, S, S + heads, dev)
        out = ops.gcp_sparse_attn(q, kv, idx, heads, 512 // heads)
        assert_close(out, _attn_ref(q, kv, idx, heads, 512 // heads), 1e-3, f"gcp_sparse_attn S={S} H={heads}")
    q, kv, idx = _attn_inputs(1, 2, 100, ops.GCP_MAX_S + 1, 5, dev)
    with pytest.raises(_lib.MqdetError, match=str(ops.GCP_MAX_S)):
        ops.gcp_sparse_attn(q, kv, idx, heads, 512 // heads)
    out = torch.empty_like(q)
    lib = _lib.load()
    rc = lib.mqdet_gcp_sparse_attn(ops._ptr(q), ops._ptr(kv), ops._ptr(idx), ops._ptr(out), 1, 2, 100, ops.GCP_MAX_S + 1, heads,
                                   512 // heads, ops._stream())
    assert rc != 0 and str(ops.GCP_MAX_S).encode() in lib.mqdet_last_error()


def test_sparse_attn_padding_slots_change_nothing(dev):
    """Padding slots add exp(-1e4 + .) = 0 to the softmax sum and get p = 0, so the same queries padded to any S give the same bits,
    across the 16-slot load chunks."""
    from mqdet_b200 import ops
    B, T, V = 2, 64, 300
    q, kv, idx = _attn_inputs(B, T, V, 300, 3, dev)
    n = torch.randint(0, 17, (B, T), generator=torch.Generator().manual_seed(4)).to(dev)
    base = torch.where(torch.arange(16, device=dev)[None, None] < n[..., None], idx[..., :16], V).int()
    want = ops.gcp_sparse_attn(q, kv, base.contiguous(), 8, 64)
    for S in (17, 48, 300):
        wide = torch.full((B, T, S), V, dtype=torch.int32, device=dev)
        wide[..., :16] = base
        assert torch.equal(ops.gcp_sparse_attn(q, kv, wide, 8, 64), want), S


def test_qvbert_model_100_queries(dev):
    """Whole language backbone with 100 queries per class (10 classes, one with 60): embeddings, PreSelect, 12 BERT layers with
    the six GCP blocks, against the oracle at the bound of test_qvbert_model_vs_oracle."""
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.language_backbone.bert_model_new import BertEncoder
    from oracle import restate, synth
    gen = synth.Gen(610)
    sd = synth.qvbert_sd(gen)
    B = 2
    ids, am, pmap = synth.prompt(10, 2, 256, gen)
    ids, am = ids.expand(B, -1).contiguous(), am.expand(B, -1).contiguous()
    vision, vmask = synth.vision_queries(pmap, 100, 256, 256, gen)
    vmask[0, 140:200] = 0
    vision = vision.expand(B, -1, -1).contiguous() + 0.1 * gen.randn(B, vision.shape[1], 256)
    vmask = vmask.expand(B, -1, -1).contiguous()
    images = gen.randn(B, 1117, 256)
    ref = restate.qvbert_model(ids, am, vision, images, vmask, sd)
    enc = BertEncoder(mq_glip_t_cfg(**{"VISION_QUERY.NUM_QUERY_PER_CLASS": 100}))
    load_sd(enc.model, sd)
    enc = enc.to(dev).eval()
    out = enc({"input_ids": ids.to(dev), "attention_mask": am.to(dev),
               "vision_inputs": {"vision": vision.to(dev), "images": images.to(dev), "vision_attention_mask": vmask.to(dev),
                                 "batched_pos_category_map": None}})
    assert_close(out["hidden"], ref["hidden"], 3e-3, "QVBertModel hidden K=100")


def _glip(sd, dev, K):
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
    model = GeneralizedVLRCNN_New(mq_glip_t_cfg(**{"VISION_QUERY.NUM_QUERY_PER_CLASS": K}))
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    return load_sd(model, full).to(dev).eval()


def _bank(pmap, K, gen, short=None):
    from oracle import synth
    bank = synth.query_bank(pmap, K, gen)
    if short is not None:
        bank[short] = bank[short][:60]
    return bank


def test_detector_forward_100_queries(dev):
    """GeneralizedVLRCNN_New.forward_device with NUM_QUERY_PER_CLASS = 100 (banks of 100 rows, one class with 60) against the
    oracle's whole forward, checked as test_detector_forward checks K = 5."""
    from mqdet_b200.structures.bounding_box import BoxList
    from mqdet_b200.structures.image_list import ImageList
    from oracle import restate, synth
    from test_detector_gpu import _iou
    gen = synth.Gen(2024)                     # the weights, prompt and images of test_detector_forward; only the bank differs
    sd = synth.detector_sd(gen, bias0=-1.5)
    ids, am, pmap = synth.prompt(10, 2, 256, gen)
    synth.query_bank(pmap, 5, gen)            # that test's K = 5 bank: keeps the generator in step for the images
    B, h, w = 2, 150, 203
    img = synth.images(gen, B, h, w)
    bank = _bank(pmap, 100, gen, short=4)
    ref = restate.detector(img, (h, w), ids, am, pmap, bank, sd, K=100)
    model = _glip(sd, dev, 100)
    model.query_selector.set_query_bank(bank)
    il = ImageList(img.to(dev), [(h, w)] * B)
    caps = {"input_ids": ids, "attention_mask": am}
    out = model.forward_device(il, caps, pmap)
    bad = []
    assert_close(out["head"]["hidden"], ref["fused_hidden"], 5e-3, "e2e K=100: fused language stream", defer=bad)
    assert_close(out["head"]["dot_product_logits"], ref["logits"], 1.5e-2, "e2e K=100: dot-product logits", defer=bad)
    assert not bad, bad
    res = model(il, captions=caps, positive_map=pmap)
    assert len(res) == B and all(isinstance(r, BoxList) for r in res)
    for b, r in enumerate(res):
        rb, rs, rl = ref["detections"][b]
        assert len(r) >= min(100, rb.shape[0]) - 5
        iou = _iou(rb, r.bbox)
        same = rl[:, None] == r.get_field("labels")[None]
        matched = ((iou > 0.9) & same & ((rs[:, None] - r.get_field("scores")[None]).abs() < 2e-2)).any(1)
        assert matched.float().mean().item() >= 0.85, f"image {b}: only {matched.float().mean().item():.2f} matched"


def test_inference_engine_replay_100_queries(dev):
    """InferenceEngine's CUDA-graph replay returns exactly the eager detections at NUM_QUERY_PER_CLASS = 100."""
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    gen = synth.Gen(177)
    sd = synth.detector_sd(gen, bias0=-1.5)
    ids, am, pmap = synth.prompt(10, 2, 256, gen)
    model = _glip(sd, dev, 100)
    model.query_selector.set_query_bank(_bank(pmap, 100, gen, short=7))
    B, h, w = 2, 150, 203
    caps = {"input_ids": ids, "attention_mask": am}
    batches = [synth.images(gen, B, h, w) for _ in range(3)]
    sizes = [(h, w)] * B
    want = [model(ImageList(b.to(dev), sizes), captions=caps, positive_map=pmap) for b in batches]
    eng = InferenceEngine(model, caps, pmap, tuple(batches[0].shape), sizes, use_graph=True, warmup=1)
    got = list(eng.run([b.pin_memory() for b in batches]))
    eng.close()
    assert len(got) == len(want)
    for g_b, w_b in zip(got, want):
        for g, r in zip(g_b, w_b):
            assert len(g) == len(r) and len(r) > 0
            assert torch.equal(g.bbox.cpu(), r.bbox.cpu())
            assert torch.equal(g.get_field("labels").cpu(), r.get_field("labels").cpu())
            assert torch.equal(g.get_field("scores").cpu(), r.get_field("scores").cpu())


def test_gdino_forward_chunked_100_queries(dev):
    """MQ-GroundingDINO-T (2 + 2 layers, 100 queries), 27 classes in chunks of 10 with 100 vision queries per class:
    ``forward_chunked_device`` packs exactly the rows of one ``forward_device`` per image and chunk."""
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    from test_gdino_chunked_gpu import _model
    el, dl, nq = 2, 2, 100
    gen = synth.Gen(2141)
    sd = synth.gdino_sd(gen, el, dl, nq)
    chunks = synth.chunked_prompts(27, 10, 256, gen)
    bank = {}
    for _, _, pm in chunks:
        bank.update(synth.query_bank(pm, 100, gen))
    bank[5] = bank[5][:60]
    B, h, w = 2, 150, 203
    img = synth.rgb_images(gen, B, h, w)
    sizes = [(h, w), (h - 22, w - 37)]
    img[1, :, sizes[1][0]:, :] = 0
    img[1, :, :, sizes[1][1]:] = 0
    model = _model(sd, el, dl, nq, dev, 28)
    model.query_selector.num_query_per_class = 100
    model.query_selector.set_query_bank(bank)
    il = ImageList(img.to(dev), sizes)
    caps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    pmaps = [pm for _, _, pm in chunks]
    pk = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)["det_packed"]
    total = 0
    for b in range(B):
        one = ImageList(img[b:b + 1].to(dev), sizes[b:b + 1])
        for c, (cap, pm) in enumerate(zip(caps, pmaps)):
            ref = model.forward_device(one, cap, pm)["det_packed"][0]
            assert torch.equal(pk[c, b], ref), f"image {b}, chunk {c}"
            total += int(ref[nq, 0])
    assert total > 20


def test_gcp_training_rejects_more_than_16(dev):
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.modeling.language_backbone.gcp_backward import GCPBlockTrain
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import GatedCrossAttentionBlock
    c = many_query_case(17)
    blk = load_sd(GatedCrossAttentionBlock(dim=768, cfg=vq_cfg()), c["sd"]).to(dev).eval()
    with pytest.raises(MqdetError, match="16"):
        GCPBlockTrain(blk).forward(c["x"].to(dev), c["vision"].to(dev), c["mask"].to(dev))
    c = many_query_case(17)
    c["mask"][:, 16::17] = 0                             # 16 queries per token: still trains
    tr = GCPBlockTrain(blk)
    y = tr.forward(c["x"].to(dev), c["vision"].to(dev), c["mask"].to(dev))
    dx, _, _ = tr.backward(torch.ones_like(y))
    assert torch.isfinite(dx).all()
