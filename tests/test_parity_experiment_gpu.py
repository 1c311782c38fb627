"""Which stage owns the end-to-end error of the 6-layer fusion tower?  (VERDICT round 1, item 1c.)

The tower of tests/test_fusion_gpu.py::test_vldyhead_tower (same seed, same deliberately lively weights) is run layer by
layer on the GPU next to the fp32 CPU oracle, twice per attention-score precision:
  * free-running  : every GPU stage consumes the previous GPU stage's output -> the accumulated error after each stage;
  * teacher-forced: every GPU stage consumes the ORACLE's input of that stage (rounded to the stage's storage type) ->
                    the error each stage adds on its own.
Score precisions (``BiMultiHeadAttention.score_precision``): "fused" = the product path, "f32" = diagnostic fp32 score
matrix in HBM.  Results go to parity_experiment.json in the run's output directory.
"""
import json
import os

import pytest
import torch

from util import ROOT, load_sd, rel_err

pytestmark = pytest.mark.gpu

SIZES = [(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)]


def _mean_rel(out, ref):
    out, ref = out.detach().float().cpu(), ref.detach().float().cpu()
    return (out - ref).abs().mean().item() / (ref.abs().mean().item() + 1e-12)


def test_tower_error_attribution_fused_and_f32(dev):
    from mqdet_b200 import ops
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.language_backbone.modeling_bert_new import BertLayer
    from mqdet_b200.modeling.rpn.vldyhead import VLDyHead
    from oracle import restate, synth
    gen = synth.Gen(78)
    nconv = 6
    sd = synth.vldyhead_sd(gen, nconv)
    B, T = 2, 256
    feats = [gen.randn(B, 256, h, w) for h, w in SIZES]
    hidden = gen.randn(B, T, 768)
    masks = torch.ones(B, T, dtype=torch.long)
    masks[0, 120:] = 0
    masks[1, 31:] = 0
    head = load_sd(VLDyHead(mq_glip_t_cfg()), sd).to(dev).eval()
    lv = ops.Levels(SIZES, dev)
    cm = masks.float().to(dev)
    report = {}
    modes = ["fused", "f32"]
    for mode in modes:
        for i in range(0, len(head.dyhead_tower), 3):
            head.dyhead_tower[i].b_attn.attn.score_precision = mode
        rows = []
        v_ref, h_ref = restate.flatten_levels(feats), hidden
        v_gpu, h_gpu = v_ref.half().to(dev).contiguous(), hidden.to(dev)
        for i in range(nconv):
            fuse, bert, dyc = head.dyhead_tower[3 * i], head.dyhead_tower[3 * i + 1], head.dyhead_tower[3 * i + 2]
            p = f"dyhead_tower.{3 * i}.b_attn."
            # oracle stages
            v1_ref, h1_ref = restate.bi_attention(v_ref, h_ref, masks, sd, p)
            h2_ref = restate.bert_layer(h1_ref, restate.extended_mask(masks), sd, f"dyhead_tower.{3 * i + 1}.", clamp=50000.0)
            v2_ref = restate.flatten_levels(restate.dyconv(restate.split_levels(v1_ref, SIZES), sd, f"dyhead_tower.{3 * i + 2}."))
            # teacher-forced GPU stages
            tv1, th1 = fuse.b_attn.forward_flat(v_ref.half().to(dev).contiguous(), h_ref.to(dev), masks.to(dev))
            th2, _ = BertLayer.forward(bert, h1_ref.to(dev).contiguous(), ops.cast_f16(h1_ref.to(dev).contiguous()), cm)
            tv2 = dyc.forward_flat(v1_ref.half().to(dev).contiguous(), lv)
            # free-running GPU stages
            v_gpu, h_gpu = fuse.b_attn.forward_flat(v_gpu, h_gpu, masks.to(dev))
            fr_v1, fr_h1 = rel_err(v_gpu, v1_ref), rel_err(h_gpu, h1_ref)
            h_gpu, _ = BertLayer.forward(bert, h_gpu, ops.cast_f16(h_gpu), cm)
            v_gpu = dyc.forward_flat(v_gpu, lv)
            rows.append(dict(layer=i,
                             forced_fusion_v=rel_err(tv1, v1_ref), forced_fusion_l=rel_err(th1, h1_ref),
                             forced_bert=rel_err(th2, h2_ref), forced_dyconv=rel_err(tv2, v2_ref),
                             free_fusion_v=fr_v1, free_fusion_l=fr_h1, free_bert=rel_err(h_gpu, h2_ref),
                             free_dyconv=rel_err(v_gpu, v2_ref), free_dyconv_mean=_mean_rel(v_gpu, v2_ref)))
            v_ref, h_ref = v2_ref, h2_ref
        ref = restate.vl_dyhead(feats, hidden, masks, sd, nconv)
        r = head.forward_flat(restate.flatten_levels(feats).half().to(dev).contiguous(), lv, hidden.to(dev), masks.to(dev))
        report[mode] = dict(layers=rows, tower_logits=rel_err(r["dot_product_logits"], ref["dot_product_logits"]),
                            tower_hidden=rel_err(r["hidden"], ref["hidden"]),
                            tower_visual=rel_err(r["visual"], restate.flatten_levels(ref["visual"])),
                            tower_visual_mean=_mean_rel(r["visual"], restate.flatten_levels(ref["visual"])))
    for i in range(0, len(head.dyhead_tower), 3):
        head.dyhead_tower[i].b_attn.attn.score_precision = "fused"
    out_dir = os.path.join(ROOT, "gpurun_out")
    if os.path.isdir(out_dir):
        with open(os.path.join(out_dir, "parity_experiment.json"), "w") as f:
            json.dump(report, f, indent=1)
    print(json.dumps({m: {k: v for k, v in rep.items() if k != "layers"} for m, rep in report.items()}))
    for rep in report.values():
        for row in rep["layers"]:
            # every stage on its own stays at the per-operator scale (fp16 operands, fp16-stored activations)
            assert row["forced_fusion_v"] < 3e-3 and row["forced_fusion_l"] < 3e-3 and row["forced_bert"] < 3e-3, row
            assert row["forced_dyconv"] < 1e-2, row
