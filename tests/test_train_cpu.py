"""CPU: pins the training-side oracle pieces against the reference's own code (live where its sources are present, else against the
results recorded from it: tests/golden/pins, refpin.py) and checks the host-side parameter-group rules of mqdet_b200.solver.build
against solver/build.py."""
import types

import pytest
import torch

from oracle import ref_loader, restate
from refpin import max_err, pinned


def test_token_focal_loss_vs_reference():
    import sys
    g = torch.Generator().manual_seed(4)
    logits = torch.randn(2, 300, 256, generator=g) * 3 - 2
    targets = (torch.rand(2, 300, 256, generator=g) > 0.95).float()
    tm = torch.ones(2, 256)
    tm[0, 200:] = 0
    tm[1, 120:] = 0

    def reference():
        ref_loader._install_shims()
        sys.modules["maskrcnn_benchmark"]._C = types.SimpleNamespace()   # the CUDA-only sigmoid focal loss op is not on this path
        m = ref_loader._load_file("ref_sigmoid_focal_loss", "maskrcnn_benchmark/layers/sigmoid_focal_loss.py")
        mod = m.TokenSigmoidFocalLoss(0.25, 2.0)
        return [mod(logits, targets, text_masks=mask, version="binary") for mask in (tm, None)]
    refs = pinned("token_focal_loss", reference)
    for mask, ref in zip((tm, None), refs):
        got = restate.token_focal_loss(logits, targets, 0.25, 2.0, mask)
        assert abs(ref.item() - got.item()) <= 1e-6 * abs(ref.item())


def test_gcp_block_autograd_oracle_vs_reference():
    """The backward oracle = autograd over restate.gcp_block: its gradients equal autograd over the reference's own block."""
    from oracle import make_golden, synth
    gen = synth.Gen(6)
    sd = synth.gcp_block_sd(gen)
    B, T = 2, 64
    _, _, pmap = synth.prompt(6, 2, T, gen)
    _, mk = synth.vision_queries(pmap, 5, T, 768, gen)
    mask = mk.expand(B, -1, -1).clone()
    mask[0, 3] = 0
    vision, x, dy = gen.randn(B, mask.shape[1], 768), gen.randn(B, T, 768), gen.randn(B, T, 768)

    def reference():
        blk = ref_loader.modeling_bert_new().GatedCrossAttentionBlock(dim=768, cfg=make_golden.ref_cfg())
        blk.load_state_dict(sd, strict=True)
        xr, vr = x.clone().requires_grad_(True), vision.clone().requires_grad_(True)
        blk(xr, vr, mask).backward(dy)
        return {"x": xr.grad, "vision": vr.grad, "params": {k: q.grad for k, q in blk.named_parameters()}}
    ref = pinned("gcp_block_grads", reference)
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    x2, v2 = x.clone().requires_grad_(True), vision.clone().requires_grad_(True)
    restate.gcp_block(x2, v2, mask, p, "").backward(dy)

    def close(a, b):
        err, bmax = max_err(a, b)
        assert err <= 2e-5 * bmax + 1e-7

    close(x2.grad, ref["x"])
    close(v2.grad, ref["vision"])
    assert set(ref["params"]) <= set(p)
    for k, g in ref["params"].items():
        close(p[k].grad.view(g.shape), g)


def test_param_group_rules():
    from mqdet_b200.solver.build import param_group_options
    NS = types.SimpleNamespace
    cfg = NS(SOLVER=NS(BASE_LR=1e-4, WEIGHT_DECAY=1e-4, LANG_LR=1e-5, BACKBONE_BODY_LR_FACTOR=1.0, BIAS_LR_FACTOR=2.0,
                       WEIGHT_DECAY_BIAS=0.0, WEIGHT_DECAY_NORM_FACTOR=1.0, GATE_LR=5e-3, QUERY_LR=1e-5))
    pre = "language_backbone.body.model."
    assert param_group_options(cfg, pre + "encoder.qv_layer.0.attn.to_q.weight") == (1e-5, 1e-4)
    assert param_group_options(cfg, pre + "encoder.qv_layer.0.ff_gate") == (1e-5, 1e-4)          # qv_layer rule wins over the gate rule
    assert param_group_options(cfg, pre + "encoder.qv_layer.0.attn.norm.bias") == (1e-5, 0.0)
    assert param_group_options(cfg, pre + "pre_select.layers.0.ff.linear1.weight") == (1e-5, 1e-4)
    assert param_group_options(cfg, "rpn.head.bias0") == (2e-4, 0.0)
