"""The part of the modulated pre-training step (maskrcnn_benchmark/engine/trainer.py:119-157) that mqdet_b200 runs natively: everything
that touches a TRAINABLE parameter.

    reference step                                      here
    ------------------------------------------------    -------------------------------------------------------------------
    loss_dict = model(images, targets, captions, ...)    language backbone forward: ``QVBertModelTrain.forward`` (training kernels)
      fusion tower forward                                ``VLDyHead.forward_flat`` (inference kernels)
      ATSS assignment, GIoU / centerness / token losses   ``VLDyHeadModule.forward_train_flat``: ``ops.atss_targets`` ->
                                                          ``parallel.all_reduce_loss_normalizers`` -> ``ops.atss_loss`` = losses +
                                                          d(logits), d(box / centerness output) on the device
      backward through the frozen fusion tower            NOT built (DESIGN.md §1 row f2) — the caller supplies dL/d(hidden)
    GroundingDINO (config 4): out = decoder outputs,     ``GroundingDINO.decoder_outputs_flat`` (all layers, one MLP chain / one
      SetCriterion(out, targets, text_mask, pos_map)      contrastive product) -> ``SetCriterion.forward_flat``: ``ops.gdino_match``
      (HungarianMatcher + scipy, L1 / GIoU / token        (cost + on-device linear sum assignment) -> ``parallel.all_reduce_loss_
      focal losses per decoder layer)                     normalizers`` -> ``ops.gdino_set_loss`` = losses + d(logits), d(boxes)
                                                          of every layer on the device; the backward into the decoder: NOT built
    scaler.scale(losses).backward()                      ``QVBertModelTrain.backward(d_hidden)`` -> gradients of all 119 trainable tensors
    DDP gradient all-reduce                               ``parallel.all_reduce_gradients`` (ONE flat NCCL all-reduce, averaged)
    clip_grad_norm_ + AdamW per parameter group           ``FusedAdamW.step`` (norm, clip coefficient, updates: all on the device)

``LanguageSideTrainer.step`` strings the native pieces together; it is exercised (forward -> focal loss on a read-out -> backward ->
optimizer) by tests/test_train_gpu.py::test_qvbert_model_backward_and_optimizer_step.
"""
import torch

from .. import parallel
from ..modeling.language_backbone.gcp_backward import QVBertModelTrain
from ..solver.build import FusedAdamW


class LanguageSideTrainer:
    def __init__(self, qvbert_model, cfg=None, name_prefix="language_backbone.body.model.", **optimizer_kw):
        """``qvbert_model``: mqdet_b200 ``QVBertModel``; trainable = ``encoder.qv_layer.*`` and ``pre_select.*`` (tools/train_net.py:70-77).
        ``name_prefix`` is the parameter path inside the detector, which the reference's lr / weight-decay rules match on."""
        self.model = qvbert_model
        self.prefix = name_prefix
        self.fb = QVBertModelTrain(qvbert_model)
        named = []
        for k, p in qvbert_model.named_parameters():
            train = k.startswith(("encoder.qv_layer", "pre_select"))
            p.requires_grad_(train)
            if train:
                named.append((name_prefix + k, p))
        self.optimizer = FusedAdamW(named, cfg=cfg, **optimizer_kw)

    @torch.no_grad()
    def forward(self, input_ids, attention_mask, vision, images, vision_attention_mask):
        return self.fb.forward(input_ids, attention_mask, vision, images, vision_attention_mask)

    @torch.no_grad()
    def step(self, d_hidden, lr_scale=1.0):
        """d_hidden fp32 [B,T,768] = dL/d(hidden) of the last forward -> (clip coefficient, gradient norm) device tensor."""
        grads = self.fb.backward(d_hidden)
        parallel.all_reduce_gradients(grads)
        return self.optimizer.step({self.prefix + k: g for k, g in grads.items()}, lr_scale=lr_scale)
