"""Optimizer of the modulated pre-training on sm_90a kernels, drop-in for maskrcnn_benchmark/solver/build.py:8-57 (``make_optimizer``
with SOLVER.OPTIMIZER "ADAMW" and full-model gradient clipping): per-parameter learning rate / weight decay groups chosen by the
reference's substring rules, ``torch.nn.utils.clip_grad_norm_`` over ALL trainable parameters, then ``torch.optim.AdamW``.

The global norm, the clip coefficient and every update stay on the device (``mqdet_sqnorm_partials`` / ``mqdet_clip_coef`` /
``mqdet_adamw_step``): no host synchronisation per step, where the reference's clip_grad_norm_ + per-tensor Python loop synchronises
and launches several ATen kernels per parameter.  Gradients are passed explicitly ({name: fp32 tensor}, e.g. from
``GCPBlockTrain.backward``) — the hot path has no autograd.
"""
import torch

from .. import ops
from .._lib import MqdetError


def param_group_options(cfg, key):
    """(lr, weight_decay) of one named parameter — the rules of solver/build.py:31-52, in the reference's order (later rules win:
    a ``qv_layer`` gate ends up with QUERY_LR, not GATE_LR, exactly like there)."""
    s = cfg.SOLVER
    lr, wd = s.BASE_LR, s.WEIGHT_DECAY
    if "language_backbone" in key:
        lr = s.LANG_LR
    if "backbone.body" in key and "language_backbone.body" not in key:
        lr = s.BASE_LR * s.BACKBONE_BODY_LR_FACTOR
    if "bias" in key:
        lr *= s.BIAS_LR_FACTOR
        wd = s.WEIGHT_DECAY_BIAS
    if "norm" in key or "Norm" in key:
        wd *= s.WEIGHT_DECAY_NORM_FACTOR
    if "attn_gate" in key or "ff_gate" in key:
        lr = s.GATE_LR
    if "pre_select" in key or "qv_layer" in key:
        lr = s.QUERY_LR
    return lr, wd


class FusedAdamW:
    """AdamW (betas (0.9, 0.999), eps 1e-8 — torch defaults, which the reference uses) + full-model gradient clipping."""

    def __init__(self, named_params, cfg=None, lr=1e-4, weight_decay=1e-4, betas=(0.9, 0.999), eps=1e-8, clip_value=None):
        self.params = {}
        for name, p in named_params:
            if not p.requires_grad:
                continue
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise MqdetError(f"FusedAdamW: parameter {name} must be contiguous fp32")
            plr, pwd = param_group_options(cfg, name) if cfg is not None else (lr, weight_decay)
            self.params[name] = dict(p=p, lr=plr, wd=pwd, m=torch.zeros_like(p), v=torch.zeros_like(p))
        self.betas, self.eps, self.steps = betas, eps, 0
        if clip_value is None and cfg is not None:
            c = cfg.SOLVER.CLIP_GRADIENTS
            clip_value = c.CLIP_VALUE if (c.ENABLED and c.CLIP_TYPE == "full_model" and c.CLIP_VALUE > 0.0) else 0.0
        self.clip_value = float(clip_value or 0.0)
        self.last_coef = None

    @torch.no_grad()
    def step(self, grads, lr_scale=1.0):
        """grads: {name: fp32 tensor} for EVERY tracked parameter.  Returns the device tensor (clip coefficient, gradient norm)."""
        missing = [k for k in self.params if k not in grads]
        if missing:
            raise MqdetError(f"FusedAdamW.step: no gradient for {missing[:3]}")
        self.steps += 1
        gl = [grads[k].float().contiguous().view(-1) for k in self.params]
        coef = ops.clip_coef(gl, self.clip_value)   # clip_value 0: coefficient 1, the norm is still reported
        for g, (name, st) in zip(gl, self.params.items()):
            ops.adamw_step_(st["p"].data.view(-1), g, st["m"].view(-1), st["v"].view(-1), self.steps, st["lr"] * lr_scale, self.betas,
                            self.eps, st["wd"], grad_scale=coef[:1])
        self.last_coef = coef
        return coef


def make_optimizer(cfg, model):
    """Reference signature (solver/build.py:8): returns the fused optimizer over ``model.named_parameters()`` with requires_grad."""
    if cfg.SOLVER.OPTIMIZER != "ADAMW":
        raise NotImplementedError("the MQ pre-training configs use SOLVER.OPTIMIZER ADAMW")
    return FusedAdamW(model.named_parameters(), cfg=cfg)
