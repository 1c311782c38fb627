"""Drop-in for groundingdino_new/models/GroundingDINO/loss.py (``SetCriterion``) on the device, with the gradients of its loss at
the decoder outputs of every layer.

``forward`` returns the reference's dict: ``loss_ce``, ``loss_bbox``, ``loss_giou`` of the last decoder layer and the same with the
suffix ``_k`` for the auxiliary layers k = 0..L-2, each already multiplied by its weight (loss.py:166-171), as 0-dim device
tensors.  ``last_train`` keeps ``d_logits`` [L, B, Q, T] / ``d_boxes`` [L, B, Q, 4], the gradient of the sum of that dict with
respect to each layer's ``pred_logits`` / ``pred_boxes`` (layer order: aux layers first, the last layer at index L-1).

Matching (``ops.gdino_match``), the normaliser all-reduce (``parallel.all_reduce_loss_normalizers``) and the losses
(``ops.gdino_set_loss``) involve no host synchronisation, so ``forward_flat`` can be captured in a CUDA graph at a fixed GT
capacity.  The rules the reference leaves open are written down in DESIGN.md §4: a GT whose token row is empty has class cost 0
and its query gets the unmatched one-hot target; an image without GTs matches nothing; assignment ties resolve as scipy resolves
them.
"""
import torch
from torch import nn

from ... import ops, parallel
from .matcher import gt_pack, indices_from_match

LOSS_NAMES = ("loss_ce", "loss_bbox", "loss_giou")


def stack_outputs(outputs):
    """The reference's ``out`` dict ({pred_logits, pred_boxes, aux_outputs: [...]}) -> (pred_logits [L, B, Q, T], pred_boxes
    [L, B, Q, 4]) fp32 contiguous, aux layers first (``GroundingDINO.decoder_outputs_flat`` gives them without the copy)."""
    layers = list(outputs.get("aux_outputs", [])) + [outputs]
    logits = torch.stack([o["pred_logits"].float() for o in layers]).contiguous()
    boxes = torch.stack([o["pred_boxes"].float() for o in layers]).contiguous()
    return logits, boxes


def loss_dict(losses):
    """losses fp32 [L, 3] -> the reference's 18-key dict (for L = 6) of 0-dim device tensors, in its insertion order."""
    L = losses.shape[0]
    out = {k: losses[L - 1, i] for i, k in enumerate(LOSS_NAMES)}
    for l in range(L - 1):
        out.update({f"{k}_{l}": losses[l, i] for i, k in enumerate(LOSS_NAMES)})
    return out


class SetCriterion(nn.Module):
    """loss.py:18-178 with the shipped losses ('labels' = token sigmoid focal loss, 'boxes' = L1 + GIoU)."""

    def __init__(self, matcher, cfg):
        super().__init__()
        self.matcher = matcher
        g = cfg.GROUNDINGDINO
        self.weight_dict = {"loss_ce": g.loss_ce_coef, "loss_bbox": g.loss_bbox_coef, "loss_giou": g.loss_giou_coef}
        self.losses = ["labels", "boxes"]
        fc = cfg.MODEL.DYHEAD.FUSE_CONFIG
        self.alpha, self.gamma = getattr(fc, "TOKEN_ALPHA", 0.25), getattr(fc, "TOKEN_GAMMA", 2.0)
        self.last_train = None

    def forward_flat(self, pred_logits, pred_boxes, gt_pack, text_mask, world=1):
        """pred_logits fp32 [L, B, Q, T], pred_boxes fp32 [L, B, Q, 4], gt_pack = (gt_boxes [B, Gmax, 4] normalised cxcywh, gt_count
        [B], gt_tokens [B, Gmax, T]), text_mask [B, T] (> 0 = in use) or None -> dict(losses [L, 3], d_logits, d_boxes, match
        [L, B, Q], cost [L, B, Q, Gmax], norm [1]).  ``world``: the number of data-parallel ranks; the GT count is all-reduced over
        the default process group between matching and losses."""
        m = self.matcher.match_flat(pred_logits, pred_boxes, *gt_pack)
        parallel.all_reduce_loss_normalizers(m["norm"])
        losses, dl, db, norm = ops.gdino_set_loss(pred_logits, pred_boxes, *gt_pack, text_mask, targets=m, world=world, alpha=self.alpha,
                                                  gamma=self.gamma, ce_coef=self.weight_dict["loss_ce"],
                                                  bbox_coef=self.weight_dict["loss_bbox"], giou_coef=self.weight_dict["loss_giou"])
        return {"losses": losses, "d_logits": dl, "d_boxes": db, "match": m["match"], "cost": m["cost"], "norm": norm}

    @torch.no_grad()
    def forward(self, outputs, targets, return_indices=False, text_mask=None, positive_map=None):
        """Reference signature (loss.py:114): outputs = {pred_logits, pred_boxes, aux_outputs}, targets = list of ``BoxList`` with a
        ``normed_cxcy_boxes`` field, text_mask [B, T] bool, positive_map [sum G, T] -> the loss dict (and with ``return_indices``
        the per-layer index lists, aux layers first, the last layer at the end, as the reference orders them)."""
        logits, boxes = stack_outputs(outputs)
        world = torch.distributed.get_world_size() if (torch.distributed.is_available() and torch.distributed.is_initialized()) else 1
        pack = gt_pack(targets, positive_map, logits.device)
        tm = None if text_mask is None else text_mask.to(device=logits.device, dtype=torch.float32)
        r = self.forward_flat(logits, boxes, pack, tm, world=world)
        self.last_train = r
        losses = loss_dict(r["losses"])
        if return_indices:
            match = r["match"]
            L = match.shape[0]
            return losses, [indices_from_match(match[l]) for l in range(L)]
        return losses
