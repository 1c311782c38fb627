"""Drop-in for groundingdino_new/models/GroundingDINO/matcher.py (``HungarianMatcher``, ``build_matcher``) on the device.

The matching cost of matcher.py:49-81 is ``ops.gdino_match``'s cost kernel, and the assignment is solved on the device by
``mqdet_linear_sum_assignment``, which returns index for index what ``scipy.optimize.linear_sum_assignment`` returns on the same
fp32 cost matrix, ties included.  The reference copies each cost matrix to the host and solves it there once per image; here
the only device-to-host copy is the final one that builds the reference's list of index tensors.
"""
import torch
from torch import nn

from ... import ops


def gt_pack(targets, positive_map, device, Gmax=None):
    """The reference's per-image targets as the fixed-capacity pack of ``ops.gdino_match``: targets = list of ``BoxList`` with a
    ``normed_cxcy_boxes`` field, positive_map [sum G, T] (rows in target order) -> (gt_boxes fp32 [B, Gmax, 4], gt_count int32 [B],
    gt_tokens fp32 [B, Gmax, T]) on ``device``; Gmax defaults to max(1, the largest G)."""
    sizes = [len(t.get_field("normed_cxcy_boxes")) for t in targets]
    if positive_map.shape[0] != sum(sizes):
        raise ValueError(f"positive_map has {positive_map.shape[0]} rows for {sum(sizes)} target boxes")
    B, T = len(targets), positive_map.shape[1]
    G = max(1, max(sizes, default=0)) if Gmax is None else int(Gmax)
    boxes = torch.zeros((B, G, 4), dtype=torch.float32, device=device)
    tokens = torch.zeros((B, G, T), dtype=torch.float32, device=device)
    pm = positive_map.to(device=device, dtype=torch.float32)
    off = 0
    for b, (t, n) in enumerate(zip(targets, sizes)):
        if n > G:
            raise ValueError(f"image {b} has {n} target boxes, more than the capacity Gmax={G}")
        if n:
            boxes[b, :n] = t.get_field("normed_cxcy_boxes").to(device=device, dtype=torch.float32)
            tokens[b, :n] = pm[off:off + n]
        off += n
    count = torch.tensor(sizes, dtype=torch.int32).to(device)
    return boxes, count, tokens


def indices_from_match(match):
    """match int32 [B, Q] (GT per query, -1) -> the reference's list of (index_i, index_j) int64 CPU tensors, sorted by query
    index like scipy's output for a tall matrix.  One device-to-host copy."""
    m = match.cpu().long()
    out = []
    for b in range(m.shape[0]):
        i = (m[b] >= 0).nonzero().squeeze(1)
        out.append((i, m[b, i]))
    return out


class HungarianMatcher(nn.Module):
    """matcher.py:8-86: ``forward(outputs, targets, positive_map)`` -> list over images of (index_i, index_j) int64 CPU tensors,
    computed on the device (cost kernel + linear sum assignment)."""

    def __init__(self, cost_class: float = 1, cost_bbox: float = 1, cost_giou: float = 1, focal_alpha=0.25):
        super().__init__()
        self.cost_class, self.cost_bbox, self.cost_giou = cost_class, cost_bbox, cost_giou
        assert cost_class != 0 or cost_bbox != 0 or cost_giou != 0, "all costs cant be 0"
        self.focal_alpha = focal_alpha

    def match_flat(self, pred_logits, pred_boxes, gt_boxes, gt_count, gt_tokens):
        """pred_logits [L, B, Q, T], pred_boxes [L, B, Q, 4] + the GT pack -> ``ops.gdino_match`` dict (cost, match, norm)."""
        return ops.gdino_match(pred_logits, pred_boxes, gt_boxes, gt_count, gt_tokens, cost_class=self.cost_class,
                               cost_bbox=self.cost_bbox, cost_giou=self.cost_giou, focal_alpha=self.focal_alpha)

    @torch.no_grad()
    def forward(self, outputs, targets, positive_map):
        logits, boxes = outputs["pred_logits"], outputs["pred_boxes"]
        pack = gt_pack(targets, positive_map, logits.device)
        m = self.match_flat(logits.float().contiguous()[None], boxes.float().contiguous()[None], *pack)
        return indices_from_match(m["match"][0])


def build_matcher(args):
    """matcher.py:169-182.  ``SimpleMinsumMatcher`` is not part of the shipped configuration and is not built."""
    assert args.matcher_type in ["HungarianMatcher", "SimpleMinsumMatcher"], "Unknown args.matcher_type: {}".format(args.matcher_type)
    if args.matcher_type == "HungarianMatcher":
        return HungarianMatcher(cost_class=args.set_cost_class, cost_bbox=args.set_cost_bbox, cost_giou=args.set_cost_giou,
                                focal_alpha=args.focal_alpha)
    raise NotImplementedError("SimpleMinsumMatcher is not implemented (the shipped configuration uses HungarianMatcher)")
