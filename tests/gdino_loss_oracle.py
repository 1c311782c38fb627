"""GroundingDINO's Hungarian matching and set-prediction losses restated in fp32 torch, plus a loader that runs the reference's own
``SetCriterion`` / ``HungarianMatcher`` (groundingdino_new/models/GroundingDINO/{loss,matcher}.py) on CPU.

The restatement is what the device kernels (mqdet_b200/csrc/gdino_loss.cu) are compared against: the matching cost as the
reference's matcher computes it, the assignment by ``scipy.optimize.linear_sum_assignment`` on that cost, and the losses, which
are differentiable, so ``torch.autograd`` gives the reference gradients.  The loader only runs where the original sources are
present (``oracle.ref_loader.available()``); tests compare against its recorded results elsewhere (tests/golden/gdino_loss_pins.pt).

Documented where the reference leaves a case open (DESIGN.md §4):
  * a GT whose token row is empty has class cost 0 (the reference's mean over no tokens is NaN, and scipy raises on it), and
    its matched query gets the unmatched one-hot target (loss.py:60 does that already);
  * an image without GTs matches nothing: all its queries are unmatched;
  * assignment ties resolve as scipy resolves them.
"""
import math
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ALPHA, GAMMA = 0.25, 2.0
COST = (1.0, 5.0, 2.0)    # set_cost_class, set_cost_bbox, set_cost_giou
COEF = (2.0, 5.0, 2.0)    # loss_ce_coef, loss_bbox_coef, loss_giou_coef


def to_xyxy(b):
    cx, cy, w, h = b.unbind(-1)
    return torch.stack((cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h), dim=-1)


def _area(b):
    return (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])


def giou_matrix(a, b):
    """generalized_box_iou (box_ops.py:22-62): xyxy [N, 4] x [M, 4] -> [N, M]"""
    area1, area2 = _area(a), _area(b)
    lt = torch.max(a[:, None, :2], b[:, :2])
    rb = torch.min(a[:, None, 2:], b[:, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[:, :, 0] * wh[:, :, 1]
    union = area1[:, None] + area2 - inter
    iou = inter / (union + 1e-6)
    lt = torch.min(a[:, None, :2], b[:, :2])
    rb = torch.max(a[:, None, 2:], b[:, 2:])
    wh = (rb - lt).clamp(min=0)
    area = wh[:, :, 0] * wh[:, :, 1]
    return iou - (area - union) / (area + 1e-6)


def giou_pairs(a, b):
    """the diagonal of giou_matrix(a, b), computed pairwise (the same gradients as torch.diag of the full matrix)"""
    area1, area2 = _area(a), _area(b)
    wh = (torch.min(a[:, 2:], b[:, 2:]) - torch.max(a[:, :2], b[:, :2])).clamp(min=0)
    inter = wh[:, 0] * wh[:, 1]
    union = area1 + area2 - inter
    iou = inter / (union + 1e-6)
    wh = (torch.max(a[:, 2:], b[:, 2:]) - torch.min(a[:, :2], b[:, :2])).clamp(min=0)
    area = wh[:, 0] * wh[:, 1]
    return iou - (area - union) / (area + 1e-6)


def match_cost(logits, boxes, gt_boxes, gt_count, gt_tokens, cost=COST, alpha=ALPHA):
    """matcher.py:49-81 per image: logits [B, Q, T], boxes [B, Q, 4] -> cost fp32 [B, Q, Gmax] (0 beyond gt_count)."""
    B, Q, _ = logits.shape
    out = torch.zeros(B, Q, gt_boxes.shape[1], device=logits.device)
    for b in range(B):
        n = int(gt_count[b])
        if n == 0:
            continue
        p = logits[b].float().sigmoid()
        neg = (1 - alpha) * (p ** 2) * (-(1 - p + 1e-8).log())
        pos = alpha * ((1 - p) ** 2) * (-(p + 1e-8).log())
        cls = []
        for row in gt_tokens[b, :n] > 0:
            cls.append((pos[:, row] - neg[:, row]).mean(-1) if row.any() else torch.zeros(Q, device=logits.device))
        cls = torch.stack(cls).transpose(1, 0)
        tgt = gt_boxes[b, :n].float()
        l1 = torch.cdist(boxes[b].float(), tgt, p=1)
        giou = -giou_matrix(to_xyxy(boxes[b].float()), to_xyxy(tgt))
        out[b, :, :n] = cost[1] * l1 + cost[0] * cls + cost[2] * giou
    return out


def assign(cost, gt_count):
    """scipy.optimize.linear_sum_assignment per image, on the host as the reference does (C.cpu(), matcher.py:82): cost [B, Q, Gmax]
    -> match int64 [B, Q] (GT per query, -1) on the cost's device."""
    from scipy.optimize import linear_sum_assignment
    B, Q, _ = cost.shape
    c = cost.cpu()
    match = torch.full((B, Q), -1, dtype=torch.long)
    for b in range(B):
        n = int(gt_count[b])
        if n:
            i, j = linear_sum_assignment(c[b, :, :n].numpy())
            match[b, torch.as_tensor(i, dtype=torch.long)] = torch.as_tensor(j, dtype=torch.long)
    return match.to(cost.device)


def match_layers(logits, boxes, gt_boxes, gt_count, gt_tokens):
    """every layer: logits [L, B, Q, T], boxes [L, B, Q, 4] -> (cost [L, B, Q, Gmax], match int64 [L, B, Q])"""
    costs = torch.stack([match_cost(logits[l], boxes[l], gt_boxes, gt_count, gt_tokens) for l in range(logits.shape[0])])
    return costs, torch.stack([assign(costs[l], gt_count) for l in range(logits.shape[0])])


def _focal(x, y, alpha=ALPHA, gamma=GAMMA):
    p = torch.sigmoid(x)
    ce = torch.nn.functional.binary_cross_entropy_with_logits(x, y, reduction="none")
    pt = p * y + (1 - p) * (1 - y)
    return (alpha * y + (1 - alpha) * (1 - y)) * ce * (1 - pt) ** gamma


def token_targets(match, gt_tokens):
    """[B, Q, T]: the matched GT's token row; one-hot at T-1 for unmatched queries and rows that sum to 0 (loss.py:55-60)"""
    B, Q = match.shape
    T = gt_tokens.shape[-1]
    rows = torch.gather(gt_tokens.float(), 1, match.clamp(min=0)[..., None].expand(B, Q, T))
    tgt = torch.where((match >= 0)[..., None], rows, torch.zeros_like(rows))
    none = torch.zeros(T, device=gt_tokens.device)
    none[-1] = 1
    tgt[tgt.sum(-1) == 0] = none
    return tgt


def set_loss(logits, boxes, match, gt_boxes, gt_count, gt_tokens, text_mask=None, world=1, num_boxes_sum=None, coef=COEF):
    """loss.py:42-171: logits [L, B, Q, T] / boxes [L, B, Q, 4] (may require grad), match [L, B, Q] -> losses [L, 3] (weighted
    loss_ce, loss_bbox, loss_giou per layer)."""
    L, B, Q, T = logits.shape
    nb = max((float(gt_count.sum()) if num_boxes_sum is None else float(num_boxes_sum)) / world, 1.0)
    out = []
    for l in range(L):
        m = match[l]
        tgt = token_targets(m, gt_tokens)
        x = logits[l]
        if text_mask is not None:
            sel = (text_mask > 0)[:, None, :].expand(B, Q, T)
            el = _focal(torch.masked_select(x, sel), torch.masked_select(tgt, sel))
        else:
            el = _focal(x, tgt)
        ce = el.sum() / nb
        bi, qi = (m >= 0).nonzero(as_tuple=True)
        src = boxes[l][bi, qi]
        tb = gt_boxes.float()[bi, m[bi, qi]]
        l1 = torch.nn.functional.l1_loss(src, tb, reduction="none").sum() / nb
        gl = (1 - giou_pairs(to_xyxy(src), to_xyxy(tb))).sum() / nb
        out.append(torch.stack([ce * coef[0], l1 * coef[1], gl * coef[2]]))
    return torch.stack(out)


def losses_and_grads(logits, boxes, match, gt_boxes, gt_count, gt_tokens, text_mask=None, **kw):
    """set_loss with autograd: -> (losses [L, 3], d_logits, d_boxes) = the gradient of the sum of every returned loss"""
    x = logits.detach().clone().requires_grad_(True)
    bx = boxes.detach().clone().requires_grad_(True)
    losses = set_loss(x, bx, match, gt_boxes, gt_count, gt_tokens, text_mask, **kw)
    dl, db = torch.autograd.grad(losses.sum(), (x, bx))
    return losses.detach(), dl, db


# ---------------------------------------------------------------------------------------------------------------------------
# the reference's own SetCriterion / HungarianMatcher on CPU
# ---------------------------------------------------------------------------------------------------------------------------
def ref_modules():
    """groundingdino_new/models/GroundingDINO/{matcher,loss}.py with the reference's own util/box_ops.py, util/misc.py and
    maskrcnn_benchmark/layers/sigmoid_focal_loss.py (installed by tests/atss_oracle.py::rpn_loss)."""
    from oracle import ref_loader
    if "gdino_loss" in ref_loader._cache:
        return ref_loader._cache["gdino_loss"]
    import warnings
    import atss_oracle
    atss_oracle.rpn_loss()            # maskrcnn_benchmark.layers with TokenSigmoidFocalLoss / SigmoidFocalLoss / IOULoss
    ref_loader.gdino_package()        # groundingdino_new.util.misc
    load = ref_loader._load_file
    top, util = sys.modules["groundingdino_new"], sys.modules["groundingdino_new.util"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        util.box_ops = load("groundingdino_new.util.box_ops", "groundingdino_new/util/box_ops.py")
        models = sys.modules.get("groundingdino_new.models") or types.ModuleType("groundingdino_new.models")
        gd = sys.modules.get("groundingdino_new.models.GroundingDINO") or types.ModuleType("groundingdino_new.models.GroundingDINO")
        models.__path__, gd.__path__ = [], []
        sys.modules.update({"groundingdino_new.models": models, "groundingdino_new.models.GroundingDINO": gd})
        top.models, models.GroundingDINO = models, gd
        gd.utils = load("groundingdino_new.models.GroundingDINO.utils", "groundingdino_new/models/GroundingDINO/utils.py")
        gd.matcher = load("groundingdino_new.models.GroundingDINO.matcher", "groundingdino_new/models/GroundingDINO/matcher.py")
        gd.loss = load("groundingdino_new.models.GroundingDINO.loss", "groundingdino_new/models/GroundingDINO/loss.py")
    ref_loader._cache["gdino_loss"] = gd
    return gd


def _ref_cfg():
    from types import SimpleNamespace as NS
    return NS(GROUNDINGDINO=NS(loss_ce_coef=COEF[0], loss_bbox_coef=COEF[1], loss_giou_coef=COEF[2],
                               matcher=NS(matcher_type="HungarianMatcher", set_cost_class=COST[0], set_cost_bbox=COST[1],
                                          set_cost_giou=COST[2], focal_alpha=ALPHA)),
              MODEL=NS(DYHEAD=NS(FUSE_CONFIG=NS(TOKEN_ALPHA=ALPHA, TOKEN_GAMMA=GAMMA))))


def ref_targets(gt_boxes, gt_count, gt_tokens):
    """the GT pack as the reference's targets (BoxList with a normed_cxcy_boxes field) + positive_map [sum G, T]"""
    from mqdet_b200.structures.bounding_box import BoxList
    targets, pm = [], []
    for b in range(gt_boxes.shape[0]):
        n = int(gt_count[b])
        t = BoxList(to_xyxy(gt_boxes[b, :n].float()), (1, 1), mode="xyxy")
        t.add_field("normed_cxcy_boxes", gt_boxes[b, :n].float())
        targets.append(t)
        pm.append(gt_tokens[b, :n].float())
    return targets, torch.cat(pm)


def reference(logits, boxes, gt_boxes, gt_count, gt_tokens, text_mask=None):
    """The reference's SetCriterion (with its HungarianMatcher) on the outputs of L layers -> dict(match int64 [L, B, Q],
    losses [L, 3] (loss_ce, loss_bbox, loss_giou; the un-suffixed keys in row L-1), d_logits, d_boxes (autograd of the sum of the
    returned dict), keys (the dict's keys in order))."""
    gd = ref_modules()
    cfg = _ref_cfg()
    crit = gd.loss.SetCriterion(gd.matcher.build_matcher(cfg.GROUNDINGDINO.matcher), cfg)
    L, B, Q, T = logits.shape
    x = logits.detach().clone().requires_grad_(True)
    bx = boxes.detach().clone().requires_grad_(True)
    out = {"pred_logits": x[L - 1], "pred_boxes": bx[L - 1],
           "aux_outputs": [{"pred_logits": x[k], "pred_boxes": bx[k]} for k in range(L - 1)]}
    targets, pm = ref_targets(gt_boxes, gt_count, gt_tokens)
    tm = None if text_mask is None else text_mask > 0
    losses, indices = crit(out, targets, return_indices=True, text_mask=tm, positive_map=pm)
    dl, db = torch.autograd.grad(sum(losses.values()), (x, bx))
    match = torch.full((L, B, Q), -1, dtype=torch.long)
    for l, ind in enumerate(indices):          # aux layers first, the last layer at the end
        for b, (i, j) in enumerate(ind):
            match[l, b, i] = j
    vals = torch.stack([torch.stack([losses[f"{k}{'' if l == L - 1 else f'_{l}'}"].detach().float() for k in ("loss_ce", "loss_bbox",
                                                                                                           "loss_giou")])
                        for l in range(L)])
    return {"match": match, "losses": vals, "d_logits": dl, "d_boxes": db, "keys": list(losses)}


# ---------------------------------------------------------------------------------------------------------------------------
# seeded fixtures shared by the CPU and GPU tests and tools/prof_gdino_loss.py
# ---------------------------------------------------------------------------------------------------------------------------
REF_CASES = ("bench", "duplicates", "same_boxes", "empty_image", "full_caption")
CASES = REF_CASES + ("empty_tokens",)


def _gt_boxes(gen, n):
    cx, cy = torch.rand(n, generator=gen) * 0.8 + 0.1, torch.rand(n, generator=gen) * 0.8 + 0.1
    w = torch.exp(torch.empty(n).uniform_(math.log(0.02), math.log(0.6), generator=gen))
    h = torch.exp(torch.empty(n).uniform_(math.log(0.02), math.log(0.6), generator=gen))
    return torch.stack((cx, cy, w.clamp(max=2 * torch.minimum(cx, 1 - cx)), h.clamp(max=2 * torch.minimum(cy, 1 - cy))), 1)


def make_case(counts, L=6, B=2, Q=900, T=256, seed=0, caption_len=None, Gmax=None):
    """A GT pack with multi-token spans inside each caption, decoder outputs of L layers (-inf outside the text mask, as
    ContrastiveEmbed gives them) and the text mask -> dict(logits [L, B, Q, T], boxes [L, B, Q, 4], gt_boxes [B, Gmax, 4],
    gt_count [B], gt_tokens [B, Gmax, T], text_mask [B, T]), CPU fp32."""
    gen = torch.Generator().manual_seed(seed)
    G = max(1, max(counts)) if Gmax is None else Gmax
    caption_len = caption_len or [T - 60 - 37 * b for b in range(B)]
    mask = torch.zeros(B, T)
    gt_boxes, gt_tokens = torch.zeros(B, G, 4), torch.zeros(B, G, T)
    for b, n in enumerate(counts):
        mask[b, :caption_len[b]] = 1.0
        if n:
            gt_boxes[b, :n] = _gt_boxes(gen, n)
        for g in range(n):
            s = int(torch.randint(1, caption_len[b] - 4, (1,), generator=gen))
            gt_tokens[b, g, s:s + 1 + int(torch.randint(0, 4, (1,), generator=gen))] = 1.0
    logits = torch.randn(L, B, Q, T, generator=gen) * 2.0 - 3.0
    logits = logits.masked_fill(mask[None, :, None, :] == 0, float("-inf"))
    cxcy = torch.rand(L, B, Q, 2, generator=gen) * 0.9 + 0.05
    wh = torch.sigmoid(torch.randn(L, B, Q, 2, generator=gen) - 1.5)
    return {"logits": logits, "boxes": torch.cat((cxcy, wh), -1), "gt_boxes": gt_boxes,
            "gt_count": torch.tensor(counts, dtype=torch.int32), "gt_tokens": gt_tokens, "text_mask": mask}


def case(name, seed=0):
    s = 100 * CASES.index(name) + seed
    if name == "bench":            # the bench geometry: about 20 GTs per image with multi-token spans, padded text masks
        return make_case([19, 21], seed=s)
    if name == "duplicates":       # GTs 4..6 repeat 0..2 in box AND token row: identical cost columns
        c = make_case([7, 5], seed=s)
        c["gt_boxes"][0, 4:7] = c["gt_boxes"][0, 0:3]
        c["gt_tokens"][0, 4:7] = c["gt_tokens"][0, 0:3]
        return c
    if name == "same_boxes":       # groups of queries with identical boxes and logits (a zero last bbox_embed layer at
        c = make_case([12, 9], seed=s)  # initialisation gives identical boxes): identical cost rows
        for k in range(0, 900, 30):
            c["boxes"][:, :, k:k + 30] = c["boxes"][:, :, k:k + 1]
            c["logits"][:, :, k:k + 30] = c["logits"][:, :, k:k + 1]
        return c
    if name == "empty_image":      # the first image has no GT: all its queries are unmatched
        return make_case([0, 6], seed=s)
    if name == "full_caption":     # a caption that fills all 256 tokens: the unmatched one-hot at token 255 counts
        return make_case([8, 5], seed=s, caption_len=[256, 256])
    if name == "empty_tokens":     # a GT whose token row is empty (class cost 0, the unmatched one-hot target)
        c = make_case([6, 4], seed=s)
        c["gt_tokens"][0, 2] = 0.0
        c["gt_tokens"][1, 0] = 0.0
        return c
    raise KeyError(name)
