"""ATSS target assignment and the MQ-GLIP pre-training detection losses restated in fp32 torch, plus a loader that runs the
reference's own ``ATSSLossComputation`` (maskrcnn_benchmark/modeling/rpn/loss.py) on CPU.

The restatement is what the device kernels (mqdet_b200/csrc/atss_loss.cu) are compared against; it is differentiable, so
``torch.autograd`` gives the reference gradients.  The loader only runs where the original sources are present
(``oracle.ref_loader.available()``); tests compare against its recorded results elsewhere (tests/golden/atss_loss_pins.pt).

Documented where the reference leaves an order unspecified:
  * the per-level top-k by centre distance keeps the lower anchor index on a tie at the cut (stable sort);
  * an anchor claimed by several GTs goes to the highest IoU, then to the lowest GT index (``torch.max``'s first occurrence);
  * an image without GT boxes is all-negative (the reference raises: max over an empty dimension).
"""
import math
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mqdet_b200.ops import base_anchor  # noqa: E402  (pure Python: the square base window of one level)

INF = 1e8
CLAMP = math.log(1000.0 / 16)
STRIDES = (8, 16, 32, 64, 128)
SIZES = (64, 128, 256, 512, 1024)


def level_sizes(h, w, nlev=5):
    """FPN grid of an (h, w) image padded to a multiple of 32 (P3..P7: stride 8 convs, then stride-2 3x3 convs for P6 / P7)."""
    H, W = -(-h // 32) * 32, -(-w // 32) * 32
    sizes = [(H // 8, W // 8)]
    for _ in range(nlev - 1):
        ph, pw = sizes[-1]
        sizes.append(((ph - 1) // 2 + 1, (pw - 1) // 2 + 1) if len(sizes) >= 3 else (ph // 2, pw // 2))
    return sizes


def anchors(sizes, strides=STRIDES, anchor_sizes=SIZES):
    """[N, 4] fp32 anchors of all levels (one per location), as AnchorGenerator.grid_anchors builds them; + level of each row."""
    out, lvl = [], []
    for l, ((h, w), s, a) in enumerate(zip(sizes, strides, anchor_sizes)):
        sx = torch.arange(0, w * s, step=s, dtype=torch.float32)
        sy = torch.arange(0, h * s, step=s, dtype=torch.float32)
        yy, xx = torch.meshgrid(sy, sx, indexing="ij")
        xx, yy = xx.reshape(-1), yy.reshape(-1)
        shifts = torch.stack((xx, yy, xx, yy), dim=1)
        out.append(shifts + torch.tensor(base_anchor(s, a), dtype=torch.float32)[None])
        lvl.append(torch.full((h * w,), l, dtype=torch.long))
    return torch.cat(out), torch.cat(lvl)


def _iou(a, g):
    """boxlist_iou (TO_REMOVE = 1): [N, 4] x [G, 4] -> [N, G]"""
    area1 = (a[:, 2] - a[:, 0] + 1) * (a[:, 3] - a[:, 1] + 1)
    area2 = (g[:, 2] - g[:, 0] + 1) * (g[:, 3] - g[:, 1] + 1)
    lt = torch.max(a[:, None, :2], g[None, :, :2])
    rb = torch.min(a[:, None, 2:], g[None, :, 2:])
    wh = (rb - lt + 1).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    return inter / (area1[:, None] + area2[None] - inter)


def encode(g, a):
    """BoxCoder.encode, weights (10, 10, 5, 5), TO_REMOVE = 1"""
    aw, ah = a[:, 2] - a[:, 0] + 1, a[:, 3] - a[:, 1] + 1
    acx, acy = (a[:, 2] + a[:, 0]) / 2, (a[:, 3] + a[:, 1]) / 2
    gw, gh = g[:, 2] - g[:, 0] + 1, g[:, 3] - g[:, 1] + 1
    gcx, gcy = (g[:, 2] + g[:, 0]) / 2, (g[:, 3] + g[:, 1]) / 2
    return torch.stack((10.0 * (gcx - acx) / aw, 10.0 * (gcy - acy) / ah, 5.0 * torch.log(gw / aw), 5.0 * torch.log(gh / ah)), 1)


def decode(p, a):
    """BoxCoder.decode, weights (10, 10, 5, 5), TO_REMOVE = 1, dw / dh clamped at log(1000 / 16)"""
    aw, ah = a[:, 2] - a[:, 0] + 1, a[:, 3] - a[:, 1] + 1
    acx, acy = (a[:, 2] + a[:, 0]) / 2, (a[:, 3] + a[:, 1]) / 2
    dx, dy = p[:, 0] / 10.0, p[:, 1] / 10.0
    dw, dh = torch.clamp(p[:, 2] / 5.0, max=CLAMP), torch.clamp(p[:, 3] / 5.0, max=CLAMP)
    cx, cy = dx * aw + acx, dy * ah + acy
    w, h = torch.exp(dw) * aw, torch.exp(dh) * ah
    return torch.stack((cx - 0.5 * (w - 1), cy - 0.5 * (h - 1), cx + 0.5 * (w - 1), cy + 0.5 * (h - 1)), 1)


def centerness(t, a):
    acx, acy = (a[:, 2] + a[:, 0]) / 2, (a[:, 3] + a[:, 1]) / 2
    l, t_, r, b = acx - t[:, 0], acy - t[:, 1], t[:, 2] - acx, t[:, 3] - acy
    lr, tb = torch.stack((l, r), 1), torch.stack((t_, b), 1)
    return torch.sqrt((lr.min(1)[0] / lr.max(1)[0]) * (tb.min(1)[0] / tb.max(1)[0]))


def assign_image(A, lvl, gt, topk=9):
    """ATSS assignment of one image: -> (match int64 [N] (-1 = unmatched), per-GT candidate IoU thresholds [G],
    candidate IoUs [sum k, G])."""
    N, G = A.shape[0], gt.shape[0]
    if G == 0:
        return torch.full((N,), -1, dtype=torch.long, device=A.device), torch.zeros(0), torch.zeros(0, 0)
    ious = _iou(A, gt)
    gc = torch.stack(((gt[:, 2] + gt[:, 0]) / 2.0, (gt[:, 3] + gt[:, 1]) / 2.0), 1)
    ac = torch.stack(((A[:, 2] + A[:, 0]) / 2.0, (A[:, 3] + A[:, 1]) / 2.0), 1)
    dist = (ac[:, None, :] - gc[None, :, :]).pow(2).sum(-1).sqrt()
    cand = []
    for l in range(int(lvl.max()) + 1):
        idx = (lvl == l).nonzero().squeeze(1)
        s, k = int(idx[0]), min(topk, idx.numel())
        cand.append(torch.sort(dist[idx], dim=0, stable=True).indices[:k] + s)
    cand = torch.cat(cand)                                          # [sum k, G]
    cols = torch.arange(G, device=A.device)[None].expand_as(cand)
    ciou = ious[cand, cols]
    thr = ciou.mean(0) + ciou.std(0)
    inside = torch.stack((ac[cand, 0] - gt[None, :, 0], ac[cand, 1] - gt[None, :, 1], gt[None, :, 2] - ac[cand, 0],
                          gt[None, :, 3] - ac[cand, 1]), 0).min(0)[0] > 0.01
    pos = (ciou >= thr[None]) & inside
    claimed = torch.full((N, G), -INF, device=A.device)
    claimed[cand[pos], cols[pos]] = ious[cand[pos], cols[pos]]
    best = claimed.max(1)[0]
    first = torch.where(claimed == best[:, None], torch.arange(G, device=A.device)[None], torch.full_like(claimed, G, dtype=torch.long)).min(1)[0]
    return torch.where(best == -INF, torch.full_like(first, -1), first), thr, ciou


def atss_targets(sizes, gt_boxes, gt_count, topk=9):
    """GT pack (gt_boxes [B, Gmax, 4], gt_count [B]) -> match int64 [B, N]"""
    A, lvl = anchors(sizes)
    return torch.stack([assign_image(A, lvl, gt_boxes[b, :int(gt_count[b])].float(), topk)[0] for b in range(gt_boxes.shape[0])])


def scale_per_anchor(sizes, reg_scales):
    _, lvl = anchors(sizes)
    return torch.tensor([float(s) for s in reg_scales], dtype=torch.float32)[lvl]


def _focal(x, y, alpha=0.25, gamma=2.0):
    p = torch.sigmoid(x)
    ce = torch.nn.functional.binary_cross_entropy_with_logits(x, y, reduction="none")
    pt = p * y + (1 - p) * (1 - y)
    return (alpha * y + (1 - alpha) * (1 - y)) * ce * (1 - pt) ** gamma


def token_targets(match, gt_tokens):
    """[B, N, T]: the matched GT's token row, one-hot at T-1 for unmatched anchors"""
    B, N = match.shape
    T = gt_tokens.shape[-1]
    rows = torch.gather(gt_tokens.float(), 1, match.clamp(min=0)[..., None].expand(B, N, T))
    none = torch.zeros(T, device=gt_tokens.device)
    none[-1] = 1
    return torch.where((match >= 0)[..., None], rows, none)


def atss_loss(logits, reg_ctr, match, sizes, gt_boxes, gt_labels, gt_tokens, reg_scales, text_mask=None, world=1,
              norm=None, reg_weight=2.0):
    """-> dict(loss_reg, loss_centerness, loss_dot_product_token, loss_cls (0-dim), pos [B, N] bool, reg_targets [P, 4],
    ctr_targets [P]).  logits [B, N, T] / reg_ctr [B, N, 5] may require grad.  ``norm`` = the all-rank (num_pos, sum ctr)
    (default: this rank's)."""
    dev = logits.device
    A = anchors(sizes)[0].to(dev)
    B, N, T = logits.shape
    sc = scale_per_anchor(sizes, reg_scales).to(dev)
    box = reg_ctr[..., :4] * sc[None, :, None]
    lab = torch.where(match >= 0, torch.gather(gt_labels.long(), 1, match.clamp(min=0)), torch.zeros_like(match))
    pos = lab > 0
    num_pos = float(pos.sum())
    tgt = token_targets(match, gt_tokens)
    el = _focal(logits, tgt)
    if text_mask is not None:
        el = el * (text_mask > 0)[:, None, :].float()
    ai = pos.nonzero()
    g = gt_boxes.float()[ai[:, 0], match[pos]]
    a = A[ai[:, 1]]
    reg_t = encode(g, a)
    tb = decode(reg_t, a)
    ctr_t = centerness(tb, a)
    np_all, ctr_all = (num_pos, float(ctr_t.sum())) if norm is None else (float(norm[0]), float(norm[1]))
    npa = max(np_all / world, 1.0)
    token = el.sum() / npa
    if num_pos > 0:
        pb = decode(box[pos], a)
        px1, py1 = pb[:, 0], pb[:, 1]
        px2, py2 = torch.max(px1, pb[:, 2]), torch.max(py1, pb[:, 3])
        pa = (px2 - px1) * (py2 - py1)
        ta = (tb[:, 2] - tb[:, 0]) * (tb[:, 3] - tb[:, 1])
        ix1, iy1 = torch.max(px1, tb[:, 0]), torch.max(py1, tb[:, 1])
        ix2, iy2 = torch.min(px2, tb[:, 2]), torch.min(py2, tb[:, 3])
        m = (iy2 > iy1) & (ix2 > ix1)
        ai_ = torch.where(m, (ix2 - ix1) * (iy2 - iy1), torch.zeros_like(ix1))
        ex1, ey1 = torch.min(px1, tb[:, 0]), torch.min(py1, tb[:, 1])
        ex2, ey2 = torch.max(px2, tb[:, 2]), torch.max(py2, tb[:, 3])
        ae = (ex2 - ex1) * (ey2 - ey1) + 1e-7
        au = pa + ta - ai_ + 1e-7
        losses = 1 - (ai_ / au - (ae - au) / ae)
        s = (losses * ctr_t).sum() if ctr_t.sum() > 0 else losses.sum()
        reg = s / (ctr_all / world) * reg_weight
        ctr = torch.nn.functional.binary_cross_entropy_with_logits(reg_ctr[..., 4][pos], ctr_t, reduction="sum") / npa
    else:
        reg = box[pos].sum()
        ctr = reg_ctr[..., 4][pos].sum()
    return {"loss_reg": reg, "loss_centerness": ctr, "loss_dot_product_token": token, "loss_cls": torch.zeros((), device=dev),
            "pos": pos, "reg_targets": reg_t, "ctr_targets": ctr_t, "num_pos": num_pos, "ctr_sum": float(ctr_t.sum())}


def losses_and_grads(logits, reg_ctr, match, sizes, gt_boxes, gt_labels, gt_tokens, reg_scales, text_mask=None, **kw):
    """atss_loss with autograd: -> (losses [4] = (reg, centerness, token, cls), d_logits, d_reg_ctr, the atss_loss dict)"""
    x = logits.detach().clone().requires_grad_(True)
    r = reg_ctr.detach().clone().requires_grad_(True)
    out = atss_loss(x, r, match, sizes, gt_boxes, gt_labels, gt_tokens, reg_scales, text_mask, **kw)
    total = out["loss_reg"] + out["loss_centerness"] + out["loss_dot_product_token"]
    dl, dr = torch.autograd.grad(total, (x, r), allow_unused=True)
    dl = torch.zeros_like(x) if dl is None else dl
    dr = torch.zeros_like(r) if dr is None else dr
    vals = torch.stack([out[k].detach().float().reshape(()) for k in ("loss_reg", "loss_centerness", "loss_dot_product_token", "loss_cls")])
    return vals, dl, dr, out


# ---------------------------------------------------------------------------------------------------------------------------
# the reference's own ATSSLossComputation on CPU
# ---------------------------------------------------------------------------------------------------------------------------
def rpn_loss():
    """maskrcnn_benchmark/modeling/rpn/loss.py with the reference's own boxlist_ops / bounding_box / matcher / sigmoid_focal_loss
    / amp files.  Shims: an empty ``_C`` (only the CUDA focal loss reaches it), ``utils.comm`` with world size 1, an empty
    ``shallow_contrastive_loss_helper`` (the shallow contrastive loss is off), and the tokenizer (captions are passed as None;
    the file only constructs one)."""
    from oracle import ref_loader
    if "rpn_loss" in ref_loader._cache:
        return ref_loader._cache["rpn_loss"]
    ref_loader.anchor_generator()  # installs the structures package (bounding_box, boxlist_ops) and modeling.utils
    load = ref_loader._load_file
    pkg = sys.modules["maskrcnn_benchmark"]
    utils = sys.modules["maskrcnn_benchmark.utils"]
    modeling = sys.modules["maskrcnn_benchmark.modeling"]
    if not hasattr(pkg, "_C"):
        pkg._C = types.ModuleType("maskrcnn_benchmark._C")
        sys.modules["maskrcnn_benchmark._C"] = pkg._C
    layers = sys.modules.get("maskrcnn_benchmark.layers")
    if layers is None:
        layers = types.ModuleType("maskrcnn_benchmark.layers")
        sys.modules["maskrcnn_benchmark.layers"] = layers
        pkg.layers = layers
    sfl = load("maskrcnn_benchmark.layers.sigmoid_focal_loss", "maskrcnn_benchmark/layers/sigmoid_focal_loss.py")
    iou = load("maskrcnn_benchmark.layers.iou_loss", "maskrcnn_benchmark/layers/iou_loss.py")
    sl1 = load("maskrcnn_benchmark.layers.smooth_l1_loss", "maskrcnn_benchmark/layers/smooth_l1_loss.py")
    layers.SigmoidFocalLoss, layers.TokenSigmoidFocalLoss = sfl.SigmoidFocalLoss, sfl.TokenSigmoidFocalLoss
    layers.IOULoss, layers.smooth_l1_loss = iou.IOULoss, sl1.smooth_l1_loss
    load("maskrcnn_benchmark.modeling.matcher", "maskrcnn_benchmark/modeling/matcher.py")
    load("maskrcnn_benchmark.modeling.balanced_positive_negative_sampler",
         "maskrcnn_benchmark/modeling/balanced_positive_negative_sampler.py")
    comm = types.ModuleType("maskrcnn_benchmark.utils.comm")
    comm.get_world_size = lambda: 1
    comm.reduce_sum = lambda t: t
    helper = types.ModuleType("maskrcnn_benchmark.utils.shallow_contrastive_loss_helper")
    sys.modules.update({"maskrcnn_benchmark.utils.comm": comm, "maskrcnn_benchmark.utils.shallow_contrastive_loss_helper": helper})
    utils.comm, utils.shallow_contrastive_loss_helper = comm, helper
    utils.amp = load("maskrcnn_benchmark.utils.amp", "maskrcnn_benchmark/utils/amp.py")
    prev = sys.modules.get("maskrcnn_benchmark.modeling.rpn.loss")
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        mod = load("maskrcnn_benchmark.modeling.rpn.loss", "maskrcnn_benchmark/modeling/rpn/loss.py")
    if prev is not None:  # ref_loader.vldyhead() keeps its stub under this name
        sys.modules["maskrcnn_benchmark.modeling.rpn.loss"] = prev

    class _NoTokenizer:
        @staticmethod
        def from_pretrained(*a, **k):
            return None

    mod.AutoTokenizer = _NoTokenizer
    ref_loader._cache["rpn_loss"] = mod
    return mod


def _ref_cfg():
    from types import SimpleNamespace as NS
    fc = NS(USE_TOKEN_LOSS=False, USE_DOT_PRODUCT_TOKEN_LOSS=True, TOKEN_ALPHA=0.25, TOKEN_GAMMA=2.0, USE_CONTRASTIVE_ALIGN_LOSS=False,
            USE_SHALLOW_CONTRASTIVE_LOSS=False, USE_BACKBONE_SHALLOW_CONTRASTIVE_LOSS=False, MLM_LOSS=False)
    return NS(MODEL=NS(FOCAL=NS(LOSS_GAMMA=2.0, LOSS_ALPHA=0.25, FG_IOU_THRESHOLD=0.5, BG_IOU_THRESHOLD=0.4),
                       DYHEAD=NS(FUSE_CONFIG=fc), LANGUAGE_BACKBONE=NS(MODEL_TYPE="bert-base-uncased", TOKENIZER_TYPE="bert-base-uncased"),
                       RPN=NS(ASPECT_RATIOS=(1.0,), SCALES_PER_OCTAVE=1), ATSS=NS(TOPK=9, REG_LOSS_WEIGHT=2.0)))


def reference(logits, reg_ctr, image_hw, sizes, gt_boxes, gt_labels, gt_count, gt_tokens, reg_scales, text_mask=None):
    """The reference's ATSSLossComputation on the same inputs (every image must have >= 1 GT) -> dict(labels [B, N],
    reg_targets [B, N, 4], token_labels [B, N, T], losses [4] = (reg, centerness, token, cls * 0), d_logits, d_reg_ctr)."""
    mod = rpn_loss()
    BoxList = sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList
    ev = mod.ATSSLossComputation(_ref_cfg(), None)
    from oracle import ref_loader
    ref_loader.vldyhead(lambda *a: None)
    ev.box_coder = sys.modules["maskrcnn_benchmark.modeling.rpn.vldyhead"].BoxCoder(None)
    B, N, T = logits.shape
    h, w = image_hw
    A, _ = anchors(sizes)
    offs = [0]
    for hh, ww in sizes:
        offs.append(offs[-1] + hh * ww)
    anc = [[BoxList(A[offs[l]:offs[l + 1]], (w, h), mode="xyxy") for l in range(len(sizes))] for _ in range(B)]
    targets, pm = [], []
    for b in range(B):
        g = int(gt_count[b])
        t = BoxList(gt_boxes[b, :g].float(), (w, h), mode="xyxy")
        t.add_field("labels", gt_labels[b, :g].long())
        targets.append(t)
        pm.append(gt_tokens[b, :g].float())
    pm = torch.cat(pm)
    x = logits.detach().clone().requires_grad_(True)
    r = reg_ctr.detach().clone().requires_grad_(True)
    sc = scale_per_anchor(sizes, reg_scales)
    box = r[..., :4] * sc[None, :, None]
    lv = lambda t, l: t[:, offs[l]:offs[l + 1]].transpose(1, 2).reshape(B, t.shape[-1], *sizes[l])  # noqa: E731
    box_l = [lv(box, l) for l in range(len(sizes))]
    ctr_l = [lv(r[..., 4:5], l) for l in range(len(sizes))]
    cls_l = [torch.zeros(B, 1, *s) for s in sizes]
    dots = [x[:, offs[l]:offs[l + 1]] for l in range(len(sizes))]
    labels, reg_t, tok_l = ev.prepare_targets(targets, anc, None, pm, None)[:3]
    out = ev(cls_l, box_l, ctr_l, targets, anc, None, pm, None, None, None, dots, text_mask, None)
    cls_loss, reg_loss, ctr_loss, dot_loss = out[0], out[1], out[2], out[5]
    dl, dr = torch.autograd.grad(reg_loss + ctr_loss + dot_loss, (x, r), allow_unused=True)
    dl = torch.zeros_like(x) if dl is None else dl
    dr = torch.zeros_like(r) if dr is None else dr
    losses = torch.stack([reg_loss.detach().float().reshape(()), ctr_loss.detach().float().reshape(()),
                          dot_loss.detach().float().reshape(()), (0.0 * cls_loss).detach().float().reshape(())])
    return {"labels": torch.stack(labels), "reg_targets": torch.stack(reg_t), "token_labels": torch.stack(tok_l).float(),
            "losses": losses, "d_logits": dl, "d_reg_ctr": dr}


# ---------------------------------------------------------------------------------------------------------------------------
# seeded fixtures shared by the CPU and GPU tests and tools/prof_atss_loss.py
# ---------------------------------------------------------------------------------------------------------------------------
CASES = ("bench2", "duplicates", "overlap", "small", "padded_mask", "zero_pos", "empty_gt", "ties")
REG_SCALES = (1.0, 0.9, 1.1, 1.2, 0.8)


def _boxes(gen, n, h, w, smin=8.0, smax=None):
    smax = smax or 0.8 * min(h, w)
    s = torch.exp(torch.empty(n).uniform_(math.log(smin), math.log(smax), generator=gen))
    ar = torch.exp(torch.empty(n).uniform_(-0.7, 0.7, generator=gen))
    bw, bh = (s * ar).clamp(max=w - 2), (s / ar).clamp(max=h - 2)
    x1 = torch.rand(n, generator=gen) * (w - 1 - bw)
    y1 = torch.rand(n, generator=gen) * (h - 1 - bh)
    return torch.stack((x1, y1, x1 + bw, y1 + bh), 1)


def threshold_margin(sizes, gt_boxes, gt_count, topk=9):
    """smallest |candidate IoU - threshold| / threshold over all GTs (the exact-assignment comparisons need it > 1e-6)"""
    A, lvl = anchors(sizes)
    m = float("inf")
    for b in range(gt_boxes.shape[0]):
        g = int(gt_count[b])
        if g:
            _, thr, ciou = assign_image(A, lvl, gt_boxes[b, :g].float(), topk)
            m = min(m, float(((ciou - thr[None]).abs() / thr[None].abs().clamp(min=1e-30)).min()))
    return m


def case(name, T=256, seed=0):
    """-> dict(image_hw, sizes, gt_boxes [B, Gmax, 4], gt_labels [B, Gmax], gt_count [B], gt_tokens [B, Gmax, T],
    logits [B, N, T], reg_ctr [B, N, 5], reg_scales, text_mask [B, T] | None), CPU fp32, seeded."""
    for attempt in range(50):
        gen = torch.Generator().manual_seed(1000 * CASES.index(name) + seed + 7919 * attempt)
        c = _case(name, T, gen)
        if name == "empty_gt" or threshold_margin(c["sizes"], c["gt_boxes"], c["gt_count"]) > 1e-6:
            return c
    raise AssertionError(f"{name}: no seed keeps every candidate IoU away from its threshold")


def _case(name, T, gen):
    h, w, B, counts = {"bench2": (800, 1344, 2, [20, 21]), "duplicates": (320, 480, 1, [6]), "overlap": (320, 480, 2, [5, 4]),
                       "small": (160, 224, 2, [3, 2]), "padded_mask": (256, 320, 2, [4, 3]), "zero_pos": (256, 320, 1, [3]),
                       "empty_gt": (256, 320, 2, [0, 3]), "ties": (320, 480, 1, [6])}[name]
    G = max(max(counts), 1)
    boxes = torch.zeros(B, G, 4)
    for b, n in enumerate(counts):
        if n:
            boxes[b, :n] = _boxes(gen, n, h, w)
    if name == "duplicates":  # boxes 3 / 4 / 5 repeat 0 / 1 / 1 (different labels and token rows)
        boxes[0, 3], boxes[0, 4], boxes[0, 5] = boxes[0, 0], boxes[0, 1], boxes[0, 1]
    if name == "overlap":  # nested and shifted copies of one box compete for the same anchors
        for b in range(B):
            base = _boxes(gen, 1, h, w, 60.0, 200.0)[0]
            for j in range(1, counts[b]):
                d = torch.rand(4, generator=gen) * 12 - 6
                boxes[b, j] = torch.stack((base[0] + d[0], base[1] + d[1], base[2] + d[2], base[3] + d[3]))
            boxes[b, 0] = base
    if name == "ties":  # centres half-way between two P3 anchor centres: equal distances at the top-9 cut
        for j in range(counts[0]):
            cx = 8.0 * (6 + 7 * j) + 7.5
            cy = 8.0 * (5 + 4 * j) + 3.5
            half = 12.0 + 4.0 * j
            boxes[0, j] = torch.tensor([cx - half, cy - half * 0.75, cx + half, cy + half * 0.75])
    labels = torch.randint(1, 81, (B, G), generator=gen, dtype=torch.int32)
    if name == "zero_pos":
        labels.zero_()
    tokens = torch.zeros(B, G, T)
    for b in range(B):
        for g in range(G):
            s = int(torch.randint(1, max(T - 40, 2), (1,), generator=gen))
            tokens[b, g, s:s + 1 + int(torch.randint(0, 3, (1,), generator=gen))] = 1.0
    sizes = level_sizes(h, w)
    N = sum(a * c for a, c in sizes)
    logits = torch.randn(B, N, T, generator=gen) * 2.0 - 3.0
    reg_ctr = torch.randn(B, N, 5, generator=gen) * 0.5
    if name == "bench2":  # predicted dw / dh past the decode clamp on a fifth of the anchors
        sel = torch.rand(B, N, generator=gen) < 0.2
        reg_ctr[..., 2][sel] = 30.0
        reg_ctr[..., 3][sel & (torch.rand(B, N, generator=gen) < 0.5)] = 25.0
    mask = None
    if name in ("padded_mask", "bench2"):
        mask = torch.zeros(B, T)
        for b in range(B):
            mask[b, :T - 37 * (b + 1)] = 1.0
            mask[b, -1] = 1.0  # the no-object token stays in use
    return {"image_hw": (h, w), "sizes": sizes, "gt_boxes": boxes, "gt_labels": labels,
            "gt_count": torch.tensor(counts, dtype=torch.int32), "gt_tokens": tokens, "logits": logits, "reg_ctr": reg_ctr,
            "reg_scales": REG_SCALES, "text_mask": mask}
