"""GPU: GroundingDINO Hungarian matching and set-prediction losses (mqdet_b200/csrc/gdino_loss.cu) against the fp32 restatement
(tests/gdino_loss_oracle.py, itself pinned to the reference's SetCriterion by tests/test_gdino_loss_cpu.py) and, for the
assignment, against scipy.optimize.linear_sum_assignment on the kernel's own cost matrix."""
import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment as scipy_lsa

import gdino_loss_oracle as go

pytestmark = pytest.mark.gpu

TIE_FREE = ("bench", "empty_image", "full_caption", "empty_tokens")


def _dev(c, dev):
    return {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in c.items()}


def _scipy_match(cost, count):
    """scipy on a [Q, >= count] cost matrix -> match int64 [Q]"""
    m = torch.full((cost.shape[0],), -1, dtype=torch.long)
    if count:
        i, j = scipy_lsa(cost[:, :count].numpy())
        m[torch.as_tensor(i, dtype=torch.long)] = torch.as_tensor(j, dtype=torch.long)
    return m


def _grad_ok(got, ref, what):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    err = (got - ref).abs().max().item()
    bound = 1e-5 * ref.abs().max().item() + 1e-7
    assert err <= bound, f"{what}: max|err| {err:.3e} > {bound:.3e}"


def _run(d):
    from mqdet_b200 import ops
    m = ops.gdino_match(d["logits"], d["boxes"], d["gt_boxes"], d["gt_count"], d["gt_tokens"])
    losses, dl, db, norm = ops.gdino_set_loss(d["logits"], d["boxes"], d["gt_boxes"], d["gt_count"], d["gt_tokens"], d["text_mask"],
                                              targets=m)
    return m, losses, dl, db, norm


@pytest.mark.parametrize("name", go.CASES)
def test_cost_assignment_losses_and_gradients(dev, name):
    c = go.case(name)
    m, losses, dl, db, norm = _run(_dev(c, dev))
    torch.cuda.synchronize()
    cost, match = m["cost"].cpu(), m["match"].cpu().long()
    L, B = cost.shape[:2]
    rcost, rmatch = go.match_layers(c["logits"], c["boxes"], c["gt_boxes"], c["gt_count"], c["gt_tokens"])
    assert torch.isfinite(cost).all()
    err = (cost - rcost).abs().max().item()
    assert err <= 1e-5 * rcost.abs().max().item(), f"{name}: cost max|err| {err:.3e}"
    # the assignment is scipy's on the kernel's own cost, index for index
    for l in range(L):
        for b in range(B):
            assert torch.equal(match[l, b], _scipy_match(cost[l, b], int(c["gt_count"][b]))), (name, l, b)
    if name in TIE_FREE:
        assert torch.equal(match, rmatch), f"{name}: assignment differs from the restatement's"
    assert float(norm[0]) == float(c["gt_count"].sum())
    vals, rdl, rdb = go.losses_and_grads(c["logits"], c["boxes"], match, c["gt_boxes"], c["gt_count"], c["gt_tokens"], c["text_mask"])
    lc = losses.cpu()
    assert ((lc - vals).abs() <= 1e-5 * vals.abs() + 1e-12).all(), (name, lc, vals)
    _grad_ok(dl, rdl, f"{name}: d_logits")
    _grad_ok(db, rdb, f"{name}: d_boxes")
    assert torch.isfinite(dl).all() and torch.isfinite(db).all()
    if name == "empty_image":
        assert (match[:, 0] == -1).all()


def test_reruns_are_bit_identical(dev):
    d = _dev(go.case("bench"), dev)
    a, b = _run(d), _run(d)
    torch.cuda.synchronize()
    for k in ("cost", "match", "norm"):
        assert torch.equal(a[0][k], b[0][k])
    for x, y in zip(a[1:], b[1:]):
        assert torch.equal(x, y)


def test_world_normaliser_divides_and_clamps(dev):
    from mqdet_b200 import ops
    c = go.case("empty_image")
    d = _dev(c, dev)
    m = ops.gdino_match(d["logits"], d["boxes"], d["gt_boxes"], d["gt_count"], d["gt_tokens"])
    match = m["match"].cpu().long()
    for total, world in ((13.0, 2), (1.0, 2)):       # 6.5; 0.5 -> clamped to 1
        m["norm"].fill_(total)
        losses, _, db, _ = ops.gdino_set_loss(d["logits"], d["boxes"], d["gt_boxes"], d["gt_count"], d["gt_tokens"], d["text_mask"],
                                              targets=m, world=world)
        vals, _, rdb = go.losses_and_grads(c["logits"], c["boxes"], match, c["gt_boxes"], c["gt_count"], c["gt_tokens"],
                                           c["text_mask"], world=world, num_boxes_sum=total)
        lc = losses.cpu()
        assert ((lc - vals).abs() <= 1e-5 * vals.abs() + 1e-12).all(), (total, lc, vals)
        _grad_ok(db, rdb, f"d_boxes at world {world}")


def _random_problems(gen, shapes, ties=False):
    """[(Q, G)] -> cost fp32 [P, Qmax, Gmax] (Q = Qmax for all; G varies through counts), counts [P]"""
    Q = max(s[0] for s in shapes)
    G = max(max(s[1] for s in shapes), 1)
    cost = torch.rand(len(shapes), Q, G, generator=gen)
    if ties:
        cost = torch.randint(0, 4, (len(shapes), Q, G), generator=gen).float()
        for p in range(len(shapes)):   # duplicated rows and columns
            cost[p, 1::3] = cost[p, 0::3][:cost[p, 1::3].shape[0]]
            cost[p, :, 1::2] = cost[p, :, 0::2][:, :cost[p, :, 1::2].shape[1]]
    return cost, torch.tensor([s[1] for s in shapes], dtype=torch.int32)


@pytest.mark.parametrize("Q,shapes,ties", [
    (64, [(64, 64), (64, 40), (64, 1), (64, 0)], False),
    (300, [(300, 300), (300, 120), (300, 7)], False),
    (900, [(900, 300), (900, 200), (900, 50), (900, 1), (900, 0)], False),
    (64, [(64, 64), (64, 33), (64, 12)], True),
    (900, [(900, 300), (900, 200), (900, 20)], True),
])
def test_linear_sum_assignment_equals_scipy(dev, Q, shapes, ties):
    from mqdet_b200 import ops
    gen = torch.Generator().manual_seed(Q * 7 + len(shapes) + int(ties))
    cost, counts = _random_problems(gen, shapes, ties)
    match = ops.linear_sum_assignment(cost.to(dev), counts.to(dev)).cpu().long()
    for p in range(cost.shape[0]):
        want = _scipy_match(cost[p], int(counts[p]))
        assert torch.equal(match[p], want), (Q, shapes[p], ties, (match[p] != want).nonzero()[:5].tolist())
        if int(counts[p]):
            i = (want >= 0).nonzero().squeeze(1)
            assert np.isclose(float(cost[p][i, want[i]].double().sum()), float(cost[p][i, match[p][i]].double().sum()))


def test_cuda_graph_replay_with_new_gt_contents(dev):
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.modeling.groundingdino.loss import SetCriterion
    from mqdet_b200.modeling.groundingdino.matcher import build_matcher
    cfg = mq_groundingdino_t_cfg()
    crit = SetCriterion(build_matcher(cfg.GROUNDINGDINO.matcher), cfg)
    G = 24
    c1 = go.make_case([19, 21], seed=5, Gmax=G)
    c2 = go.make_case([7, 23], seed=6, Gmax=G)
    d1, d2 = _dev(c1, dev), _dev(c2, dev)
    keys = ("logits", "boxes", "gt_boxes", "gt_count", "gt_tokens", "text_mask")
    static = {k: d1[k].clone() for k in keys}

    def step():
        r = crit.forward_flat(static["logits"], static["boxes"], (static["gt_boxes"], static["gt_count"], static["gt_tokens"]),
                              static["text_mask"])
        return [r[k] for k in ("losses", "d_logits", "d_boxes", "match", "cost")]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step()
    for k in keys:
        static[k].copy_(d2[k])
    g.replay()
    torch.cuda.synchronize()
    r = crit.forward_flat(d2["logits"], d2["boxes"], (d2["gt_boxes"], d2["gt_count"], d2["gt_tokens"]), d2["text_mask"])
    torch.cuda.synchronize()
    for x, k in zip(out, ("losses", "d_logits", "d_boxes", "match", "cost")):
        assert torch.equal(x, r[k]), k


def test_decoder_outputs_and_loss_evaluator(dev):
    from test_gdino_asm_gpu import _build_model, _gdino_case
    from mqdet_b200 import ops
    from mqdet_b200.structures.bounding_box import BoxList
    from mqdet_b200.structures.image_list import ImageList
    B, h, w, el, dl, nq = 2, 150, 203, 2, 3, 100
    sd, ids, am, pmap, bank, img = _gdino_case(2031, B, h, w, 13, el, dl, nq)
    model = _build_model(sd, el, dl, nq, dev)
    model.query_selector.set_query_bank(bank)
    sizes = [(h, w), (h - 22, w - 37)]
    out = model.forward_device(ImageList(img.to(dev), sizes), {"input_ids": ids, "attention_mask": am}, pmap, all_layers=True)
    logits, boxes = model.decoder_outputs_flat(out)
    assert logits.shape == (dl, B, nq, 256) and boxes.shape == (dl, B, nq, 4)
    assert torch.equal(logits[-1], out["pred_logits"]) and torch.equal(boxes[-1], out["pred_boxes"])
    o = model.decoder_outputs(out)
    assert set(o) == {"pred_logits", "pred_boxes", "aux_outputs"} and len(o["aux_outputs"]) == dl - 1
    # GTs: boxes and token rows of a seeded case, the text mask of the prompt padded to 256
    gen = torch.Generator().manual_seed(11)
    counts = [5, 3]
    gt_boxes = torch.zeros(B, 5, 4)
    gt_tokens = torch.zeros(B, 5, 256)
    targets, rows = [], []
    T = int(am.shape[1])
    for b, n in enumerate(counts):
        gt_boxes[b, :n] = go._gt_boxes(gen, n)
        for g in range(n):
            s = int(torch.randint(1, int(am[0].sum()) - 3, (1,), generator=gen))
            gt_tokens[b, g, s:s + 2] = 1.0
        bl = BoxList(go.to_xyxy(gt_boxes[b, :n]), (w, h), mode="xyxy")
        bl.add_field("normed_cxcy_boxes", gt_boxes[b, :n].clone())
        targets.append(bl)
        rows.append(gt_tokens[b, :n])
    text_mask = torch.zeros(B, 256, dtype=torch.bool)
    text_mask[:, :T] = am.bool().expand(B, T)
    losses = model.loss_evaluator(o, targets, text_mask=text_mask.to(dev), positive_map=torch.cat(rows).to(dev))
    torch.cuda.synchronize()
    assert len(losses) == 3 * dl and all(v.dim() == 0 and v.is_cuda for v in losses.values())
    d = {"gt_boxes": gt_boxes.to(dev), "gt_count": torch.tensor(counts, dtype=torch.int32, device=dev), "gt_tokens": gt_tokens.to(dev)}
    own, odl, odb, _ = ops.gdino_set_loss(logits, boxes, d["gt_boxes"], d["gt_count"], d["gt_tokens"], text_mask.float().to(dev))
    for l in range(dl):
        sfx = "" if l == dl - 1 else f"_{l}"
        got = torch.stack([losses[f"loss_ce{sfx}"], losses[f"loss_bbox{sfx}"], losses[f"loss_giou{sfx}"]])
        assert torch.equal(got, own[l]), (l, got, own[l])
    assert torch.equal(model.loss_evaluator.last_train["d_logits"], odl)
    assert torch.equal(model.loss_evaluator.last_train["d_boxes"], odb)
    assert torch.isfinite(odl).all() and torch.isfinite(odb).all()
