"""GPU: ATSS assignment and the pre-training detection losses (mqdet_b200/csrc/atss_loss.cu) against the fp32 restatement
(tests/atss_oracle.py, itself pinned to the reference's ATSSLossComputation by tests/test_atss_loss_cpu.py)."""
import pytest
import torch

import atss_oracle as ao
from util import load_sd

pytestmark = pytest.mark.gpu

CASES = ("bench2", "duplicates", "overlap", "small", "padded_mask", "zero_pos", "empty_gt", "ties")


def _dev(c, dev):
    return {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in c.items()}


def _run(c, dev):
    from mqdet_b200 import ops
    d = _dev(c, dev)
    lv = ops.get_levels(c["sizes"], dev)
    t = ops.atss_targets(d["gt_boxes"], d["gt_labels"], d["gt_count"], lv, ao.STRIDES, ao.SIZES)
    losses, dl, dr = ops.atss_loss(d["logits"], d["reg_ctr"], d["gt_boxes"], d["gt_labels"], d["gt_count"], d["gt_tokens"], lv,
                                   ao.STRIDES, ao.SIZES, c["reg_scales"], d["text_mask"], targets=t)
    return t, losses, dl, dr


def _grad_ok(got, ref, what):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    err = (got - ref).abs().max().item()
    bound = 1e-5 * ref.abs().max().item() + 1e-7
    assert err <= bound, f"{what}: max|err| {err:.3e} > {bound:.3e}"


@pytest.mark.parametrize("name", CASES)
def test_assignment_losses_and_gradients_match_restatement(dev, name):
    c = ao.case(name)
    t, losses, dl, dr = _run(c, dev)
    torch.cuda.synchronize()
    match = ao.atss_targets(c["sizes"], c["gt_boxes"], c["gt_count"])
    assert torch.equal(t["match"].cpu().long(), match), f"{name}: assignment differs"
    vals, rdl, rdr, out = ao.losses_and_grads(c["logits"], c["reg_ctr"], match, c["sizes"], c["gt_boxes"], c["gt_labels"],
                                              c["gt_tokens"], c["reg_scales"], c["text_mask"])
    norm = t["norm"].cpu()
    assert norm[0] == out["num_pos"] and norm[2] == out["num_pos"]
    assert abs(float(norm[1]) - out["ctr_sum"]) <= 1e-5 * abs(out["ctr_sum"]) + 1e-12
    lc = losses.cpu()
    for i in range(4):
        assert abs(float(lc[i]) - float(vals[i])) <= 1e-5 * abs(float(vals[i])) + 1e-12, (name, i, float(lc[i]), float(vals[i]))
    assert float(lc[3]) == 0.0
    _grad_ok(dl, rdl, f"{name}: d_logits")
    _grad_ok(dr, rdr, f"{name}: d_reg_ctr")
    if name == "zero_pos":
        assert float(lc[0]) == 0.0 and float(lc[1]) == 0.0 and float(dr.abs().max()) == 0.0


def test_two_runs_are_bit_identical(dev):
    c = ao.case("bench2")
    a = _run(c, dev)
    b = _run(c, dev)
    torch.cuda.synchronize()
    assert torch.equal(a[0]["match"], b[0]["match"]) and torch.equal(a[0]["norm"], b[0]["norm"])
    for x, y in zip(a[1:], b[1:]):
        assert torch.equal(x, y)


def test_cuda_graph_replay_with_new_gt_contents(dev):
    from mqdet_b200 import ops
    c1, c2 = ao.case("overlap"), ao.case("overlap", seed=1)
    G = max(c1["gt_boxes"].shape[1], c2["gt_boxes"].shape[1])

    def padded(c):
        B, g, T = c["gt_tokens"].shape
        out = dict(c)
        out["gt_boxes"] = torch.zeros(B, G, 4)
        out["gt_boxes"][:, :g] = c["gt_boxes"]
        out["gt_labels"] = torch.zeros(B, G, dtype=torch.int32)
        out["gt_labels"][:, :g] = c["gt_labels"]
        out["gt_tokens"] = torch.zeros(B, G, T)
        out["gt_tokens"][:, :g] = c["gt_tokens"]
        return _dev(out, dev)

    d1, d2 = padded(c1), padded(c2)
    lv = ops.get_levels(c1["sizes"], dev)
    static = {k: d1[k].clone() for k in ("gt_boxes", "gt_labels", "gt_count", "gt_tokens", "logits", "reg_ctr")}
    mask = d1["text_mask"]

    def step():
        return ops.atss_loss(static["logits"], static["reg_ctr"], static["gt_boxes"], static["gt_labels"], static["gt_count"],
                             static["gt_tokens"], lv, ao.STRIDES, ao.SIZES, c1["reg_scales"], mask)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step()
    for k in static:
        static[k].copy_(d2[k])
    g.replay()
    torch.cuda.synchronize()
    eager = ops.atss_loss(d2["logits"], d2["reg_ctr"], d2["gt_boxes"], d2["gt_labels"], d2["gt_count"], d2["gt_tokens"], lv,
                          ao.STRIDES, ao.SIZES, c1["reg_scales"], mask)
    torch.cuda.synchronize()
    for x, y in zip(out, eager):
        assert torch.equal(x, y)


def test_vldyhead_module_train_forward(dev):
    from mqdet_b200 import ops
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.rpn.vldyhead import VLDyHeadModule
    from mqdet_b200.structures.bounding_box import BoxList
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    gen = synth.Gen(4242)
    sd = synth.vldyhead_sd(gen, 6)
    c = ao.case("small")
    B, T = 2, 256
    mod = VLDyHeadModule(mq_glip_t_cfg())
    load_sd(mod.head, sd)
    mod = mod.to(dev).train()
    feats = [gen.randn(B, 256, h, w).to(dev) for h, w in c["sizes"]]
    hidden = gen.randn(B, T, 768).to(dev)
    masks = torch.ones(B, T, dtype=torch.long, device=dev)
    masks[1, 100:-1] = 0
    h, w = c["image_hw"]
    targets, pmap = [], []
    for b in range(B):
        n = int(c["gt_count"][b])
        bl = BoxList(c["gt_boxes"][b, :n].to(dev), (w, h), mode="xyxy")
        bl.add_field("labels", c["gt_labels"][b, :n].long().to(dev))
        targets.append(bl)
        pmap.append(c["gt_tokens"][b, :n])
    pmap = torch.cat(pmap).to(dev)
    images = ImageList(torch.zeros(B, 3, h, w, device=dev), [(h, w)] * B)
    res = mod(images, feats, targets, {"hidden": hidden, "masks": masks}, pmap)
    torch.cuda.synchronize()
    assert res[0] is None and res[2] is None
    losses = res[1]
    assert set(losses) == {"loss_reg", "loss_centerness", "loss_cls", "loss_dot_product_token"}
    assert all(v.dim() == 0 and v.is_cuda for v in losses.values())
    r = mod.last_train["head"]
    scales = [float(sd[f"scales.{l}.scale"]) for l in range(5)]
    d = _dev(c, dev)
    own, dl, dr = ops.atss_loss(r["dot_product_logits"], r["reg_ctr"], d["gt_boxes"], d["gt_labels"], d["gt_count"], d["gt_tokens"],
                                ops.get_levels(c["sizes"], dev), ao.STRIDES, ao.SIZES, scales, masks)
    got = torch.stack([losses["loss_reg"], losses["loss_centerness"], losses["loss_dot_product_token"], losses["loss_cls"]])
    assert torch.equal(got, own)
    assert torch.equal(mod.last_train["d_logits"], dl) and torch.equal(mod.last_train["d_reg_ctr"], dr)
    match = ao.atss_targets(c["sizes"], c["gt_boxes"], c["gt_count"])
    vals, _, _, _ = ao.losses_and_grads(r["dot_product_logits"].cpu(), r["reg_ctr"].cpu(), match, c["sizes"], c["gt_boxes"],
                                        c["gt_labels"], c["gt_tokens"], scales, masks.cpu())
    gc = got.cpu()
    for i in range(4):
        assert abs(float(gc[i]) - float(vals[i])) <= 1e-5 * abs(float(vals[i])) + 1e-12, (i, float(gc[i]), float(vals[i]))
