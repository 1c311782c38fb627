"""CPU: the GroundingDINO matching / set-loss restatement (tests/gdino_loss_oracle.py) against the reference's own SetCriterion and
HungarianMatcher run on CPU (live where the original sources are present, else its recorded results in
tests/golden/gdino_loss_pins.pt), the rules the reference leaves open, the argument validation of the new ops and C-ABI entries,
the matcher-type policy and the data-parallel normaliser all-reduce."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import gdino_loss_oracle as go
import refpin
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "gdino_loss_pins.pt")
_live = {}
_store = None


def _pinned(name, fn, full=False):
    """``refpin.pinned`` with the GroundingDINO loss results in a file of their own (same storage format): fn() where the original
    sources are present (stored under `name` when MQDET_RECORD_PINS=1), else the stored result."""
    global _store
    if _store is None:
        _store = torch.load(PIN_FILE, weights_only=True) if os.path.exists(PIN_FILE) else {}
    if ref_loader.available():
        val = fn()
        if os.environ.get("MQDET_RECORD_PINS") == "1":
            _store[name] = refpin._shrink(val, full)
            torch.save(_store, PIN_FILE)
        return val
    assert name in _store, f"{name}: no recorded result in {PIN_FILE}"
    return refpin._expand(_store[name])


def _reference(name):
    if name not in _live:
        c = go.case(name)
        _live[name] = go.reference(c["logits"], c["boxes"], c["gt_boxes"], c["gt_count"], c["gt_tokens"], c["text_mask"])
    return _live[name]


def _pairs(match):
    """match [L, B, Q] -> [K, 4] int32 rows (layer, image, query, GT) of the matched pairs"""
    idx = (match >= 0).nonzero()
    return torch.cat((idx, match[match >= 0][:, None]), 1).int()


def _ref_summary(name):
    r = _reference(name)
    matched = r["match"] >= 0
    return {"pairs": _pairs(r["match"]), "losses": r["losses"], "d_boxes_matched": r["d_boxes"][matched],
            "d_boxes_other_absmax": r["d_boxes"][~matched].abs().max(), "keys": torch.tensor([len(r["keys"])])}


@pytest.mark.parametrize("name", go.REF_CASES)
def test_restatement_matches_reference(name):
    c = go.case(name)
    want = _pinned(f"gdino_loss/{name}/summary", lambda: _ref_summary(name), full=True)
    want_dl = _pinned(f"gdino_loss/{name}/d_logits", lambda: _reference(name)["d_logits"])
    cost, match = go.match_layers(c["logits"], c["boxes"], c["gt_boxes"], c["gt_count"], c["gt_tokens"])
    assert torch.isfinite(cost).all()
    # identical indices (every layer, every image)
    assert torch.equal(_pairs(match), want["pairs"])
    vals, dl, db = go.losses_and_grads(c["logits"], c["boxes"], match, c["gt_boxes"], c["gt_count"], c["gt_tokens"], c["text_mask"])
    wl = want["losses"]
    assert ((vals - wl).abs() <= 1e-5 * wl.abs() + 1e-12).all(), (vals, wl)
    err, bmax = refpin.max_err(dl, want_dl)
    assert err <= 1e-5 * bmax + 1e-7, ("d_logits", err, bmax)
    wd = want["d_boxes_matched"]
    assert (db[match >= 0] - wd).abs().max() <= 1e-5 * float(wd.abs().max()) + 1e-7
    assert float(want["d_boxes_other_absmax"]) == 0.0 and float(db[match < 0].abs().max()) == 0.0
    assert int(want["keys"][0]) == 18
    if name == "empty_image":
        assert (match[:, 0] == -1).all() and (match[:, 1] >= 0).any()
    if name == "full_caption":  # token 255 is inside the mask: the unmatched one-hot contributes, with a gradient there
        assert (dl[..., 255] != 0).any()
    if name in ("duplicates", "same_boxes"):  # the fixtures do produce tied cost entries
        for l in range(cost.shape[0]):
            n = int(c["gt_count"][0])
            k = cost[l, 0, :, :n]
            assert (torch.unique(k.reshape(-1)).numel() < k.numel())


def test_empty_token_row_rule():
    c = go.case("empty_tokens")
    cost, match = go.match_layers(c["logits"], c["boxes"], c["gt_boxes"], c["gt_count"], c["gt_tokens"])
    assert torch.isfinite(cost).all()
    # class cost 0: the column is the box terms alone
    l1 = torch.cdist(c["boxes"][0, 0], c["gt_boxes"][0, 2:3], p=1)[:, 0]
    giou = go.giou_matrix(go.to_xyxy(c["boxes"][0, 0]), go.to_xyxy(c["gt_boxes"][0, 2:3]))[:, 0]
    assert torch.allclose(cost[0, 0, :, 2], 5.0 * l1 - 2.0 * giou, rtol=0, atol=1e-6)
    # the query matched to that GT gets the unmatched one-hot target
    q = int((match[0, 0] == 2).nonzero()[0, 0])
    tgt = go.token_targets(match[0], c["gt_tokens"])
    assert tgt[0, q, -1] == 1 and float(tgt[0, q, :-1].abs().sum()) == 0.0
    vals, dl, db = go.losses_and_grads(c["logits"], c["boxes"], match, c["gt_boxes"], c["gt_count"], c["gt_tokens"], c["text_mask"])
    assert torch.isfinite(vals).all() and torch.isfinite(dl).all() and torch.isfinite(db).all()


def test_ops_reject_cpu_tensors_and_bad_shapes():
    from mqdet_b200 import ops
    from mqdet_b200._lib import MqdetError
    c = go.case("empty_image")
    args = (c["logits"], c["boxes"], c["gt_boxes"], c["gt_count"], c["gt_tokens"])
    with pytest.raises(MqdetError):
        ops.gdino_match(*args)
    with pytest.raises(MqdetError):
        ops.gdino_set_loss(*args, c["text_mask"])
    with pytest.raises(MqdetError):
        ops.linear_sum_assignment(torch.zeros(2, 8, 4), torch.zeros(2, dtype=torch.int32))


def test_abi_argument_validation_without_gpu():
    import ctypes
    from mqdet_b200 import _lib
    lib = _lib.load()
    nul, one = ctypes.c_void_p(0), ctypes.c_void_p(16)

    def expect(rc, needle):
        assert rc < 0
        msg = lib.mqdet_last_error().decode()
        assert needle in msg, msg

    expect(lib.mqdet_gdino_match_cost(nul, one, one, one, one, 6, 2, 900, 256, 20, 0.25, 1.0, 5.0, 2.0, one, one, nul), "null pointer")
    expect(lib.mqdet_gdino_match_cost(one, one, one, one, one, 6, 2, 900, 256, 901, 0.25, 1.0, 5.0, 2.0, one, one, nul), "Gmax")
    expect(lib.mqdet_gdino_match_cost(one, one, one, one, one, 6, 2, 900, 0, 20, 0.25, 1.0, 5.0, 2.0, one, one, nul), "token count")
    expect(lib.mqdet_linear_sum_assignment(one, one, 2, 12, 900, 901, one, one, nul), "Gmax")
    expect(lib.mqdet_linear_sum_assignment(one, one, 2, 12, 5000, 10, one, one, nul), "Q=")
    expect(lib.mqdet_linear_sum_assignment(one, nul, 2, 12, 900, 20, one, one, nul), "null pointer")
    args = [one] * 5 + [6, 2, 900, 256, 20, nul, one, 1.0, 0.25, 2.0, 2.0, 5.0, 2.0, one, one, one, one, nul]
    bad = list(args)
    bad[9] = 901
    expect(lib.mqdet_gdino_set_loss(*bad), "Gmax")
    bad = list(args)
    bad[12] = 0.5
    expect(lib.mqdet_gdino_set_loss(*bad), "world size")
    bad = list(args)
    bad[2] = nul
    expect(lib.mqdet_gdino_set_loss(*bad), "null pointer")
    assert lib.mqdet_linear_sum_assignment_workspace_bytes(12, 900, 200) == 12 * 900 * 200 * 4
    assert lib.mqdet_gdino_set_loss_workspace_floats(6, 2, 900) > 0


def test_matcher_policy_and_config():
    from types import SimpleNamespace as NS
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.modeling.groundingdino.loss import SetCriterion, loss_dict
    from mqdet_b200.modeling.groundingdino.matcher import HungarianMatcher, build_matcher
    g = mq_groundingdino_t_cfg().GROUNDINGDINO
    assert (g.loss_ce_coef, g.loss_bbox_coef, g.loss_giou_coef) == (2.0, 5.0, 2.0)
    m = build_matcher(g.matcher)
    assert isinstance(m, HungarianMatcher) and (m.cost_class, m.cost_bbox, m.cost_giou, m.focal_alpha) == (1.0, 5.0, 2.0, 0.25)
    with pytest.raises(NotImplementedError):
        build_matcher(NS(matcher_type="SimpleMinsumMatcher", set_cost_class=1.0, set_cost_bbox=5.0, set_cost_giou=2.0, focal_alpha=0.25))
    with pytest.raises(AssertionError):
        build_matcher(NS(matcher_type="Other", set_cost_class=1.0, set_cost_bbox=5.0, set_cost_giou=2.0, focal_alpha=0.25))
    crit = SetCriterion(m, mq_groundingdino_t_cfg())
    assert not list(crit.parameters()) and not crit.state_dict()
    d = loss_dict(torch.arange(18, dtype=torch.float32).view(6, 3))
    assert list(d)[:3] == ["loss_ce", "loss_bbox", "loss_giou"] and len(d) == 18
    assert float(d["loss_giou"]) == 17.0 and float(d["loss_ce_0"]) == 0.0 and float(d["loss_bbox_4"]) == 13.0


def _norm_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    from mqdet_b200 import parallel
    dist.init_process_group("gloo", rank=rank, world_size=world)
    calls = []
    orig = dist.all_reduce
    dist.all_reduce = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    ok = True
    for local, total in (((5.0, 2.0), 7.0), ((1.0, 0.0), 1.0)):   # the second: 1 / world = 0.5 -> clamped to 1
        norm = torch.tensor([local[rank]])
        parallel.all_reduce_loss_normalizers(norm)
        ok &= float(norm[0]) == total
    ret[rank] = bool(ok and len(calls) == 2)
    dist.barrier()
    dist.destroy_process_group()


def test_gdino_normalizer_all_reduce_world2():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 35500 + (os.getpid() % 2000)
    mp.spawn(_norm_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}
    # num_boxes = max(sum over ranks / world, 1): the restatement divides by exactly that
    c = go.case("empty_image")
    cost, match = go.match_layers(c["logits"], c["boxes"], c["gt_boxes"], c["gt_count"], c["gt_tokens"])
    args = (c["logits"], c["boxes"], match, c["gt_boxes"], c["gt_count"], c["gt_tokens"], c["text_mask"])
    base = go.set_loss(*args, num_boxes_sum=1.0)
    assert torch.equal(go.set_loss(*args, world=2, num_boxes_sum=1.0), base)            # 0.5 -> 1
    assert torch.allclose(go.set_loss(*args, world=2, num_boxes_sum=7.0), base / 3.5, rtol=1e-6, atol=0)
