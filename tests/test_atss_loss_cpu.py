"""CPU: the ATSS assignment / loss restatement (tests/atss_oracle.py) against the reference's own ATSSLossComputation run on CPU
(live where the original sources are present, else its recorded results in tests/golden/atss_loss_pins.pt), the argument validation of the
new C-ABI entries, the loss-flag policy and the data-parallel normaliser all-reduce."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import atss_oracle as ao
import refpin
from oracle import ref_loader
from util import ROOT

REF_CASES = ("bench2", "duplicates", "overlap", "small", "padded_mask", "zero_pos")
PIN_FILE = os.path.join(ROOT, "tests", "golden", "atss_loss_pins.pt")
_live = {}
_store = None


def _pinned(name, fn, full=False):
    """``refpin.pinned`` (same storage format: whole tensors up to refpin.FULL elements or with `full`, else a seeded sample plus
    max |value|) with the ATSS results in a file of their own: fn() where the original sources are present (stored under `name`
    when MQDET_RECORD_PINS=1), else the stored result."""
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
        c = ao.case(name)
        _live[name] = (c, ao.reference(c["logits"], c["reg_ctr"], c["image_hw"], c["sizes"], c["gt_boxes"], c["gt_labels"],
                                       c["gt_count"], c["gt_tokens"], c["reg_scales"], c["text_mask"]))
    return _live[name]


def _ref_summary(name):
    """the reference's assignment in compact form, and its losses / gradients at the positives (whole tensors)"""
    _, r = _reference(name)
    lab = r["labels"]
    pos = lab > 0
    T = r["token_labels"].shape[-1]
    none = torch.zeros(T)
    none[-1] = 1
    matched = ~(r["token_labels"] == none).all(-1)
    sig = (r["token_labels"].double() * torch.arange(1, T + 1, dtype=torch.float64)).sum(-1)
    return {"pos_idx": pos.reshape(-1).nonzero().squeeze(1).int(), "labels_pos": lab[pos].int(),
            "matched_idx": matched.reshape(-1).nonzero().squeeze(1).int(), "token_sig": sig[matched],
            "reg_targets_pos": r["reg_targets"][pos], "losses": r["losses"], "d_reg_ctr_pos": r["d_reg_ctr"][pos],
            "d_reg_ctr_other_absmax": r["d_reg_ctr"][~pos].abs().max() if (~pos).any() else torch.zeros(())}


def _restated(c):
    match = ao.atss_targets(c["sizes"], c["gt_boxes"], c["gt_count"])
    vals, dl, dr, out = ao.losses_and_grads(c["logits"], c["reg_ctr"], match, c["sizes"], c["gt_boxes"], c["gt_labels"], c["gt_tokens"],
                                            c["reg_scales"], c["text_mask"])
    return match, vals, dl, dr, out


@pytest.mark.parametrize("name", REF_CASES)
def test_restatement_matches_reference(name):
    c = ao.case(name)
    want = _pinned(f"atss_loss/{name}/summary", lambda: _ref_summary(name), full=True)
    want_dl = _pinned(f"atss_loss/{name}/d_logits", lambda: _reference(name)[1]["d_logits"])
    match, vals, dl, dr, out = _restated(c)
    B, N = match.shape
    lab = torch.where(match >= 0, torch.gather(c["gt_labels"].long(), 1, match.clamp(min=0)), torch.zeros_like(match))
    pos = lab > 0
    # identical assignment: positive set, labels, matched set and the token row of every matched anchor
    assert torch.equal(pos.reshape(-1).nonzero().squeeze(1).int(), want["pos_idx"])
    assert torch.equal(lab[pos].int(), want["labels_pos"])
    assert torch.equal((match >= 0).reshape(-1).nonzero().squeeze(1).int(), want["matched_idx"])
    tgt = ao.token_targets(match, c["gt_tokens"])
    T = tgt.shape[-1]
    sig = (tgt.double() * torch.arange(1, T + 1, dtype=torch.float64)).sum(-1)
    assert torch.equal(sig[match >= 0], want["token_sig"])
    # regression targets
    rt = out["reg_targets"]
    assert rt.shape == want["reg_targets_pos"].shape
    if rt.numel():
        assert (rt - want["reg_targets_pos"]).abs().max() <= 1e-6 * max(1.0, float(want["reg_targets_pos"].abs().max()))
    # losses
    for i, k in enumerate(("loss_reg", "loss_centerness", "loss_dot_product_token", "loss_cls")):
        w = float(want["losses"][i])
        assert abs(float(vals[i]) - w) <= 1e-5 * abs(w) + 1e-12, (k, float(vals[i]), w)
    assert float(vals[3]) == 0.0
    # gradients: restatement autograd against autograd through the reference's code
    err, bmax = refpin.max_err(dl, want_dl)
    assert err <= 1e-5 * bmax + 1e-7, ("d_logits", err, bmax)
    wd = want["d_reg_ctr_pos"]
    if wd.numel():
        assert (dr[pos] - wd).abs().max() <= 1e-5 * float(wd.abs().max()) + 1e-7
    assert float(want["d_reg_ctr_other_absmax"]) == 0.0 and float(dr[~pos].abs().max()) == 0.0
    if name == "zero_pos":
        assert not pos.any() and (match >= 0).any() and float(vals[0]) == 0.0 and float(vals[1]) == 0.0
    if name == "bench2":  # the clamp case is exercised: positives with dw past the clamp get no dw gradient
        sc = ao.scale_per_anchor(c["sizes"], c["reg_scales"])[None].expand(B, N)
        past = pos & (c["reg_ctr"][..., 2] * sc / 5.0 > ao.CLAMP)
        assert past.any() and float(dr[..., 2][past].abs().max()) == 0.0
    if name == "small":
        assert c["sizes"][-1][0] * c["sizes"][-1][1] < 9


def test_duplicate_gts_go_to_the_lowest_index():
    c = ao.case("duplicates")
    match = ao.atss_targets(c["sizes"], c["gt_boxes"], c["gt_count"])[0]
    # boxes 3 / 4 / 5 repeat 0 / 1 / 1: every anchor they would claim goes to the lower index with the same IoU
    assert (match >= 0).any()
    assert not ((match == 3) | (match == 4) | (match == 5)).any()


def test_overlapping_gts_compete_for_anchors():
    c = ao.case("overlap")
    A, lvl = ao.anchors(c["sizes"])
    g = c["gt_boxes"][0, :int(c["gt_count"][0])]
    claims = torch.zeros(A.shape[0], dtype=torch.int32)
    for j in range(g.shape[0]):
        claims += (ao.assign_image(A, lvl, g[j:j + 1])[0] >= 0).int()
    assert (claims > 1).any()   # at least one anchor is a positive candidate of several GTs
    match = ao.atss_targets(c["sizes"], c["gt_boxes"], c["gt_count"])[0]
    ious = ao._iou(A, g)
    contested = (claims > 1) & (match >= 0)
    best = ious[contested].max(1)[0]
    # the winner has the highest IoU among the GTs that claimed the anchor (here: among all GTs that kept it positive)
    assert torch.all(ious[contested, match[contested]] <= best)


def test_empty_gt_image_is_all_negative():
    c = ao.case("empty_gt")
    match = ao.atss_targets(c["sizes"], c["gt_boxes"], c["gt_count"])
    assert (match[0] == -1).all() and (match[1] >= 0).any()
    tgt = ao.token_targets(match, c["gt_tokens"])
    assert torch.all(tgt[0, :, -1] == 1) and float(tgt[0, :, :-1].abs().sum()) == 0.0
    vals, dl, dr, out = ao.losses_and_grads(c["logits"], c["reg_ctr"], match, c["sizes"], c["gt_boxes"], c["gt_labels"], c["gt_tokens"],
                                            c["reg_scales"], c["text_mask"])
    assert torch.isfinite(vals).all() and float(dr[0].abs().max()) == 0.0


def test_topk_tie_rule_keeps_the_lower_anchor_index():
    c = ao.case("ties")
    A, lvl = ao.anchors(c["sizes"])
    g = c["gt_boxes"][0, :1]
    ac = torch.stack(((A[:, 2] + A[:, 0]) / 2.0, (A[:, 3] + A[:, 1]) / 2.0), 1)
    gc = torch.stack(((g[:, 2] + g[:, 0]) / 2.0, (g[:, 3] + g[:, 1]) / 2.0), 1)
    d = (ac[lvl == 0] - gc).pow(2).sum(-1).sqrt()
    srt = torch.sort(d, stable=True)
    assert srt.values[8] == srt.values[9]          # the fixture does tie at the cut
    tied = (d == srt.values[8]).nonzero().squeeze(1)
    kept = srt.indices[:9]
    assert set(kept.tolist()) & set(tied.tolist()) == set(tied[:int((srt.values[:9] == srt.values[8]).sum())].tolist())


def test_fixtures_keep_candidates_away_from_the_threshold():
    for name in ao.CASES:
        c = ao.case(name)
        if name != "empty_gt":
            assert ao.threshold_margin(c["sizes"], c["gt_boxes"], c["gt_count"]) > 1e-6


def test_atss_abi_argument_validation_without_gpu():
    import ctypes
    from mqdet_b200 import _lib
    lib = _lib.load()
    nul, one = ctypes.c_void_p(0), ctypes.c_void_p(16)
    hw = (ctypes.c_int32 * 4)(10, 10, 5, 5)
    f = (ctypes.c_float * 8)()

    def expect(rc, needle):
        assert rc < 0
        msg = lib.mqdet_last_error().decode()
        assert needle in msg, msg

    hwp, fp = ctypes.cast(hw, ctypes.c_void_p), ctypes.cast(f, ctypes.c_void_p)
    expect(lib.mqdet_atss_assign(nul, one, one, 2, 8, hwp, 2, fp, fp, 9, one, one, nul, one, nul), "null pointer")
    expect(lib.mqdet_atss_assign(one, one, one, 2, 0, hwp, 2, fp, fp, 9, one, one, nul, one, nul), "Gmax")
    expect(lib.mqdet_atss_assign(one, one, one, 2, 8, hwp, 2, fp, fp, 17, one, one, nul, one, nul), "topk")
    expect(lib.mqdet_atss_assign(one, one, one, 2, 8, hwp, 0, fp, fp, 9, one, one, nul, one, nul), "level table")
    expect(lib.mqdet_atss_assign(one, one, one, 0, 8, hwp, 2, fp, fp, 9, one, one, nul, one, nul), "B=")
    args = [one] * 6 + [2, 8, 256, nul, hwp, 2, fp, fp, fp, one, 1.0, 0.25, 2.0, 2.0, 1.0, one, one, one, one, nul]
    bad = list(args)
    bad[0] = nul
    expect(lib.mqdet_atss_loss(*bad), "null pointer")
    bad = list(args)
    bad[8] = 0
    expect(lib.mqdet_atss_loss(*bad), "token count")
    bad = list(args)
    bad[16] = 0.0
    expect(lib.mqdet_atss_loss(*bad), "world size")
    # GT capacities far above 1000 per image are accepted by the argument checks (they fail only on the fake pointers' level table)
    expect(lib.mqdet_atss_assign(one, one, one, 2, 5000, hwp, 0, fp, fp, 9, one, one, nul, one, nul), "level table")
    assert lib.mqdet_atss_assign_workspace_bytes(2, 100) >= 2 * 100 * 8
    assert lib.mqdet_atss_loss_workspace_floats(2, 100) > 0


@pytest.mark.parametrize("flag", ["USE_CLASSIFICATION_LOSS", "USE_TOKEN_LOSS", "USE_CONTRASTIVE_ALIGN_LOSS",
                                  "USE_SHALLOW_CONTRASTIVE_LOSS", "USE_BACKBONE_SHALLOW_CONTRASTIVE_LOSS", "MLM_LOSS"])
def test_unshipped_loss_flags_raise(flag):
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.rpn.vldyhead import check_loss_config
    check_loss_config(mq_glip_t_cfg())
    with pytest.raises(NotImplementedError):
        check_loss_config(mq_glip_t_cfg(**{f"MODEL.DYHEAD.FUSE_CONFIG.{flag}": True}))


def _norm_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    from mqdet_b200 import parallel
    dist.init_process_group("gloo", rank=rank, world_size=world)
    calls = []
    orig = dist.all_reduce
    dist.all_reduce = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    norm = torch.tensor([3.0 + rank, 1.5 * (rank + 1), 3.0 + rank, 1.5 * (rank + 1)])
    parallel.all_reduce_loss_normalizers(norm[:2])
    ret[rank] = bool(torch.equal(norm, torch.tensor([7.0, 4.5, 3.0 + rank, 1.5 * (rank + 1)])) and len(calls) == 1)
    dist.barrier()
    dist.destroy_process_group()


def test_loss_normalizer_all_reduce_world2_one_collective():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_norm_worker, args=(world, port, ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}
    from mqdet_b200 import parallel
    buf = torch.ones(2)
    assert parallel.all_reduce_loss_normalizers(buf) is buf and torch.equal(buf, torch.ones(2))
