"""CPU: the test-time vision-query update.

* tests/online_update_oracle.py pinned to the reference's own ``online_update`` (maskrcnn_benchmark/engine/inference.py:383-497),
  ``expand_bbox`` and ``GeneralizedVLRCNN_New.extract_query`` (generalized_vl_rcnn_new.py:32-49, :231-288), compiled from source as
  tests/test_bbox_aug_cpu.py does and driven by a stub detector whose detections are fixed per image and per bank, and a stub pooler.
  Cases: 1 and 3 turns, a starting bank from a file and none, labels reaching the cap in the middle of an image, near-duplicates
  within one call, boxes clipped to empty.  Results are recorded under tests/golden/online_update_pins.pt so that the comparison
  also runs where the reference is absent.
* The host logic of ``engine/online_update`` over the ops test double (tests/hostlogic), in its own process.
"""
import ast
import os
import subprocess
import sys
import tempfile
import types
from collections import defaultdict
from types import SimpleNamespace as NS

import pytest
import torch
import torch.nn.functional as F

import online_update_oracle as ou
import refpin
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "online_update_pins.pt")
_store = None
C = 16


def pinned(name, fn):
    global _store
    if _store is None:
        _store = torch.load(PIN_FILE, weights_only=True) if os.path.exists(PIN_FILE) else {}
    if ref_loader.available():
        val = fn()
        if os.environ.get("MQDET_RECORD_PINS") == "1":
            _store[name] = refpin._shrink(val, True)
            torch.save(_store, PIN_FILE)
        return val
    assert name in _store, f"{name}: no recorded result in {PIN_FILE}"
    return refpin._expand(_store[name])


# ---- the stub detector and pooler, shared by the reference run and the restatement -------------------------------------------
def bank_rows(bank):
    return sum(len(v) for v in bank.values()) if bank else 0


def detect(case, im, held):
    """Packed rows [M + 1, 6] of image ``im`` while the model holds ``held``: the scores move with the size of the held bank, so each
    turn sees different detections.  Rows 0-1 share a label and a cluster (near-duplicates), row 2 lies outside the image (clipped
    to empty), row 3 scores exactly the threshold (dropped)."""
    g = torch.Generator().manual_seed(1000 * case["seed"] + im)
    M, (w, h) = case["M"], case["sizes"][im]
    n = M - (im % 3)
    x1 = torch.rand(n, generator=g) * (w - 20)
    y1 = torch.rand(n, generator=g) * (h - 20)
    bw = 4 + torch.rand(n, generator=g) * w * 0.6
    bh = 4 + torch.rand(n, generator=g) * h * 0.6
    boxes = torch.stack([x1, y1, x1 + bw, y1 + bh], 1)
    scores = 0.3 + 0.7 * torch.rand(n, generator=g) + 0.2 * (1 - 1 / (1 + bank_rows(held)))
    scores = scores.clamp(max=0.99)
    labels = torch.randint(1, case["K"] + 1, (n,), generator=g).float()
    labels[1] = labels[0]
    boxes[1] = boxes[0] + 0.5
    boxes[2] = torch.tensor([w + 5.0, 3.0, w + 30.0, 20.0])
    scores[:2] = 0.9
    scores[3] = 0.6
    out = torch.zeros(M + 1, 6)
    out[:n, :4], out[:n, 4], out[:n, 5] = boxes, scores, labels
    out[M, 0] = n
    return out


def pool(case, im, boxes):
    """Features [R, C]: a cluster direction (from the box position) plus a small perturbation: boxes of one cluster are near-duplicates
    (cosine well above 0.85), boxes of different clusters are not."""
    g = torch.Generator().manual_seed(case["seed"])
    dirs = torch.randn(24, C, generator=g)
    W = torch.randn(4, C, generator=g)
    cl = ((boxes[:, 0] + boxes[:, 1]) / 7).floor().long() % 24
    return dirs[cl] + case["noise"] * torch.sin(boxes @ W / 7 + im)


def pin_cases():
    sizes = [(96, 80)] * 4 + [(128, 72)] * 3 + [(96, 80)] * 2
    start = defaultdict(list)
    g = torch.Generator().manual_seed(3)
    for k in (1, 2):
        start[k] = torch.randn(2, 1, C, generator=g)
    return {
        "one_turn_no_bank": dict(seed=1, M=10, K=3, sizes=sizes, turns=1, start=None, max_query=100, noise=0.4),
        "three_turns_no_bank": dict(seed=2, M=10, K=3, sizes=sizes, turns=3, start=None, max_query=100, noise=0.4),
        "three_turns_file_bank_cap": dict(seed=4, M=12, K=2, sizes=sizes, turns=3, start=start, max_query=4, noise=0.3),
        "one_turn_file_bank": dict(seed=5, M=8, K=3, sizes=sizes, turns=1, start=start, max_query=100, noise=0.5),
    }


def _cfg(case, bank_path):
    vq = NS(QUERY_BANK_PATH=bank_path, DATASET_NAME="odinw_stub", MAX_TEST_QUERY_NUMBER=case["max_query"], SELECT_FPN_LEVEL=True,
            SCORE_THRESHOLD=0.6, EXPAND_RATIO=1.5, SIMILARITY_THRESHOLD=0.85, MAX_QUERY_NUMBER=5000)
    return NS(TEST=NS(EVAL_TASK="detection", SUBSET=-1, USE_MULTISCALE=False), VISION_QUERY=vq, DATASETS=NS(TEST=("odinw_stub_val",)),
              MODEL=NS(ROI_BOX_HEAD=NS(POOLER_RESOLUTION=1)))


def _functions(rel, names, cls=None):
    path = os.path.join(ref_loader.REF, rel)
    tree = ast.parse(open(path).read())
    body = tree.body
    if cls is not None:
        body = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls][0].body
    fns = [n for n in body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(fns) == len(names), (rel, names)
    for f in fns:
        f.decorator_list = []
    return ast.Module(body=fns, type_ignores=[]), path


def _run_reference(case):
    """The reference's online_update on the stub detector: the bank saved after every turn and the bank the model holds at the end."""
    ref_loader.rpn_inference(lambda *a, **k: None)        # installs the reference's structures package
    BoxList = sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList
    saved = []

    class TorchProxy(types.ModuleType):
        def __getattr__(self, n):
            return getattr(torch, n)

        @staticmethod
        def load(*a, **k):                                  # the reference predates torch.load(weights_only=True)
            return torch.load(*a, weights_only=False, **k)

        @staticmethod
        def save(obj, path):
            saved.append(ou.copy_bank(obj))
            torch.save(obj, path)

    tp = TorchProxy("torch")
    ns = {"torch": tp, "os": os, "F": F, "einsum": torch.einsum, "defaultdict": defaultdict, "tqdm": lambda x: x, "BoxList": BoxList,
          "print": lambda *a, **k: None, "to_image_list": None,
          "create_queries_and_maps_from_dataset": lambda ds, cfg, disable_print=True: (["caption"], [{1: [1], 2: [3], 3: [5]}])}
    for rel, names, cls in (("maskrcnn_benchmark/engine/inference.py", ("online_update",), None),
                            ("maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py", ("expand_bbox",), None),
                            ("maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py", ("extract_query",), "GeneralizedVLRCNN_New")):
        mod, path = _functions(rel, names, cls)
        exec(compile(mod, path, "exec"), ns)

    with tempfile.TemporaryDirectory() as d:
        bank_path = os.path.join(d, "bank.pth") if case["start"] is not None else os.path.join(d, "absent.pth")
        if case["start"] is not None:
            torch.save(case["start"], bank_path)
        cfg = _cfg(case, bank_path)

        class Stub:
            def __init__(self):
                self.cfg = cfg
                self.held = tp.load(bank_path) if case["start"] is not None else None

            def eval(self):
                return self

            def load_query_bank(self, path):
                self.held = tp.load(path)

            def pooler(self, visual_features, targets):
                im = int(visual_features[0].flatten()[0])
                return torch.cat([pool(case, im, t.bbox) for t in targets])[:, :, None, None]

            def __call__(self, images, captions=None, positive_map=None, return_backbone_features=False):
                im = int(images.flatten()[0])
                pk = detect(case, im, self.held)
                n = int(pk[-1, 0])
                bl = BoxList(pk[:n, :4].clone(), case["sizes"][im], mode="xyxy")
                bl.add_field("scores", pk[:n, 4].clone())
                bl.add_field("labels", pk[:n, 5].long())
                return [bl], [torch.full((1, 1, 1, 1), float(im))]

        model = Stub()
        model.extract_query = types.MethodType(ns["extract_query"], model)
        batches = []
        for im, wh in enumerate(case["sizes"]):
            t = BoxList(torch.zeros(1, 4), wh, mode="xyxy")
            batches.append((torch.full((1, 1), float(im)), [t], [im]))

        class Loader(list):
            dataset = None

        ns["online_update"](model, Loader(batches), device="cpu", cfg=cfg, num_turns=case["turns"], save_name=os.path.join(d, "out.pth"))
        return {"banks": [dict(b) for b in saved], "eval": dict(model.held) if model.held is not None else {}}


def _restated(case):
    start = case["start"]
    return ou.online_update(lambda im, held: detect(case, im, held), lambda im, b: pool(case, im, b), list(range(len(case["sizes"]))),
                            case["sizes"], start, ou.copy_bank(start) if start is not None else None, case["turns"],
                            max_query=case["max_query"])


def _same_bank(a, b):
    ka = sorted(k for k, v in a.items() if len(v))
    kb = sorted(k for k, v in b.items() if len(v))
    return ka == kb and all(torch.equal(a[k], b[k]) for k in ka)


@pytest.mark.parametrize("name", sorted(pin_cases()))
def test_restatement_vs_reference_online_update(name):
    case = pin_cases()[name]
    want = pinned(name, lambda: _run_reference(case))
    banks, held, _ = _restated(case)
    assert len(banks) == len(want["banks"]) == case["turns"]
    for t, (got, ref) in enumerate(zip(banks, want["banks"])):
        assert _same_bank(got, {int(k): v for k, v in ref.items()}), (name, t)
    assert _same_bank(held or {}, {int(k): v for k, v in want["eval"].items()}), name


def test_cases_cover_what_they_claim():
    cs = pin_cases()
    for name, case in cs.items():
        banks, held, margin = _restated(case)
        assert margin > 1e-3, name                                        # no similarity within 1e-3 of the threshold
        if case["turns"] == 3:
            assert _same_bank(held, banks[1])                              # the evaluation uses the bank after turn 2
            assert bank_rows(banks[2]) >= bank_rows(banks[1]) >= bank_rows(banks[0])
        else:
            assert _same_bank(held or {}, case["start"] or {})             # one turn: the update does not reach the evaluation
    banks, held, _ = _restated(cs["three_turns_no_bank"])
    assert bank_rows(banks[1]) > bank_rows(banks[0]) and _same_bank(held, banks[1])   # turn 2 grew the bank the evaluation uses
    c = cs["three_turns_file_bank_cap"]
    banks, _, _ = _restated(c)
    assert max(len(v) for v in banks[0].values()) == c["max_query"]        # the cap engaged
    # the cap is reached in the middle of an image: some image has a kept box of a full label after one that was appended
    full_mid = False
    bank = ou.copy_bank(c["start"])
    for im, wh in enumerate(c["sizes"]):
        boxes, labels = ou.candidates(detect(c, im, c["start"]), wh, 0.6, 1.5)
        before = {k: len(bank[k]) for k in set(labels.tolist())}
        ou.bank_update(bank, labels, pool(c, im, boxes), c["max_query"], 0.85)
        full_mid |= any(before[k] < c["max_query"] <= len(bank[k]) and (labels == k).sum() > len(bank[k]) - before[k] for k in before)
    assert full_mid
    # rows 0 and 1 of every image are near-duplicates: the second never enters the bank in the same call
    case = cs["one_turn_no_bank"]
    for im, wh in enumerate(case["sizes"][:3]):
        boxes, labels = ou.candidates(detect(case, im, None), wh, 0.6, 1.5)
        f = pool(case, im, boxes[:2])
        assert labels[0] == labels[1] and float(F.cosine_similarity(f[0], f[1], dim=0)) > 0.86
        b = defaultdict(list)
        ou.bank_update(b, labels[:2], f, 100, 0.85)
        assert len(b[int(labels[0])]) == 1
    # the box outside the image is clipped to empty, the one at exactly the threshold is dropped
    pk = detect(case, 0, None)
    n = int(pk[-1, 0])
    boxes, labels = ou.candidates(pk, case["sizes"][0], 0.6, 1.5)
    assert boxes.shape[0] < int((pk[:n, 4] > 0.6).sum()) + 1 and (pk[:n, 4] == 0.6).sum() == 1
    assert not any(torch.equal(b, torch.tensor([95.0, 0.0, 95.0, 26.25])) for b in boxes)


def test_restated_candidates_bad_count_row():
    pk = torch.zeros(5, 6)
    pk[4, 0] = 4.5
    assert ou.candidates(pk, (10, 10), 0.6, 1.5) is ou.BAD_COUNT
    pk[4, 0] = 5
    assert ou.candidates(pk, (10, 10), 0.6, 1.5) is ou.BAD_COUNT


def test_config_keys_and_unsupported_paths():
    from mqdet_b200.config import mq_glip_l_cfg, mq_glip_t_cfg, mq_groundingdino_t_cfg
    from mqdet_b200.engine.online_update import check_config
    for cfg in (mq_glip_t_cfg(), mq_glip_l_cfg(), mq_groundingdino_t_cfg()):
        vq = cfg.VISION_QUERY
        assert (vq.SCORE_THRESHOLD, vq.MAX_TEST_QUERY_NUMBER, vq.NUM_TURNS, vq.OFFLINE_WITH_ONLINE) == (0.6, 100, 1, False)
        check_config(cfg)
    with pytest.raises(NotImplementedError, match="TEST.USE_MULTISCALE"):
        check_config(mq_glip_t_cfg(**{"TEST.USE_MULTISCALE": True}))
    cfg = mq_glip_t_cfg()
    cfg.TEST.EVAL_TASK = "grounding"
    with pytest.raises(NotImplementedError, match="TEST.EVAL_TASK"):
        check_config(cfg)
    with pytest.raises(NotImplementedError, match="VISION_QUERY.SELECT_FPN_LEVEL"):
        check_config(mq_glip_t_cfg(**{"VISION_QUERY.SELECT_FPN_LEVEL": False}))
    cfg = mq_glip_t_cfg()
    cfg.DATASETS = NS(TEST=("lvis_evaluation_mini_val",))
    with pytest.raises(NotImplementedError, match="DATASETS.TEST"):
        check_config(cfg)


def test_online_update_host_logic():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostlogic", "online_update_case.py")], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PASS online_update" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
