"""CPU: the vision-query bank extraction over a dataset.

tests/query_extract_oracle.py pinned to the reference's own loop: ``extract_query`` of tools/train_net.py:256-336 over
``GeneralizedVLRCNN_New.extract_query`` and ``expand_bbox`` (generalized_vl_rcnn_new.py:32-49, :231-288), compiled from source as
tests/test_online_update_cpu.py does, fed by a stub loader whose targets the reference's ``BoxList.resize`` takes to the test size,
with a stub backbone and pooler.  Cases: the cap reached in the middle of a batch, boxes that clip to empty, boxes on the image
borders, images without boxes, mixed sizes, aspect-grouped and plain batch order.  Results are recorded under
tests/golden/query_extract_pins.pt so that the comparison also runs where the reference is absent.  The several-rank restatement
equals the one-rank bank for G = 1, 2, 3 and 8.
"""
import ast
import os
import sys
import types
from collections import defaultdict
from types import SimpleNamespace as NS

import pytest
import torch
import torch.nn.functional as F

import query_extract_oracle as qo
import refpin
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "query_extract_pins.pt")
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


SIZES = [(480, 640), (640, 427), (375, 500), (500, 375), (333, 500), (612, 612), (427, 640), (480, 640), (640, 480), (360, 640),
         (500, 333), (480, 640), (424, 640), (640, 512), (375, 500), (480, 640), (612, 612), (333, 500)]


def gts_of(seed, labels, max_boxes):
    """Per image (boxes [n, 4], labels [n], (w, h)): every fourth image without boxes; on the others a box over the whole image
    (both borders), one outside the image (clipped to empty), one on the right border, then random ones."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, (h, w) in enumerate(SIZES):
        n = 0 if i % 4 == 3 else 3 + int(torch.randint(0, max_boxes - 2, (1,), generator=g))
        x1 = torch.rand(n, generator=g) * w * 0.9
        y1 = torch.rand(n, generator=g) * h * 0.9
        b = torch.stack([x1, y1, x1 + 1 + torch.rand(n, generator=g) * w * 0.4, y1 + 1 + torch.rand(n, generator=g) * h * 0.4], 1)
        if n:
            b[0] = torch.tensor([0.0, 0.0, float(w), float(h)])
            b[1] = torch.tensor([float(w) + 40, 2.0, float(w) + 60, 20.0])
            b[2, 2] = float(w - 1)
        out.append((b, torch.randint(1, labels + 1, (n,), generator=g), (w, h)))
    return out


def resized_wh():
    from mqdet_b200.engine.transforms import get_size
    return [tuple(reversed(get_size((w, h), 800, 1333))) for h, w in SIZES]


def pool(seed, i, boxes):
    """The stub pooler: a feature of each (expanded, clipped) box and its image, in fp32."""
    W = torch.randn(4, C, generator=torch.Generator().manual_seed(seed))
    return torch.sin(boxes.float() @ W / 50 + float(i))


def pin_cases():
    return {
        "cap_mid_batch_grouped": dict(seed=1, labels=3, max_boxes=9, max_query=4, ims=4, grouping=True),
        "grouped_big_cap": dict(seed=2, labels=6, max_boxes=7, max_query=5000, ims=3, grouping=True),
        "plain_order_cap5": dict(seed=3, labels=5, max_boxes=8, max_query=5, ims=8, grouping=False),
        "one_per_batch": dict(seed=4, labels=4, max_boxes=6, max_query=2, ims=1, grouping=True),
    }


def batches_of(case):
    from mqdet_b200.engine.batches import reference_test_batches
    return reference_test_batches(SIZES, case["ims"], case["grouping"])


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
    """tools/train_net.py's extract_query over a stub loader of the case's batches -> the bank it saves."""
    ref_loader.rpn_inference(lambda *a, **k: None)        # installs the reference's structures package
    BoxList = sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList
    saved = []

    class TorchProxy(types.ModuleType):
        def __getattr__(self, n):
            return getattr(torch, n)

        @staticmethod
        def save(obj, path):
            saved.append({int(k): v.clone() for k, v in obj.items()})

    gts, rwh = gts_of(case["seed"], case["labels"], case["max_boxes"]), resized_wh()
    vq = NS(MAX_QUERY_NUMBER=case["max_query"], EXPAND_RATIO=1.5, SELECT_FPN_LEVEL=True, QUERY_BANK_SAVE_PATH="bank.pth",
            SIMILARITY_THRESHOLD=0.85)
    cfg = NS(DATASETS=NS(FEW_SHOT=0), VISION_QUERY=vq, MODEL=NS(DEVICE="cpu", WEIGHT="w", SWINT=NS(VERSION="swint")), num_gpus=1)

    class Images:
        def __init__(self, ids):
            self.tensors = torch.tensor(ids, dtype=torch.float32)

        def to(self, device):
            return self

    class Stub:
        def __init__(self):
            self.cfg = cfg

        def to(self, device):
            return self

        def eval(self):
            return self

        def backbone(self, x):
            return [x]

        def pooler(self, visual_features, targets):
            ids = visual_features[0].tolist()
            return torch.cat([pool(case["seed"], int(i), t.bbox) for i, t in zip(ids, targets)])[:, :, None, None]

    loader = []
    for idx in batches_of(case):
        tg = []
        for i in idx:
            b, l, wh = gts[i]
            t = BoxList(b.clone(), wh, mode="xyxy")
            t.add_field("labels", l.clone())
            tg.append(t.resize(rwh[i]))                    # the test loader's Resize transform
        loader.append((Images(idx), tg, idx))

    model = Stub()
    ns = {"torch": TorchProxy("torch"), "F": F, "einsum": torch.einsum, "defaultdict": defaultdict, "tqdm": lambda x: x,
          "BoxList": BoxList, "print": lambda *a, **k: None, "to_image_list": lambda x: x, "build_detection_model": lambda c: model,
          "DetectronCheckpointer": lambda c, m: NS(load=lambda *a: None), "try_to_find": lambda p: p,
          "make_data_loader": lambda *a, **k: [loader]}
    for rel, names, cls in (("tools/train_net.py", ("extract_query",), None),
                            ("maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py", ("expand_bbox",), None)):
        mod, path = _functions(rel, names, cls)
        exec(compile(mod, path, "exec"), ns)
    train_extract = ns["extract_query"]
    mod, path = _functions("maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py", ("extract_query",), "GeneralizedVLRCNN_New")
    exec(compile(mod, path, "exec"), ns)
    model.extract_query = types.MethodType(ns["extract_query"], model)
    train_extract(cfg)
    assert len(saved) == 1
    return saved[0]


def _restated(case, G=None):
    gts = gts_of(case["seed"], case["labels"], case["max_boxes"])
    args = (gts, batches_of(case), resized_wh(), lambda i, b: pool(case["seed"], i, b), case["max_query"])
    return qo.extract(*args) if G is None else qo.extract_ranks(*args, G)


@pytest.mark.parametrize("name", sorted(pin_cases()))
def test_restatement_vs_reference_extract_query(name):
    case = pin_cases()[name]
    want = pinned(name, lambda: _run_reference(case))
    assert qo.same_bank(_restated(case), {int(k): v for k, v in want.items()}), name


@pytest.mark.parametrize("G", [1, 2, 3, 8])
@pytest.mark.parametrize("name", sorted(pin_cases()))
def test_several_ranks_give_the_one_rank_bank(name, G):
    case = pin_cases()[name]
    assert qo.same_bank(_restated(case, G), _restated(case)), (name, G)


def test_cases_cover_what_they_claim():
    rwh = resized_wh()
    assert len(set(rwh)) > 3                                             # mixed sizes
    for name, case in pin_cases().items():
        gts = gts_of(case["seed"], case["labels"], case["max_boxes"])
        assert any(b.shape[0] == 0 for b, _, _ in gts)                   # images without boxes
        first = qo.first_boxes(gts, batches_of(case))
        kept = sum(qo.batch_rois(gts, [i], [rwh[i]], 1.5, first)[0].shape[0] for i in range(len(gts)))
        assert kept < sum(b.shape[0] for b, _, _ in gts)                 # boxes clipped to empty
        rois = torch.cat([qo.batch_rois(gts, [i], [rwh[i]], 1.5, first)[0] for i in range(len(gts))])
        assert (rois[:, 1] == 0).any() and (rois[:, 3] == torch.tensor([float(w - 1) for w, _ in rwh]).max()).any() or \
            any((qo.batch_rois(gts, [i], [rwh[i]], 1.5, first)[0][:, 3] == rwh[i][0] - 1).any() for i in range(len(gts)))
    grouped = batches_of(pin_cases()["cap_mid_batch_grouped"])
    assert grouped != sorted(grouped) or any(b != list(range(b[0], b[0] + len(b))) for b in grouped)   # aspect grouping reorders
    # the cap is reached in the middle of a batch: some batch appends a label's last row and then skips a later box of it
    case = pin_cases()["cap_mid_batch_grouped"]
    gts = gts_of(case["seed"], case["labels"], case["max_boxes"])
    first, bank, mid = qo.first_boxes(gts, grouped), defaultdict(list), False
    for idx in grouped:
        _, labels, _ = qo.batch_rois(gts, idx, [rwh[i] for i in idx], 1.5, first)
        before = {k: len(bank[k]) for k in set(labels.tolist())}
        qo.cap_append(bank, labels, torch.zeros(labels.shape[0], C), case["max_query"])
        mid |= any(before[k] < case["max_query"] == len(bank[k]) and int((labels == k).sum()) > len(bank[k]) - before[k]
                   for k in before)
    assert mid
    assert max(len(v) for v in _restated(pin_cases()["grouped_big_cap"]).values()) < 5000


def test_config_checks():
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.engine.query_extract import check_config
    cfg = mq_glip_t_cfg()
    check_config(cfg)
    cfg.DATASETS = NS(FEW_SHOT=5)
    with pytest.raises(ValueError, match="DATASETS.FEW_SHOT"):
        check_config(cfg)
    cfg.VISION_QUERY.MAX_QUERY_NUMBER = 5
    check_config(cfg)
    with pytest.raises(NotImplementedError, match="SELECT_FPN_LEVEL"):
        check_config(mq_glip_t_cfg(**{"VISION_QUERY.SELECT_FPN_LEVEL": False}))


def test_engine_refuses_a_cpu_model():
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.engine.query_extract import extract_query_bank
    from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
    cfg = mq_glip_t_cfg()
    with pytest.raises(MqdetError, match="CUDA"):
        extract_query_bank(GeneralizedVLRCNN_New(cfg), [], [], cfg)
