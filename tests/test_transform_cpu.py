"""CPU: tests/transform_oracle.py (the restatement the GPU tests compare the kernel against) pinned to the reference's own
test transform, and its resampler compared with PIL.

The reference classes Resize, ToTensor and Normalize are compiled as they are from maskrcnn_benchmark/data/transforms/transforms.py
and run on PIL images, followed by the reference's to_image_list; BoxList.resize is pinned to the reference's BoxList.  Results
are recorded under tests/golden/transform_pins.pt so that the comparison also runs where the reference is absent.  PIL and
torchvision are installed packages, not the reference, and are called directly."""
import ast
import os

import numpy as np
import pytest
import torch
from PIL import Image

import refpin
import transform_oracle as to
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "transform_pins.pt")
_store = None

GLIP = dict(mean=[103.530, 116.280, 123.675], std=[57.375, 57.120, 58.395], fmt="bgr255")
GDINO = dict(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225], fmt="rgb")

# (name, image sizes (h, w), size, max_size, normalisation, SIZE_DIVISIBILITY): small enough to store whole
PIN_CASES = [
    ("up_bgr255", [(17, 23)], 30, 60, GLIP, 32),
    ("down_bgr255", [(61, 47)], 20, 33, GLIP, 32),
    ("clamp_rgb", [(13, 90)], 24, 50, GDINO, 32),
    ("equal_short_side_rgb", [(24, 31)], 24, 100, GDINO, 8),
    ("batch_two_sources_bgr255", [(20, 30), (40, 60)], 26, 1000, GLIP, 32),
    ("tall_rgb_no_pad", [(75, 11)], 9, 80, GDINO, 0),
]


def pinned(name, fn):
    """``refpin.pinned`` with the results in a file of their own (whole tensors)."""
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


def _reference_transforms():
    import random

    import torchvision.transforms.functional as F
    path = os.path.join(ref_loader.REF, "maskrcnn_benchmark", "data", "transforms", "transforms.py")
    want = ("Compose", "Resize", "ToTensor", "Normalize")
    tree = ast.parse(open(path).read())
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name in want]
    assert len(cls) == len(want)
    ns = {"np": np, "F": F, "random": random, "torch": torch, "cv2": None}
    exec(compile(ast.Module(body=cls, type_ignores=[]), path, "exec"), ns)
    return ns


def _images(sizes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]


def _run_reference(sizes, size, max_size, norm, div, seed):
    T = _reference_transforms()
    tf = T["Compose"]([T["Resize"](size, max_size), T["ToTensor"](), T["Normalize"](norm["mean"], norm["std"], norm["fmt"])])
    out = [tf(Image.fromarray(im)) for im in _images(sizes, seed)]
    il = ref_loader.image_list().to_image_list(out, div)
    return {"batch": il.tensors, "sizes": torch.tensor(il.image_sizes)}


@pytest.mark.parametrize("case", PIN_CASES, ids=[c[0] for c in PIN_CASES])
def test_restatement_vs_reference_transform(case):
    name, sizes, size, max_size, norm, div = case
    want = pinned(name, lambda: _run_reference(sizes, size, max_size, norm, div, seed=len(name)))
    batch, resized = to.transform(_images(sizes, len(name)), size, max_size, norm["mean"], norm["std"], norm["fmt"], div)
    assert torch.equal(batch, want["batch"])
    assert [tuple(r.shape[:2]) for r in resized] == [tuple(s) for s in want["sizes"].tolist()]


def _size_triples():
    """(w, h, size, max_size): random sizes, the max-size clamp, shorter side equal to size, extreme aspect ratios."""
    rng = np.random.default_rng(7)
    out = [(int(w), int(h), int(s), int(m)) for w, h, s, m in zip(rng.integers(1, 5000, 300), rng.integers(1, 5000, 300),
                                                                 rng.integers(100, 1500, 300), rng.integers(500, 3000, 300))]
    out += [(640, 480, 800, 1333), (480, 640, 800, 1333), (4000, 3000, 800, 1333), (1333, 800, 800, 1333), (800, 1333, 800, 1333),
            (800, 800, 800, 1333), (1, 5000, 800, 1333), (5000, 1, 800, 1333), (3, 2000, 400, 2500), (2000, 3, 1800, 2500),
            (1066, 800, 800, 1333), (999, 1000, 1000, 1333), (1000, 999, 1000, 1333), (500, 1250, 400, 1000)]
    for s in (400, 500, 600, 640, 700, 900, 1000, 1100, 1200, 1300, 1400, 1800):   # TEST.SCALES at TEST.MAX_SIZE
        out += [(640, 480, s, 2500), (427, 640, s, 2500), (1024, 683, s, 2500), (4032, 3024, s, 2500)]
    return out


def test_get_size_vs_reference():
    triples = _size_triples()

    def run():
        T = _reference_transforms()
        return torch.tensor([T["Resize"](s, m).get_size((w, h)) for w, h, s, m in triples])
    want = pinned("get_size", run)
    got = torch.tensor([to.get_size((w, h), s, m) for w, h, s, m in triples])
    assert torch.equal(got, want)


def test_get_size_package_equals_restatement():
    from mqdet_b200.engine import transforms as tr
    for w, h, s, m in _size_triples():
        assert tr.get_size((w, h), s, m) == to.get_size((w, h), s, m)
    assert tr.get_size((1333, 800), 800, 1333) == (800, 1333)          # shorter side already equal: kept
    assert tr.get_size((4000, 1000), 800, 1333) == (333, 1332)         # clamped to round(1333 / 4) = 333; int(333 * 4.0) = 1332
    assert to.get_size((640, 480), 800, None) == (800, 1066)           # long side truncated


def _resample_pairs():
    rng = np.random.default_rng(11)
    pairs = [(4000, 1333), (3000, 1000), (1333, 4000), (480, 1066), (640, 800), (1, 1), (1, 2), (2, 1), (1, 5), (5, 1), (2, 7),
             (7, 2), (9, 9), (10000, 10), (997, 3), (3, 997), (1001, 999), (999, 1001), (6000, 1500), (333, 1000)]
    pairs += [(int(a), int(b)) for a, b in zip(rng.integers(1, 700, 200), rng.integers(1, 700, 200))]
    pairs += [(int(a), int(b)) for a, b in zip(rng.integers(1000, 6000, 40), rng.integers(50, 1400, 40))]   # large downscales
    pairs += [(int(a), int(b)) for a, b in zip(rng.integers(2, 60, 40) * 2 + 1, rng.integers(300, 2000, 40))]  # odd, large up
    return pairs


@pytest.mark.parametrize("axis", ["horizontal", "vertical"])
def test_resample_vs_pil(axis):
    """Each (in, out) pair on a thin image (3 pixels across the other axis), so hundreds of pairs run in seconds."""
    rng = np.random.default_rng(5 if axis == "horizontal" else 6)
    bad = []
    for n_in, n_out in _resample_pairs():
        shape = (3, n_in, 3) if axis == "horizontal" else (n_in, 3, 3)
        im = rng.integers(0, 256, shape, dtype=np.uint8)
        oh, ow = (3, n_out) if axis == "horizontal" else (n_out, 3)
        ref = np.asarray(Image.fromarray(im).resize((ow, oh), Image.BILINEAR))
        if not np.array_equal(to.resize(im, oh, ow), ref):
            bad.append((n_in, n_out))
    assert not bad, bad


def test_resize_2d_vs_pil():
    """Both passes together (the uint8 intermediate), including one dimension unchanged and large factors."""
    rng = np.random.default_rng(3)
    cases = [((480, 640), (800, 1066)), ((300, 400), (1000, 1333)), ((37, 53), (37, 91)), ((53, 37), (91, 37)),
             ((1, 1), (5, 3)), ((2, 2), (1, 1)), ((301, 199), (17, 11)), ((600, 4000), (200, 1333))]
    for (h, w), (oh, ow) in cases:
        im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = np.asarray(Image.fromarray(im).resize((ow, oh), Image.BILINEAR))
        assert np.array_equal(to.resize(im, oh, ow), ref), ((h, w), (oh, ow))


def test_normalize_vs_torchvision():
    import torchvision.transforms.functional as F
    rng = np.random.default_rng(9)
    im = rng.integers(0, 256, (19, 29, 3), dtype=np.uint8)
    im[0, :3] = [[0, 0, 0], [255, 255, 255], [1, 128, 254]]
    t = F.to_tensor(Image.fromarray(im))
    want = F.normalize(t[[2, 1, 0]] * 255, mean=GLIP["mean"], std=GLIP["std"])
    assert torch.equal(to.normalize(im, GLIP["mean"], GLIP["std"], "bgr255"), want)
    want = F.normalize(t, mean=GDINO["mean"], std=GDINO["std"])
    assert torch.equal(to.normalize(im, GDINO["mean"], GDINO["std"], "rgb"), want)


def test_boxlist_resize_vs_reference():
    from mqdet_b200.structures.bounding_box import BoxList
    g = torch.Generator().manual_seed(4)
    xy = torch.rand((12, 2), generator=g) * 500
    boxes = torch.cat((xy, xy + torch.rand((12, 2), generator=g) * 300), 1)
    cases = [((640, 480), (1066, 800), "xyxy"), ((1333, 1000), (4000, 3000), "xyxy"), ((640, 480), (1066, 799), "xyxy"),
             ((100, 60), (33, 61), "xywh")]

    def run():
        RB = ref_loader.bounding_box().BoxList
        out = []
        for size, new, mode in cases:
            bl = RB(boxes.clone(), size, mode="xyxy").convert(mode)
            bl.add_field("scores", torch.arange(12.0))
            r = bl.resize(new)
            out.append({"bbox": r.bbox, "scores": r.get_field("scores")})
        return out
    want = pinned("boxlist_resize", run)
    for (size, new, mode), w in zip(cases, want):
        bl = BoxList(boxes.clone(), size, mode="xyxy").convert(mode)
        bl.add_field("scores", torch.arange(12.0))
        r = bl.resize(new)
        assert r.size == new and r.mode == mode
        assert torch.equal(r.bbox, w["bbox"]) and torch.equal(r.get_field("scores"), w["scores"])


def test_config_keys_and_errors():
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.config import mq_glip_t_cfg, mq_groundingdino_t_cfg
    from mqdet_b200.engine import transforms as tr
    g = tr.TestTransform(mq_glip_t_cfg())
    assert (g.size, g.max_size, g.bgr, g.times255, g.div) == (800, 1333, True, True, 32)
    d = tr.TestTransform(mq_groundingdino_t_cfg())
    assert (d.size, d.max_size, d.bgr, d.times255) == (800, 1333, False, False)
    assert tr.TestTransform(mq_glip_t_cfg(), 400, 2500).size == 400
    with pytest.raises(ValueError, match="TO_BGR255"):
        tr.TestTransform(mq_glip_t_cfg(**{"INPUT.TO_BGR255": False}))
    with pytest.raises(ValueError, match="random"):
        tr.TestTransform(mq_glip_t_cfg(**{"INPUT.MIN_SIZE_TEST": (640, 800)}))
    with pytest.raises(MqdetError, match="uint8"):
        tr.upload([np.zeros((4, 4, 3), np.float32)], "cpu")
    with pytest.raises(MqdetError, match="uint8"):
        tr.upload([np.zeros((4, 4), np.uint8)], "cpu")


def test_abi_rejects_bad_arguments_without_gpu():
    import ctypes
    from mqdet_b200 import _lib
    lib = _lib.load()
    assert lib.mqdet_resize_coeffs_ksize(4000, 1333) == 2 * 4 + 1                   # support 3.0008 -> ceil 4
    assert lib.mqdet_resize_coeffs_ksize(480, 800) == 3
    assert lib.mqdet_resize_coeffs_ksize(0, 5) == 0
    for n_in, n_out in ((4000, 1333), (480, 800), (1, 7), (10000, 10)):
        assert lib.mqdet_resize_coeffs_ksize(n_in, n_out) == to.ksize(n_in, n_out)
    nul = ctypes.c_void_p(0)
    assert lib.mqdet_resize_coeffs(5, 3, nul, nul) < 0
    assert "null pointer" in lib.mqdet_last_error().decode()
    assert lib.mqdet_resize_coeffs(0, 3, ctypes.c_void_p(16), nul) < 0
    assert "bad lengths" in lib.mqdet_last_error().decode()
    one = (ctypes.c_void_p * 1)(16)
    hw = (ctypes.c_int64 * 2)(0, 5)
    ms = (ctypes.c_float * 3)(0.0, 0.0, 0.0)
    sd = (ctypes.c_float * 3)(1.0, 1.0, 1.0)
    assert lib.mqdet_test_transform(one, hw, one, one, 1, 4, 4, 4, 4, 0, 0, ms, sd, ctypes.c_void_p(16), nul, nul) < 0
    assert "bad size" in lib.mqdet_last_error().decode()
    hw = (ctypes.c_int64 * 2)(3, 5)
    assert lib.mqdet_test_transform(one, hw, one, one, 1, 4, 4, 3, 4, 0, 0, ms, sd, ctypes.c_void_p(16), nul, nul) < 0
    assert "padded" in lib.mqdet_last_error().decode()
    sd = (ctypes.c_float * 3)(1.0, 0.0, 1.0)
    assert lib.mqdet_test_transform(one, hw, one, one, 1, 4, 4, 4, 4, 0, 0, ms, sd, ctypes.c_void_p(16), nul, nul) < 0
    assert "std[1] is zero" in lib.mqdet_last_error().decode()
