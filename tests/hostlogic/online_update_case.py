"""Host-logic dry run of ``engine/online_update.py`` (CPU, throw-away process): ``online_update`` composed over torch stand-ins of
``ops.QueryBank`` / ``ops.query_candidates`` / ``ops.roi_align_levels_counted`` / ``ops.query_bank_update`` (each restating its
kernel's specification in include/mqdet_b200.h through tests/online_update_oracle.py) and a stand-in MQ-GLIP whose ``forward_device``
returns fixed packed rows per image and per installed bank.  Every tensor the stand-ins hand to the engine records host reads, so the
run shows the launches per batch, that nothing is read on the host inside a turn, and which bank the evaluation is left with.

    python tests/hostlogic/online_update_case.py
"""
import os
import sys
from types import SimpleNamespace as NS

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_double  # noqa: F401,E402  (patches mqdet_b200.ops; must come first)
import torch  # noqa: E402

import online_update_oracle as ou  # noqa: E402
from mqdet_b200 import ops  # noqa: E402
from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New  # noqa: E402

LOG = []
_HOST_READS = {"item", "tolist", "cpu", "numpy", "__int__", "__float__", "__bool__", "__index__"}
C, M = 8, 12


class Dev(torch.Tensor):
    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        name = getattr(func, "__name__", "")
        if name in _HOST_READS or (name == "to" and any(str(a) == "cpu" for a in list(args[1:]) + list((kwargs or {}).values()))):
            LOG.append(("host read", name))
        return super().__torch_function__(func, types, args, kwargs or {})


def plain(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, Dev) else t


class QueryBank(ops.QueryBank):
    @classmethod
    def from_dict(cls, bank, L, min_cap, C, device):
        items = {int(k): v for k, v in (bank or {}).items() if torch.is_tensor(v) and len(v)}
        qb = cls(L, max([min_cap] + [len(v) for v in items.values()]), C, device)
        for k, v in items.items():
            qb.rows[k, :len(v)] = v[:, 0]
            qb.count[k] = len(v)
        qb.count = qb.count.as_subclass(Dev)
        return qb


def query_candidates(packed, img_wh, score_thr, expand_ratio, bad):
    LOG.append(("candidates", tuple(img_wh)))
    packed = plain(packed)
    B = packed.shape[0]
    rois, labels = torch.zeros(B * M, 5), torch.zeros(B * M, dtype=torch.int32)
    n = 0
    for b in range(B):
        c = ou.candidates(packed[b], img_wh, score_thr, expand_ratio)
        if c is ou.BAD_COUNT:
            bad += 1
            continue
        k = c[0].shape[0]
        rois[n:n + k, 0], rois[n:n + k, 1:], labels[n:n + k] = float(b), c[0], c[1].int()
        n += k
    return rois.as_subclass(Dev), labels.as_subclass(Dev), torch.tensor([n], dtype=torch.int32).as_subclass(Dev)


def roi_align_levels_counted(pyr16, levels, scales, rois, count, pooled=7, sampling_ratio=0):
    LOG.append(("pool",))
    rois, n, tags = plain(rois), int(plain(count)), plain(pyr16)[:, 0, 0]
    out = torch.full((rois.shape[0], C), float("nan"))
    out[:n] = pool(tags[rois[:n, 0].long()], rois[:n, 1:])
    return out.as_subclass(Dev)


def query_bank_update(bank, feats, labels, count, max_query, sim_thr):
    LOG.append(("update", max_query))
    n = int(plain(count))
    d = bank.as_dict(plain(bank.count))
    ou.bank_update(d, plain(labels)[:n].long(), plain(feats)[:n], max_query, sim_thr)
    for k, v in d.items():
        bank.rows[k, :len(v)] = plain(v)[:, 0]
        bank.count[k] = len(v)
    return bank


ops.QueryBank, ops.query_candidates, ops.roi_align_levels_counted, ops.query_bank_update = \
    QueryBank, query_candidates, roi_align_levels_counted, query_bank_update


def pool(img_tags, boxes):
    """Features of boxes [R, 4] of the images tagged ``img_tags`` [R]: a cluster direction from the box position plus a perturbation."""
    g = torch.Generator().manual_seed(11)
    dirs, W = torch.randn(24, C, generator=g), torch.randn(4, C, generator=g)
    cl = ((boxes[:, 0] + boxes[:, 1]) / 7).floor().long() % 24
    return dirs[cl] + 0.3 * torch.sin(boxes @ W / 7 + img_tags[:, None])


def detect(im, held, wh):
    g = torch.Generator().manual_seed(im)
    w, h = wh
    x1, y1 = torch.rand(M, generator=g) * (w - 20), torch.rand(M, generator=g) * (h - 20)
    out = torch.zeros(M + 1, 6)
    out[:M, 0], out[:M, 1] = x1, y1
    out[:M, 2], out[:M, 3] = x1 + 4 + torch.rand(M, generator=g) * w * 0.5, y1 + 4 + torch.rand(M, generator=g) * h * 0.5
    rows = sum(len(v) for v in held.values()) if held else 0
    out[:M, 4] = (0.3 + 0.7 * torch.rand(M, generator=g) + 0.2 * (1 - 1 / (1 + rows))).clamp(max=0.99)
    out[:M, 5] = torch.randint(1, 4, (M,), generator=g).float()
    out[M, 0] = M
    return out


class Selector:
    def __init__(self, bank):
        self.query_bank = bank

    def set_query_bank(self, bank):
        LOG.append(("install",))
        self.query_bank = bank


class Detector(GeneralizedVLRCNN_New):
    def __init__(self, cfg, bank):
        torch.nn.Module.__init__(self)
        self.cfg, self.query_selector, self.rpn, self._prompt = cfg, Selector(bank), NS(_tokmap=None), None
        self.pooler = NS(scales=(0.125, 0.0625), output_size=(7, 7), sampling_ratio=0)

    def forward_device(self, images, captions, positive_map, max_out=None):
        x = plain(images.tensors)
        h, w = images.image_sizes[0]
        tags = x[:, 0, 0, 0]
        LOG.append(("forward", x.shape[0]))
        held = self.query_selector.query_bank
        pk = torch.stack([detect(int(t), held, (w, h)) for t in tags])
        pyr = tags[:, None, None].expand(-1, 5, C).contiguous()
        return {"det_packed": pk.as_subclass(Dev), "pyramid16": pyr.as_subclass(Dev), "levels": NS(n=2, sizes=[(2, 2), (1, 1)]),
                "image_sizes": images.image_sizes}


def main():
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.engine.online_update import make_batches, online_update
    sizes = [(80, 96)] * 5 + [(72, 128)] * 2 + [(80, 96)] * 2
    imgs = []
    for i, (h, w) in enumerate(sizes):
        x = torch.zeros(3, h, w)
        x[0, 0, 0] = i
        imgs.append(x)
    g = torch.Generator().manual_seed(3)
    start = {1: torch.randn(2, 1, C, generator=g), 3: torch.randn(1, 1, C, generator=g)}
    for turns in (1, 3):
        for B in (1, 4):
            cfg = mq_glip_t_cfg(**{"VISION_QUERY.NUM_TURNS": turns, "VISION_QUERY.MAX_TEST_QUERY_NUMBER": 5, "MODEL.BACKBONE.OUT_CHANNELS": C})
            model = Detector(cfg, ou.copy_bank(start))
            batches = make_batches(imgs, B)
            assert [len(b.image_sizes) for b in batches] == ([1] * 9 if B == 1 else [4, 1, 2, 2])
            LOG.clear()
            res = online_update(model, batches, "caption", {1: [1], 2: [3], 3: [5]}, cfg, bank=start)
            log = []
            for e in LOG:                               # the host reads at the end of a turn collapse to one entry
                if not (e[0] == "host read" and log and log[-1] == "host read"):
                    log.append("host read" if e[0] == "host read" else e)
            per_batch = []
            for b in batches:
                h, w = b.image_sizes[0]
                per_batch += [("forward", len(b.image_sizes)), ("candidates", (w, h)), ("pool",), ("update", 5)]
            want = (per_batch + ["host read"]) + ([("install",)] + per_batch + ["host read"]) * (turns - 1)
            assert log == want, (turns, B, log)
            banks, held, _ = ou.online_update(lambda im, hb: detect(im, hb, (sizes[im][1], sizes[im][0])),
                                              lambda im, bx: pool(torch.full((bx.shape[0],), float(im)), bx), list(range(9)),
                                              [(w, h) for h, w in sizes], start, ou.copy_bank(start), turns, max_query=5)
            for got, ref in zip(res["banks"], banks):
                assert sorted(k for k, v in got.items() if len(v)) == sorted(k for k, v in ref.items() if len(v))
                for k, v in ref.items():
                    assert torch.equal(plain(got[k]), v), (turns, B, k)
            ev = res["eval_bank"]
            assert ev is model.query_selector.query_bank
            if turns == 1:
                assert all(torch.equal(ev[k], start[k]) for k in start) and len(ev) == len(start)
            else:
                assert ev is res["banks"][1]                # the evaluation uses the bank after turn 2
            assert sum(len(v) for v in banks[-1].values()) > 3
    # bank=None: the starting bank is read from VISION_QUERY.QUERY_BANK_PATH, a file in the reference's format (torch.save of a
    # defaultdict(list), as engine/inference.py and tools/train_net.py write it)
    import tempfile
    from collections import defaultdict
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "bank.pth")
        ref_bank = defaultdict(list)
        ref_bank.update(start)
        ref_bank[2]                                        # a label looked up without exemplars: saved as []
        torch.save(ref_bank, path)
        cfg = mq_glip_t_cfg(**{"VISION_QUERY.NUM_TURNS": 3, "VISION_QUERY.MAX_TEST_QUERY_NUMBER": 5, "MODEL.BACKBONE.OUT_CHANNELS": C,
                               "VISION_QUERY.QUERY_BANK_PATH": path})
        from_file = online_update(Detector(cfg, ou.copy_bank(start)), make_batches(imgs, 4), "caption", {1: [1], 2: [3], 3: [5]}, cfg)
        explicit = online_update(Detector(cfg, ou.copy_bank(start)), make_batches(imgs, 4), "caption", {1: [1], 2: [3], 3: [5]}, cfg,
                                 bank=start)
        for a, b in zip(from_file["banks"], explicit["banks"]):
            assert sorted(a) == sorted(b) and all(torch.equal(plain(a[k]), plain(b[k])) for k in a)
    print("PASS online_update")


if __name__ == "__main__":
    main()
