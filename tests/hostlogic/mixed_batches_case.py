"""Host-logic dry run of ``engine/online_update.py`` over the reference's padded batches of differently sized images (CPU, throw-away
process).  It reuses the stand-ins of online_update_case.py (ops test double, packed rows per image and per installed bank) with two
changes: ``ops.query_candidates`` takes one size or one size per image, and the stand-in MQ-GLIP runs the detector's real
``_prompt_state`` cache, its query selector logging every rebuild.  The run shows the launches per batch, the sizes each batch hands
to the candidates, that nothing is read on the host inside a turn, that the prompt state is rebuilt only after a bank install or when
the batch count changes, and that the bank equals the one-image restatement over the images in batch order.

    python tests/hostlogic/mixed_batches_case.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import online_update_case as oc  # noqa: E402  (patches mqdet_b200.ops with its stand-ins)
import torch  # noqa: E402

import online_update_oracle as ou  # noqa: E402
from mqdet_b200 import ops  # noqa: E402

LOG, Dev, plain, C, M = oc.LOG, oc.Dev, oc.plain, oc.C, oc.M


def query_candidates(packed, img_wh, score_thr, expand_ratio, bad):
    per_image = isinstance(img_wh[0], (tuple, list))
    LOG.append(("candidates", [tuple(s) for s in img_wh] if per_image else tuple(img_wh)))
    packed = plain(packed)
    B = packed.shape[0]
    rois, labels = torch.zeros(B * M, 5), torch.zeros(B * M, dtype=torch.int32)
    n = 0
    for b in range(B):
        c = ou.candidates(packed[b], img_wh[b] if per_image else img_wh, score_thr, expand_ratio)
        k = c[0].shape[0]
        rois[n:n + k, 0], rois[n:n + k, 1:], labels[n:n + k] = float(b), c[0], c[1].int()
        n += k
    return rois.as_subclass(Dev), labels.as_subclass(Dev), torch.tensor([n], dtype=torch.int32).as_subclass(Dev)


ops.query_candidates = query_candidates


class Selector(oc.Selector):
    bank_version = 0

    def set_query_bank(self, bank):
        super().set_query_bank(bank)
        self.bank_version += 1

    def __call__(self, labels, maps, _):
        LOG.append(("prompt rebuild", len(labels)))
        B = len(labels)
        return torch.zeros(B, 1, 256), torch.zeros(B, 1, 256), [[1] * len(labels[0])] * B


class Detector(oc.Detector):
    def __init__(self, cfg, bank):
        super().__init__(cfg, bank)
        self.query_selector = Selector(bank)

    def forward_device(self, images, captions, positive_map, max_out=None):
        x = plain(images.tensors)
        B = x.shape[0]
        self._prompt_state(captions, positive_map, B, torch.device("cpu"))     # the detector's real prompt cache
        tags = x[:, 0, 0, 0]
        LOG.append(("forward", B))
        held = self.query_selector.query_bank
        pk = torch.stack([oc.detect(int(t), held, (w, h)) for t, (h, w) in zip(tags, images.image_sizes)])
        pyr = tags[:, None, None].expand(-1, 5, C).contiguous()
        return {"det_packed": pk.as_subclass(Dev), "pyramid16": pyr.as_subclass(Dev), "levels": oc.NS(n=2, sizes=[(2, 2), (1, 1)]),
                "image_sizes": images.image_sizes}


def main():
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.engine.batches import reference_test_batches
    from mqdet_b200.engine.online_update import make_batches, online_update
    sizes = [(80, 96), (96, 72), (72, 128), (80, 96), (80, 96), (96, 80), (72, 128), (80, 96), (72, 128), (80, 96), (96, 72)]
    imgs = []
    for i, (h, w) in enumerate(sizes):
        x = torch.zeros(3, h, w)
        x[0, 0, 0] = i
        imgs.append(x)
    g = torch.Generator().manual_seed(3)
    start = {1: torch.randn(2, 1, C, generator=g), 3: torch.randn(1, 1, C, generator=g)}
    caps = {"input_ids": torch.tensor([[101, 1037, 1038, 1039, 1040, 1041, 102]]), "attention_mask": torch.ones(1, 7, dtype=torch.long)}
    pmap = {1: [1], 2: [3], 3: [5]}
    for turns in (1, 3):
        for grouping in (True, False):
            idx = reference_test_batches(sizes, 4, grouping)
            assert [len(b) for b in idx] == ([4, 3, 4] if grouping else [4, 4, 3]), idx
            cfg = mq_glip_t_cfg(**{"VISION_QUERY.NUM_TURNS": turns, "VISION_QUERY.MAX_TEST_QUERY_NUMBER": 5,
                                   "MODEL.BACKBONE.OUT_CHANNELS": C})
            model = Detector(cfg, ou.copy_bank(start))
            batches = make_batches(imgs, 4, 32, orig_hw=sizes, aspect_grouping=grouping)
            assert [il.image_sizes for il in batches] == [[sizes[i] for i in b] for b in idx]
            assert all(len(set(il.image_sizes)) > 1 for il in batches)              # every batch mixes sizes
            LOG.clear()
            res = online_update(model, batches, caps, pmap, cfg, bank=start)
            log = []
            for e in LOG:                               # the host reads at the end of a turn collapse to one entry
                if not (e[0] == "host read" and log and log[-1] == "host read"):
                    log.append("host read" if e[0] == "host read" else e)
            want, prev = [], None
            for turn in range(turns):
                if turn > 0:
                    want.append(("install",))
                    prev = None
                for il in batches:
                    B = len(il.image_sizes)
                    if B != prev:                       # the prompt cache holds one batch count (and one bank)
                        want.append(("prompt rebuild", B))
                    prev = B
                    want += [("forward", B), ("candidates", [(w, h) for h, w in il.image_sizes]), ("pool",), ("update", 5)]
                want.append("host read")
            assert log == want, (turns, grouping, log)
            order = [i for b in idx for i in b]
            banks, _, _ = ou.online_update(lambda im, hb: oc.detect(im, hb, (sizes[im][1], sizes[im][0])),
                                           lambda im, bx: oc.pool(torch.full((bx.shape[0],), float(im)), bx), order,
                                           [(sizes[i][1], sizes[i][0]) for i in order], start, ou.copy_bank(start), turns, max_query=5)
            for got, ref in zip(res["banks"], banks):
                assert sorted(k for k, v in got.items() if len(v)) == sorted(k for k, v in ref.items() if len(v))
                for k, v in ref.items():
                    assert torch.equal(plain(got[k]), v), (turns, grouping, k)
            assert sum(len(v) for v in banks[-1].values()) > 3
    print("PASS mixed online_update")


if __name__ == "__main__":
    main()
