"""Host-logic dry run of ``engine/bbox_aug.py`` (CPU, throw-away process): ``im_detect_bbox_aug`` composed over torch stand-ins of
``ops.hflip_pad`` / ``ops.bbox_aug_collect`` / ``ops.nms_by_class`` (each restating its kernel's specification in
include/mqdet_b200.h through tests/bbox_aug_oracle.py) and a stand-in detector that returns fixed candidates per pass.  It checks
the pass order, the flip / range / size handed to every collect, the padded batch shapes and the unpacking — not the kernels.

    python tests/hostlogic/bbox_aug_case.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_double  # noqa: F401,E402  (patches mqdet_b200.ops; must come first)
import torch  # noqa: E402

import bbox_aug_oracle as bo  # noqa: E402
from mqdet_b200 import ops  # noqa: E402


def hflip_pad(images, out_hw):
    B, C, h, w = images.shape
    out = torch.zeros(B, C, *out_hw)
    out[..., :h, :w] = torch.flip(images, dims=[-1])
    return out


def bbox_aug_collect(merged, cb, cs, cl, totals, pass_size, orig_size, *, flip=False, keep_range=None):
    for b in range(merged.B):
        n = int(totals[b])
        bx, sc, lb = bo.collect_pass(cb[b, :n], cs[b, :n], cl[b, :n], pass_size, orig_size, flip, keep_range)
        c, k = int(merged.count[b]), min(bx.shape[0], merged.cap - int(merged.count[b]))
        merged.boxes[b, c:c + k], merged.scores[b, c:c + k], merged.labels[b, c:c + k] = bx[:k], sc[:k], lb[:k].int()
        merged.count[b] += k
        merged.overflow[b] += bx.shape[0] - k
    return merged


def nms_by_class(boxes, scores, labels, count, classes, thresh, *, mode="nms", top_n=0, max_out, overflow=None):
    B = scores.shape[0]
    out = torch.zeros(B, max_out + 1, 6)
    for b in range(B):
        n = int(count[b])
        rb, rs, rl = bo.merge(boxes[b, :n], scores[b, :n], labels[b, :n].long(), classes.tolist(), thresh, mode, top_n)
        k = min(rb.shape[0], max_out)
        out[b, :k, :4], out[b, :k, 4], out[b, :k, 5] = rb[:k], rs[:k], rl[:k].float()
        out[b, max_out, 0] = rb.shape[0]
        out[b, max_out, 1] = 0 if overflow is None else float(overflow[b])
    return out


ops.hflip_pad, ops.bbox_aug_collect, ops.nms_by_class = hflip_pad, bbox_aug_collect, nms_by_class


class Detector:
    """forward_device stand-in: candidates that depend on the pass (its size and whether the batch arrived flipped)"""

    def __init__(self, cfg, B):
        self.cfg, self.B, self.calls = cfg, B, []

    def candidates(self, size, flipped, b):
        g = torch.Generator().manual_seed(size[0] * 4 + 2 * int(flipped) + b)
        return bo._objects(g, 5, 8, size, 5)

    def forward_device(self, images, captions, positive_map):
        x = images.tensors
        h, w = images.image_sizes[0]
        assert x.shape[-2] % 32 == 0 and x.shape[-1] % 32 == 0 and (x[..., h:, :] == 0).all() and (x[..., w:] == 0).all()
        flipped = bool(x[0, 0, 0, 0] < 0)          # the un-flipped test images carry a negative right edge
        self.calls.append(((w, h), flipped))
        S = 64
        cb, cs, cl = torch.zeros(self.B, S, 4), torch.zeros(self.B, S), torch.zeros(self.B, S)
        tot = torch.zeros(self.B, dtype=torch.int32)
        for b in range(self.B):
            bx, sc, lb = self.candidates((w, h), flipped, b)
            n = bx.shape[0]
            cb[b, :n], cs[b, :n], cl[b, :n], tot[b] = bx, sc, lb.float(), n
        return {"cand_boxes": cb, "cand_scores": cs, "cand_labels": cl, "cand_totals": tot}


def main():
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.engine import bbox_aug
    B, orig = 2, (203, 150)
    sizes = [(162, 120), (203, 150), (244, 180)]
    for special in ("none", "vote"):
        cfg = mq_glip_t_cfg(**{"TEST.SCALES": (120, 150, 180), "TEST.RANGES": ((24, 10000), (0, 10000), (0, 120)), "TEST.FLIP": True,
                               "TEST.SPECIAL_NMS": special, "TEST.NUM_CLASSES": 6, "TEST.PRE_NMS_TOP_N": 40})
        imgs = []
        for w, h in sizes:
            x = torch.rand(B, 3, h, w) + 0.5
            x[..., -1] = -1.0
            imgs.append(x)
        det = Detector(cfg, B)
        res = bbox_aug.im_detect_bbox_aug(det, imgs, [orig] * B, None, None)
        assert det.calls == [(s, f) for s in sizes for f in (False, True)], det.calls
        per_pass = [(s, f, r, [det.candidates(s, f, b) for b in range(B)])
                    for s, r in zip(sizes, cfg.TEST.RANGES) for f in (False, True)]
        want, union = bo.merge_candidates(per_pass, [orig] * B, cfg.TEST)
        for r, (wb, ws, wl) in zip(res, want):
            assert r.size == orig and torch.equal(r.bbox, wb) and torch.equal(r.get_field("scores"), ws)
            assert torch.equal(r.get_field("labels"), wl) and 0 < len(r)
        try:
            bbox_aug.im_detect_bbox_aug(Detector(cfg, B), imgs, [orig] * B, None, None, cap=union[0][0].shape[0] - 1)
            raise AssertionError("a full merged buffer must raise")
        except MqdetError as e:
            assert "did not fit" in str(e)
    print("PASS bbox_aug")


if __name__ == "__main__":
    main()
