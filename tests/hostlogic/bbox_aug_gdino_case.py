"""Host-logic dry run of ``engine/bbox_aug.py`` for a ``GroundingDINO`` model (CPU, throw-away process): ``im_detect_bbox_aug``
composed over torch stand-ins of ``ops.hflip_pad`` / ``ops.bbox_aug_collect_packed`` / ``ops.nms_by_class`` (each restating its
kernel's specification in include/mqdet_b200.h through tests/bbox_aug_gdino_oracle.py and tests/bbox_aug_oracle.py) and a
stand-in GroundingDINO whose ``forward_chunked_device`` returns fixed packed rows per pass.  Every tensor the stand-ins hand to
the engine records host reads (``item``, ``cpu``, ``int()`` ...), so the run shows the order of the launches and that the engine
reads nothing on the host before ``unpack`` — not the kernels.

    python tests/hostlogic/bbox_aug_gdino_case.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_double  # noqa: F401,E402  (patches mqdet_b200.ops; must come first)
import torch  # noqa: E402

import bbox_aug_gdino_oracle as go  # noqa: E402
import bbox_aug_oracle as bo  # noqa: E402
from mqdet_b200 import ops  # noqa: E402
from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO  # noqa: E402

LOG = []
_HOST_READS = {"item", "tolist", "cpu", "numpy", "__int__", "__float__", "__bool__", "__index__"}


class Dev(torch.Tensor):
    """A tensor the engine receives from a device op: reading it on the host is logged."""

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        name = getattr(func, "__name__", "")
        if name in _HOST_READS or (name == "to" and any(str(a) == "cpu" for a in list(args[1:]) + list((kwargs or {}).values()))):
            LOG.append(("host read", name))
        return super().__torch_function__(func, types, args, kwargs or {})


def plain(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, Dev) else t


def hflip_pad(images, out_hw):
    images = plain(images)
    B, C, h, w = images.shape
    out = torch.zeros(B, C, *out_hw)
    out[..., :h, :w] = torch.flip(images, dims=[-1])
    return out.as_subclass(Dev)


def bbox_aug_collect(*a, **k):
    raise AssertionError("the GroundingDINO branch must not use the cand_* collect")


def bbox_aug_collect_packed(merged, packed, pass_size, orig_size, *, flip=False, keep_range=None):
    LOG.append(("collect", tuple(pass_size), flip, keep_range))
    packed = plain(packed)
    assert packed.is_contiguous() and packed.dim() == 3 and packed.shape[0] == merged.B
    rest = [dict(boxes=merged.boxes[b, :int(merged.count[b])], scores=merged.scores[b, :int(merged.count[b])],
                 labels=merged.labels[b, :int(merged.count[b])].long(), overflow=int(merged.overflow[b]), cap=merged.cap)
            for b in range(merged.B)]
    go.collect_packed(rest, packed, pass_size, orig_size, flip, keep_range)
    for b, m in enumerate(rest):
        n = m["boxes"].shape[0]
        merged.boxes[b, :n], merged.scores[b, :n], merged.labels[b, :n] = m["boxes"], m["scores"], m["labels"].int()
        merged.count[b], merged.overflow[b] = n, m["overflow"]
    return merged


def nms_by_class(boxes, scores, labels, count, classes, thresh, *, mode="nms", top_n=0, max_out, overflow=None):
    LOG.append(("merge", mode))
    B = scores.shape[0]
    out = torch.zeros(B, max_out + 1, 6)
    for b in range(B):
        n = int(count[b])
        rb, rs, rl = bo.merge(boxes[b, :n], scores[b, :n], labels[b, :n].long(), classes.tolist(), thresh, mode, top_n)
        k = min(rb.shape[0], max_out)
        out[b, :k, :4], out[b, :k, 4], out[b, :k, 5] = rb[:k], rs[:k], rl[:k].float()
        out[b, max_out, 0] = rb.shape[0]
        out[b, max_out, 1] = 0 if overflow is None else float(overflow[b])
    return out.as_subclass(Dev)


ops.hflip_pad, ops.bbox_aug_collect, ops.bbox_aug_collect_packed, ops.nms_by_class = \
    hflip_pad, bbox_aug_collect, bbox_aug_collect_packed, nms_by_class


class Detector(GroundingDINO):
    """GroundingDINO stand-in: packed rows that depend on the pass (its size and whether the batch arrived flipped)."""

    M = 60

    def __init__(self, cfg, B, bad_count=False):
        torch.nn.Module.__init__(self)
        self.cfg, self.B, self.bad_count = cfg, B, bad_count

    def rows(self, size, flipped, b):
        g = torch.Generator().manual_seed(size[0] * 4 + 2 * int(flipped) + b)
        n = 0 if (size[0] == 244 and flipped and b == 1) else (self.M if b == 0 else 17)
        return go.gdino_rows(g, n, size, 5)

    def forward_device(self, *a, **k):
        raise AssertionError("forward_device takes one stable-softmax maximum over the batch; TTA runs the chunked path")

    def forward_chunked_device(self, images, chunk_captions, chunk_positive_maps, chunks_per_pass=8, chunk_ids=None):
        x = plain(images.tensors)
        h, w = images.image_sizes[0]
        assert x.shape[-2] % 32 == 0 and x.shape[-1] % 32 == 0 and (x[..., h:, :] == 0).all() and (x[..., w:] == 0).all()
        assert chunk_captions == ["caption"] and chunk_positive_maps == ["pmap"] and chunk_ids is None
        flipped = bool(x[0, 0, 0, 0] < 0)          # the un-flipped test images carry a negative right edge
        LOG.append(("forward", (w, h), flipped))
        pk = torch.stack([go.pack(*self.rows((w, h), flipped, b), self.M) for b in range(self.B)])
        if self.bad_count:
            pk[1, self.M, 0] = 0.5
        return {"det_packed": pk[None].contiguous().as_subclass(Dev), "chunks": [0]}


def main():
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.engine import bbox_aug
    B, orig = 2, (203, 150)
    sizes = [(162, 120), (203, 150), (244, 180)]
    ranges = ((24, 10000), (0, 10000), (0, 120))
    for special in ("none", "vote"):
        cfg = mq_groundingdino_t_cfg(**{"TEST.SCALES": (120, 150, 180), "TEST.RANGES": ranges, "TEST.FLIP": True,
                                        "TEST.SPECIAL_NMS": special, "TEST.NUM_CLASSES": 6, "TEST.PRE_NMS_TOP_N": 40})
        imgs = []
        for w, h in sizes:
            x = torch.rand(B, 3, h, w) + 0.5
            x[..., -1] = -1.0
            imgs.append(x.as_subclass(Dev))
        det = Detector(cfg, B)
        LOG.clear()
        packed, merged = bbox_aug.im_detect_bbox_aug_device(det, imgs, [orig] * B, "caption", "pmap")
        want_log = []
        for s, r in zip(sizes, ranges):
            for f in (False, True):
                want_log += [("forward", s, f), ("collect", s, f, r)]
        want_log.append(("merge", "vote" if special == "vote" else "nms"))
        assert LOG == want_log, LOG                   # one forward + one collect per pass, one merge, no host read
        assert merged.cap == len(want_log) // 2 * Detector.M
        res = bbox_aug.unpack(packed, [orig] * B)
        assert LOG[len(want_log)] == ("host read", "cpu")
        per_pass = [(s, f, r, [det.rows(s, f, b) for b in range(B)]) for s, r in zip(sizes, ranges) for f in (False, True)]
        want, union = bo.merge_candidates(per_pass, [orig] * B, cfg.TEST)
        for r, (wb, ws, wl) in zip(res, want):
            assert r.size == orig and torch.equal(r.bbox, wb) and torch.equal(r.get_field("scores"), ws)
            assert torch.equal(r.get_field("labels"), wl) and 0 < len(r)
        try:
            bbox_aug.im_detect_bbox_aug(Detector(cfg, B), imgs, [orig] * B, "caption", "pmap", cap=union[0][0].shape[0] - 1)
            raise AssertionError("a full merged buffer must raise")
        except MqdetError as e:
            assert "did not fit" in str(e)
        try:
            bbox_aug.im_detect_bbox_aug(Detector(cfg, B, bad_count=True), imgs, [orig] * B, "caption", "pmap")
            raise AssertionError("a bad count row must raise")
        except MqdetError as e:
            assert "image 1" in str(e) and "count row" in str(e)
        try:
            bbox_aug.im_detect_bbox_aug(Detector(cfg, B), imgs, [orig, (204, 150)], "caption", "pmap")
            raise AssertionError("images of different original sizes must raise")
        except NotImplementedError:
            pass
    print("PASS bbox_aug_gdino")


if __name__ == "__main__":
    main()
