"""BoxList — the output type of the drop-in boundary (maskrcnn_benchmark/structures/bounding_box.py:19-285).

Only the part of the interface that crosses the hot-path boundary: construction, per-box fields, indexing, device moves,
xyxy <-> xywh with the reference's inclusive-pixel (+1) convention, resizing, clipping, area.  The reference's class is a superset
and can be passed wherever this one is accepted; tests/test_host_cpu.py pins the shared behaviour against it.  ``boxlists_from_packed``
turns the detectors' packed fixed-shape results into BoxLists.
"""
import torch

_MODES = ("xyxy", "xywh")
_PIX = 1  # widths / heights count both end pixels (the reference's TO_REMOVE)


class BoxList(object):
    def __init__(self, bbox, image_size, mode="xyxy"):
        dev = bbox.device if torch.is_tensor(bbox) else torch.device("cpu")
        bbox = torch.as_tensor(bbox, dtype=torch.float32, device=dev)
        if bbox.ndimension() != 2 or bbox.size(-1) != 4:
            raise ValueError("bbox must be [n, 4], got shape {}".format(tuple(bbox.shape)))
        if mode not in _MODES:
            raise ValueError("mode should be 'xyxy' or 'xywh'")
        self.bbox, self.size, self.mode = bbox, image_size, mode  # size = (image_width, image_height)
        self.extra_fields = {}

    # ---- per-box fields ----
    def add_field(self, field, field_data):
        self.extra_fields[field] = field_data

    def get_field(self, field):
        return self.extra_fields[field]

    def has_field(self, field):
        return field in self.extra_fields

    def fields(self):
        return list(self.extra_fields)

    def _with(self, bbox, mode=None, fields=None):
        """New BoxList on `bbox` carrying `fields` (default: all of mine), each passed through unchanged."""
        out = BoxList(bbox, self.size, self.mode if mode is None else mode)
        out.extra_fields.update(self.extra_fields if fields is None else fields)
        return out

    def _copy_extra_fields(self, other):
        self.extra_fields.update(other.extra_fields)

    # ---- geometry ----
    def convert(self, mode):
        if mode not in _MODES:
            raise ValueError("mode should be 'xyxy' or 'xywh'")
        if mode == self.mode:
            return self
        b = self.bbox
        if mode == "xywh":
            wh = b[:, 2:] - b[:, :2] + _PIX
            return self._with(torch.cat((b[:, :2], wh), dim=-1), mode)
        far = b[:, :2] + (b[:, 2:] - _PIX).clamp(min=0)
        return self._with(torch.cat((b[:, :2], far), dim=-1), mode)

    def clip_to_image(self, remove_empty=True):
        w, h = self.size
        for col, hi in ((0, w), (1, h), (2, w), (3, h)):
            self.bbox[:, col].clamp_(min=0, max=hi - _PIX)
        if not remove_empty:
            return self
        b = self.bbox
        return self[(b[:, 3] > b[:, 1]) & (b[:, 2] > b[:, 0])]

    def resize(self, size):
        """Boxes scaled from ``self.size`` to ``size`` = (width, height): one tensor-times-ratio product when both ratios are
        equal, else per coordinate on the xyxy form; fields are carried over (those that are not tensors resized too)."""
        rw, rh = (float(s) / float(s0) for s, s0 in zip(size, self.size))
        fields = {k: (v if torch.is_tensor(v) else v.resize(size)) for k, v in self.extra_fields.items()}
        if rw == rh:
            out = BoxList(self.bbox * rw, size, self.mode)
        else:
            b = self.convert("xyxy").bbox
            out = BoxList(torch.cat((b[:, 0:1] * rw, b[:, 1:2] * rh, b[:, 2:3] * rw, b[:, 3:4] * rh), dim=-1), size, "xyxy")
        out.extra_fields.update(fields)
        return out.convert(self.mode)

    def area(self):
        b = self.bbox
        if self.mode == "xywh":
            return b[:, 2] * b[:, 3]
        return (b[:, 2] - b[:, 0] + _PIX) * (b[:, 3] - b[:, 1] + _PIX)

    # ---- container behaviour ----
    def to(self, device):
        moved = {k: (v.to(device) if hasattr(v, "to") else v) for k, v in self.extra_fields.items()}
        return self._with(self.bbox.to(device), fields=moved)

    def __getitem__(self, item):
        return self._with(self.bbox[item], fields={k: v[item] for k, v in self.extra_fields.items()})

    def __len__(self):
        return self.bbox.shape[0]

    def copy_with_fields(self, fields, skip_missing=False):
        names = fields if isinstance(fields, (list, tuple)) else [fields]
        picked = {}
        for f in names:
            if f in self.extra_fields:
                picked[f] = self.extra_fields[f]
            elif not skip_missing:
                raise KeyError("Field '{}' not found in {}".format(f, self))
        return self._with(self.bbox, fields=picked)

    def __repr__(self):
        return "BoxList(num_boxes={}, image_width={}, image_height={}, mode={})".format(len(self), self.size[0],
                                                                                         self.size[1], self.mode)


def boxlists_from_packed(packed, image_sizes, n_chunks=1):
    """Packed detections fp32 [B, n_chunks * rows, 6], on the host or the device -> one BoxList per image at its (h, w) of
    ``image_sizes``, mode xyxy, fields ``labels`` then ``scores``.  Per image, chunk c holds rows c * rows .. (c + 1) * rows - 1:
    its detections (x1, y1, x2, y2, score, label), then a count row (count, ...); the chunks' detections are concatenated in chunk
    order.  One device->host copy.  A count above its chunk's rows - 1 is an error, never a silent truncation: the rows kept are
    in candidate order, not score order."""
    from .._lib import MqdetError
    pk = packed.cpu()
    pk = pk.reshape(pk.shape[0], n_chunks, -1, 6)
    n_rows = pk.shape[2] - 1
    res = []
    for b, (h, w) in enumerate(image_sizes):
        parts = []
        for c in range(n_chunks):
            n = int(round(float(pk[b, c, n_rows, 0])))
            if n > n_rows:
                where = f"image {b}, chunk {c}" if n_chunks > 1 else f"image {b}"
                raise MqdetError(f"{where}: {n} detections exceed the {n_rows}-row result buffer")
            parts.append(pk[b, c, :n])
        d = torch.cat(parts) if n_chunks > 1 else parts[0]
        bl = BoxList(d[:, :4].clone(), (w, h), mode="xyxy")
        bl.add_field("labels", d[:, 5].long())
        bl.add_field("scores", d[:, 4].clone())
        res.append(bl)
    return res
