"""The test transform on the device: decoded uint8 images -> the normalised, padded batch the detectors take.

Drop-in for the inference side of maskrcnn_benchmark/data/transforms (build_transforms(cfg, is_train=False): Resize(MIN_SIZE_TEST,
MAX_SIZE_TEST) -> ToTensor -> Normalize(PIXEL_MEAN, PIXEL_STD, format)) followed by to_image_list(SIZE_DIVISIBILITY).  The
reference resizes a PIL image with PIL's bilinear resampler; ``ops.test_transform`` reproduces it bit for bit, together with
the fp32 rounding of ToTensor and Normalize, in one launch per batch (csrc/transform.cu, DESIGN.md section 4).  Each image
crosses to the device once, as uint8 from pinned staging, instead of the resized fp32 batch the host path uploads (11x fewer
bytes for a 640 x 480 image resized to 800 x 1066).
"""
import numpy as np
import torch

from .. import ops
from .._lib import MqdetError
from ..structures.image_list import ImageList


def get_size(image_size, size, max_size):
    """Resize.get_size (restrict=False): (w, h) -> (oh, ow).  The shorter side becomes ``size`` unless the longer side would
    exceed ``max_size``; then ``size`` is round(max_size * short / long).  The longer side is truncated, and an image whose
    shorter side already equals ``size`` keeps its size."""
    w, h = image_size
    short, long_ = float(min(w, h)), float(max(w, h))
    if max_size is not None and long_ / short * size > max_size:
        size = int(round(max_size * short / long_))
    if min(w, h) == size:
        return h, w
    if w < h:
        return int(size * h / w), size
    return size, int(size * w / h)


def _format(inp):
    """INPUT.FORMAT when set, else 'bgr255' under INPUT.TO_BGR255 (build_transforms)."""
    if inp.FORMAT != "":
        return inp.FORMAT.lower()
    if inp.TO_BGR255:
        return "bgr255"
    raise ValueError("INPUT.FORMAT is empty and INPUT.TO_BGR255 is off: the reference defines no input format for that")


def _cuda_device(device):
    device = torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if device.type == "cuda" and device.index is None else device


def upload(images, device):
    """uint8 HWC RGB images (numpy arrays or tensors) -> contiguous uint8 CUDA tensors [h, w, 3].  Host images are staged in
    one pinned buffer and cross to the device in one asynchronous copy; images already on ``device`` are used as they are."""
    device = _cuda_device(device)
    out, host = [], []
    for i, im in enumerate(images):
        if not torch.is_tensor(im):
            im = np.asarray(im)
        u8 = im.dtype == torch.uint8 if torch.is_tensor(im) else im.dtype == np.uint8
        if not u8 or im.ndim != 3 or im.shape[2] != 3 or min(im.shape[:2]) < 1:
            raise MqdetError(f"image {i}: uint8 [h, w, 3] RGB required (got {im.dtype} {tuple(im.shape)})")
        if torch.is_tensor(im) and im.is_cuda:
            if im.device != device:
                raise MqdetError(f"image {i} is on {im.device}, not {device}")
            out.append(im.contiguous())
        else:
            out.append(None)
            host.append((i, im))
    if host:
        n = sum(int(np.prod(im.shape)) for _, im in host)
        staging = torch.empty((n,), dtype=torch.uint8, pin_memory=True)
        flat = staging.numpy()
        off = 0
        for _, im in host:
            k = int(np.prod(im.shape))
            flat[off:off + k].reshape(im.shape)[...] = im.numpy() if torch.is_tensor(im) else im
            off += k
        dst = torch.empty((n,), dtype=torch.uint8, device=device)
        dst.copy_(staging, non_blocking=True)
        off = 0
        for i, im in host:
            k = int(np.prod(im.shape))
            out[i] = dst[off:off + k].view(tuple(im.shape))
            off += k
    return out


class TestTransform:
    """build_transforms(cfg, is_train=False) + to_image_list on the device.  ``scale`` / ``max_size`` replace
    INPUT.MIN_SIZE_TEST / MAX_SIZE_TEST (the per-scale transforms of box_aug.py)."""

    __test__ = False   # not a pytest class

    def __init__(self, cfg, scale=None, max_size=None):
        inp = cfg.INPUT
        size = inp.MIN_SIZE_TEST if scale is None else scale
        if isinstance(size, (list, tuple)):
            if len(size) != 1:
                raise ValueError(f"one test size required (got {tuple(size)}): Resize would pick one at random")
            size = size[0]
        self.size = int(size)
        self.max_size = inp.MAX_SIZE_TEST if max_size is None else max_size
        fmt = _format(inp)
        self.bgr, self.times255 = "bgr" in fmt, "255" in fmt
        self.mean = [float(np.float32(v)) for v in inp.PIXEL_MEAN]
        self.std = [float(np.float32(v)) for v in inp.PIXEL_STD]
        if len(self.mean) != 3 or len(self.std) != 3:
            raise ValueError("INPUT.PIXEL_MEAN and INPUT.PIXEL_STD need three channels")
        if 0.0 in self.std:
            raise ValueError(f"INPUT.PIXEL_STD {tuple(inp.PIXEL_STD)} is zero in fp32 (Normalize divides by it)")
        self.div = int(cfg.DATALOADER.SIZE_DIVISIBILITY)

    def target_size(self, h, w):
        return get_size((w, h), self.size, self.max_size)

    def __call__(self, images, device, pad=True, want_resized=False, mixed_sizes=False, out=None):
        """images: uint8 HWC RGB numpy arrays or tensors (host or ``device``) -> (ImageList, orig_sizes [(w, h)]).  By default all
        images must resize to one size, so that a batch holds no padding beyond SIZE_DIVISIBILITY and ``want_resized`` has one
        shape.  ``pad=False`` leaves the batch at the resized size; ``want_resized`` adds the resized uint8 images [B, oh, ow, 3]
        as a third result.

        ``mixed_sizes=True`` takes images that resize to different sizes, as the reference's test loader batches them: each is
        resized to its own target size and the batch is zero-padded to the largest, rounded up to SIZE_DIVISIBILITY (its
        ``to_image_list``); ``image_sizes`` holds every image's own target size.  ``want_resized`` is then refused.

        ``out``: a flat fp32 buffer on ``device`` to write the batch into (its leading B * 3 * Hp * Wp elements, which the returned
        ImageList's tensor views), e.g. a staging buffer a captured graph reads."""
        if len(images) == 0:
            raise MqdetError("TestTransform: no images")
        device = _cuda_device(device)
        dev_images = upload(images, device)
        sizes = [tuple(im.shape[:2]) for im in dev_images]
        per_image = [self.target_size(h, w) for h, w in sizes]
        targets = set(per_image)
        if len(targets) != 1 and not mixed_sizes:
            raise MqdetError(f"TestTransform: the images resize to different sizes {sorted(targets)}; batch images of one target "
                             "size together, or pass mixed_sizes=True for one padded batch")
        if mixed_sizes and want_resized:
            raise MqdetError("TestTransform: want_resized needs one target size; it is not available with mixed_sizes=True")
        oh, ow = max(h for h, _ in per_image), max(w for _, w in per_image)
        div = self.div if pad else 0
        Hp, Wp = (-(-oh // div) * div, -(-ow // div) * div) if div > 0 else (oh, ow)
        dst = None
        if out is not None:
            need = len(dev_images) * 3 * Hp * Wp
            if out.dtype != torch.float32 or out.dim() != 1 or out.numel() < need or out.device != device:
                raise MqdetError(f"TestTransform: out must be a flat fp32 buffer on {device} of at least {need} elements for a "
                                 f"[{len(dev_images)}, 3, {Hp}, {Wp}] batch (got {out.dtype} {tuple(out.shape)} on {out.device})")
            dst = out[:need].view(len(dev_images), 3, Hp, Wp)
        tables = {}

        def table(n_in, n_out):
            if (n_in, n_out) not in tables:
                tables[(n_in, n_out)] = ops.resize_coeffs(n_in, n_out, device)
            return tables[(n_in, n_out)]

        if mixed_sizes:
            res = ops.test_transform(dev_images, [table(w, t[1]) for (_, w), t in zip(sizes, per_image)],
                                     [table(h, t[0]) for (h, _), t in zip(sizes, per_image)], per_image, (Hp, Wp), self.mean, self.std,
                                     bgr=self.bgr, times255=self.times255, out=dst)
        else:
            res = ops.test_transform(dev_images, [table(w, ow) for _, w in sizes], [table(h, oh) for h, _ in sizes], (oh, ow),
                                     (Hp, Wp), self.mean, self.std, bgr=self.bgr, times255=self.times255, want_resized=want_resized,
                                     out=dst)
        batch, resized = res if want_resized else (res, None)
        il = ImageList(batch, list(per_image))
        orig = [(w, h) for h, w in sizes]
        return (il, orig, resized) if want_resized else (il, orig)


def model_device(model):
    return next(model.parameters()).device


@torch.no_grad()
def predict(model, images_u8, captions, positive_map, mixed_sizes=False):
    """Decoded uint8 RGB images -> list[BoxList] in original-image coordinates, for MQ-GLIP and MQ-GroundingDINO: the test
    transform on the device, the detector's forward, and BoxList.resize back to each image's size (as the reference's
    evaluators map the results).  ``mixed_sizes=True``: images of different target sizes form one padded batch (see
    ``TestTransform``)."""
    il, orig = TestTransform(model.cfg)(images_u8, model_device(model), mixed_sizes=mixed_sizes)
    res = model(il, captions=captions, positive_map=positive_map)
    return [bl.resize(size) for bl, size in zip(res, orig)]
