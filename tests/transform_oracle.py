"""numpy / torch restatement of the reference's test transform (data/transforms: Resize -> ToTensor -> Normalize, then
to_image_list), the thing the GPU tests compare the kernel against.

* ``get_size``: Resize.get_size with restrict=False.
* ``resize``: PIL ``Image.resize((ow, oh), BILINEAR)`` of an RGB image, restated from the published description of Pillow's
  separable resampler: per output index, in float64, scale = in / out, filterscale = max(scale, 1), support = filterscale,
  center = (i + 0.5) * scale, first tap = int(center - support + 0.5) (truncation, clamped to 0), end = int(center + support + 0.5)
  (clamped to in), weight = triangle((x + first - center + 0.5) * (1 / filterscale)) normalised by the sequential sum; weights in
  22-bit fixed point rounded half away from zero; a pixel is (1 << 21 + sum of value * weight) >> 22 clipped to [0, 255].  The
  horizontal pass runs first (uint8 intermediate), then the vertical pass; a pass whose length does not change is skipped.
* ``normalize``: ToTensor (uint8 -> fp32 / 255) and Normalize ('bgr' reorders the channels, '255' multiplies by 255, then
  (x - mean) / std with mean and std in fp32), one rounded fp32 operation at a time, in torch on the CPU.
"""
import math

import numpy as np
import torch

PRECISION_BITS = 22


def get_size(image_size, size, max_size):
    """(w, h) -> (oh, ow) of the shorter side scaled to ``size``, the longer side capped by ``max_size`` (None: no cap)."""
    w, h = image_size
    short, long_ = float(min(w, h)), float(max(w, h))
    if max_size is not None and long_ / short * size > max_size:
        size = int(round(max_size * short / long_))
    if min(w, h) == size:
        return h, w
    if w < h:
        return int(size * h / w), size
    return size, int(size * w / h)


def ksize(n_in, n_out):
    """Taps per output index in the coefficient table (Pillow's ksize = 2 * ceil(support) + 1)."""
    return int(math.ceil(max(n_in / n_out, 1.0))) * 2 + 1


def coeffs(n_in, n_out):
    """-> (first tap int64 [n_out], taps int64 [n_out], fixed-point weights int64 [n_out, ksize] (zero past taps))."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support, ss = fs, 1.0 / fs
    K = ksize(n_in, n_out)
    center = (np.arange(n_out, dtype=np.float64) + 0.5) * scale
    lo = np.maximum(np.trunc(center - support + 0.5).astype(np.int64), 0)
    hi = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), n_in)
    n = hi - lo
    w = np.zeros((n_out, K), np.float64)
    total = np.zeros(n_out, np.float64)
    for t in range(K):
        d = np.abs(((t + lo).astype(np.float64) - center + 0.5) * ss)
        wt = np.where(d < 1.0, 1.0 - d, 0.0)
        wt = np.where(t < n, wt, 0.0)
        w[:, t] = wt
        total = total + wt                  # sequential, as the C loop (not math.fsum / Python 3.12's compensated sum)
    w = np.where(total[:, None] != 0.0, w / np.where(total == 0.0, 1.0, total)[:, None], w)
    f = w * float(1 << PRECISION_BITS)
    k = np.where(w < 0, np.trunc(f - 0.5), np.trunc(f + 0.5)).astype(np.int64)
    return lo, n, k


def resample_axis(a, n_out, axis):
    """One pass of the integer resampler along ``axis`` of a uint8 array."""
    n_in = a.shape[axis]
    if n_in == n_out:
        return a
    lo, n, k = coeffs(n_in, n_out)
    src = np.moveaxis(a, axis, 0).astype(np.int64)
    acc = np.full((n_out,) + src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    shape = (n_out,) + (1,) * (src.ndim - 1)
    for t in range(k.shape[1]):
        idx = np.minimum(lo + t, n_in - 1)
        acc += src[idx] * k[:, t].reshape(shape)      # weight 0 past the taps
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img, oh, ow):
    """uint8 [h, w, C] -> uint8 [oh, ow, C]: horizontal pass, then vertical pass."""
    return resample_axis(resample_axis(np.asarray(img), ow, 1), oh, 0)


def normalize(u8, mean, std, fmt):
    """uint8 HWC -> fp32 [3, H, W] as ToTensor + Normalize(mean, std, format) compute it on the CPU."""
    x = torch.from_numpy(np.array(u8, dtype=np.uint8)).permute(2, 0, 1).float().div(255)
    fmt = fmt.lower()
    if "bgr" in fmt:
        x = x[[2, 1, 0]]
    if "255" in fmt:
        x = x * 255
    m = torch.tensor(mean, dtype=torch.float32).view(-1, 1, 1)
    s = torch.tensor(std, dtype=torch.float32).view(-1, 1, 1)
    return (x - m) / s


def pad_batch(chw_list, size_divisible):
    """to_image_list: zero-padded [B, 3, Hp, Wp], Hp / Wp rounded up to a multiple of size_divisible."""
    H = max(x.shape[1] for x in chw_list)
    W = max(x.shape[2] for x in chw_list)
    if size_divisible > 0:
        H, W = -(-H // size_divisible) * size_divisible, -(-W // size_divisible) * size_divisible
    out = torch.zeros((len(chw_list), 3, H, W), dtype=torch.float32)
    for o, x in zip(out, chw_list):
        o[:, :x.shape[1], :x.shape[2]] = x
    return out


def transform(images, size, max_size, mean, std, fmt, size_divisible):
    """uint8 HWC images -> (padded fp32 batch, resized uint8 images): the whole test transform."""
    resized = []
    for im in images:
        h, w = im.shape[:2]
        oh, ow = get_size((w, h), size, max_size)
        resized.append(resize(im, oh, ow))
    return pad_batch([normalize(r, mean, std, fmt) for r in resized], size_divisible), resized
