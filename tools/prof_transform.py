"""Cost of the test transform on the device (engine/transforms.py, csrc/transform.cu) against the reference's host pipeline.
    python tools/prof_transform.py [--batch 8] [--reps 50] [--host-images 4] [--out FILE]
For two inputs, 640 x 480 -> 800 x 1066 (LVIS / COCO-like, padded to 800 x 1088) and 4000 x 3000 -> 1333 x 1000 (a camera photo at
MIN_SIZE_TEST 1000, padded to 1024 x 1344), with the MQ-GLIP-T format (bgr255):
1. ops.test_transform alone (the two coefficient tables built once): us per image from CUDA events around `reps` launches of
   a batch of `batch` images already on the device.
2. TestTransform.__call__ from host uint8 arrays (pinned staging, one upload, tables, kernel): us per image over `reps` calls
   ending in a synchronise.
3. The bytes that cross to the device per image: the uint8 source here, the padded fp32 batch row on the host path.
4. The host path per image: PIL resize + torchvision to_tensor / normalize + zero padding on the CPU, over `host-images` images
   (a single-process data loader's work), wall clock.
The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout (and to --out)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from mqdet_b200 import ops
from mqdet_b200.config import mq_glip_t_cfg
from mqdet_b200.engine.transforms import TestTransform, upload

INPUTS = {"640x480_to_800x1066": ((480, 640), 800), "4000x3000_to_1333x1000": ((3000, 4000), 1000)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def images(hw, n, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (hw[0], hw[1], 3), dtype=np.uint8) for _ in range(n)]


def host_path(imgs, size, cfg):
    """Resize -> ToTensor -> Normalize (bgr255) -> to_image_list on the CPU, as the reference's data loader runs it."""
    import torchvision.transforms.functional as F
    from PIL import Image
    from mqdet_b200.engine.transforms import get_size
    inp, div = cfg.INPUT, cfg.DATALOADER.SIZE_DIVISIBILITY
    out = []
    for im in imgs:
        h, w = im.shape[:2]
        pil = F.resize(Image.fromarray(im), list(get_size((w, h), size, inp.MAX_SIZE_TEST)))
        t = F.normalize(F.to_tensor(pil)[[2, 1, 0]] * 255, mean=inp.PIXEL_MEAN, std=inp.PIXEL_STD)
        H, W = -(-t.shape[1] // div) * div, -(-t.shape[2] // div) * div
        pad = t.new_zeros((3, H, W))
        pad[:, :t.shape[1], :t.shape[2]] = t
        out.append(pad)
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-images", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    cfg = mq_glip_t_cfg()
    res = {"card": card(), "batch": a.batch, "reps": a.reps, "inputs": {}}
    for name, (hw, size) in INPUTS.items():
        tf = TestTransform(cfg, size)
        host = images(hw, a.batch, 1)
        oh, ow = tf.target_size(*hw)
        Hp, Wp = -(-oh // 32) * 32, -(-ow // 32) * 32
        d_imgs = upload(host, dev)
        xt, yt = ops.resize_coeffs(hw[1], ow, dev), ops.resize_coeffs(hw[0], oh, dev)

        def kernel():
            return ops.test_transform(d_imgs, [xt] * a.batch, [yt] * a.batch, (oh, ow), (Hp, Wp), tf.mean, tf.std, bgr=True, times255=True)
        for _ in range(3):
            kernel()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            kernel()
        e1.record()
        torch.cuda.synchronize()
        k_us = e0.elapsed_time(e1) * 1e3 / (a.reps * a.batch)

        for _ in range(3):
            tf(host, dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            tf(host, dev)
        torch.cuda.synchronize()
        call_us = (time.perf_counter() - t0) * 1e6 / (a.reps * a.batch)

        n_host = min(a.host_images, a.batch)
        host_path(host[:1], size, cfg)
        t0 = time.perf_counter()
        ref = host_path(host[:n_host], size, cfg)
        host_us = (time.perf_counter() - t0) * 1e6 / n_host
        same = bool(torch.equal(tf(host[:n_host], dev)[0].tensors.cpu(), ref))

        src_bytes = hw[0] * hw[1] * 3
        moved = Hp * Wp * 3 * 4
        res["inputs"][name] = {"source_hw": hw, "resized_hw": (oh, ow), "padded_hw": (Hp, Wp), "kernel_us_per_image": round(k_us, 2),
                               "transform_call_us_per_image": round(call_us, 1), "h2d_bytes_per_image": src_bytes,
                               "h2d_bytes_per_image_fp32_path": moved, "h2d_ratio": round(moved / src_bytes, 2),
                               "kernel_gb_per_s": round((src_bytes + moved) / (k_us * 1e-6) / 1e9, 1),
                               "host_pil_torchvision_us_per_image": round(host_us, 1), "bit_identical_to_host_path": same}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
