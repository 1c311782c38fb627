"""CPU: what every launching wrapper of ``mqdet_b200.ops`` passes across the C ABI, pinned against tests/golden/ops_calls.json.

The library is replaced by a recorder (``_lib._lib``), the stream by a null one and the CUDA-tensor check by a no-op, so the
wrappers run on small CPU tensors.  For each wrapper call the pin holds the symbol sequence, the scalar arguments, every pointer as
the order of its first appearance in that call (None = null), ``GemmArgs`` fields and ctypes arrays expanded, the ``launch_count``
delta, and the error message of each launching call when that call fails.  The kernels themselves are checked by the ``-m gpu`` tests.

    python tests/test_ops_calls_cpu.py --write     # regenerate the golden file (only when the ABI traffic is meant to change)
"""
import ctypes
import json
import os
import re
import sys
from types import SimpleNamespace

import pytest
import torch

from util import ROOT

from mqdet_b200 import _lib, ops  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "ops_calls.json")

# entry points that return a size or a capability instead of launching work
_QUERY = re.compile(r"_workspace_|_floats$|_chunks$|_ksize$|_supported$")
_QUERY_RESULT = {"mqdet_dyconv_combine_chunks": 4, "mqdet_resize_coeffs_ksize": 3}
WORKSPACE = 4096
N_WRITTEN = 3   # what the recorder writes to the byref int64 out-parameter of mqdet_sqnorm_partials

# wrapper paths the recorder cannot reach on the CPU (covered by the -m gpu suite)
NOT_DRIVEN = {
    "atss_postprocess with a device size table (mqdet_atss_candidates_sizes_dev)":
        "the entry point is chosen by img_w.is_cuda, which a CPU tensor never is",
}


class Recorder:
    """Stands in for the CDLL: records each call and returns 0 (or a fixed size for the queries)."""

    def __init__(self, shifted_supported=1, fail_at=None):
        self.calls, self.launches = [], 0
        self.shifted_supported, self.fail_at = shifted_supported, fail_at

    def __getattr__(self, name):
        if not name.startswith("mqdet_"):
            raise AttributeError(name)

        def fn(*args):
            if name == "mqdet_last_error":
                return b"recorded failure"
            self.calls.append(_encode(name, args))
            if name == "mqdet_softmax_rows_shifted_supported":
                return self.shifted_supported
            if _QUERY.search(name):
                return _QUERY_RESULT.get(name, WORKSPACE)
            for a in args:
                if type(a).__name__ == "CArgObject" and isinstance(a._obj, ctypes.c_int64):
                    a._obj.value = N_WRITTEN
            self.launches += 1
            return -1 if self.launches - 1 == self.fail_at else 0
        return fn


I32, F32, PTR = ctypes.c_int32, ctypes.c_float, ctypes.c_void_p
# host tables passed as plain pointers: symbol -> [(argument index, element type, element count from the arguments)]
_HOST_ARRAYS = {
    "mqdet_dcn_conv": [(3, I32, lambda a: 2 * a[4])] + [(i, t, lambda a: a[7]) for i, t in ((8, I32), (9, PTR), (10, PTR), (11, PTR))],
    "mqdet_dcn_cols": [(3, I32, lambda a: 2 * a[4])],
    "mqdet_conv3x3_small": [(3, I32, lambda a: 2 * a[4])],
    "mqdet_dyconv_combine": [(9, I32, lambda a: 2 * a[10])],
    "mqdet_dyrelu_apply": [(2, I32, lambda a: 2 * a[3])],
    "mqdet_roi_align_levels": [(1, I32, lambda a: 2 * a[2]), (3, F32, lambda a: a[2])],
    "mqdet_roi_align_levels_counted": [(1, I32, lambda a: 2 * a[2]), (3, F32, lambda a: a[2])],
    "mqdet_avgpool2_levels": [(1, I32, lambda a: 2 * a[2])],
    "mqdet_ms_deform_attn": [(6, I32, lambda a: 2 * a[7])],
    "mqdet_atss_workspace_bytes": [(0, I32, lambda a: 2 * a[1])],
    "mqdet_atss_candidates": [(10, I32, lambda a: 2 * a[11]), (12, F32, lambda a: a[11]), (13, F32, lambda a: 4 * a[11]),
                              (14, F32, lambda a: a[11]), (19, F32, lambda a: 2 * a[20])],
    "mqdet_atss_assign": [(5, I32, lambda a: 2 * a[6]), (7, F32, lambda a: a[6]), (8, F32, lambda a: 4 * a[6])],
    "mqdet_atss_loss": [(10, I32, lambda a: 2 * a[11]), (12, F32, lambda a: a[11]), (13, F32, lambda a: 4 * a[11]),
                        (14, F32, lambda a: a[11])],
    "mqdet_anchors": [(5, F32, lambda a: 4)],
}


def _encode(name, args):
    """One call as JSON-able data, taken when the call is made."""
    ptrs = {}

    def ptr(v):
        if not v:
            return None
        return {"ptr": ptrs.setdefault(v, len(ptrs))}

    def enc(a):
        if a is None:
            return None
        if isinstance(a, ctypes.c_void_p):
            return ptr(a.value)
        if isinstance(a, (int, float)) and not isinstance(a, bool):
            return a
        if isinstance(a, ctypes.Array):
            return [ptr(v) if a._type_ is ctypes.c_void_p else v for v in a]
        if type(a).__name__ == "CArgObject":
            obj = a._obj
            if isinstance(obj, ctypes.Structure):
                return {f: (ptr(getattr(obj, f)) if t is ctypes.c_void_p else getattr(obj, f)) for f, t in obj._fields_}
            return {"byref": obj.value}
        raise TypeError(f"{name}: unrecorded argument type {type(a).__name__}")

    out = [enc(a) for a in args]
    for i, t, n in _HOST_ARRAYS.get(name, ()):
        out[i] = {"host": enc((t * n(args)).from_address(args[i].value))}
    return [name, out]


# ---------------------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------------------
def f32(*s):
    return torch.rand(s, dtype=torch.float32)


def f16(*s):
    return torch.rand(s, dtype=torch.float32).half()


def i32(*s):
    return torch.zeros(s, dtype=torch.int32)


def i64(*s):
    return torch.zeros(s, dtype=torch.int64)


def lv():
    return ops.Levels([(4, 4), (2, 2)], "cpu")   # N = 20, N1 = 4


def lvis_gt(coco):
    t = {"gt_pair": i32(6), "gt_box": f32(6, 4), "gt_area": f32(6), "gt_ignore": i32(6), "gt_id": i64(6), "num_gt": i32(4),
         "iou_thrs": f32(10), "rec_thrs": f32(101), "area_rng": f32(4, 2)}
    if coco:
        t.update(gt_crowd=i32(6), max_dets=i32(3))
    else:
        t.update(pos_pairs=i32(4), neg_pairs=i32(2), nel_pairs=i32(2))
    return SimpleNamespace(cat_ids=[1, 2], dev=t, det_area_filter=coco)


def transform_case(B, per_image):
    images = [torch.zeros((6 + i % 3, 8, 3), dtype=torch.uint8) for i in range(B)]
    sizes = [(4, 4) if i % 2 == 0 else (3, 4) for i in range(B)] if per_image else [(4, 4)] * B
    xt = [torch.zeros((ow, 5), dtype=torch.int32) for _, ow in sizes]
    yt = [torch.zeros((oh, 5), dtype=torch.int32) for oh, _ in sizes]
    return ops.test_transform(images, xt, yt, sizes if per_image else (4, 4), (8, 8), (0.4, 0.5, 0.6), (0.2, 0.25, 0.3),
                              bgr=True, times255=per_image, want_resized=not per_image)


CASES = {
    "gemm": lambda: ops.gemm(f16(2, 3, 16), f16(8, 16), bias=f32(8), act=_lib.ACT_GELU, clamp=5.0, gate=f32(8),
                             gate_mode=_lib.VEC_PER_COL, gate_tanh=True, residual=f16(2, 3, 8), alpha=0.5),
    "gemm_batched_f32": lambda: ops.gemm(f16(2, 4, 3, 16), f16(4, 8, 16), out_dtype=torch.float32, bias=f32(4, 8),
                                         scale_after_bias=True, residual=f32(2, 4, 3, 8), impl=_lib.IMPL_SIMT),
    "layernorm": lambda: ops.layernorm(f16(2, 3, 8), f32(8), f32(8), 1e-6, out32=True, zero_row_period=3),
    "swin_mlp": lambda: ops.swin_mlp(f32(4, 96), f32(96), f32(96), 1e-5, f16(384, 96), f32(384), f16(96, 384), f32(96)),
    "add_layernorm": lambda: ops.add_layernorm(f32(3, 8), f32(3, 8), f32(8), f32(8), 1e-5, clamp=4.0),
    "softmax_rows": lambda: ops.softmax_rows(f32(2, 3, 16), n=12, scale=0.5, colmask=f32(2, 16), rows_per_batch=3,
                                             mask_value=-1.0, keep_add=0.25),
    "sum_splits_cast": lambda: ops.sum_splits_cast(f32(1, 2, 3, 4, 8), torch.zeros((1, 2, 4, 16), dtype=torch.float16)[..., :8]),
    "softmax_rows_shifted": lambda: ops.softmax_rows_shifted(f32(2, 3, 16), f32(2), -3.0, 3.0, n=12, colmask=f32(2, 16),
                                                             rows_per_batch=3, mask_value=-2.0, keep_add=0.5, rows_per_shift=3),
    "softmax_rows_shifted_unfused": lambda: ops.softmax_rows_shifted(f32(2, 3, 16), f32(2), -3.0, 3.0, n=12, rows_per_shift=3),
    "global_max": lambda: ops.global_max(f32(4, 8), segments=2),
    "shift_clamp_": lambda: ops.shift_clamp_(f32(2, 8), f32(2), -1.0, 1.0, rows_per_shift=1),
    "row_max": lambda: ops.row_max(f32(3, 8)),
    "topk_desc": lambda: ops.topk_desc(f32(2, 10), 3),
    "gather_rows": lambda: ops.gather_rows(f32(2, 5, 4), i64(2, 3), sigmoid=True),
    "l2_normalize": lambda: ops.l2_normalize(f32(3, 8), f32(8), f32(1), eps=1e-6),
    "biattn_image": lambda: ops.biattn_image(f16(1, 16, 256), f16(1, 2, 8, 256), f32(1, 2, 8, 4), f16(1, 2, 256, 8), f32(256),
                                             f32(256), f16(1, 16, 256), f32(1, 8), 50.0, 2),
    "biattn_text_vn": lambda: ops.biattn_text_vn(f16(1, 2, 8, 32), f16(1, 2, 16, 32), f16(1, 16, 256), f32(2, 8), 50.0,
                                                 torch.zeros((1, 8, 2, 256), dtype=torch.float16).transpose(1, 2), f32(1, 2, 8, 4)),
    "cast_f16": lambda: ops.cast_f16(f32(3, 4)),
    "cast_f16_noop": lambda: ops.cast_f16(f16(3, 4)),
    "cast_f32": lambda: ops.cast_f32(f16(3, 4)),
    "contrastive_embed": lambda: ops.contrastive_embed(f16(1, 4, 16), f16(1, 3, 16), torch.ones((1, 3), dtype=torch.bool), 8),
    "dense_cross_attn": lambda: ops.dense_cross_attn(f16(1, 4, 64), f16(1, 6, 128), 2, 32),
    "gcp_build_index": lambda: ops.gcp_build_index(f32(1, 3, 4), 2),
    "gcp_sparse_attn": lambda: ops.gcp_sparse_attn(f16(1, 4, 64), f16(1, 4, 128), i32(1, 4, 2), 2, 32),
    "gcp_gate_residual_ln": lambda: ops.gcp_gate_residual_ln(f16(4, 16), f32(16), f32(4, 8), f32(4, 8), f32(8), f32(8), 1e-6,
                                                             want_gate=True),
    "argsort_desc": lambda: ops.argsort_desc(f32(5)),
    "argsort_desc_empty": lambda: ops.argsort_desc(f32(0)),
    "ml_nms_device": lambda: ops.ml_nms_device(f32(4, 4), f32(4), f32(4), 0.5, max_det=3),
    "ml_nms": lambda: ops.ml_nms(f32(4, 4), f32(4), f32(4), 0.6),
    "hflip_pad": lambda: ops.hflip_pad(f32(1, 3, 4, 5), (8, 8)),
    "bbox_aug_collect": lambda: ops.bbox_aug_collect(ops.MergedBoxes(2, 16, "cpu"), f32(2, 4, 4), f32(2, 4), f32(2, 4), i32(2),
                                                     (100, 80), (200, 170), flip=True, keep_range=(0, 64)),
    "bbox_aug_collect_packed": lambda: ops.bbox_aug_collect_packed(ops.MergedBoxes(2, 16, "cpu"), f32(2, 5, 6), (100, 80),
                                                                   (150, 120)),
    "nms_by_class": lambda: ops.nms_by_class(f32(2, 16, 4), f32(2, 16), i32(2, 16), i32(2), i32(3), 0.6, mode="vote", top_n=5,
                                             max_out=4, overflow=i32(2)),
    "nms_by_class_passes": lambda: ops.nms_by_class(f32(1, 4097, 4), f32(1, 4097), i32(1, 4097), i32(1), i32(3), 0.5, max_out=4),
    "resize_coeffs": lambda: ops.resize_coeffs(10, 6, "cpu"),
    "test_transform": lambda: transform_case(2, False),
    "test_transform_sizes": lambda: transform_case(3, True),
    "test_transform_65": lambda: transform_case(65, False),
    "mask_prompt_tokens": lambda: ops.mask_prompt_tokens(i64(2, 5), i32(2, 5), torch.zeros((2, 3), dtype=torch.uint8), 103),
    "mask_prompt_tokens_no_flags": lambda: ops.mask_prompt_tokens(i64(2, 5), i32(2, 5), torch.zeros((2, 0), dtype=torch.uint8),
                                                                  103, out=i64(2, 5)),
    "query_bank_from_dict": lambda: ops.QueryBank.from_dict({1: f32(2, 1, 8)}, 3, 4, 8, "cpu"),
    "query_candidates": lambda: ops.query_candidates(f32(2, 5, 6), [(100, 80), (90, 70)], 0.3, 1.5, i32(1)),
    "roi_align_levels_counted": lambda: ops.roi_align_levels_counted(f16(1, 20, 8), lv(), [0.25, 0.125], f32(6, 5), i32(1),
                                                                     pooled=5, sampling_ratio=2),
    "query_bank_update": lambda: ops.query_bank_update(ops.QueryBank(3, 4, 8, "cpu"), f32(6, 8), i32(6), i32(1), 4, 0.9),
    "dcn_cols": lambda: ops.dcn_cols(f16(1, 20, 256), f32(1, 20, 32), lv(), 1),
    "dcn_cols_tail": lambda: ops.dcn_cols(f16(1, 20, 256), None, lv(), 0),
    "dcn_conv": lambda: ops.dcn_conv(f16(1, 20, 256), f32(1, 20, 32), lv(), [0, 1], [f16(256, 2304), f16(256, 2304)],
                                     [f32(256), None]),
    "conv3x3_small": lambda: ops.conv3x3_small(f16(1, 20, 256), f16(27, 2304), f32(27), lv()),
    "chan_stats": lambda: ops.chan_stats(f16(1, 20, 8), i32(3), 1, 20, f32(20)),
    "gn_attn": lambda: ops.gn_attn(f32(64), i32(3), 1, 8, 2, True, f32(8), f32(8), 1e-5, f32(8), f32(1)),
    "dyconv_combine": lambda: ops.dyconv_combine(f16(20, 8), f16(4, 8), f16(4, 8), f32(2), f32(2), f32(2), f32(2), f32(2), f32(2),
                                                 lv(), 1),
    "dyrelu": lambda: ops.dyrelu(f16(1, 20, 8), lv(), f32(2, 8), f32(2), f32(32, 2), f32(32)),
    "dyrelu_sums": lambda: ops.dyrelu(f16(1, 20, 8), lv(), f32(2, 8), f32(2), f32(32, 2), f32(32), mid_sums=f32(1, 2, 4, 8)),
    "atss_postprocess": lambda: ops.atss_postprocess(f32(1, 20, 6), f32(1, 20, 5), i32(3, 2), lv(), [8, 16], [64, 128], [1.0, 0.5],
                                                     100, 80, pre_nms_top_n=10, want_keys=True, class_labels=i32(3)),
    "atss_postprocess_per_image": lambda: ops.atss_postprocess(f32(2, 20, 6), f32(2, 20, 5), i32(2, 3, 2), lv(), [8, 16], [64, 128],
                                                               [1.0, 1.0], [100, 90], [80, 70], pre_nms_thresh=0.1, nms_thresh=0.5,
                                                               max_det=50, max_out=16),
    "atss_targets": lambda: ops.atss_targets(f32(1, 3, 4), i32(1, 3), i32(1), lv(), [8, 16], [64, 128], topk=5),
    "atss_loss": lambda: ops.atss_loss(f32(1, 20, 6), f32(1, 20, 5), f32(1, 3, 4), i32(1, 3), i32(1), f32(1, 3, 6), lv(), [8, 16],
                                       [64, 128], [1.0, 0.5], f32(1, 6), world=2),
    "linear_sum_assignment": lambda: ops.linear_sum_assignment(f32(2, 4, 3), i32(2)),
    "gdino_match": lambda: ops.gdino_match(f32(2, 1, 4, 6), f32(2, 1, 4, 4), f32(1, 3, 4), i32(1), f32(1, 3, 6), cost_bbox=4.0),
    "gdino_set_loss": lambda: ops.gdino_set_loss(f32(2, 1, 4, 6), f32(2, 1, 4, 4), f32(1, 3, 4), i32(1), f32(1, 3, 6), f32(1, 6),
                                                 world=2, giou_coef=3.0),
    "anchors": lambda: ops.anchors(2, 3, 8, 64, 100, 80, "cpu"),
    "patchify4": lambda: ops.patchify4(f32(1, 3, 8, 10)),
    "swin_window_attn": lambda: ops.swin_window_attn(f16(49, 96), f32(96), f32(169), 1, 7, 7, 1, 7, 3, 0.125),
    "patch_merge_ln": lambda: ops.patch_merge_ln(f32(16, 8), 1, 4, 4, f32(32), f32(32), 1e-5),
    "upsample_add": lambda: ops.upsample_add(f16(1, 16, 8), f16(1, 4, 8), 1, 4, 4, 2, 2),
    "im2col3x3": lambda: ops.im2col3x3(f16(1, 16, 8), 1, 4, 4, stride=2, relu_in=True),
    "avgpool2_levels": lambda: ops.avgpool2_levels(f16(1, 20, 8), lv()),
    "roi_align_levels": lambda: ops.roi_align_levels(f16(1, 20, 8), lv(), [0.25, 0.125], f32(3, 5), mean_only=False),
    "ms_deform_attn": lambda: ops.ms_deform_attn(f16(1, 20, 64), f32(3, 24), 16, f32(1, 3, 2, 2), lv(), 2, 2,
                                                 out_dtype=torch.float32),
    "add_cast": lambda: ops.add_cast(f32(3, 8), f32(3, 8), f32(3), out32=True),
    "groupnorm_rows": lambda: ops.groupnorm_rows(f32(1, 4, 8), 2, f32(8), f32(8), 1e-6, out16=False, out32=True),
    "box_refine_sine": lambda: ops.box_refine_sine(f32(1, 3, 4), f32(1, 2, 2), delta=f32(1, 3, 8), ref_is_logit=True),
    "box_refine_sine_plain": lambda: ops.box_refine_sine(f32(1, 3, 4), f32(1, 2, 2), want_sine=False),
    "gdino_detections": lambda: ops.gdino_detections(f32(2, 4, 6), f32(2, 4, 4), i32(2, 3, 2), f32(2, 2), 0.3, 3,
                                                     class_labels=i32(2, 3)),
    "transpose_cast": lambda: ops.transpose_cast(f32(5, 8), scale=0.5),
    "transpose_cast_batched": lambda: ops.transpose_cast_batched(f16(1, 2, 5, 8)),
    "softmax_bwd_rows": lambda: ops.softmax_bwd_rows(f16(3, 8), f32(3, 8), scale=0.25),
    "layernorm_bwd": lambda: ops.layernorm_bwd(f32(3, 8), f32(3, 8), f32(8), 1e-5, dx=f32(3, 8), x2=f32(3, 8)),
    "layernorm_bwd_plain": lambda: ops.layernorm_bwd(f32(3, 8), f32(3, 8), f32(8), 1e-6, want_param_grads=False),
    "gelu_bwd": lambda: ops.gelu_bwd(f16(3, 8), f32(3, 8)),
    "gcp_gate_bwd": lambda: ops.gcp_gate_bwd(f32(4, 8), f32(4, 8), f32(4), f32(16)),
    "colsum_weighted": lambda: ops.colsum_weighted(f16(4, 8), f32(4)),
    "gcp_sparse_attn_bwd": lambda: ops.gcp_sparse_attn_bwd(f16(1, 4, 64), f16(1, 4, 128), i32(1, 4, 2), f16(1, 4, 64), 2, 32),
    "dot_sum": lambda: ops.dot_sum(f32(8), f32(8), f32(1), mul=0.5),
    "dot_sum_sq": lambda: ops.dot_sum(f32(8)),
    "scale_cast": lambda: ops.scale_cast(f32(3, 8), f32(1), tanh_scalar=True, alpha=2.0, out32=True),
    "token_focal_loss": lambda: ops.token_focal_loss(f32(1, 4, 6), f32(1, 4, 6), f32(1, 6), grad_scale=0.5),
    "clip_coef": lambda: ops.clip_coef([f32(8), f32(4, 3), f32(2)], 1.0),
    "adamw_step_": lambda: ops.adamw_step_(f32(8), f32(8), f32(8), f32(8), 3, 1e-3, weight_decay=0.05, grad_scale=f32(2)),
    "lvis_collect": lambda: ops.lvis_collect(ops.LvisPool(64, "cpu"), 4, 5, f32(2, 2, 4, 6), i32(2), f32(2, 2), i32(3),
                                             label_map=i32(5), need_img=True, bad=i32(1), wh_plus_one=True, bad_img=i32(1)),
    "lvis_cut": lambda: ops.lvis_cut(ops.LvisPool(64, "cpu"), 10, ops.LvisPool(64, "cpu"), n_groups=6, k=5, group=ops.CUT_BY_PAIR,
                                     n_cat=2),
    "lvis_cut_by_image": lambda: ops.lvis_cut(ops.LvisPool(64, "cpu"), 10, ops.LvisPool(64, "cpu"), n_groups=3, k=300,
                                              by_image=True),
    "lvis_evaluate": lambda: ops.lvis_evaluate(ops.LvisPool(64, "cpu"), 10, lvis_gt(False)),
    "lvis_evaluate_coco": lambda: ops.lvis_evaluate(ops.LvisPool(64, "cpu"), 10, lvis_gt(True), want_match=True),
}


def record(case):
    """Runs one case against the recorder -> {"calls", "launches", "errors"}."""
    saved = (_lib._lib, ops._stream, ops._need_cuda, ops.launch_count)
    ops._stream = lambda: ctypes.c_void_p(0)
    ops._need_cuda = lambda *ts: None
    supported = 0 if case.endswith("_unfused") else 1
    try:
        torch.manual_seed(0)
        rec = _lib._lib = Recorder(supported)
        ops.launch_count = 0
        CASES[case]()
        out = {"calls": rec.calls, "launches": ops.launch_count, "errors": []}
        for i in range(rec.launches):   # each launching call failing in turn: the message names the failed step
            _lib._lib = Recorder(supported, fail_at=i)
            with pytest.raises(_lib.MqdetError) as e:
                CASES[case]()
            out["errors"].append(str(e.value))
        return out
    finally:
        _lib._lib, ops._stream, ops._need_cuda, ops.launch_count = saved


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_case(golden):
    assert sorted(golden) == sorted(CASES)


@pytest.mark.parametrize("case", sorted(CASES))
def test_abi_calls_match_golden(case, golden):
    assert json.loads(json.dumps(record(case))) == golden[case]


if __name__ == "__main__" and sys.argv[1:] == ["--write"]:
    with open(GOLDEN, "w") as f:
        json.dump({c: record(c) for c in sorted(CASES)}, f, indent=0, sort_keys=True)
        f.write("\n")
