"""VL deep-fusion head (VLDyHead) on sm_90a kernels.

Drop-in for the hot-path slice of maskrcnn_benchmark/modeling/rpn/vldyhead.py: ``Conv3x3Norm`` (:111-152), ``DyConv``
(:155-247), ``BertEncoderLayer`` (:250-301), ``VLFuse`` (MHA-B, :364-574), ``VLDyHead`` (:594-900) with the
reference's parameter names (``dyhead_tower.{3i,3i+1,3i+2}``, ``DyConv.{0,1,2}.{conv,bn}``, ``AttnConv.1``,
``relu.fc.{0,2}``, ``offset``, ``b_attn...``, ``dot_product_projection_text``, ``bias_lang``, ``bias0``, ``log_scale``,
``scales.N.scale``, ``bbox_pred``, ``centerness``, ``cls_logits``); ``VLDyHeadModule`` also computes the ATSS training
losses and their gradients at the head outputs (the tower itself has no backward here).

Layout: the visual pyramid is ONE fp16 tensor [B, N, 256] (all levels concatenated, NHWC rows) through the whole
tower; NCHW appears only at the reference-facing ``forward`` boundary.
"""
import math

import torch
from torch import nn

from ... import ops
from ..._lib import MqdetError
from ...structures.bounding_box import boxlists_from_packed
from ...utils.fuse_helper import BiAttentionBlockForCheckpoint, _flatten_levels, _split_levels
from ...utils.weights import f32, w16
from ..language_backbone.modeling_bert_new import BertLayer

_derived = {}


def _conv_w16(conv_weight):
    """[O, C, 3, 3] conv weight -> fp16 [O, 9*C] with k = tap*C + c (matches the column matrix of dcn_cols)."""
    ent = _derived.get(id(conv_weight))
    ver = (conv_weight.data_ptr(), conv_weight._version)
    if ent is not None and ent[0] == ver and ent[2]() is conv_weight:
        return ent[1]
    import weakref
    O = conv_weight.shape[0]
    w = conv_weight.detach().float().permute(0, 2, 3, 1).reshape(O, -1).contiguous()
    h = ops.cast_f16(w)
    _derived[id(conv_weight)] = (ver, h, weakref.ref(conv_weight, lambda _r, k=id(conv_weight): _derived.pop(k, None)))
    return h


class h_sigmoid(nn.Module):
    def __init__(self, inplace=True, h_max=1):
        super().__init__()
        self.h_max = h_max


class ModulatedDeformConv(nn.Module):
    """Parameter container for maskrcnn_benchmark/layers/deform_conv.py:340-382 (weight [O, C, 3, 3], bias [O])."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, groups=1):
        super().__init__()
        self.stride, self.padding = stride, padding
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, kernel_size, kernel_size))
        self.bias = nn.Parameter(torch.zeros(out_channels))
        n = in_channels * kernel_size * kernel_size
        self.weight.data.uniform_(-1.0 / math.sqrt(n), 1.0 / math.sqrt(n))


class Conv3x3Norm(nn.Module):
    def __init__(self, in_channels, out_channels, stride, groups=1, deformable=False, bn_type=None):
        super().__init__()
        if not deformable or not (isinstance(bn_type, (list, tuple)) and bn_type[0] == "gn"):
            raise NotImplementedError("MQ-GLIP configs use deformable convs with GroupNorm (USE_DFCONV, USE_GN)")
        self.conv = ModulatedDeformConv(in_channels, out_channels, 3, stride=stride, padding=1, groups=groups)
        self.bn = nn.GroupNorm(num_groups=bn_type[1], num_channels=out_channels)


class DYReLU(nn.Module):
    """Parameter container for maskrcnn_benchmark/layers/dyrelu.py:38-78 (K2, use_bias, reduction 4)."""

    def __init__(self, inp, oup, reduction=4):
        super().__init__()
        self.oup = oup
        squeeze = inp // reduction
        self.fc = nn.Sequential(nn.Linear(inp, squeeze), nn.ReLU(inplace=True), nn.Linear(squeeze, oup * 4), h_sigmoid())


class DyConv(nn.Module):
    def __init__(self, in_channels=256, out_channels=256, conv_func=None, use_dyfuse=True, use_dyrelu=False,
                 use_deform=False):
        super().__init__()
        if not (use_dyfuse and use_dyrelu and use_deform):
            raise NotImplementedError("MQ-GLIP configs enable USE_DYFUSE, USE_DYRELU and USE_DFCONV")
        self.DyConv = nn.ModuleList([conv_func(in_channels, out_channels, 1), conv_func(in_channels, out_channels, 1),
                                     conv_func(in_channels, out_channels, 2)])
        self.AttnConv = nn.Sequential(nn.AdaptiveAvgPool2d(1), nn.Conv2d(in_channels, 1, kernel_size=1),
                                      nn.ReLU(inplace=True))
        self.h_sigmoid = h_sigmoid()
        self.relu = DYReLU(in_channels, out_channels)
        self.offset = nn.Conv2d(in_channels, 27, kernel_size=3, stride=1, padding=1)
        self.implicit_dcn = True
        self.init_weights()

    def init_weights(self):
        for m in self.DyConv.modules():
            if isinstance(m, ModulatedDeformConv):
                nn.init.normal_(m.weight.data, 0, 0.01)
                m.bias.data.zero_()
        for m in self.AttnConv.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight.data, 0, 0.01)
                m.bias.data.zero_()

    @torch.no_grad()
    def forward_flat(self, x16, levels):
        """x16 [B, N, 256] fp16 -> next pyramid [B, N, 256] fp16 (vldyhead.py:205-247)."""
        B, N, C = x16.shape
        L = levels.n
        # offset/mask conv (plain 3x3, 27 channels) for every level in one implicit-GEMM launch; pixel-major [B*N, 32] fp32
        om3 = ops.conv3x3_small(x16, _conv_w16(self.offset.weight), f32(self.offset.bias), levels).view(B, N, 32)
        aw = f32(self.AttnConv[1].weight).view(-1)
        ab = f32(self.AttnConv[1].bias)

        # the three DCNv2 convolutions: one implicit-GEMM launch (no column matrix); implicit_dcn = False keeps the
        # sampling kernel + GEMM pair (dcn_cols -> gemm), the path the comparison tests check the implicit one against
        ks = [1, 2, 0] if L > 1 else [1]
        if self.implicit_dcn:
            ys = dict(zip(ks, ops.dcn_conv(x16, om3, levels, ks, [_conv_w16(self.DyConv[k].conv.weight) for k in ks],
                                           [f32(self.DyConv[k].conv.bias) for k in ks])))

        def branch(k, rows, seg, weights=None):
            conv, gn = self.DyConv[k].conv, self.DyConv[k].bn
            if self.implicit_dcn:
                y = ys[k]
            else:
                c = ops.dcn_cols(x16, om3, levels, k)
                y = ops.gemm(c, _conv_w16(conv.weight), bias=f32(conv.bias))
            part = ops.chan_stats(y, seg, B, rows, weights)
            aff, at = ops.gn_attn(part, seg, B, C, gn.num_groups, weights is not None, f32(gn.weight), f32(gn.bias),
                                  gn.eps, aw, ab)
            return y, aff, at

        y1, aff1, at1 = branch(1, N, levels.seg_all)
        if L > 1:
            y2, aff2, at2 = branch(2, levels.N1, levels.seg_tail)
            y0, aff0, at0 = branch(0, levels.N1, levels.seg_tail, levels.up_w)
        else:
            y2 = y0 = aff2 = aff0 = at2 = at0 = None
        mid, mid_sums = ops.dyconv_combine(y1, y2, y0, aff1, aff2, aff0, at1, at2, at0, levels, B)
        fc = self.relu.fc
        return ops.dyrelu(mid, levels, f32(fc[0].weight), f32(fc[0].bias), f32(fc[2].weight), f32(fc[2].bias), mid_sums=mid_sums)

    def forward(self, inputs):
        """Reference signature: {"visual": [B,256,h,w] x L, "lang": ...} -> same dict structure."""
        feats = inputs["visual"]
        if not feats[0].is_cuda:
            raise MqdetError("DyConv: CUDA tensors required (no CPU fallback)")
        levels = ops.get_levels([(f.shape[2], f.shape[3]) for f in feats], feats[0].device)
        x16 = ops.cast_f16(_flatten_levels(feats))
        out = ops.cast_f32(self.forward_flat(x16, levels))
        return {"visual": _split_levels(out, levels.sizes), "lang": inputs["lang"]}


class BertEncoderLayer(BertLayer):
    """vldyhead.py:250-301 — in-repo BERT layer (rpn/modeling_bert.py) with the +-5e4 clamps, on the fused text stream."""

    def __init__(self, config, clamp_min_for_underflow=False, clamp_max_for_overflow=False):
        super().__init__(config.hidden_size, config.num_attention_heads, config.intermediate_size,
                         config.layer_norm_eps, clamp=50000.0 if (clamp_min_for_underflow or clamp_max_for_overflow) else 0.0)

    def forward(self, inputs):
        lang = inputs["lang"]
        h32 = lang["hidden"].float().contiguous()
        o32, _ = BertLayer.forward(self, h32, ops.cast_f16(h32), lang["masks"].float().contiguous())
        lang["hidden"] = o32
        return {"visual": inputs["visual"], "lang": lang}


class VLFuse(nn.Module):
    """vldyhead.py:364-574, TYPE == "MHA-B" only (configs/pretrain/mq-glip-t.yaml:47)."""

    def __init__(self, cfg):
        super().__init__()
        fc = cfg.MODEL.DYHEAD.FUSE_CONFIG
        if fc.TYPE != "MHA-B":
            raise NotImplementedError(f"fusion type {fc.TYPE}: only MHA-B is used by the MQ configs")
        self.cfg = cfg
        self.b_attn = BiAttentionBlockForCheckpoint(v_dim=fc.JOINT_EMB_SIZE, l_dim=cfg.MODEL.LANGUAGE_BACKBONE.LANG_DIM,
                                                    embed_dim=2048, num_heads=8, hidden_dim=3072, dropout=0.1,
                                                    drop_path=.0, init_values=1.0 / cfg.MODEL.DYHEAD.NUM_CONVS, cfg=cfg)

    def forward(self, x):
        lang = x["lang"]
        q = self.b_attn(*x["visual"], lang["hidden"], lang["masks"], None)
        lang["hidden"] = q[5]
        x.update({"visual": list(q[:5]), "lang": lang})
        return x


class Scale(nn.Module):
    def __init__(self, init_value=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.FloatTensor([init_value]))


class VLDyHead(nn.Module):
    """vldyhead.py:594-900 for the MQ-GLIP configuration: 6 x [VLFuse(MHA-B), BertEncoderLayer, DyConv] + dot-product
    token head + 1x1 bbox / centerness heads."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        from types import SimpleNamespace
        lang_cfg = SimpleNamespace(hidden_size=cfg.MODEL.LANGUAGE_BACKBONE.LANG_DIM, num_attention_heads=12,
                                   intermediate_size=3072, layer_norm_eps=1e-12)
        num_classes = cfg.MODEL.DYHEAD.NUM_CLASSES - 1
        num_anchors = len(cfg.MODEL.RPN.ASPECT_RATIOS) * cfg.MODEL.RPN.SCALES_PER_OCTAVE
        channels = cfg.MODEL.DYHEAD.CHANNELS
        fc = cfg.MODEL.DYHEAD.FUSE_CONFIG
        if num_anchors != 1 or not fc.USE_DOT_PRODUCT_TOKEN_LOSS or not fc.USE_FUSED_FEATURES_DOT_PRODUCT:
            raise NotImplementedError("only the MQ-GLIP head (1 anchor, fused-feature dot-product token head)")
        # flags the reference reads on this path whose non-shipped value would change the arithmetic: refuse, never ignore
        if not getattr(fc, "CLAMP_DOT_PRODUCT", True):
            raise NotImplementedError("FUSE_CONFIG.CLAMP_DOT_PRODUCT=False (vldyhead.py:884-886): the +-5e4 clamp is fused")
        if getattr(cfg.VISION_QUERY, "QUERY_FUSION", False):
            raise NotImplementedError("VISION_QUERY.QUERY_FUSION (SupportFuse, vldyhead.py:576-591) is off in every MQ config")
        if getattr(getattr(cfg, "DATASETS", None), "ONE_HOT", False):
            raise NotImplementedError("DATASETS.ONE_HOT is off in every MQ config")
        if getattr(cfg.MODEL.LANGUAGE_BACKBONE, "MASK_SPECIAL", False):
            raise NotImplementedError("LANGUAGE_BACKBONE.MASK_SPECIAL is off in every MQ config")
        bn_type = ["gn", cfg.MODEL.GROUP_NORM.NUM_GROUPS]
        conv_func = lambda i, o, s: Conv3x3Norm(i, o, s, deformable=cfg.MODEL.DYHEAD.USE_DFCONV, bn_type=bn_type)  # noqa: E731
        tower = []
        for i in range(cfg.MODEL.DYHEAD.NUM_CONVS):
            tower.append(VLFuse(cfg))
            tower.append(BertEncoderLayer(lang_cfg, clamp_min_for_underflow=fc.CLAMP_BERTATTN_MIN_FOR_UNDERFLOW,
                                          clamp_max_for_overflow=fc.CLAMP_BERTATTN_MAX_FOR_OVERFLOW))
            tower.append(DyConv(channels, channels, conv_func=conv_func, use_dyrelu=cfg.MODEL.DYHEAD.USE_DYRELU,
                                use_dyfuse=cfg.MODEL.DYHEAD.USE_DYFUSE, use_deform=cfg.MODEL.DYHEAD.USE_DFCONV))
        self.add_module("dyhead_tower", nn.Sequential(*tower))
        self.cls_logits = nn.Conv2d(channels, num_anchors * num_classes, kernel_size=1)
        self.bbox_pred = nn.Conv2d(channels, num_anchors * 4, kernel_size=1)
        self.centerness = nn.Conv2d(channels, num_anchors * 1, kernel_size=1)
        bias_value = -math.log((1 - cfg.MODEL.DYHEAD.PRIOR_PROB) / cfg.MODEL.DYHEAD.PRIOR_PROB)
        self.dot_product_projection_image = nn.Identity()
        self.dot_product_projection_text = nn.Linear(cfg.MODEL.LANGUAGE_BACKBONE.LANG_DIM, num_anchors * channels, bias=True)
        self.log_scale = nn.Parameter(torch.Tensor([cfg.MODEL.DYHEAD.LOG_SCALE]), requires_grad=True)
        self.bias_lang = nn.Parameter(torch.zeros(cfg.MODEL.LANGUAGE_BACKBONE.LANG_DIM), requires_grad=True)
        self.bias0 = nn.Parameter(torch.Tensor([bias_value]), requires_grad=True)
        for m in (self.cls_logits, self.bbox_pred, self.centerness):
            torch.nn.init.normal_(m.weight, std=0.01)
            torch.nn.init.constant_(m.bias, 0)
        self.scales = nn.ModuleList([Scale(init_value=1.0) for _ in range(5)])
        torch.nn.init.constant_(self.cls_logits.bias, bias_value)
        self._head = None
        self.overlap_text_stream = True   # run the text branch of every tower layer on a second stream next to DyConv
        self._side = {}

    def _side_stream(self, device):
        s = self._side.get(device)
        if s is None:
            s = self._side[device] = torch.cuda.Stream(device=device)
        return s

    def _head_weights(self):
        """[4 bbox + 1 centerness, 256] fused 1x1 head (+ bias); log_scale read once (it is a constant at inference)."""
        ps = (self.bbox_pred.weight, self.centerness.weight, self.bbox_pred.bias, self.centerness.bias, self.log_scale)
        key = tuple((p.data_ptr(), p._version) for p in ps)
        if self._head is None or self._head[0] != key:
            w = torch.cat([self.bbox_pred.weight.detach().flatten(1), self.centerness.weight.detach().flatten(1)], 0)
            b = torch.cat([self.bbox_pred.bias.detach(), self.centerness.bias.detach()], 0).float().contiguous()
            self._head = (key, ops.cast_f16(w.float().contiguous()), b, float(torch.exp(-self.log_scale.detach()).item()))
        return self._head[1:]

    @torch.no_grad()
    def forward_flat(self, v16, levels, lang_hidden32, lang_masks):
        """v16 [B,N,256] fp16, language hidden fp32 [B,T,768], masks [B,T] ->
        dict(dot_product_logits [B,N,T] fp32, bbox_reg [B,N,4] fp32 (level Scale applied), centerness [B,N] fp32,
             visual [B,N,256] fp16, hidden [B,T,768] fp32)."""
        B, N, C = v16.shape
        T = lang_hidden32.shape[1]
        cm = lang_masks.float().contiguous()
        h32 = lang_hidden32.float().contiguous()
        main = torch.cuda.current_stream(v16.device)
        for i in range(0, len(self.dyhead_tower), 3):
            fuse, bert, dyconv = self.dyhead_tower[i], self.dyhead_tower[i + 1], self.dyhead_tower[i + 2]
            split = fuse.b_attn.forward_flat_split(v16, h32, cm) if self.overlap_text_stream else None
            if split is None:
                v16, h32 = fuse.b_attn.forward_flat(v16, h32, cm)
                h32, _ = BertLayer.forward(bert, h32, ops.cast_f16(h32), cm)
                v16 = dyconv.forward_flat(v16, levels)
                continue
            # Two branches that do not depend on each other until the next fusion layer:
            #   text branch  : text->image attention over all image tokens -> value / output projections -> BertEncoderLayer
            #   visual branch: DyConv on the fused pyramid
            # The text branch (128 CTAs, then GEMMs with a few dozen tiles) leaves most SMs idle; on a second stream it fills in
            # next to the DyConv kernels.  Fork / join by events (capturable into the CUDA graph as two branches).  Every tensor
            # that crosses streams is kept alive until the join, so the caching allocator never hands a block to one stream
            # while the other may still touch it.
            v_new, ctx = split
            side = self._side_stream(v16.device)
            fork, join = torch.cuda.Event(), torch.cuda.Event()
            fork.record(main)
            with torch.cuda.stream(side):
                side.wait_event(fork)
                h_new = fuse.b_attn.finish_text(ctx)
                h_new, _ = BertLayer.forward(bert, h_new, ops.cast_f16(h_new), cm)
                join.record(side)
            v16 = dyconv.forward_flat(v_new, levels)
            main.wait_event(join)
            keep_alive = (ctx, h32)   # released only now: after the join both streams are done with them
            h32 = h_new
            del keep_alive
        # dot-product token head (:806-818, :871-888): tok = Linear(normalize(h)/2), bias = normalize(h).bias_lang + bias0
        e16, _, beta = ops.l2_normalize(h32, f32(self.bias_lang), f32(self.bias0))  # beta [B,T] fp32
        pt = self.dot_product_projection_text
        tok = ops.gemm(e16.view(B * T, -1), w16(pt.weight), alpha=0.5, bias=f32(pt.bias)).view(B, T, C)
        hw16, hb, inv_scale = self._head_weights()
        logits = torch.empty((B, N, T), dtype=torch.float32, device=v16.device)
        ops.gemm(v16, tok, out=logits, alpha=inv_scale, bias=beta, clamp=50000.0)
        reg_ctr = ops.gemm(v16.view(B * N, C), hw16, bias=hb, out_dtype=torch.float32).view(B, N, 5)
        return {"dot_product_logits": logits, "reg_ctr": reg_ctr, "visual": v16, "hidden": h32}

    @torch.no_grad()
    def forward(self, x, language_dict_features=None, embedding=None, swint_feature_c4=None):
        """Reference signature (:769): x = list of [B,256,h,w]; returns the reference's 10-tuple of per-level lists."""
        if not x[0].is_cuda:
            raise MqdetError("VLDyHead: CUDA tensors required (no CPU fallback)")
        levels = ops.get_levels([(f.shape[2], f.shape[3]) for f in x], x[0].device)
        v16 = ops.cast_f16(_flatten_levels(x))
        r = self.forward_flat(v16, levels, language_dict_features["hidden"], language_dict_features["masks"])
        B = v16.shape[0]
        logits, bbox_reg, centerness, dots, fused = [], [], [], [], []
        vis32 = ops.cast_f32(r["visual"])
        cw = w16(self.cls_logits.weight, view=(self.cls_logits.weight.shape[0], -1))
        for l, (h, w) in enumerate(levels.sizes):
            s, e = levels.off[l], levels.off[l + 1]
            rc = r["reg_ctr"][:, s:e]
            bbox_reg.append((rc[..., :4] * self.scales[l].scale.detach()).transpose(1, 2).reshape(B, 4, h, w))
            centerness.append(rc[..., 4:5].transpose(1, 2).reshape(B, 1, h, w))
            dots.append(r["dot_product_logits"][:, s:e])
            cl = ops.gemm(r["visual"][:, s:e].reshape(B * (e - s), -1), cw, bias=f32(self.cls_logits.bias),
                          out_dtype=torch.float32)
            logits.append(cl.view(B, e - s, -1).transpose(1, 2).reshape(B, -1, h, w))
            fused.append(vis32[:, s:e].transpose(1, 2).reshape(B, -1, h, w))
        language_dict_features["hidden"] = r["hidden"]
        fused_out = fused if getattr(self.cfg.MODEL.RPN, "RETURN_FUSED_FEATURES", False) else None
        return logits, bbox_reg, centerness, None, None, None, dots, None, None, fused_out


_UNSHIPPED_LOSS_FLAGS = ("USE_CLASSIFICATION_LOSS", "USE_TOKEN_LOSS", "USE_CONTRASTIVE_ALIGN_LOSS", "USE_SHALLOW_CONTRASTIVE_LOSS",
                         "USE_BACKBONE_SHALLOW_CONTRASTIVE_LOSS", "MLM_LOSS")


def check_loss_config(cfg):
    """The training losses are those of the MQ-GLIP pre-training configs (dot-product token loss, GIoU, centerness): refuse a
    loss flag whose non-shipped value would add or change a term, never ignore it."""
    fc = cfg.MODEL.DYHEAD.FUSE_CONFIG
    for flag in _UNSHIPPED_LOSS_FLAGS:
        if getattr(fc, flag, False):
            raise NotImplementedError(f"FUSE_CONFIG.{flag}=True: only the MQ-GLIP pre-training losses (dot-product token focal loss, "
                                      "GIoU, centerness) are implemented")
    if not fc.USE_DOT_PRODUCT_TOKEN_LOSS:
        raise NotImplementedError("FUSE_CONFIG.USE_DOT_PRODUCT_TOKEN_LOSS=False is not an MQ-GLIP configuration")


class VLDyHeadModule(nn.Module):
    """vldyhead.py:903-1077: head -> anchors -> ATSS post-processing -> list[BoxList] at inference; in ``train()`` mode head ->
    ATSS assignment -> losses + their gradients at the head outputs (``RPN_ONLY`` branch, :1017-1045)."""

    def __init__(self, cfg, **kwargs):
        super().__init__()
        self.cfg = cfg
        self.head = VLDyHead(cfg)
        self._scales = None
        self._tokmap = None
        self.last_train = None

    def _reg_scales(self):
        ps = [s.scale for s in self.head.scales]
        key = tuple((p.data_ptr(), p._version) for p in ps)
        if self._scales is None or self._scales[0] != key:
            self._scales = (key, [float(p.detach().item()) for p in ps])
        return self._scales[1]

    @torch.no_grad()
    def forward_flat(self, pyr16, levels, image_sizes, lang_hidden, lang_masks, positive_map, max_out=None, tokmap=None,
                     class_labels=None, img_wh=None):
        """pyr16 [B,N,256] fp16 -> device-resident detections: dict(det [B,max_out,6], num [B], ...).
        ``image_sizes``: the (h, w) of every element, or of the B images when the elements are chunks of them (e = chunk * B + image);
        each element's boxes are clipped to its own image, as the reference's post-processor clips each BoxList.
        ``tokmap`` int32 [B,C,max_tok] (+ ``class_labels`` int32 [B,C]): explicit per-element positive maps (batched prompt
        chunks) instead of the one ``positive_map`` dict shared by the batch.  ``img_wh``: fp32 [B, 2] device table of (w, h) per
        image; when given, the clip reads it and ``image_sizes`` is not read."""
        cfg = self.cfg
        if max_out is None:
            max_out = (int(cfg.MODEL.ATSS.DETECTIONS_PER_IMG) + 28 + 31) // 32 * 32
        r = self.head.forward_flat(pyr16, levels, lang_hidden, lang_masks)
        if tokmap is None:
            pkey = tuple((int(k), tuple(v) if not isinstance(v, int) else (v,)) for k, v in sorted(positive_map.items()))
            if self._tokmap is None or self._tokmap[0] != pkey:
                self._tokmap = (pkey, ops.make_tokmap(positive_map, cfg.MODEL.DYHEAD.NUM_CLASSES - 1, pyr16.device))
            tokmap = self._tokmap[1]
        if img_wh is not None:
            iw, ih = img_wh, None
        else:
            ih, iw = image_sizes[0]
            if any(tuple(s) != (ih, iw) for s in image_sizes):   # a padded batch: each element clips to its own image size
                ih, iw = [float(h) for h, _ in image_sizes], [float(w) for _, w in image_sizes]
        out = ops.atss_postprocess(r["dot_product_logits"], r["reg_ctr"], tokmap, levels, cfg.MODEL.RPN.ANCHOR_STRIDE,
                                   cfg.MODEL.RPN.ANCHOR_SIZES, self._reg_scales()[:levels.n], iw, ih,
                                   pre_nms_thresh=cfg.MODEL.ATSS.INFERENCE_TH, pre_nms_top_n=cfg.MODEL.ATSS.PRE_NMS_TOP_N,
                                   nms_thresh=cfg.MODEL.ATSS.NMS_TH, max_det=cfg.MODEL.ATSS.DETECTIONS_PER_IMG,
                                   max_out=max_out, class_labels=class_labels)
        out["head"] = r
        return out

    @torch.no_grad()
    def forward_train_flat(self, pyr16, levels, image_sizes, lang_hidden, lang_masks, gt_pack):
        """pyr16 [B,N,256] fp16 + the GT pack dict(boxes [B,Gmax,4] xyxy, labels [B,Gmax], count [B], tokens [B,Gmax,T]) ->
        dict(losses fp32 [4] = (loss_reg, loss_centerness, loss_dot_product_token, loss_cls = 0), d_logits fp32 [B,N,T],
        d_reg_ctr fp32 [B,N,5] (channels 0-3 w.r.t. the raw box output, before the frozen level Scale), head = the head outputs).
        The loss normalisers are summed over the data-parallel ranks (one collective); nothing synchronises the host."""
        import torch.distributed as dist
        from ... import parallel
        cfg = self.cfg
        check_loss_config(cfg)
        fc, atss = cfg.MODEL.DYHEAD.FUSE_CONFIG, cfg.MODEL.ATSS
        r = self.head.forward_flat(pyr16, levels, lang_hidden, lang_masks)
        strides, sizes = cfg.MODEL.RPN.ANCHOR_STRIDE[:levels.n], cfg.MODEL.RPN.ANCHOR_SIZES[:levels.n]
        t = ops.atss_targets(gt_pack["boxes"], gt_pack["labels"], gt_pack["count"], levels, strides, sizes,
                             topk=getattr(atss, "TOPK", 9))
        parallel.all_reduce_loss_normalizers(t["norm"][:2])
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        losses, d_logits, d_reg_ctr = ops.atss_loss(
            r["dot_product_logits"], r["reg_ctr"], gt_pack["boxes"], gt_pack["labels"], gt_pack["count"], gt_pack["tokens"], levels,
            strides, sizes, self._reg_scales()[:levels.n], lang_masks, targets=t, world=world, alpha=getattr(fc, "TOKEN_ALPHA", 0.25),
            gamma=getattr(fc, "TOKEN_GAMMA", 2.0), reg_weight=getattr(atss, "REG_LOSS_WEIGHT", 2.0),
            token_weight=getattr(fc, "DOT_PRODUCT_TOKEN_LOSS_WEIGHT", 1.0))
        return {"losses": losses, "d_logits": d_logits, "d_reg_ctr": d_reg_ctr, "head": r}

    @staticmethod
    def pack_targets(targets, positive_map, T, device):
        """list of BoxList (field ``labels``) + positive_map [sum G, T] (the reference trainer's inputs) -> the fixed-capacity GT pack
        of ``forward_train_flat`` (Gmax = the largest GT count of the batch, at least 1)."""
        counts = [len(t) for t in targets]
        B, G = len(targets), max(counts + [1])
        boxes = torch.zeros((B, G, 4), dtype=torch.float32, device=device)
        labels = torch.zeros((B, G), dtype=torch.int32, device=device)
        tokens = torch.zeros((B, G, T), dtype=torch.float32, device=device)
        off = 0
        for b, t in enumerate(targets):
            g = counts[b]
            if g:
                boxes[b, :g] = t.convert("xyxy").bbox.to(device=device, dtype=torch.float32)
                labels[b, :g] = t.get_field("labels").to(device=device, dtype=torch.int32)
                tokens[b, :g] = positive_map[off:off + g].to(device=device, dtype=torch.float32)
            off += g
        if positive_map.shape[0] != off:
            raise ValueError(f"positive_map has {positive_map.shape[0]} rows for {off} GT boxes")
        return {"boxes": boxes, "labels": labels, "count": torch.tensor(counts, dtype=torch.int32).to(device), "tokens": tokens}

    @torch.no_grad()
    def forward(self, images, features, targets=None, language_dict_features=None, positive_map=None, captions=None,
                swint_feature_c4=None):
        """Reference signature: features = list of [B,256,h,w]; returns (list[BoxList], {}, fused_visual_features) at inference and
        (None, {loss_reg, loss_centerness, loss_cls, loss_dot_product_token} as 0-dim device tensors, None) in ``train()`` mode, with
        ``targets`` = list of BoxList (field ``labels``) and ``positive_map`` [sum G, T]; the gradients at the head outputs are in
        ``self.last_train`` (see ``forward_train_flat``)."""
        sizes = images.image_sizes if hasattr(images, "image_sizes") else [tuple(images.shape[-2:])] * features[0].shape[0]
        levels = ops.get_levels([(f.shape[2], f.shape[3]) for f in features], features[0].device)
        v16 = ops.cast_f16(_flatten_levels(features))
        if self.training:
            hidden = language_dict_features["hidden"]
            pack = self.pack_targets(targets, positive_map, hidden.shape[1], hidden.device)
            out = self.forward_train_flat(v16, levels, sizes, hidden, language_dict_features["masks"], pack)
            language_dict_features["hidden"] = out["head"]["hidden"]
            self.last_train = out
            l = out["losses"]
            return None, {"loss_reg": l[0], "loss_centerness": l[1], "loss_cls": l[3], "loss_dot_product_token": l[2]}, None
        out = self.forward_flat(v16, levels, sizes, language_dict_features["hidden"], language_dict_features["masks"],
                                positive_map)
        language_dict_features["hidden"] = out["head"]["hidden"]
        return boxlists_from_packed(out["det_packed"], sizes), {}, None
