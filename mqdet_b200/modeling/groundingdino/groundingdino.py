"""MQ-GroundingDINO-T forward on sm_90a kernels, drop-in for groundingdino_new/models/GroundingDINO/groundingdino.py:93-709
(``GroundingDINO``), backbone/backbone.py:155-221 (``Joiner`` of Swin-T + ``PositionEmbeddingSineHW``) and bertwarper.py:28-223
(``BertModelWarper`` around the vision-conditioned ``QVBertModel``), inference (BASELINE config 4), plus the decoder outputs of every
layer and the set-prediction losses of the training branch (``decoder_outputs``, ``loss_evaluator``; groundingdino.py:590-641).

    images -> Swin-T (3 outputs) -> input_proj (1x1 conv + GroupNorm(32); one extra 3x3 stride-2 level) -> 4 levels of 256 channels
    prompt -> QuerySelector (vision queries) + token ids -> per-category text masks -> QVBertModel (PreSelect + GCP) -> feat_map
    Transformer: 6 x [BiAttention fusion, text enhancer, deformable encoder layer] -> two-stage top-900 -> 6 decoder layers
    heads: ContrastiveEmbed class logits, iterative box refinement -> convert_groundingdino_to_glip_output -> list[BoxList]

Same module / parameter names as the reference (``backbone.0.*``, ``input_proj.N.{0,1}``, ``bert.*``, ``feat_map``,
``transformer.*``, ``bbox_embed.N.layers.M`` shared across the decoder layers, ``transformer.enc_out_bbox_embed``), so its
checkpoints load unchanged.  Differences from the reference's inference path, all outside the arithmetic: string captions need an
attached tokenizer (pre-tokenised ``{"input_ids", "attention_mask"}`` are accepted, no vocabulary offline); batches larger than 1 are
supported when the images share one prompt (the reference asserts B == 1, groundingdino.py:543); everything that depends only on
the prompt or on the padding geometry is cached (``_prompt_state`` / ``_geometry``).  Many-category vocabularies (LVIS) run
through ``forward_chunked``: the backbone once per image batch, the prompt chunks as batch elements.
"""
import math

import torch
from torch import nn

from ... import ops
from ..._lib import MqdetError
from ...structures.image_list import to_image_list
from ...utils.weights import f32, w16
from ..backbone.swint import SwinTransformer
from ..language_backbone.bert_model_new import bert_base_config
from ..language_backbone.modeling_bert_new import QVBertModel
from ..query_selector.query_selector import QuerySelector
from ..rpn.vldyhead import _conv_w16
from .bertwarper import generate_masks_with_special_tokens_and_transfer_map
from .loss import SetCriterion
from .matcher import build_matcher
from .transformer import Transformer
from .utils import MLP, ContrastiveEmbed


class PositionEmbeddingSineHW(nn.Module):
    """backbone/position_encoding.py:78-128 with normalize=True (build_position_encoding :171-178): depends only on the padding
    mask, i.e. on the input geometry — evaluated once per geometry by ``GroundingDINO._geometry`` (torch index arithmetic)."""

    def __init__(self, num_pos_feats=128, temperatureH=20, temperatureW=20, normalize=True, scale=None):
        super().__init__()
        self.num_pos_feats, self.temperatureH, self.temperatureW, self.normalize = num_pos_feats, temperatureH, temperatureW, normalize
        self.scale = 2 * math.pi if scale is None else scale

    @torch.no_grad()
    def forward(self, mask):
        """mask bool [B,H,W] (True = padding) -> fp32 [B, 2*num_pos_feats, H, W]."""
        not_mask = ~mask
        y_embed = not_mask.cumsum(1, dtype=torch.float32)
        x_embed = not_mask.cumsum(2, dtype=torch.float32)
        if self.normalize:
            eps = 1e-6
            y_embed = y_embed / (y_embed[:, -1:, :] + eps) * self.scale
            x_embed = x_embed / (x_embed[:, :, -1:] + eps) * self.scale
        d = torch.arange(self.num_pos_feats, dtype=torch.float32, device=mask.device)
        dim_tx = self.temperatureW ** (2 * torch.div(d, 2, rounding_mode="floor") / self.num_pos_feats)
        dim_ty = self.temperatureH ** (2 * torch.div(d, 2, rounding_mode="floor") / self.num_pos_feats)
        pos_x = x_embed[:, :, :, None] / dim_tx
        pos_y = y_embed[:, :, :, None] / dim_ty
        pos_x = torch.stack((pos_x[..., 0::2].sin(), pos_x[..., 1::2].cos()), dim=4).flatten(3)
        pos_y = torch.stack((pos_y[..., 0::2].sin(), pos_y[..., 1::2].cos()), dim=4).flatten(3)
        return torch.cat((pos_y, pos_x), dim=3).permute(0, 3, 1, 2)


class _Pooler(nn.Module):
    """``bert.pooler.dense`` of the reference checkpoint (BertModelWarper keeps it, bertwarper.py:35); its output is never used at
    inference, so it is a parameter container only."""

    def __init__(self, D):
        super().__init__()
        self.dense = nn.Linear(D, D)


class GroundingDINO(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        g = cfg.GROUNDINGDINO
        if g.two_stage_type != "standard" or not g.dec_pred_bbox_embed_share or g.two_stage_bbox_embed_share or \
                g.two_stage_class_embed_share or not g.sub_sentence_present or g.num_feature_levels != 4:
            raise NotImplementedError("only the shipped MQ-GroundingDINO-T configuration (config/defaults.py:944-987) is implemented")
        self.box_threshold = g.box_threshold
        self.num_queries, self.hidden_dim, self.num_feature_levels = g.num_queries, g.hidden_dim, g.num_feature_levels
        self.max_text_len = g.max_text_len
        sw = cfg.MODEL.SWINT
        body = SwinTransformer(sw.EMBED_DIM, tuple(sw.DEPTHS), tuple(sw.NUM_HEADS), sw.WINDOW_SIZE, sw.MLP_RATIO,
                               out_features=("stage3", "stage4", "stage5"))
        pos = PositionEmbeddingSineHW(g.hidden_dim // 2, g.pe_temperatureH, g.pe_temperatureW, normalize=True)
        self.backbone = nn.Sequential(body, pos)   # Joiner: keys backbone.0.* (position embedding has no parameters)
        self.backbone.num_channels = body.num_features[1:]
        self.transformer = Transformer(
            d_model=g.hidden_dim, dropout=g.dropout, nhead=g.nheads, num_queries=g.num_queries, dim_feedforward=g.dim_feedforward,
            num_encoder_layers=g.enc_layers, num_decoder_layers=g.dec_layers, normalize_before=g.pre_norm,
            return_intermediate_dec=True, query_dim=g.query_dim, activation=g.transformer_activation, num_patterns=g.num_patterns,
            num_feature_levels=g.num_feature_levels, enc_n_points=g.enc_n_points, dec_n_points=g.dec_n_points,
            learnable_tgt_init=True, two_stage_type=g.two_stage_type, embed_init_tgt=g.embed_init_tgt,
            use_text_enhancer=g.use_text_enhancer, use_fusion_layer=g.use_fusion_layer, use_text_cross_attention=g.use_text_cross_attention,
            text_dropout=g.text_dropout, fusion_dropout=g.fusion_dropout, fusion_droppath=g.fusion_droppath)
        self.query_selector = None if getattr(cfg.VISION_QUERY, "DISABLE_SELECTOR", False) else QuerySelector(cfg)
        config = bert_base_config()
        self.bert = QVBertModel(config, dim_t=config.hidden_size, dim_v=self.hidden_dim, share_kv=cfg.VISION_QUERY.SHARE_KV, cfg=cfg)
        self.bert.pooler = _Pooler(config.hidden_size)
        self.feat_map = nn.Linear(config.hidden_size, self.hidden_dim, bias=True)
        nn.init.constant_(self.feat_map.bias.data, 0)
        nn.init.xavier_uniform_(self.feat_map.weight.data)
        self.tokenizer = None
        self.specical_tokens = [101, 102, 1012, 1029]  # [CLS], [SEP], '.', '?' of bert-base-uncased (groundingdino.py:206)
        proj = []
        for c in self.backbone.num_channels:
            proj.append(nn.Sequential(nn.Conv2d(c, self.hidden_dim, kernel_size=1), nn.GroupNorm(32, self.hidden_dim)))
        in_c = self.backbone.num_channels[-1]
        for _ in range(self.num_feature_levels - len(self.backbone.num_channels)):
            proj.append(nn.Sequential(nn.Conv2d(in_c, self.hidden_dim, kernel_size=3, stride=2, padding=1), nn.GroupNorm(32, self.hidden_dim)))
            in_c = self.hidden_dim
        self.input_proj = nn.ModuleList(proj)
        for p in self.input_proj:
            nn.init.xavier_uniform_(p[0].weight, gain=1)
            nn.init.constant_(p[0].bias, 0)
        _bbox_embed = MLP(self.hidden_dim, self.hidden_dim, 4, 3)
        nn.init.constant_(_bbox_embed.layers[-1].weight.data, 0)
        nn.init.constant_(_bbox_embed.layers[-1].bias.data, 0)
        self.bbox_embed = nn.ModuleList([_bbox_embed for _ in range(g.dec_layers)])           # shared (groundingdino.py:247-252)
        self.class_embed = nn.ModuleList([ContrastiveEmbed(self.max_text_len) for _ in range(g.dec_layers)])
        self.transformer.decoder.bbox_embed = self.bbox_embed
        self.transformer.decoder.class_embed = self.class_embed
        import copy
        self.transformer.enc_out_bbox_embed = copy.deepcopy(_bbox_embed)                       # two_stage_bbox_embed_share False
        self.transformer.enc_out_class_embed = ContrastiveEmbed(self.max_text_len)
        rb = getattr(cfg.MODEL, "ROI_BOX_HEAD", None)
        self.pooler = None
        if rb is not None:
            from ..poolers import Pooler
            self.pooler = Pooler(output_size=(rb.POOLER_RESOLUTION, rb.POOLER_RESOLUTION), scales=rb.POOLER_SCALES,
                                 sampling_ratio=rb.POOLER_SAMPLING_RATIO, use_v2=True)
        self._prompt = None
        self._geo = None
        # loss criterion (groundingdino.py:152); no parameters, so the state_dict keys are unchanged
        self.loss_evaluator = SetCriterion(build_matcher(g.matcher), cfg)

    # ---- vision-query bank extraction (groundingdino.py:340-430) ------------------------------------------------------
    @torch.no_grad()
    def extract_query(self, samples=None, targets=None, query_images=None, visual_features=None, exclude_similar=False, device=None,
                      max_query_number=None):
        """Expand every ground-truth box x EXPAND_RATIO, pool it from its level of the 4-level ``input_proj`` pyramid (aligned ROIAlign
        POOLER_RESOLUTION^2, mean over the bins) and append it to ``query_images[label]`` ([n, 1, C]) — the GroundingDINO flavour of
        ``GeneralizedVLRCNN_New.extract_query`` (same ``mqdet_roi_align_levels`` kernel, same bank bookkeeping)."""
        from collections import defaultdict
        from ..detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New, append_to_bank
        if self.pooler is None:
            raise MqdetError("extract_query needs cfg.MODEL.ROI_BOX_HEAD (POOLER_RESOLUTION / POOLER_SCALES / POOLER_SAMPLING_RATIO)")
        if not getattr(self.cfg.VISION_QUERY, "SELECT_FPN_LEVEL", True):
            raise NotImplementedError("VISION_QUERY.SELECT_FPN_LEVEL is True in every MQ config (CustomPooler over all levels is unused)")
        query_images = defaultdict(list) if query_images is None else query_images
        targets = GeneralizedVLRCNN_New.expand_bbox([t for t in targets if t is not None], self.cfg.VISION_QUERY.EXPAND_RATIO)
        if visual_features is None:
            images = to_image_list(samples, self.cfg.DATALOADER.SIZE_DIVISIBILITY)
            if not images.tensors.is_cuda:
                raise MqdetError("GroundingDINO.extract_query: CUDA images required (no CPU fallback)")
            _, pyr16, sizes = self.visual_features(images.tensors)
            levels = ops.get_levels(sizes, images.tensors.device)
        else:
            levels = ops.get_levels([(f.shape[2], f.shape[3]) for f in visual_features], visual_features[0].device)
            pyr16 = ops.cast_f16(torch.cat([f.flatten(2).transpose(1, 2) for f in visual_features], dim=1).float().contiguous())
        feats, _ = self.pooler.forward_flat(pyr16, levels, targets, mean_only=True)      # [num_boxes, C]
        query_feats = feats[:, None, :].cpu()
        labels = torch.cat([t.get_field("labels") for t in targets]) if targets else torch.zeros(0, dtype=torch.long)
        assert len(labels) == len(query_feats)
        return append_to_bank(query_images, labels, query_feats, self.cfg, exclude_similar, max_query_number)

    def save_query_bank(self, query_images, path):
        """The on-disk bank format of tools/extract_vision_query.py: torch.save of {label: FloatTensor[n, n_scales, C]}."""
        torch.save({int(k): v.detach().cpu() for k, v in query_images.items()}, path)

    # ---- prompt / geometry state ------------------------------------------------------------------------------------
    def load_query_bank(self, query_path):
        self.query_selector.load_query_bank(query_path)
        self._prompt = None

    def set_query_bank(self, bank):
        """In-memory bank {label: tensor[n, scales, C]} (device tensors are used in place): ``load_query_bank`` without the file."""
        self.query_selector.set_query_bank(bank)
        self._prompt = None

    @torch.no_grad()
    def get_labels_and_maps_from_positive_map(self, positive_map, dtype=torch.float):
        """groundingdino.py:436-445."""
        labels = [k for k, v in positive_map.items() if len(v) != 0]
        all_map = torch.zeros((len(labels), self.cfg.MODEL.LANGUAGE_BACKBONE.MAX_QUERY_LEN), dtype=dtype)
        for j, label in enumerate(labels):
            all_map[j, positive_map[label]] = 1
        return labels, all_map / (all_map.sum(-1)[:, None] + 1e-6)

    def _tokenize(self, captions):
        if isinstance(captions, dict):
            return captions["input_ids"], captions["attention_mask"]
        if self.tokenizer is None:
            raise MqdetError("string captions need a tokenizer (bert-base-uncased vocabulary is not available offline): "
                             "pass {'input_ids', 'attention_mask'} or set model.tokenizer")
        caps = [c.lower().strip() if c.lower().strip().endswith(".") else c.lower().strip() + "." for c in captions]
        tok = self.tokenizer(caps, padding="max_length", return_tensors="pt")
        return tok["input_ids"], tok["attention_mask"]

    @torch.no_grad()
    def _prompt_state(self, captions, positive_map, B, dev):
        """Token ids, per-category text masks / position ids (bertwarper.py:271-320), selected vision queries and the class ->
        token table: everything that depends on the prompt only, rebuilt when its CONTENT (or the query bank) changes."""
        from ..detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
        bank_version = self.query_selector.bank_version if self.query_selector is not None else 0
        # content key (token ids / strings, positive map entries, batch size, bank version); device-resident ids are keyed by storage
        # identity + version counter, so the hot path never synchronises to compare prompts
        key = GeneralizedVLRCNN_New._prompt_key(captions, positive_map, B, bank_version)
        st = self._prompt
        if st is not None and st["key"] == key:
            return st
        ids, am = self._tokenize(captions)
        ids, am = ids[:, : self.max_text_len].cpu(), am[:, : self.max_text_len].cpu()
        sam, pid, _ = generate_masks_with_special_tokens_and_transfer_map({"input_ids": ids}, self.specical_tokens, self.tokenizer)
        if ids.shape[0] == 1 and B > 1:
            ids, am, sam, pid = (t.expand(B, *t.shape[1:]).contiguous() for t in (ids, am, sam, pid))
        vision = vmask = None
        if self.cfg.VISION_QUERY.ENABLED and self.query_selector is not None and self.query_selector.query_bank is not None:
            labels, all_map = self.get_labels_and_maps_from_positive_map(positive_map)
            vision, vmask, _ = self.query_selector([labels] * B, [all_map] * B, None)
            vision, vmask = vision.float().to(dev).contiguous(), vmask.float().to(dev).contiguous()
        C = self.cfg.MODEL.DYHEAD.NUM_CLASSES - 1
        self._prompt = dict(key=key, ids=ids.to(dev), token_mask=am.bool().to(dev), self_mask=sam.to(dev), position_ids=pid.to(dev),
                            bert_mask=sam.float().to(dev).contiguous(), vision=vision, vmask=vmask,
                            tokmap=ops.make_tokmap(positive_map, C, dev))
        self._geo = None
        return self._prompt

    def _image_key(self, image_sizes, padded_hw, level_hw):
        le = self.transformer.level_embed   # folded into the cached level position embeddings: a reloaded checkpoint invalidates them
        return (tuple(tuple(int(v) for v in s) for s in image_sizes), tuple(padded_hw), tuple(level_hw), le.data_ptr(), le._version)

    @torch.no_grad()
    def _level_masks(self, image_sizes, padded_hw, level_hw, B, dev):
        """Padding masks per level (backbone.py:103-111, groundingdino.py:513-516) and their position embeddings."""
        Hp, Wp = padded_hw
        m = torch.zeros((B, Hp, Wp), dtype=torch.float32, device=dev)
        for b, (h, w) in enumerate(image_sizes):
            m[b, int(h):, :] = 1
            m[b, :, int(w):] = 1
        masks = [torch.nn.functional.interpolate(m[None], size=hw).to(torch.bool)[0] for hw in level_hw]
        return masks, [self.backbone[1](mk) for mk in masks]

    @torch.no_grad()
    def _geometry(self, image_sizes, padded_hw, level_hw, B, dev, st):
        """Padding masks per level, position embeddings, encoder reference points, valid ratios, anchor proposals, text position
        embeddings: functions of the image sizes and the prompt only."""
        key = self._image_key(image_sizes, padded_hw, level_hw) + (st["key"],)
        if self._geo is not None and self._geo["key"] == key:
            return self._geo
        masks, poss = self._level_masks(image_sizes, padded_hw, level_hw, B, dev)
        geo = self.transformer.prepare(masks, poss, st["token_mask"], st["position_ids"], st["self_mask"])
        geo["key"] = key
        geo["levels"] = ops.get_levels(list(level_hw), dev)
        geo["img_wh"] = torch.tensor([[float(w), float(h)] for h, w in image_sizes], dtype=torch.float32, device=dev)
        self._geo = geo
        return geo

    # ---- forward ----------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def visual_features(self, x):
        """images [B,3,H,W] -> (src32 fp32 [B, N, 256] of the 4 levels concatenated, src16, level sizes): Swin-T, then per level
        Conv2d + GroupNorm(32) (groundingdino.py:486-511; the 4th level is a 3x3 stride-2 conv of the last Swin stage)."""
        B = x.shape[0]
        feats = self.backbone[0].forward_flat(x, want=(1, 2, 3))
        E = self.hidden_dim
        srcs, sizes = [], []
        for l, i in enumerate((1, 2, 3)):
            t16, h, w = feats[i]
            conv, gn = self.input_proj[l]
            y = ops.gemm(t16.reshape(B * h * w, -1), w16(conv.weight, view=(E, -1)), bias=f32(conv.bias), out_dtype=torch.float32)
            srcs.append(ops.groupnorm_rows(y.view(B, h * w, E), gn.num_groups, f32(gn.weight), f32(gn.bias), gn.eps, out16=False, out32=True))
            sizes.append((h, w))
        t16, h, w = feats[3]
        for l in range(3, self.num_feature_levels):
            conv, gn = self.input_proj[l]
            cols, h, w = ops.im2col3x3(t16, B, h, w, stride=2)
            y = ops.gemm(cols, _conv_w16(conv.weight), bias=f32(conv.bias), out_dtype=torch.float32)
            s32 = ops.groupnorm_rows(y.view(B, h * w, E), gn.num_groups, f32(gn.weight), f32(gn.bias), gn.eps, out16=False, out32=True)
            srcs.append(s32)
            sizes.append((h, w))
            t16 = ops.cast_f16(s32)
        src32 = torch.cat(srcs, dim=1)
        return src32, ops.cast_f16(src32), sizes

    @torch.no_grad()
    def forward_device(self, samples, captions, positive_map, all_layers=False, proposals=None):
        """-> dict(det_packed [B, nq+1, 6] on the device, pred_logits (raw) [B,nq,T], pred_boxes [B,nq,4], ...)."""
        if self.training:
            raise NotImplementedError("training is SURVEY.md §8(f2)")
        images = to_image_list(samples, self.cfg.DATALOADER.SIZE_DIVISIBILITY)
        x = images.tensors
        if not x.is_cuda:
            raise MqdetError("GroundingDINO: CUDA images required (no CPU fallback)")
        B, dev = x.shape[0], x.device
        st = self._prompt_state(captions, positive_map, B, dev)
        src32, src16, sizes = self.visual_features(x)
        geo = self._geometry(images.image_sizes, tuple(x.shape[-2:]), tuple(sizes), B, dev, st)
        pooled = ops.avgpool2_levels(src16, geo["levels"]) if st["vision"] is not None else None   # flatten_fpn_features (:432-434)
        bert = self.bert(input_ids=st["ids"], attention_mask=st["bert_mask"], position_ids=st["position_ids"], vision=st["vision"],
                         images=pooled, vision_attention_mask=st["vmask"], batched_pos_category_map=None)
        h = bert["last_hidden_state"]
        T = h.shape[1]
        enc_text = ops.gemm(ops.cast_f16(h).view(B * T, -1), w16(self.feat_map.weight), bias=f32(self.feat_map.bias),
                            out_dtype=torch.float32).view(B, T, self.hidden_dim)
        tr = self.transformer.forward_flat(src32, geo, enc_text, all_layers=all_layers, proposals=proposals)
        hs, refs = tr["hs"], tr["references"]
        nq = hs[-1].shape[1]
        logits, boxes = self._last_layer_heads(tr, geo["valid_ratios"], st["token_mask"])
        packed = ops.gdino_detections(logits, boxes, st["tokmap"], geo["img_wh"], self.box_threshold)
        return {"det_packed": packed, "det": packed[:, :nq], "num": packed[:, nq, 0], "pred_logits": logits, "pred_boxes": boxes,
                "image_sizes": images.image_sizes, "hs": hs, "references": refs, "srcs": src32, "level_sizes": sizes,
                "encoded_text": enc_text, "bert_hidden": h, "transformer": tr,
                "vision_query_gates": bert["vision_query_gates"], "valid_ratios": geo["valid_ratios"],
                "text_token_mask": st["token_mask"]}

    def _last_layer_heads(self, tr, valid_ratios, token_mask):
        """Class logits [B, nq, 256] and boxes [B, nq, 4] of the last decoder layer: deformable-detr-like anchor update on the
        normed hidden state (groundingdino.py:618-627) and the contrastive class head."""
        h = tr["hs"][-1]
        B, nq = h.shape[:2]
        hs16 = ops.cast_f16(h)
        delta = self.bbox_embed[-1](hs16.view(B * nq, -1), out_dtype=torch.float32)
        boxes, _, _ = ops.box_refine_sine(tr["references"][-2], valid_ratios, delta=delta.view(B, nq, -1), want_sine=False)
        text_dict = {"encoded_text": tr["memory_text"], "encoded_text16": tr["memory_text16"], "text_token_mask": token_mask}
        return self.class_embed[-1](hs16, text_dict), boxes

    # ---- many-category prompts: chunked evaluation (LVIS) --------------------------------------------------------------
    CHUNK_STATE_CAPACITY = 4096    # distinct chunk prompts kept (LVIS: 31)
    CHUNK_GROUP_CAPACITY = 16      # passes of one image geometry kept (LVIS at 8 chunks per pass: 4)

    @torch.no_grad()
    def _chunk_state(self, captions, positive_map, dev):
        """Per-chunk prompt state, cached by content like ``_prompt_state``: token ids, attention mask, per-category self-attention
        mask and restarted position ids (bertwarper.py:271-320), selected vision queries + their token mask, and the chunk's
        classes in ascending label order with their token lists (its score columns)."""
        from ..detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
        bank_version = self.query_selector.bank_version if self.query_selector is not None else 0
        key = GeneralizedVLRCNN_New._prompt_key(captions, positive_map, 1, bank_version)
        cache = self.__dict__.setdefault("_chunk_cache", {})
        st = cache.get(key)
        if st is not None:
            return st
        ids, am = self._tokenize(captions)
        ids, am = ids[:1, : self.max_text_len].cpu(), am[:1, : self.max_text_len].cpu()
        sam, pid, _ = generate_masks_with_special_tokens_and_transfer_map({"input_ids": ids}, self.specical_tokens, self.tokenizer)
        vision = vmask = None
        if self.cfg.VISION_QUERY.ENABLED and self.query_selector is not None and self.query_selector.query_bank is not None:
            labels, all_map = self.get_labels_and_maps_from_positive_map(positive_map)
            vision, vmask, _ = self.query_selector([labels], [all_map], None)
            vision, vmask = vision[0].float().to(dev).contiguous(), vmask[0].float().to(dev).contiguous()
        cols = sorted(int(k) for k in positive_map)
        toks = [([positive_map[c]] if isinstance(positive_map[c], int) else list(positive_map[c])) for c in cols]
        if len(cache) >= self.CHUNK_STATE_CAPACITY:
            cache.clear()
        st = cache[key] = dict(key=key, ids=ids.to(dev), token_mask=am.bool().to(dev), self_mask=sam.to(dev), position_ids=pid.to(dev),
                               vision=vision, vmask=vmask, cols=cols, toks=toks)
        return st

    @torch.no_grad()
    def _chunk_pass_state(self, image_sizes, padded_hw, level_hw, B, dev, sts):
        """Everything one pass of ``forward_chunked_device`` needs besides the image features, for elements e = chunk * B + image:
        the image half of the geometry (computed once per image geometry, repeated per chunk) and the text half of
        ``_chunk_text_state``.  Cached per (image geometry, chunk group); the cache holds the passes of the current image geometry
        only.  Building it uploads nothing that waits for the stream, so a new geometry (the next scale of test-time
        augmentation) does not stall the host."""
        ikey = self._image_key(image_sizes, padded_hw, level_hw)
        cache = self.__dict__.get("_chunk_pass_cache")
        if cache is None or cache["ikey"] != ikey:
            masks, poss = self._level_masks(image_sizes, padded_hw, level_hw, B, dev)
            img_geo = self.transformer.prepare_image(masks, poss)
            img_geo["levels"] = ops.get_levels(list(level_hw), dev)
            wh = torch.tensor([[float(w), float(h)] for h, w in image_sizes], dtype=torch.float32)
            img_geo["img_wh"] = ops.upload_async(wh, dev)
            cache = self._chunk_pass_cache = dict(ikey=ikey, img_geo=img_geo, passes={})
        gkey = tuple(st["key"] for st in sts)
        ps = cache["passes"].get(gkey)
        if ps is not None:
            return ps
        G = len(sts)
        img_geo = cache["img_geo"]
        ps = Transformer.repeat_image_geometry(img_geo, G)
        ps["levels"] = img_geo["levels"]
        ps["img_wh"] = img_geo["img_wh"].repeat(G, 1).contiguous()
        ps.update(self._chunk_text_state(sts, B, dev))
        if len(cache["passes"]) >= self.CHUNK_GROUP_CAPACITY:
            cache["passes"].clear()
        cache["passes"][gkey] = ps
        return ps

    @torch.no_grad()
    def _chunk_text_state(self, sts, B, dev):
        """The text half of a pass, a function of the chunk group and the batch size only: the text half of the geometry and the
        BERT inputs of the chunks, the vision queries zero-padded to the group's largest count (the pad_sequence padding of
        QuerySelector.forward, query_selector.py:112-116), and the per-element class tables.  Cached apart from the image
        geometry, so every geometry's pass shares these tensors (the GCP index table is built once per vision mask tensor)."""
        key = (tuple(st["key"] for st in sts), B)
        cache = self.__dict__.setdefault("_chunk_text_cache", {})
        ts = cache.get(key)
        if ts is not None:
            return ts
        G = len(sts)

        def per_element(ts):   # [1, ...] per chunk -> [G * B, ...], element e = chunk * B + image
            return torch.cat(ts).repeat_interleave(B, dim=0).contiguous()

        token_mask = per_element([st["token_mask"] for st in sts])
        self_mask, position_ids = per_element([st["self_mask"] for st in sts]), per_element([st["position_ids"] for st in sts])
        ts = dict(self.transformer.prepare_text(token_mask, position_ids, self_mask))
        ts["per_element_max"] = True   # each chunk's fusion scores are shifted by their own maximum (one chunk per reference forward)
        ts["ids"], ts["bert_mask"], ts["position_ids"] = per_element([st["ids"] for st in sts]), self_mask.float().contiguous(), position_ids
        ts["vision"] = ts["vmask"] = None
        if sts[0]["vision"] is not None:
            Vmax = max(st["vision"].shape[0] for st in sts)
            vision = torch.zeros((G, Vmax, sts[0]["vision"].shape[1]), dtype=torch.float32, device=dev)
            vmask = torch.zeros((G, Vmax, sts[0]["vmask"].shape[1]), dtype=torch.float32, device=dev)
            for g, st in enumerate(sts):
                vision[g, :st["vision"].shape[0]] = st["vision"]
                vmask[g, :st["vmask"].shape[0]] = st["vmask"]
            ts["vision"] = vision.repeat_interleave(B, dim=0).contiguous()
            ts["vmask"] = vmask.repeat_interleave(B, dim=0).contiguous()
        Cmax = max(max(len(st["cols"]) for st in sts), 1)
        mt = max(max((len(t) for t in st["toks"]), default=1) for st in sts)
        tok_h = torch.full((G, Cmax, mt), -1, dtype=torch.int32)
        lab_h = torch.zeros((G, Cmax), dtype=torch.int32)
        for g, st in enumerate(sts):
            for j, (c, tk) in enumerate(zip(st["cols"], st["toks"])):
                tok_h[g, j, :len(tk)] = torch.tensor(tk, dtype=torch.int32)
                lab_h[g, j] = c
        ts["tokmap"] = ops.upload_async(tok_h, dev).repeat_interleave(B, dim=0).contiguous()
        ts["class_labels"] = ops.upload_async(lab_h, dev).repeat_interleave(B, dim=0).contiguous()
        if len(cache) >= self.CHUNK_GROUP_CAPACITY:
            cache.clear()
        cache[key] = ts
        return ts

    @torch.no_grad()
    def forward_chunked_device(self, images, chunk_captions, chunk_positive_maps, chunks_per_pass=8, chunk_ids=None):
        """Chunked evaluation of a many-category vocabulary (LVIS: 1203 classes as 31 prompts of 40 classes,
        maskrcnn_benchmark/engine/inference.py:600-660 with TEST.CHUNKED_EVALUATION).  The reference runs the WHOLE model once per
        chunk and image; here Swin-T + ``input_proj`` run ONCE per image batch and the chunks travel as extra batch elements
        (element e = chunk * B + image) through the vision-conditioned BERT, ``feat_map``, the transformer and the heads,
        ``chunks_per_pass`` chunks at a time.  The stable-softmax maximum of the fusion layers is taken per element, so a chunk's
        detections do not depend on which chunks share its pass.  Score columns of a chunk are its classes in ascending label
        order; the emitted labels are the global class ids (ties to the lowest label, as the reference's ``topk(1)`` over the
        zero-filled full-vocabulary scores).  ``chunk_ids``: the subset of chunks THIS rank evaluates, default all.
        Returns {"det_packed": [n_chunks_local, B, num_queries + 1, 6] device tensor, "chunks": [chunk index ...], ...}."""
        if self.training:
            raise NotImplementedError("training is SURVEY.md §8(f2)")
        if int(chunks_per_pass) < 1:
            raise ValueError(f"chunks_per_pass must be >= 1, got {chunks_per_pass}")
        chunks_per_pass = int(chunks_per_pass)
        images = to_image_list(images, self.cfg.DATALOADER.SIZE_DIVISIBILITY)
        x = images.tensors
        if not x.is_cuda:
            raise MqdetError("GroundingDINO: CUDA images required (no CPU fallback)")
        if len(chunk_captions) != len(chunk_positive_maps):
            raise ValueError("one positive map per chunk caption required")
        B, dev = x.shape[0], x.device
        chunk_ids = list(range(len(chunk_captions))) if chunk_ids is None else [int(c) for c in chunk_ids]
        src32, src16, sizes = self.visual_features(x)     # ONCE per image batch, shared by all chunks
        nq = self.num_queries
        packed = torch.empty((len(chunk_ids), B, nq + 1, 6), dtype=torch.float32, device=dev)
        pooled = None
        for p0 in range(0, len(chunk_ids), chunks_per_pass):
            group = chunk_ids[p0:p0 + chunks_per_pass]
            G = len(group)
            sts = [self._chunk_state(chunk_captions[c], chunk_positive_maps[c], dev) for c in group]
            ps = self._chunk_pass_state(images.image_sizes, tuple(x.shape[-2:]), tuple(sizes), B, dev, sts)
            if ps["vision"] is not None and pooled is None:
                pooled = ops.avgpool2_levels(src16, ps["levels"])   # flatten_fpn_features (:432-434)
            bert = self.bert(input_ids=ps["ids"], attention_mask=ps["bert_mask"], position_ids=ps["position_ids"], vision=ps["vision"],
                             images=pooled.repeat(G, 1, 1) if ps["vision"] is not None else None,
                             vision_attention_mask=ps["vmask"], batched_pos_category_map=None)
            h = bert["last_hidden_state"]
            E, T = h.shape[:2]
            enc_text = ops.gemm(ops.cast_f16(h).view(E * T, -1), w16(self.feat_map.weight), bias=f32(self.feat_map.bias),
                                out_dtype=torch.float32).view(E, T, self.hidden_dim)
            tr = self.transformer.forward_flat(src32.repeat(G, 1, 1) if G > 1 else src32, ps, enc_text)
            logits, boxes = self._last_layer_heads(tr, ps["valid_ratios"], ps["text_token_mask"])
            det = ops.gdino_detections(logits, boxes, ps["tokmap"], ps["img_wh"], self.box_threshold, class_labels=ps["class_labels"])
            packed[p0:p0 + G] = det.view(G, B, nq + 1, 6)
        return {"det_packed": packed, "chunks": chunk_ids, "image_sizes": images.image_sizes, "srcs": src32, "pyramid16": src16,
                "levels": ops.get_levels(sizes, dev)}

    def forward_chunked(self, images, chunk_captions, chunk_positive_maps, chunks_per_pass=8, chunk_ids=None):
        """-> list[BoxList] (mode xyxy, fields labels / scores): per image, the per-chunk detections concatenated in chunk order
        with their global labels (``BoxList.concate_box_list``, engine/inference.py:704-706)."""
        from ...structures.bounding_box import BoxList
        out = self.forward_chunked_device(images, chunk_captions, chunk_positive_maps, chunks_per_pass, chunk_ids)
        pk = out["det_packed"].cpu()
        nq = pk.shape[2] - 1
        res = []
        for b, (h, w) in enumerate(out["image_sizes"]):
            parts = [pk[g, b, :int(pk[g, b, nq, 0])] for g in range(pk.shape[0])]
            d = torch.cat(parts) if parts else torch.zeros((0, 6))
            bl = BoxList(d[:, :4].clone(), (w, h), mode="xyxy")
            bl.add_field("labels", d[:, 5].long())
            bl.add_field("scores", d[:, 4].clone())
            res.append(bl)
        return res

    @torch.no_grad()
    def decoder_outputs_flat(self, out):
        """Class logits and boxes of EVERY decoder layer from ``forward_device(..., all_layers=True)`` (groundingdino.py:590-607)
        -> (pred_logits fp32 [L, B, Q, 256], -inf outside the text mask; pred_boxes fp32 [L, B, Q, 4], sigmoid cxcywh, layer k =
        sigmoid(bbox_embed(hs[k]) + inverse_sigmoid(references[k]))).  ``bbox_embed`` is shared across the layers and the text
        operand of ``ContrastiveEmbed`` is the same for all of them, so the L layers' rows go through ONE MLP chain and ONE
        contrastive product per image.  Layer L-1 equals ``out["pred_logits"]`` / ``out["pred_boxes"]`` bit for bit."""
        hs, refs = out["hs"], out["references"]
        L = len(hs)
        if L != len(refs) - 1:
            raise ValueError("decoder_outputs needs the hidden states of every layer: call forward_device(..., all_layers=True)")
        B, nq, E = hs[0].shape
        hs16 = ops.cast_f16(torch.stack(hs, 1).contiguous())                                 # [B, L, nq, E], rows (b, l, q)
        delta = self.bbox_embed[-1](hs16.view(B * L * nq, E), out_dtype=torch.float32)
        ref = torch.stack(refs[:L], 1).contiguous().view(B * L, nq, 4)
        vr = out["valid_ratios"].repeat_interleave(L, dim=0)
        boxes, _, _ = ops.box_refine_sine(ref, vr, delta=delta.view(B * L, nq, -1), want_sine=False)
        tr = out["transformer"]
        text_dict = {"encoded_text": tr["memory_text"], "encoded_text16": tr["memory_text16"], "text_token_mask": out["text_token_mask"]}
        logits = self.class_embed[-1](hs16.view(B, L * nq, E), text_dict)                      # [B, L*nq, 256]
        logits = logits.view(B, L, nq, -1).transpose(0, 1).contiguous()
        boxes = boxes.view(B, L, nq, 4).transpose(0, 1).contiguous()
        return logits, boxes

    def decoder_outputs(self, out):
        """The reference's training-branch ``out`` dict (groundingdino.py:609-611): {"pred_logits" [B, Q, 256], "pred_boxes"
        [B, Q, 4] of the last layer, "aux_outputs": [{"pred_logits", "pred_boxes"} of layers 0..L-2]}, views of
        ``decoder_outputs_flat``."""
        logits, boxes = self.decoder_outputs_flat(out)
        L = logits.shape[0]
        return {"pred_logits": logits[L - 1], "pred_boxes": boxes[L - 1],
                "aux_outputs": [{"pred_logits": logits[k], "pred_boxes": boxes[k]} for k in range(L - 1)]}

    @staticmethod
    def to_boxlists(packed, image_sizes):
        """One device->host copy of the packed result, then BoxList(mode xyxy, fields labels / scores) per image."""
        from ...structures.bounding_box import BoxList
        h = packed.cpu()
        nq = h.shape[1] - 1
        res = []
        for b, (ih, iw) in enumerate(image_sizes):
            k = int(h[b, nq, 0])
            bl = BoxList(h[b, :k, :4].clone(), (iw, ih), mode="xyxy")
            bl.add_field("labels", h[b, :k, 5].long())
            bl.add_field("scores", h[b, :k, 4].clone())
            res.append(bl)
        return res

    def forward(self, samples, targets=None, **kw):
        """Reference signature (groundingdino.py:447): eval -> list[BoxList] (or (result, srcs) with return_backbone_features)."""
        out = self.forward_device(samples, kw["captions"], kw["positive_map"])
        res = self.to_boxlists(out["det_packed"], out["image_sizes"])
        if kw.get("return_backbone_features", False):
            B = out["srcs"].shape[0]
            off, maps = 0, []
            for h, w in out["level_sizes"]:
                maps.append(out["srcs"][:, off:off + h * w].transpose(1, 2).reshape(B, -1, h, w).contiguous())
                off += h * w
            return res, maps
        return res
