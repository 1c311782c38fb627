"""MQ-GLIP detector meta-architecture (inference), drop-in for
maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py:90-667 (``GeneralizedVLRCNN_New``).

    images -> Swin-T -> FPN -> [B, N, 256] pyramid ---------------------------------------------+
    positive_map -> QuerySelector -> vision queries -> PreSelect(queries x pooled pyramid) ----+ |
    token ids -> BERT layers 0..5 -> [GCP_i -> BERT layer 6+i] x 6 -> text stream [B,T,768] --+-+-> VLDyHead -> ATSS
                                                                                                   post-processing -> BoxList

Parameter names follow the reference (``backbone.body.*``, ``backbone.fpn.*``, ``language_backbone.body.model.*``,
``rpn.head.*``) so its checkpoints load unchanged.  Differences from the reference, all at the host boundary:
  * captions may be given pre-tokenised ({"input_ids", "attention_mask"}) — no tokenizer vocabulary is available
    offline; with an HF tokenizer attached (``self.tokenizer``) plain strings work as in the reference;
  * the eval-time ``assert B == 1`` (:354) is lifted: a batch shares one prompt (the training-branch tensor layout).
"""
import random
from collections import OrderedDict

import torch
from torch import nn

from ... import ops
from ..._lib import MqdetError
from ...structures.bounding_box import boxlists_from_packed
from ...structures.image_list import to_image_list
from ...utils import reserve_entries
from ..backbone.fpn import FPN, LastLevelP6P7
from ..backbone.swint import SwinTransformer
from ..chunk_prompts import cached_chunk_state, chunk_columns, chunk_group_tables, group_key, per_element, prompt_key
from ..language_backbone.bert_model_new import BertEncoder
from ..poolers import Pooler
from ..query_selector.query_selector import QuerySelector
from ..rpn.vldyhead import VLDyHeadModule

MASK_TOKEN_ID = 103   # [MASK] of the bert-base-uncased vocabulary (tokenizer.mask_token_id)


def build_backbone(cfg):
    """SWINT-FPN-RETINANET (modeling/backbone/__init__.py:37-80)."""
    sw = cfg.MODEL.SWINT
    body = SwinTransformer(embed_dim=sw.EMBED_DIM, depths=tuple(sw.DEPTHS), num_heads=tuple(sw.NUM_HEADS),
                           window_size=sw.WINDOW_SIZE, mlp_ratio=sw.MLP_RATIO)
    oc = cfg.MODEL.BACKBONE.OUT_CHANNELS
    fpn = FPN([0, sw.OUT_CHANNELS[-3], sw.OUT_CHANNELS[-2], sw.OUT_CHANNELS[-1]], oc, top_blocks=LastLevelP6P7(oc, oc))
    return nn.Sequential(OrderedDict([("body", body), ("fpn", fpn)]))


def append_to_bank(query_images, labels, query_feats, cfg, exclude_similar=False, max_query_number=None):
    """The bank bookkeeping shared by ``GeneralizedVLRCNN_New.extract_query`` (generalized_vl_rcnn_new.py:268-288) and
    ``GroundingDINO.extract_query`` (groundingdino.py:411-430): append each box's pooled feature [n_scales, C] to ``query_images[label]``
    up to MAX_QUERY_NUMBER per label, optionally skipping near-duplicates (cosine similarity above SIMILARITY_THRESHOLD).  Host-side
    list handling on a handful of ground-truth boxes."""
    import torch.nn.functional as F
    max_query_number = cfg.VISION_QUERY.MAX_QUERY_NUMBER if max_query_number is None else max_query_number
    for label, feat in zip(labels.tolist(), query_feats):
        n = len(query_images[label])
        if n >= max_query_number:
            continue
        if exclude_similar and n > 0:
            bank = F.normalize(query_images[label], p=2, dim=-1)                    # [n, 1, C]
            new = F.normalize(feat, p=2, dim=-1)                                     # [1, C]
            if ((bank * new[None]).sum(-1) > cfg.VISION_QUERY.SIMILARITY_THRESHOLD).sum() > 0:
                continue
        query_images[label] = feat[None] if n == 0 else torch.cat([query_images[label], feat[None]])
    return query_images


class GeneralizedVLRCNN_New(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.backbone = build_backbone(cfg)
        self.language_backbone = nn.Sequential(OrderedDict([("body", BertEncoder(cfg))]))
        self.rpn = VLDyHeadModule(cfg)
        self.roi_heads = None  # RPN_ONLY: True (configs/pretrain/mq-glip-t.yaml:6)
        self.query_selector = QuerySelector(cfg) if cfg.VISION_QUERY.ENABLED else None
        # box pooler for extracting the vision-query bank (:108-122; SELECT_FPN_LEVEL True in every MQ config)
        rb = getattr(cfg.MODEL, "ROI_BOX_HEAD", None)
        self.pooler = None
        if rb is not None:
            if not cfg.VISION_QUERY.SELECT_FPN_LEVEL:
                raise NotImplementedError("VISION_QUERY.SELECT_FPN_LEVEL=False (CustomPooler) is off in every MQ config")
            self.pooler = Pooler(output_size=(rb.POOLER_RESOLUTION, rb.POOLER_RESOLUTION), scales=rb.POOLER_SCALES,
                                 sampling_ratio=rb.POOLER_SAMPLING_RATIO, use_v2=True)
        self.tokenizer = None  # attach an HF tokenizer to accept string captions
        self.DEBUG = False
        self._prompt = None
        self.overlap_text_prefix = True   # image-independent BERT layers on a second stream next to the visual backbone
        self.cache_chunk_groups = True    # keep the prompt side of each chunked pass, BERT prefix included (False: rebuild per pass)
        self._chunk_read = None
        self._side = {}

    def _side_stream(self, device):
        s = self._side.get(device)
        if s is None:
            s = self._side[device] = torch.cuda.Stream(device=device)
        return s

    def load_query_bank(self, path):
        self.query_selector.load_query_bank(path)
        self.invalidate_prompt_cache()

    def set_query_bank(self, bank):
        """In-memory bank {label: tensor[n, scales, C]} (device tensors are used in place): ``load_query_bank`` without the file."""
        self.query_selector.set_query_bank(bank)
        self.invalidate_prompt_cache()

    def save_query_bank(self, query_images, path):
        """The on-disk bank format of tools/extract_vision_query.py: torch.save of {label: FloatTensor[n, n_scales, C]}."""
        torch.save({int(k): v.detach().cpu() for k, v in query_images.items()}, path)

    @staticmethod
    def expand_bbox(box_list, expand_ratio=1.5):
        """generalized_vl_rcnn_new.py:32-49: boxes grown by ``expand_ratio`` about their centre, clipped to the image, empty
        ones removed (host-side box bookkeeping on a handful of ground-truth boxes)."""
        from ...structures.bounding_box import BoxList
        out = []
        for boxes in box_list:
            assert boxes.mode == "xyxy"
            bb = boxes.bbox.float()
            bw, bh = bb[:, 2] - bb[:, 0], bb[:, 3] - bb[:, 1]
            dw, dh = (bw * expand_ratio - bw) / 2, (bh * expand_ratio - bh) / 2
            nb = BoxList(bb + torch.stack([-dw, -dh, dw, dh], dim=1), boxes.size, mode="xyxy")
            nb.add_field("labels", boxes.get_field("labels"))
            out.append(nb.clip_to_image(remove_empty=True))
        return out

    @torch.no_grad()
    def extract_query(self, images=None, targets=None, query_images=None, visual_features=None, exclude_similar=False,
                      device=None, max_query_number=None):
        """Vision-query bank extraction (:232-288): expand every ground-truth box x EXPAND_RATIO, pool it from its FPN level
        (aligned ROIAlign POOLER_RESOLUTION^2, mean over the bins -> one 256-vector per box) and append it to
        ``query_images[label]`` ([n, 1, C]) up to MAX_QUERY_NUMBER per label, optionally skipping near-duplicates."""
        from collections import defaultdict
        import torch.nn.functional as F
        if self.pooler is None:
            raise MqdetError("extract_query needs cfg.MODEL.ROI_BOX_HEAD (POOLER_RESOLUTION / POOLER_SCALES / POOLER_SAMPLING_RATIO)")
        query_images = defaultdict(list) if query_images is None else query_images
        targets = self.expand_bbox([t for t in targets if t is not None], self.cfg.VISION_QUERY.EXPAND_RATIO)
        if visual_features is None:
            images = to_image_list(images)
            x = images.tensors
            if not x.is_cuda:
                raise MqdetError("GeneralizedVLRCNN_New.extract_query: CUDA images required (no CPU fallback)")
            feats = self.backbone.body.forward_flat(x)
            pyr16, levels = self.backbone.fpn.forward_flat([feats[i] for i in (1, 2, 3)])
        else:
            levels = ops.get_levels([(f.shape[2], f.shape[3]) for f in visual_features], visual_features[0].device)
            pyr16 = ops.cast_f16(torch.cat([f.flatten(2).transpose(1, 2) for f in visual_features], dim=1).contiguous())
        feats, _ = self.pooler.forward_flat(pyr16, levels, targets, mean_only=True)     # [num_boxes, C]
        query_feats = feats[:, None, :].cpu()                                            # [num_boxes, 1 scale, C]
        labels = torch.cat([t.get_field("labels") for t in targets]) if targets else torch.zeros(0, dtype=torch.long)
        assert len(labels) == len(query_feats)
        return append_to_bank(query_images, labels, query_feats, self.cfg, exclude_similar, max_query_number)

    def graph_state(self):
        """The cached tensors a forward just read (prompt state, the head's token map, the GCP index and padded-query tables, and
        the chunk and chunk-group states of the last chunked forward): whoever captures that forward in a CUDA graph keeps this
        object as long as the graph, because the next prompt, batch size or chunk grouping replaces or clears these caches and
        would free memory the graph still reads."""
        from ..language_backbone import modeling_bert_new
        return (self._prompt, self.rpn._tokmap) + modeling_bert_new.cache_entries() + (self._chunk_read,)

    def invalidate_prompt_cache(self):
        """Drop everything cached per prompt (token ids, selected queries, masks, the head's token map)."""
        self._prompt = None
        self.rpn._tokmap = None

    def text_mask_rate(self):
        """Vision-only evaluation (generalized_vl_rcnn_new.py:397-407): VISION_QUERY.TEXT_DROPOUT when MASK_DURING_INFERENCE
        masks prompt tokens at inference, else 0.  Each forward draws one ``random.random()`` per category per image; the
        tokens of a category whose draw is below the rate and that has vision queries become [MASK]."""
        vq = self.cfg.VISION_QUERY
        if not (vq.ENABLED and getattr(vq, "MASK_DURING_INFERENCE", False) and vq.TEXT_DROPOUT > 0):
            return 0.0
        if vq.PURE_TEXT_RATE != 0:
            raise NotImplementedError("VISION_QUERY.MASK_DURING_INFERENCE needs VISION_QUERY.PURE_TEXT_RATE == 0 (the reference "
                                      f"asserts it), got {vq.PURE_TEXT_RATE}")
        if vq.NEW_MASK_TOKEN:
            raise NotImplementedError("VISION_QUERY.NEW_MASK_TOKEN=True with VISION_QUERY.MASK_DURING_INFERENCE: the reference's "
                                      "learned mask token branch is disabled; use the [MASK] token (NEW_MASK_TOKEN=False)")
        if self.query_selector.query_bank is None:
            raise MqdetError("VISION_QUERY.MASK_DURING_INFERENCE: vision-only evaluation needs a query bank")
        return float(vq.TEXT_DROPOUT)

    def _mask_tables(self, ids, all_map, has, rate):
        """Per-prompt tables of the token masking: ``tok_cat`` int32 [E, T] (row of ``all_map`` each token belongs to, -1 for
        none) and the per-image has-query lists; at rate >= 1 every draw is below the rate, so the masked ids are cached too."""
        E, T = ids.shape
        pos = all_map != 0
        if pos.shape[1] != T:
            raise MqdetError(f"MASK_DURING_INFERENCE: {T} token ids per prompt but MAX_QUERY_LEN = {pos.shape[1]}")
        if (pos.sum(0) > 1).any():
            raise MqdetError("MASK_DURING_INFERENCE: a token belongs to two categories of the positive map")
        cat = torch.full((T,), -1, dtype=torch.int32)
        rows, toks = pos.nonzero(as_tuple=True)
        cat[toks] = rows.to(torch.int32)
        tok_cat = ops.upload_async(cat[None].expand(E, -1).contiguous(), ids.device)
        tab = dict(tok_cat=tok_cat, has=has, mask_rate=rate)
        if rate >= 1.0:
            tab["ids_masked"] = ops.mask_prompt_tokens(ids, tok_cat, ops.upload_async(torch.tensor(has, dtype=torch.uint8), ids.device),
                                                       self.mask_token_id())
        return tab

    def mask_token_id(self):
        return getattr(self.tokenizer, "mask_token_id", None) or MASK_TOKEN_ID

    @staticmethod
    def draw_text_masks(has, rate):
        """:402-406 for the images of ``has`` (one has-query list per image) in order: one ``random.random()`` per category,
        drawn for every category -> [len(has)][C] flags, 1 = mask the category's tokens."""
        return [[int(random.random() < rate and h == 1) for h in row] for row in has]

    @classmethod
    def draw_chunk_text_masks(cls, states, B, rate):
        """The draws of a chunked forward over B images: the reference's forwards run images outer, chunks inner
        (inference.py:600-625) -> [B][chunk][C] flags."""
        return [[cls.draw_text_masks(st["has"], rate)[0] for st in states] for _ in range(B)]

    def max_out(self):
        """Rows of the fixed-shape per-image result: DETECTIONS_PER_IMG plus head-room for the reference's `>= kth score`
        ties (rpn/inference.py:757-767), rounded up to a multiple of 32 (100 -> 128, LVIS 300 -> 352)."""
        d = int(self.cfg.MODEL.ATSS.DETECTIONS_PER_IMG)
        return (d + 28 + 31) // 32 * 32

    @torch.no_grad()
    def get_labels_and_maps_from_positive_map(self, positive_map, dtype=torch.float):
        """:295-305 — labels with at least one token and their normalised token-location rows."""
        labels = [k for k, v in positive_map.items() if len(v) != 0]
        T = self.cfg.MODEL.LANGUAGE_BACKBONE.MAX_QUERY_LEN
        all_map = torch.zeros((len(labels), T), dtype=dtype)
        for j, label in enumerate(labels):
            all_map[j, positive_map[label]] = 1
        all_map = all_map / (all_map.sum(-1)[:, None] + 1e-6)
        return labels, all_map

    def _tokenize(self, captions, device):
        if isinstance(captions, dict):
            return captions["input_ids"].to(device), captions["attention_mask"].to(device)
        if self.tokenizer is None:
            raise MqdetError("string captions need a tokenizer (bert-base-uncased vocabulary is not available offline): "
                             "pass {'input_ids', 'attention_mask'} or set model.tokenizer")
        L = self.cfg.MODEL.LANGUAGE_BACKBONE
        encode = getattr(self.tokenizer, "batch_encode_plus", None) or self.tokenizer   # transformers >= 5 dropped the alias of __call__
        tok = encode(captions, max_length=L.MAX_QUERY_LEN, padding="max_length" if L.PAD_MAX else "longest",
                     return_special_tokens_mask=True, return_tensors="pt", truncation=True)
        return tok.input_ids.to(device), tok.attention_mask.to(device)

    @torch.no_grad()
    def _prompt_state(self, captions, positive_map, B, dev):
        """Everything that depends only on the prompt (token ids, selected vision queries, their token mask) is built
        once per (captions, positive_map) object pair and batch size — the reference rebuilds it in every forward
        (Python loops over classes in QuerySelector.forward :57-100 and a tokenizer call :378-383)."""
        st = self._prompt
        bank_version = self.query_selector.bank_version if self.query_selector is not None else 0
        same_objects = st is not None and st["captions"] is captions and st["positive_map"] is positive_map
        rate = self.text_mask_rate()
        key = prompt_key(captions, positive_map, B, bank_version) + (rate,)
        if st is not None and st["key"] == key:
            if not same_objects:
                st["captions"], st["positive_map"] = captions, positive_map
            return st
        self.rpn._tokmap = None
        ids, am = self._tokenize(captions, dev)
        if ids.shape[0] == 1 and B > 1:
            ids, am = ids.expand(B, -1).contiguous(), am.expand(B, -1).contiguous()
        vision = vmask = None
        self._prompt = dict(key=key, captions=captions, positive_map=positive_map, B=B, ids=ids, am=am, mask_rate=0.0)
        if self.query_selector is not None and self.query_selector.query_bank is not None:
            labels, all_map = self.get_labels_and_maps_from_positive_map(positive_map)
            vision, vmask, has = self.query_selector([labels] * B, [all_map] * B, None)
            vision, vmask = vision.float().contiguous(), vmask.float().contiguous()
            if rate > 0:
                self._prompt.update(self._mask_tables(ids, all_map, has, rate))
        self._prompt.update(vision=vision, vmask=vmask)
        return self._prompt

    def _prompt_ids(self, st):
        """The token ids of one forward: the prompt's own, or those of vision-only evaluation.  At rate >= 1 the cached masked
        ids; below, this forward's draws are uploaded (pinned, asynchronous) and masked on the device.  The draws advance
        Python's ``random`` exactly as the reference's per-image forwards do, in both cases."""
        rate = st["mask_rate"]
        if rate == 0:
            return st["ids"]
        flags = self.draw_text_masks(st["has"], rate)
        if rate >= 1.0:
            return st["ids_masked"]
        dev = st["ids"].device
        flags = ops.upload_async(torch.tensor(flags, dtype=torch.uint8), dev)
        return ops.mask_prompt_tokens(st["ids"], st["tok_cat"], flags, self.mask_token_id())

    @torch.no_grad()
    def forward_device(self, images, captions, positive_map, max_out=None, img_wh=None):
        """Everything up to (and excluding) the device->host copy: returns the device-resident result dict.
        ``max_out`` (rows of the fixed-shape detections) defaults to ``self.max_out()`` (from DETECTIONS_PER_IMG).
        ``img_wh``: optional fp32 [B, 2] device table of the images' (w, h); the clip then reads it instead of
        ``images.image_sizes``, so a captured graph serves any image sizes at its padded shape."""
        max_out = self.max_out() if max_out is None else int(max_out)
        if self.training:
            raise NotImplementedError("training is SURVEY.md §8f")
        images = to_image_list(images, self.cfg.DATALOADER.SIZE_DIVISIBILITY)
        x = images.tensors
        if not x.is_cuda:
            raise MqdetError("GeneralizedVLRCNN_New: CUDA images required (no CPU fallback)")
        B = x.shape[0]
        st = self._prompt_state(captions, positive_map, B, x.device)
        ids = self._prompt_ids(st)
        # The embeddings and the BERT layers before the first GCP block depend on the prompt only: they run on a second
        # stream next to the visual backbone (fork / join by events; capturable as a second graph branch).
        prefix = None
        if self.overlap_text_prefix:
            main = torch.cuda.current_stream(x.device)
            side = self._side_stream(x.device)
            fork, join = torch.cuda.Event(), torch.cuda.Event()
            fork.record(main)
            with torch.cuda.stream(side):
                side.wait_event(fork)
                prefix = self.language_backbone.body.model.text_prefix(ids, st["am"])
                join.record(side)
        feats = self.backbone.body.forward_flat(x)
        pyr16, levels = self.backbone.fpn.forward_flat([feats[i] for i in (1, 2, 3)])
        if prefix is not None:
            main.wait_event(join)
        pooled = ops.avgpool2_levels(pyr16, levels) if st["vision"] is not None else None  # flatten_fpn_features (:291-293)
        lang = self.language_backbone.body({"input_ids": ids, "attention_mask": st["am"], "text_prefix": prefix,
                                            "vision_inputs": {"vision": st["vision"], "images": pooled,
                                                              "vision_attention_mask": st["vmask"],
                                                              "batched_pos_category_map": None}})
        out = self.rpn.forward_flat(pyr16, levels, images.image_sizes, lang["hidden"], lang["masks"], positive_map, max_out,
                                    img_wh=img_wh)
        out["image_sizes"], out["levels"] = images.image_sizes, levels
        out["pyramid16"], out["lang_hidden"] = pyr16, lang["hidden"]  # inputs of the fusion tower (parity tests read them)
        out["vision_query_gates"] = lang["vision_query_gates"]
        return out

    # ---- many-category prompts: chunked evaluation (LVIS) --------------------------------------------------------------
    @torch.no_grad()
    def _chunk_state(self, captions, positive_map, dev):
        """Per-chunk prompt state (token ids, selected vision queries + token mask, class columns in ascending label order,
        the token masking tables of vision-only evaluation), cached by content like ``_prompt_state``."""
        bank_version = self.query_selector.bank_version if self.query_selector is not None else 0
        rate = self.text_mask_rate()

        def build():
            ids, am = self._tokenize(captions, dev)
            ids, am = ids[:1], am[:1]
            vision = vmask = None
            tab = dict(mask_rate=0.0)
            if self.query_selector is not None and self.query_selector.query_bank is not None:
                labels, all_map = self.get_labels_and_maps_from_positive_map(positive_map)
                vision, vmask, has = self.query_selector([labels], [all_map], None)
                vision, vmask = vision[0].float().contiguous(), vmask[0].float().contiguous()
                if rate > 0:
                    tab = self._mask_tables(ids.contiguous(), all_map, has, rate)
            cols, toks = chunk_columns(positive_map)
            return dict(ids=ids, am=am, vision=vision, vmask=vmask, cols=cols, toks=toks, **tab)

        return cached_chunk_state(self, prompt_key(captions, positive_map, 1, bank_version) + (rate,), build)

    CHUNK_GROUP_CAPACITY = 16      # chunk groups x batch sizes kept (LVIS at 8 chunks per pass: 4 per batch size); more when one
                                   # forward has more groups (``reserve_entries``)

    @torch.no_grad()
    def _chunk_group_state(self, sts, B, dev, key):
        """The prompt side of one pass of ``forward_chunked_device`` over elements e = chunk * B + image, a function of the chunk
        group and the batch size only, built once on the device and cached by (chunk keys, B): token ids and attention mask, the
        padded vision queries, GCP index and class tables of ``chunk_group_tables``, and the embeddings + BERT layers before the
        first GCP block (they read the token ids only), computed at the pass's own element count.  At 0 < TEXT_DROPOUT < 1 every
        forward masks other ids, so that path has no prefix.  ``key`` (``chunk_prompts.group_key``) carries the (data_ptr,
        _version) of the prefix's weights, so reloaded weights rebuild it; the forward makes room for all its groups before the
        first (``reserve_entries``), so nothing is evicted here."""
        cache = self.__dict__.setdefault("_chunk_group_cache", {})
        gs = cache.get(key)
        if gs is not None and self.cache_chunk_groups:
            return gs
        rate = sts[0]["mask_rate"]
        gs = dict(ids=per_element([st["ids_masked" if rate >= 1.0 else "ids"] for st in sts], B),
                  am=per_element([st["am"] for st in sts], B), prefix=None)
        if 0 < rate < 1.0:
            gs["tok_cat"] = per_element([st["tok_cat"] for st in sts], B)
            gs["n_cats"] = max(len(st["has"][0]) for st in sts)
        gs.update(chunk_group_tables(sts, B, dev))
        if not self.cache_chunk_groups:
            return gs
        if not 0 < rate < 1.0:
            gs["prefix"] = self.language_backbone.body.model.text_prefix(gs["ids"], gs["am"], output_hidden_states=False)
        cache[key] = gs
        return gs

    @torch.no_grad()
    def forward_chunked_device(self, images, chunk_captions, chunk_positive_maps, chunks_per_pass=8, chunk_ids=None, img_wh=None):
        """Chunked evaluation of a many-category vocabulary (LVIS: 1203 classes as 31 prompts of 40 classes,
        maskrcnn_benchmark/engine/inference.py:165-283,605-625).  The reference runs the WHOLE model once per chunk and
        concatenates the per-chunk detections; here Swin + FPN run ONCE per image and the chunks travel as extra batch
        elements (element e = chunk * B + image) through the language backbone, the fusion tower and the post-processing,
        ``chunks_per_pass`` chunks at a time.  Score columns of a chunk are its classes in ascending label order and carry
        their own label table (convert_grounding_to_od_logits_v2 semantics, rpn/inference.py:793-824).
        ``chunk_ids``: the subset of chunks THIS rank evaluates (text-column sharding over ranks), default all.
        ``img_wh``: optional fp32 [B, 2] device table of the images' (w, h); the clip then reads it instead of
        ``images.image_sizes``, so a captured graph serves any image sizes at its padded shape.
        Returns {"det_packed": [n_chunks_local, B, max_out + 1, 6] device tensor, "chunks": [chunk index ...], ...}."""
        from ..language_backbone import modeling_bert_new
        if self.training:
            raise NotImplementedError("training is SURVEY.md §8f")
        images = to_image_list(images, self.cfg.DATALOADER.SIZE_DIVISIBILITY)
        x = images.tensors
        if not x.is_cuda:
            raise MqdetError("GeneralizedVLRCNN_New: CUDA images required (no CPU fallback)")
        dev = x.device
        B = x.shape[0]
        chunk_ids = list(range(len(chunk_captions))) if chunk_ids is None else list(chunk_ids)
        feats = self.backbone.body.forward_flat(x)
        pyr16, levels = self.backbone.fpn.forward_flat([feats[i] for i in (1, 2, 3)])   # ONCE per image, shared by all chunks
        max_out = self.max_out()
        packed = torch.empty((len(chunk_ids), B, max_out + 1, 6), dtype=torch.float32, device=dev)
        pooled = None
        states = [self._chunk_state(chunk_captions[c], chunk_positive_maps[c], dev) for c in chunk_ids]
        rate = states[0]["mask_rate"] if states else 0.0
        if rate > 0:   # vision-only evaluation: the draws of the reference's forwards
            flags = self.draw_chunk_text_masks(states, B, rate)
        wkey = self.language_backbone.body.model.prefix_weights_key()
        keys = [group_key(states[p0:p0 + chunks_per_pass], B, wkey) for p0 in range(0, len(chunk_ids), chunks_per_pass)]
        reserve_entries(self.__dict__.setdefault("_chunk_group_cache", {}), keys, self.CHUNK_GROUP_CAPACITY)
        groups = []
        for p0, key in zip(range(0, len(chunk_ids), chunks_per_pass), keys):
            sts = states[p0:p0 + chunks_per_pass]
            G = len(sts)
            gs = self._chunk_group_state(sts, B, dev, key)
            groups.append(gs)
            ids = gs["ids"]
            if 0 < rate < 1.0:
                C = gs["n_cats"]
                fl = torch.tensor([flags[b][p0 + g] + [0] * (C - len(flags[b][p0 + g])) for g in range(G) for b in range(B)],
                                  dtype=torch.uint8)
                ids = ops.mask_prompt_tokens(ids, gs["tok_cat"], ops.upload_async(fl, dev), self.mask_token_id())
            if gs["vision"] is not None:
                modeling_bert_new.use_sparse_index(gs["vmask"], gs["vidx"])
                if pooled is None:
                    pooled = ops.avgpool2_levels(pyr16, levels)
            lang = self.language_backbone.body({"input_ids": ids, "attention_mask": gs["am"], "text_prefix": gs["prefix"],
                                                "vision_inputs": {"vision": gs["vision"],
                                                                  "images": pooled.repeat(G, 1, 1) if gs["vision"] is not None else None,
                                                                  "vision_attention_mask": gs["vmask"],
                                                                  "batched_pos_category_map": None}})
            out = self.rpn.forward_flat(pyr16.repeat(G, 1, 1), levels, images.image_sizes, lang["hidden"], lang["masks"],
                                        None, max_out, tokmap=gs["tokmap"], class_labels=gs["class_labels"], img_wh=img_wh)
            packed[p0:p0 + G] = out["det_packed"].view(G, B, max_out + 1, 6)
        self._chunk_read = dict(states=states, groups=groups, B=B)
        return {"det_packed": packed, "chunks": chunk_ids, "image_sizes": images.image_sizes, "pyramid16": pyr16}

    def forward_chunked(self, images, chunk_captions, chunk_positive_maps, chunks_per_pass=8):
        """-> list[BoxList]: per image, the per-chunk detections concatenated (``BoxList.concate_box_list``,
        structures/bounding_box.py:273-285; engine/inference.py:704-706), chunk order preserved."""
        out = self.forward_chunked_device(images, chunk_captions, chunk_positive_maps, chunks_per_pass)
        pk = out["det_packed"].cpu()
        return boxlists_from_packed(pk.transpose(0, 1).reshape(pk.shape[1], -1, 6), out["image_sizes"], pk.shape[0])

    def forward(self, images, targets=None, captions=None, positive_map=None, greenlight_map=None,
                return_backbone_features=False):
        """Reference signature (:307-314), eval: returns list[BoxList] (fields ``labels``, ``scores``; mode xyxy)."""
        out = self.forward_device(images, captions, positive_map)
        return boxlists_from_packed(out["det_packed"], out["image_sizes"])
