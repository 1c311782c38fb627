"""Language backbone wrapper, drop-in for maskrcnn_benchmark/modeling/language_backbone/bert_model_new.py:13-104.

``BertEncoder(cfg).forward({"input_ids", "attention_mask", "vision_inputs"})`` ->
``{"aggregate", "embedded", "masks", "hidden", "vision_query_gates"}`` (N_LAYERS == 1, dot-product token loss layout).
No checkpoint download: ``from_pretrained`` needs the network; weights come from ``load_state_dict``.
"""
from types import SimpleNamespace

import torch
from torch import nn

from .modeling_bert_new import QVBertModel


def bert_base_config():
    """bert-base-uncased dimensions (what BertConfig.from_pretrained('bert-base-uncased') returns)."""
    return SimpleNamespace(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                           intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12,
                           pad_token_id=0)


class BertEncoder(nn.Module):
    def __init__(self, cfg, config=None):
        super().__init__()
        self.cfg = cfg
        config = config or bert_base_config()
        self.model = QVBertModel(config, dim_t=config.hidden_size, dim_v=cfg.MODEL.BACKBONE.OUT_CHANNELS,
                                 share_kv=cfg.VISION_QUERY.SHARE_KV, cfg=cfg)
        self.language_dim = config.hidden_size
        self.num_layers = cfg.MODEL.LANGUAGE_BACKBONE.N_LAYERS
        if self.num_layers != 1:
            raise NotImplementedError("LANGUAGE_BACKBONE.N_LAYERS == 1 in every MQ config")

    @torch.no_grad()
    def forward(self, x):
        ids, mask, vi = x["input_ids"], x["attention_mask"], x["vision_inputs"]
        # only the last hidden state is read, so a cached prompt prefix needs no per-layer states
        out = self.model(input_ids=ids, attention_mask=mask, output_hidden_states=False, vision=vi["vision"],
                         images=vi["images"], vision_attention_mask=vi["vision_attention_mask"],
                         batched_pos_category_map=vi.get("batched_pos_category_map"), text_prefix=x.get("text_prefix"))
        hidden = out.last_hidden_state
        # features = mean of the last N_LAYERS(=1) states / 1; embedded/aggregate are unused by the MHA-B fusion path
        # (bert_model_new.py:61-69) but part of the returned dict — a masked row-scale and a masked mean.
        m = mask.unsqueeze(-1).float()
        embedded = hidden * m
        ret = {"aggregate": embedded.sum(1) / mask.sum(-1).unsqueeze(-1).float(), "embedded": embedded, "masks": mask,
               "hidden": hidden, "vision_query_gates": out.vision_query_gates}
        if self.cfg.VISION_QUERY.QUERY_FUSION:
            ret["augmented_vision"] = out.augmented_vision
            ret["vision_attention_mask"] = out.vision_attention_mask
        return ret
