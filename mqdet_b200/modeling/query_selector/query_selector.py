"""Vision-query selection (host-side gather, no arithmetic).

Drop-in for maskrcnn_benchmark/modeling/query_selector/query_selector.py:8-116: picks <= NUM_QUERY_PER_CLASS rows of
the query bank ``{label: FloatTensor[n, n_scales, C]}`` per class, flattens scales, expands the class's token-location
row to each query, pads over the batch and binarises the mask.
"""
import os
import random
from collections import defaultdict

import numpy as np
import torch
from torch import nn
from torch.nn.utils.rnn import pad_sequence


class QuerySelector(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.device = torch.device(cfg.MODEL.DEVICE)
        path = cfg.VISION_QUERY.QUERY_BANK_PATH
        if path and os.path.exists(path):
            self.query_bank = torch.load(path, map_location=self.device)
        else:
            assert path == "", "query bank path {} not exists".format(path)
            self.query_bank = None
        if cfg.VISION_QUERY.LEARNABLE_BANK or cfg.VISION_QUERY.ADD_VISION_LAYER:
            raise NotImplementedError("LEARNABLE_BANK / ADD_VISION_LAYER are off in every shipped MQ config")
        self.pure_text_rate = cfg.VISION_QUERY.PURE_TEXT_RATE
        self.num_query_per_class = cfg.VISION_QUERY.NUM_QUERY_PER_CLASS
        self.cfg = cfg
        self.bank_version = 0  # bumped whenever the bank changes: per-prompt caches of the detector key on it

    def load_query_bank(self, bank_path):
        self.query_bank = torch.load(bank_path, map_location=self.device)
        self.bank_version += 1

    def set_query_bank(self, bank):
        """In-memory bank {label: tensor[n, scales, C]} (no file on disk).  A ``defaultdict(list)`` stays one, as ``torch.load`` of
        the reference's saved banks keeps it: a label without exemplars reads as ``[]``."""
        q = defaultdict(list) if isinstance(bank, defaultdict) else {}
        for k, v in bank.items():
            q[k] = v.to(self.device) if torch.is_tensor(v) else v
        self.query_bank = q
        self.bank_version += 1

    def _pick(self, label):
        """Rows of the class's bank entry to use (the reference's sampler, same RNG calls in the same order)."""
        cand = self.query_bank[label]
        k = self.num_query_per_class
        if self.cfg.VISION_QUERY.RANDOM_KSHOT and self.training:
            k = np.random.choice(range(1, k + 1))
        nq = min(len(cand), k)
        if (random.random() < self.pure_text_rate) and self.training:
            nq = 0
        rows = np.random.choice(len(cand), nq, replace=False).tolist()
        return cand, (rows if self.training else sorted(rows))

    def forward(self, batched_label_list, batched_location_map, batched_pos_labels=None):
        """-> (queries [B, Q, C], masks [B, Q, T] in {0,1}, per-image has-query flags); (None,)*3 without a bank."""
        if self.query_bank is None:
            return None, None, None
        per_q, per_m, per_has = [], [], []
        for b, (labels, loc_maps) in enumerate(zip(batched_label_list, batched_location_map)):
            feats, rows_of_mask, has = [], [], []
            for label, loc_map in zip(labels, loc_maps):
                cand, rows = self._pick(label)
                if isinstance(cand, list):  # class without exemplars
                    assert not rows
                else:
                    q = cand[rows]  # [nq, scales, C]
                    feats.append(q.reshape(-1, q.shape[-1]))
                    rows_of_mask.append(loc_map.to(self.device)[None].expand(q.shape[0] * q.shape[1], -1))
                if batched_pos_labels is None or label in batched_pos_labels[b]:
                    has.append(int(len(rows) > 0))
            per_q.append(torch.cat(feats))
            per_m.append(torch.cat(rows_of_mask))
            per_has.append(has)
        masks = pad_sequence(per_m, batch_first=True)
        return pad_sequence(per_q, batch_first=True), (masks != 0).to(masks.dtype), per_has
