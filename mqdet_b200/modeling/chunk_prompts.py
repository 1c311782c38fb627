"""The prompt bookkeeping that MQ-GLIP (``GeneralizedVLRCNN_New``) and MQ-GroundingDINO share: the content key of a prompt, and for
chunked evaluation of a many-category vocabulary (LVIS) the per-chunk state cache and the per-pass tables of a chunk group, whose
elements are e = chunk * B + image.  Each detector keeps what differs: its tokenisation, its text masks and its BERT prefix."""
import torch

from .. import ops

CHUNK_STATE_CAPACITY = 4096    # distinct chunk prompts kept per model (LVIS: 31)


def prompt_key(captions, positive_map, B, bank_version):
    """Content key of a prompt: token ids / caption strings, the positive map's entries, batch size and the query bank version — an
    in-place edit of ``positive_map`` or a swapped bank is a different prompt."""
    if isinstance(captions, dict):
        ids = captions["input_ids"]
        am = captions["attention_mask"]
        if ids.is_cuda:  # no device->host sync on the hot path: storage identity + version counters
            ck = (tuple(ids.shape), ids.data_ptr(), ids._version, am.data_ptr(), am._version)
        else:
            ck = (tuple(ids.shape), ids.detach().numpy().tobytes(), am.detach().numpy().tobytes())
    else:
        ck = tuple(captions) if isinstance(captions, (list, tuple)) else captions
    pk = tuple((int(k), tuple(int(t) for t in (v if not isinstance(v, int) else [v]))) for k, v in sorted(positive_map.items()))
    return (ck, pk, int(B), int(bank_version))


def cached_chunk_state(model, key, build):
    """The state of one chunk prompt from ``model._chunk_cache``; on a miss ``build()`` makes its dict, stored with ``key``.  The
    cache is cleared when it holds CHUNK_STATE_CAPACITY chunks."""
    cache = model.__dict__.setdefault("_chunk_cache", {})
    st = cache.get(key)
    if st is None:
        if len(cache) >= CHUNK_STATE_CAPACITY:
            cache.clear()
        st = cache[key] = dict(key=key, **build())
    return st


def chunk_columns(positive_map):
    """A chunk's score columns: its classes in ascending label order (``cols``) and each one's token list (``toks``)."""
    cols = sorted(int(k) for k in positive_map)
    return cols, [([positive_map[c]] if isinstance(positive_map[c], int) else list(positive_map[c])) for c in cols]


def group_key(states, B, wkey):
    """Cache key of a chunk group's per-pass state: its chunks, the batch size and the BERT prefix weights' key."""
    return (tuple(st["key"] for st in states), int(B), wkey)


def per_element(tensors, B):
    """One [1, ...] tensor per chunk -> [G * B, ...], element e = chunk * B + image."""
    return torch.cat(tensors).repeat_interleave(B, dim=0).contiguous()


def chunk_group_tables(states, B, dev):
    """The per-element tables of one pass over the chunks of ``states`` (each with ``vision`` [V, D] / ``vmask`` [V, T] or None,
    ``cols``, ``toks``): the vision queries and their token mask zero-padded to the group's largest query count (the pad_sequence
    padding of QuerySelector.forward, query_selector.py:112-116) with the GCP index of that mask (``vidx``), the token map int32
    [G * B, C, max_tok] (-1 padded) and the class labels int32 [G * B, C] of the score columns, C the group's largest class count
    and at least 1: a chunk with an empty positive map has one column without tokens, so it scores nothing and detects nothing."""
    from .language_backbone import modeling_bert_new
    G = len(states)
    tabs = dict(vision=None, vmask=None, vidx=None)
    if states[0]["vision"] is not None:
        Vmax = max(st["vision"].shape[0] for st in states)
        vision = torch.zeros((G, Vmax, states[0]["vision"].shape[1]), dtype=torch.float32, device=dev)
        vmask = torch.zeros((G, Vmax, states[0]["vmask"].shape[1]), dtype=torch.float32, device=dev)
        for g, st in enumerate(states):
            vision[g, :st["vision"].shape[0]] = st["vision"]
            vmask[g, :st["vmask"].shape[0]] = st["vmask"]
        tabs["vision"] = vision.repeat_interleave(B, dim=0).contiguous()
        tabs["vmask"] = vmask.repeat_interleave(B, dim=0).contiguous()
        tabs["vidx"] = modeling_bert_new.sparse_index(tabs["vmask"])
    Cmax = max(max(len(st["cols"]) for st in states), 1)
    mt = max(max((len(t) for t in st["toks"]), default=1) for st in states)
    tok_h = torch.full((G, Cmax, mt), -1, dtype=torch.int32)
    lab_h = torch.zeros((G, Cmax), dtype=torch.int32)
    for g, st in enumerate(states):
        for j, (c, tk) in enumerate(zip(st["cols"], st["toks"])):
            tok_h[g, j, :len(tk)] = torch.tensor(tk, dtype=torch.int32)
            lab_h[g, j] = c
    tabs["tokmap"] = ops.upload_async(tok_h, dev).repeat_interleave(B, dim=0).contiguous()
    tabs["class_labels"] = ops.upload_async(lab_h, dev).repeat_interleave(B, dim=0).contiguous()
    return tabs
