def reserve_entries(cache, keys, capacity):
    """Make room in a bounded cache for the entries one forward is about to read (``keys``), before it reads any of them:
    the cache is cleared when the missing ones would not fit, and it may then grow to ``len(keys)`` even above ``capacity``.
    So a forward never evicts an entry it built itself, and a forward whose entries are all cached builds nothing, which
    is what a CUDA-graph capture of it needs (building can read the host or upload from temporary pinned memory)."""
    missing = sum(1 for k in set(keys) if k not in cache)
    if missing and len(cache) + missing > max(int(capacity), len(set(keys))):
        cache.clear()
