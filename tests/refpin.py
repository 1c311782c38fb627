"""Results of the original project's own code that the pinning tests compare the oracle against.

Where the original sources are present (``oracle.ref_loader.available()``) a test runs them and compares against the live result;
with ``MQDET_RECORD_PINS=1`` it also stores that result under <name> in ``tests/golden/pins.pt``.  Elsewhere the test compares
against the stored result, so the comparison runs on every machine.  Stored tensors above ``FULL`` elements keep a fixed seeded sample of
``SAMPLE`` elements plus the max |value| of the whole tensor, so that tolerance bounds relative to max |ref| stay the same; the
helpers below compare a full tensor against either form."""
import os

import torch

from oracle import ref_loader

PIN_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pins.pt")
FULL = 1024
SAMPLE = 256
_store = None


class Sampled:
    """A stored sample of a larger tensor: flat indices, values, the full tensor's shape and max |finite value|."""

    def __init__(self, d):
        self.idx, self.val, self.shape, self.absmax = d["idx"].long(), d["val"], tuple(d["shape"]), float(d["absmax"])


def _absmax(v):
    """max |finite value| of a floating tensor (0 for other dtypes and empty tensors)"""
    if not v.is_floating_point():
        return 0.0
    fin = v[torch.isfinite(v)]
    return fin.abs().max().item() if fin.numel() else 0.0


def _shrink(v, full=False):
    if isinstance(v, torch.Tensor):
        v = v.detach().cpu()
        if full or v.numel() <= FULL:
            return v.clone()
        g = torch.Generator().manual_seed(v.numel())
        idx = torch.randperm(v.numel(), generator=g)[:SAMPLE].sort().values
        absmax = _absmax(v)
        return {"__sampled__": True, "idx": idx.int(), "val": v.reshape(-1)[idx].clone(), "shape": list(v.shape), "absmax": absmax}
    if isinstance(v, dict):
        return {k: _shrink(x, full) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return type(v)(_shrink(x, full) for x in v)
    return v


def _expand(v):
    if isinstance(v, dict):
        if v.get("__sampled__"):
            return Sampled(v)
        return {k: _expand(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return type(v)(_expand(x) for x in v)
    return v


def pinned(name, fn, full=False, live=None):
    """fn() where the original sources are present (`live`, default: ``ref_loader.available()``; stored when MQDET_RECORD_PINS=1,
    whole tensors with `full`), else the stored result of fn()."""
    global _store
    if _store is None:
        _store = torch.load(PIN_FILE, weights_only=True) if os.path.exists(PIN_FILE) else {}
    if ref_loader.available() if live is None else live:
        val = fn()
        if os.environ.get("MQDET_RECORD_PINS") == "1":
            _store[name] = _shrink(val, full)
            torch.save(_store, PIN_FILE)
        return val
    assert name in _store, f"{name}: no recorded result in {PIN_FILE}"
    return _expand(_store[name])


def align(got, want):
    """(got values, want values, max |want|) over what `want` holds: the whole tensor, or the stored sample of it."""
    got = got.detach().cpu()
    if isinstance(want, Sampled):
        assert tuple(got.shape) == want.shape, (tuple(got.shape), want.shape)
        return got.reshape(-1)[want.idx], want.val, want.absmax
    want = want.detach().cpu()
    assert got.shape == want.shape, (tuple(got.shape), tuple(want.shape))
    return got, want, _absmax(want)


def max_err(got, want):
    a, b, bmax = align(got, want)
    return (a.double() - b.double()).abs().max().item(), bmax


def equal(got, want):
    a, b, _ = align(got, want)
    return torch.equal(a, b)
