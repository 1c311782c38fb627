"""CPU: the host side of ``ChunkedEngine`` — the per-image concatenation of the packed chunk rows (what ``forward_chunked`` and the
reference's ``concate_box_list`` return), the decoding of single-prompt results, the per-pass tables of a chunk group
(tests/hostlogic/chunk_tables_case.py) and the refusals made before anything touches a device."""
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

from util import ROOT


def _packed(counts, rows=5, seed=0):
    """[B, n_chunks * rows, 6] with counts[b][c] valid rows in chunk c of image b, junk after them, the count in the last row."""
    g = torch.Generator().manual_seed(seed)
    B, n = len(counts), len(counts[0])
    pk = torch.rand((B, n, rows, 6), generator=g) * 100
    for b in range(B):
        for c in range(n):
            pk[b, c, rows - 1] = 0
            pk[b, c, rows - 1, 0] = counts[b][c]
            pk[b, c, :, 5] = torch.arange(rows, dtype=torch.float32) + 10 * c + 1
    return pk.view(B, n * rows, 6)


def test_boxlists_from_packed_concatenates_in_chunk_order():
    from mqdet_b200.structures.bounding_box import boxlists_from_packed
    counts = [[2, 0, 4], [0, 0, 1]]
    pk = _packed(counts)
    sizes = [(120, 200), (90, 64)]
    res = boxlists_from_packed(pk, sizes, 3)
    full = pk.view(2, 3, 5, 6)
    for b, bl in enumerate(res):
        want = torch.cat([full[b, c, :counts[b][c]] for c in range(3)])
        assert bl.size == (sizes[b][1], sizes[b][0]) and bl.mode == "xyxy" and len(bl) == sum(counts[b])
        assert torch.equal(bl.bbox, want[:, :4]) and torch.equal(bl.get_field("scores"), want[:, 4])
        assert torch.equal(bl.get_field("labels"), want[:, 5].long())
    assert res[0].get_field("labels").tolist() == [1, 2, 21, 22, 23, 24]


@pytest.mark.parametrize("rows", [5, 101], ids=["one_chunk", "gdino_num_queries_plus_one"])
def test_boxlists_from_packed_one_chunk(rows):
    """A single-prompt result [B, rows, 6], MQ-GLIP's max_out + 1 or MQ-GroundingDINO's num_queries + 1 rows: each image's first
    count rows, fields labels then scores, each a copy rather than a view of the (reused) packed buffer."""
    from mqdet_b200.structures.bounding_box import boxlists_from_packed
    counts = [[3], [0], [rows - 1]]
    pk = _packed(counts, rows=rows, seed=1)
    sizes = [(120, 200), (90, 64), (33, 47)]
    res = boxlists_from_packed(pk, sizes)
    for b, bl in enumerate(res):
        n = counts[b][0]
        assert bl.size == (sizes[b][1], sizes[b][0]) and bl.mode == "xyxy" and len(bl) == n
        assert bl.fields() == ["labels", "scores"]
        assert torch.equal(bl.bbox, pk[b, :n, :4]) and torch.equal(bl.get_field("scores"), pk[b, :n, 4])
        assert torch.equal(bl.get_field("labels"), pk[b, :n, 5].long())
    kept = [bl.bbox.clone() for bl in res]
    pk.zero_()
    assert all(torch.equal(bl.bbox, k) for bl, k in zip(res, kept))


def test_boxlists_from_packed_refuses_an_overfull_result():
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.structures.bounding_box import boxlists_from_packed
    with pytest.raises(MqdetError, match="chunk 1: 5 detections exceed the 4-row"):
        boxlists_from_packed(_packed([[1, 5]]), [(10, 10)], 2)
    with pytest.raises(MqdetError, match="image 1: 5 detections exceed the 4-row"):
        boxlists_from_packed(_packed([[1], [5]]), [(10, 10), (10, 10)])


def test_chunk_group_tables_host_logic():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostlogic", "chunk_tables_case.py")], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PASS chunk_tables" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])


class _Stub(torch.nn.Module):
    """Stands in for a detector: the refusals come before any use of the model's device or forward."""

    def __init__(self, rate=0.0, cached=True):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.rate = rate
        self.cache_chunk_groups = cached

    def text_mask_rate(self):
        return self.rate

    def forward_chunked_device(self, *a, **k):
        raise AssertionError("not reached")


def test_refuses_partial_text_dropout():
    from mqdet_b200.engine.inference import ChunkedEngine
    with pytest.raises(NotImplementedError, match="TEXT_DROPOUT < 1"):
        ChunkedEngine(_Stub(0.5), [{}], [{1: [1]}])


def test_refuses_a_model_without_a_chunked_forward():
    from mqdet_b200.engine.inference import ChunkedEngine
    with pytest.raises(TypeError, match="forward_chunked_device"):
        ChunkedEngine(torch.nn.Linear(1, 1), [{}], [{1: [1]}])


def test_refuses_a_multi_gpu_world(monkeypatch):
    from mqdet_b200.engine.inference import ChunkedEngine
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda *a, **k: 2)
    with pytest.raises(NotImplementedError, match="one GPU"):
        ChunkedEngine(_Stub(), [{}], [{1: [1]}])


def test_refuses_mismatched_chunks_and_a_cpu_model():
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.engine.inference import ChunkedEngine
    with pytest.raises(ValueError, match="one positive map per chunk"):
        ChunkedEngine(_Stub(), [{}, {}], [{1: [1]}])
    with pytest.raises(ValueError, match="chunks_per_pass"):
        ChunkedEngine(_Stub(), [{}], [{1: [1]}], chunks_per_pass=0)
    with pytest.raises(MqdetError, match="CUDA device"):
        ChunkedEngine(_Stub(), [{}], [{1: [1]}])


def test_refuses_a_model_that_rebuilds_its_chunk_groups():
    from mqdet_b200.engine.inference import ChunkedEngine
    with pytest.raises(NotImplementedError, match="cache_chunk_groups"):
        ChunkedEngine(_Stub(cached=False), [{}], [{1: [1]}])


def test_reserve_entries_evicts_only_before_a_forward():
    from mqdet_b200.utils import reserve_entries
    cache = {k: k for k in "abc"}
    reserve_entries(cache, ["a", "b"], 3)                 # all present: nothing built, nothing dropped
    assert set(cache) == set("abc")
    reserve_entries(cache, ["a", "d"], 3)                 # one missing, no room: cleared before the forward builds
    assert cache == {}
    cache.update({k: k for k in "uvwxyz"})                # one forward's 6 groups above a capacity of 3
    reserve_entries(cache, list("uvwxyz"), 3)
    assert set(cache) == set("uvwxyz")
