"""Host-logic dry run of the per-pass tables of a chunk group (``mqdet_b200.modeling.chunk_prompts``), which MQ-GLIP's
``_chunk_group_state`` and MQ-GroundingDINO's ``_chunk_text_state`` both build (CPU, throw-away process: the ops double stands in
for ``ops.gcp_build_index``).  Chunks with different vision-query counts, class counts and token-list lengths: the zero padding of
the queries and their mask to the group's largest count, the GCP index of that mask, the class columns in ascending label order
with their -1-padded token lists, and element e = chunk * B + image throughout; a chunk with an empty positive map gets one column
without tokens.

    python tests/hostlogic/chunk_tables_case.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_double  # noqa: F401,E402  (patches mqdet_b200.ops; must come first)
import torch  # noqa: E402

from mqdet_b200.modeling import chunk_prompts as cp  # noqa: E402

CPU = torch.device("cpu")


def state(pmap, V, T, D, g):
    """A chunk state as the detectors' ``_chunk_state`` makes it: vision queries [V, D] and their 0/1 token mask [V, T] (None
    without a bank), the class columns and token lists."""
    cols, toks = cp.chunk_columns(pmap)
    st = dict(cols=cols, toks=toks, vision=None, vmask=None)
    if V is not None:
        st["vision"] = torch.randn(V, D, generator=g)
        st["vmask"] = (torch.rand(V, T, generator=g) < 0.3).float()
    return st


def check(states, B, T):
    tabs = cp.chunk_group_tables(states, B, CPU)
    G = len(states)
    Cmax = max([len(st["cols"]) for st in states] + [1])
    mt = max([len(t) for st in states for t in st["toks"]] + [1])
    assert tabs["tokmap"].shape == (G * B, Cmax, mt) and tabs["tokmap"].dtype == torch.int32
    assert tabs["class_labels"].shape == (G * B, Cmax) and tabs["class_labels"].dtype == torch.int32
    if states[0]["vision"] is not None:
        Vmax = max(st["vision"].shape[0] for st in states)
        D = states[0]["vision"].shape[1]
        assert tabs["vision"].shape == (G * B, Vmax, D) and tabs["vmask"].shape == (G * B, Vmax, T)
        S = max(int(tabs["vmask"][e].sum(0).max()) for e in range(G * B))
        assert tabs["vidx"].shape == (G * B, T, S)
    else:
        assert tabs["vision"] is None and tabs["vmask"] is None and tabs["vidx"] is None
    for g, st in enumerate(states):
        for b in range(B):
            e = g * B + b
            for j in range(Cmax):
                label, toks = (st["cols"][j], st["toks"][j]) if j < len(st["cols"]) else (0, [])
                assert int(tabs["class_labels"][e, j]) == label, (g, b, j)
                assert tabs["tokmap"][e, j].tolist() == toks + [-1] * (mt - len(toks)), (g, b, j)
            if st["vision"] is None:
                continue
            V = st["vision"].shape[0]
            assert torch.equal(tabs["vision"][e, :V], st["vision"]) and not tabs["vision"][e, V:].any()
            assert torch.equal(tabs["vmask"][e, :V], st["vmask"]) and not tabs["vmask"][e, V:].any()
            for t in range(T):
                q = st["vmask"][:, t].nonzero().flatten().tolist()     # ascending query indices, padded with Vmax
                assert tabs["vidx"][e, t].tolist() == q + [Vmax] * (S - len(q)), (g, b, t)
    return tabs


def main():
    g = torch.Generator().manual_seed(5)
    T, D, B = 16, 8, 3
    pmaps = [{7: [1, 2], 3: [4]}, {12: 9}, {11: [2, 5, 6, 13], 9: [8], 10: [1, 3]}]
    assert cp.chunk_columns(pmaps[2]) == ([9, 10, 11], [[8], [1, 3], [2, 5, 6, 13]])
    assert cp.chunk_columns(pmaps[1]) == ([12], [[9]])
    # with vision queries: 4, 1 and 6 per chunk
    check([state(pm, V, T, D, g) for pm, V in zip(pmaps, (4, 1, 6))], B, T)
    # without: an empty positive map alone in its pass, and next to other chunks
    tabs = check([state({}, None, T, D, g)], B, T)
    assert tabs["tokmap"].shape == (B, 1, 1) and (tabs["tokmap"] == -1).all() and not tabs["class_labels"].any()
    check([state(pmaps[0], None, T, D, g), state({}, None, T, D, g), state(pmaps[2], None, T, D, g)], 2, T)
    # per_element: one [1, ...] tensor per chunk -> element e = chunk * B + image
    a, b = torch.tensor([[1, 2]]), torch.tensor([[3, 4]])
    assert cp.per_element([a, b], 2).tolist() == [[1, 2], [1, 2], [3, 4], [3, 4]]
    print("PASS chunk_tables")


if __name__ == "__main__":
    main()
