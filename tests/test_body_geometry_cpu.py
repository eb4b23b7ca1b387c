"""CPU: the limit ladder and the chunk-edge bodies of tests/body_geometry_cases.py through the host build of body_fast.cuh
(phases run thread by thread), against the sequential machine and the oracle.  The device runs the same bodies in
tests/test_body_geometry_gpu.py; here a change to the kernel source that moves a limit, or breaks an edge, shows up without a GPU."""
import collections

import pytest

import body_geometry_cases as G
import host_machine as hm
from llmapigateway_b200 import rewrite as rw


@pytest.fixture(scope="module")
def tables():
    return G.plan_tables()


def _run(raw, table, pi, mode, ops, tally):
    """fast path (when it does not hand the body back) == sequential machine == oracle; tally["fast"] counts the fast answers"""
    plans, o, blob = table.packed()
    fst, fout, fneed = hm.rewrite_body_fast(raw, plans, o, blob, pi, cap=1 << 17)
    st, out, need = hm.rewrite_body(raw, plans, o, blob, pi, cap=1 << 17)
    if fst != G.FAST_IRREGULAR:
        assert (fst, fout, fneed) == (st, out if st == rw.BODY_OK else b"", need), (raw[:120], mode)
        tally["fast"] += 1
    else:
        tally["irregular"] += 1
    G.check_against_reference(raw, st, out, ops, mode, tally)
    return fst != G.FAST_IRREGULAR


def test_limit_ladder_host(tables):
    """every ladder body under every plan of both tables; the fast path switches to the exact machine exactly at each limit"""
    t028 = tables["httpx028"]
    pi0 = t028.plan_index("gw/chain", 0, stream=True)
    ladder = G.ladder_bodies()
    tally = collections.Counter()
    for name, raw, fast, exotic in ladder:
        if fast is not None:
            assert G.is_fast(raw, t028.packed(), pi0) == fast, name
        for table in tables.values():
            for pi, mode, ops in G.plan_variants(table):
                n_exotic = tally["exotic"]
                _run(raw, table, pi, mode, ops, tally)
                if exotic is not None:
                    assert (tally["exotic"] > n_exotic) == exotic, (name, mode)
    assert tally["fast"] >= 1500 and tally["irregular"] >= 600, tally


@pytest.mark.parametrize("n", G.CHUNK_LENGTHS)
def test_chunk_edges_host(tables, n):
    """every hard piece at every offset around several per-thread chunk edges, in the three render modes (attempts rotate).
    Where a piece sits must not change whether the data-parallel path takes the body: a chunk-start state that goes wrong at an
    edge (an escape carried in, a UTF-8 sequence continued) shows up as a body handed back at some offsets only."""
    modes = G.mode_plans(tables)
    tally = {k: collections.Counter() for k in ("str", "bad", "struct")}
    decided = collections.defaultdict(set)
    for i, ((kind, name), raw) in enumerate(G.chunk_edge_bodies([n])):
        for per_att in modes:
            table, pi, mode, ops = per_att[i % len(per_att)]
            decided[(name, mode)].add(_run(raw, table, pi, mode, ops, tally[kind]))
    bad, good = tally["bad"], tally["str"] + tally["struct"]
    assert bad["fast"] == 0 and bad[rw.BODY_PARSE_ERROR] == bad["irregular"], bad          # invalid UTF-8 is never the fast path's
    assert good["fast"] >= 0.85 * (good["fast"] + good["irregular"]) and good["exotic"] == 0, good
    assert tally["struct"]["fast"] >= 0.95 * (tally["struct"]["fast"] + tally["struct"]["irregular"]), tally["struct"]
    assert not [k for k, v in decided.items() if len(v) > 1], [k for k, v in decided.items() if len(v) > 1]
