"""The request-body rewrite (k_body_fast -> k_body_rewrite -> k_body_offsets -> k_body_pack, csrc/body_kernels.cuh) and the
document kernels that share its staging buffers (k_docs_usage, k_docs_error_detail, k_body_scan) at production geometry.

Every body is checked three ways: against the oracle (the reference's json.loads + key assignments + encoder), against the exact
machine alone (engine mode 1: status, length, bytes, matched keys and root kind identical), and -- through the host build of the
same kernel source -- for whether the data-parallel path took it, so that each case family proves it exercised that path.
Families: the limit ladder and the per-thread chunk edges of tests/body_geometry_cases.py; production batches of 1 024 to 16 384
bodies (config-2 bodies, chat bodies with non-ASCII text, 8 - 64 KiB bodies, damaged and empty ones) with the irregular bodies
first, last, interleaved, alone and absent; packed output around k_body_offsets' blocks of 1 024 and k_body_pack's unaligned
slots; the device entry point; one warm engine whose grow-only buffers serve calls of every kind and size; the scan's model cap;
documents on both sides of the 6 144-byte stage and past one grid-stride lap."""
from __future__ import annotations

import collections
import ctypes as C
import json
import random

import numpy as np
import pytest

import body_cases as bc
import body_geometry_cases as G
from golden_io import canon_rows
from llmapigateway_b200 import rewrite as rw
from llmapigateway_b200.synth import chat_bodies
from oracle import body_oracle as bo

pytestmark = pytest.mark.gpu


def new_engine():
    import llmapigateway_b200 as L
    return L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)


@pytest.fixture(scope="module")
def warm():
    e = new_engine()
    yield e
    e.close_engine()


@pytest.fixture
def engine(request, warm):
    """"warm": the module's engine (buffers grown by every earlier test); "cold": a fresh one"""
    if request.param == "warm":
        yield warm
        return
    e = new_engine()
    yield e
    e.close_engine()


@pytest.fixture(scope="module")
def tables():
    return G.plan_tables()


def both_modes(engine, bodies, pis, slot_cap=None):
    """mode 0 (data-parallel path + exact machine for the rest) must equal mode 1 (exact machine only) on every body"""
    try:
        engine.set_mode(1)
        exact = engine.rewrite_bodies(bodies, pis, slot_cap=slot_cap, with_matched=True)
        engine.set_mode(0)
        fast = engine.rewrite_bodies(bodies, pis, slot_cap=slot_cap, with_matched=True)
    finally:
        engine.set_mode(0)
    diff = [i for i in range(len(bodies)) if fast[i] != exact[i]]
    assert not diff, (len(diff), bodies[diff[0]][:200], fast[diff[0]][0], exact[diff[0]][0])
    return fast


def run_checked(engine, table, items, tally):
    """items: [(body, plan index, mode name, ops)] -> engine results, each checked against the oracle and mode 1"""
    engine.load_rules(table)
    got = both_modes(engine, [it[0] for it in items], [it[1] for it in items])
    packed = table.packed()
    for (raw, pi, mode, ops), (st, out, _, _) in zip(items, got):
        G.check_against_reference(raw, st, out, ops, mode, tally)
        tally["fast" if G.is_fast(raw, packed, pi) else "irregular"] += 1
    return got


# ---- 1. limit ladder -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("engine", ["cold", "warm"], indirect=True)
def test_limit_ladder(engine, tables):
    ladder = G.ladder_bodies()
    tally = collections.Counter()
    for table in tables.values():
        items, names = [], []
        for name, raw, fast, exotic in ladder:
            for pi, mode, ops in G.plan_variants(table):
                items.append((raw, pi, mode, ops))
                names.append((name, exotic))
        got = run_checked(engine, table, items, tally)
        for (name, exotic), (st, _, _, _) in zip(names, got):
            if exotic is not None:
                assert (st == rw.BODY_EXOTIC) == exotic, name
    t028 = tables["httpx028"]
    pi0 = t028.plan_index("gw/chain", 0, stream=True)
    for name, raw, fast, _ in ladder:
        if fast is not None:
            assert G.is_fast(raw, t028.packed(), pi0) == fast, name
    assert tally["fast"] >= 1500 and tally["irregular"] >= 600, tally


# ---- 2. chunk edges ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", G.CHUNK_LENGTHS)
def test_chunk_edges(warm, tables, n):
    bodies = G.chunk_edge_bodies([n])
    modes = G.mode_plans(tables)
    tally = {k: collections.Counter() for k in ("str", "bad", "struct")}
    for tname in ("httpx028", "httpx027"):
        items, kinds = [], []
        for i, ((kind, _), raw) in enumerate(bodies):
            for per_att in modes:
                table, pi, mode, ops = per_att[i % len(per_att)]
                if table is tables[tname]:
                    items.append((raw, pi, mode, ops))
                    kinds.append(kind)
        sub = {k: collections.Counter() for k in tally}
        for k in tally:
            sel = [it for it, kk in zip(items, kinds) if kk == k]
            run_checked(warm, tables[tname], sel, sub[k])
            tally[k] += sub[k]
    bad, good = tally["bad"], tally["str"] + tally["struct"]
    assert bad["fast"] == 0 and bad[rw.BODY_PARSE_ERROR] == bad["irregular"], bad
    assert good["fast"] >= 0.85 * (good["fast"] + good["irregular"]) and good["exotic"] == 0, good


# ---- 3. production batches ------------------------------------------------------------------------------------------------------

class Pool:
    """distinct bodies; an item is (body index, plan variant index) of the httpx028 table, with its reference cached"""

    def __init__(self, table):
        rng = np.random.default_rng(4321)
        self.table, self.packed = table, table.packed()
        self.variants = G.plan_variants(table)
        b = list(chat_bodies(1024, 4096, seed=2))                                            # config 2
        for k, tgt in enumerate((300, 700, 1500, 3000, 4500, 5800, 6100)):
            b += chat_bodies(160, tgt, seed=40 + k, non_ascii=0.3)
        for k, tgt in enumerate((8192, 12000, 16384, 32768, 65536)):
            b += chat_bodies(4, tgt, seed=60 + k, non_ascii=0.1)
        b += [raw for _, raw, _, _ in G.ladder_bodies()]
        edges = G.chunk_edge_bodies()
        b += [edges[int(i)][1] for i in rng.choice(len(edges), 600, replace=False)]
        b += [G.damaged(b[int(i)], rng) for i in rng.choice(len(b), 400, replace=False)]
        b += [b""] * 6
        self.bodies = b
        self._want, self._fast = {}, {}

    def item(self, k):
        """the k-th item of a batch: the bodies in a scattered order (each once per lap), the plan variant shifted on every lap"""
        j = k * 7919 % len(self.bodies)                  # (7 919 is prime and does not divide the pool size)
        return j, (k // len(self.bodies) + j) % len(self.variants)

    def fast(self, it):
        if it not in self._fast:
            raw = self.bodies[it[0]]
            self._fast[it] = G.is_fast(raw, self.packed, self.variants[it[1]][0])
        return self._fast[it]

    def check(self, items, got, tally):
        for it, (st, out, _, _) in zip(items, got):
            if it not in self._want:
                _, mode, ops = self.variants[it[1]]
                self._want[it] = G.want(self.bodies[it[0]], ops, mode)
            wst, w = self._want[it]
            if st == rw.BODY_EXOTIC:
                assert wst in (None, rw.BODY_OK, rw.BODY_ENCODE_ERROR)
                tally["exotic"] += 1
                continue
            assert st == wst and out == w, (self.bodies[it[0]][:200], self.variants[it[1]][1], st, wst)
            tally[st] += 1
            tally["fast" if self.fast(it) else "irregular"] += 1

    def run(self, engine, items, tally):
        engine.load_rules(self.table)
        got = both_modes(engine, [self.bodies[j] for j, _ in items], [self.variants[v][0] for _, v in items])
        self.check(items, got, tally)
        return got


@pytest.fixture(scope="module")
def pool(tables):
    return Pool(tables["httpx028"])


def _layout(pool, items, layout):
    irr = [it for it in items if not pool.fast(it)]
    fast = [it for it in items if pool.fast(it)]
    if layout == "irregular_first":
        return irr + fast
    if layout == "irregular_last":
        return fast + irr
    out, k = [], max(1, len(items) // max(1, len(irr)))        # spread the irregular bodies evenly
    fi = iter(fast)
    for x in irr:
        out += [next(fi, None) for _ in range(k - 1)] + [x]
    return [x for x in out if x is not None] + list(fi)


@pytest.mark.parametrize("n", [1024, 8192, 16384])
@pytest.mark.parametrize("layout", ["irregular_first", "irregular_last", "interleaved"])
def test_production_batch(warm, pool, n, layout):
    items = _layout(pool, [pool.item(k) for k in range(n)], layout)
    assert len(items) == n
    tally = collections.Counter()
    pool.run(warm, items, tally)
    assert tally["fast"] >= 0.6 * n and tally["irregular"] >= 0.05 * n and tally[rw.BODY_PARSE_ERROR] >= 0.02 * n, tally
    assert tally["exotic"] <= 0.02 * n, tally


@pytest.mark.parametrize("which", ["all_irregular", "none_irregular"])
def test_production_batch_redo_list_full_or_empty(warm, pool, which):
    items = [pool.item(k) for k in range(12000)]
    items = [it for it in items if pool.fast(it) == (which == "none_irregular")][:4096]
    assert len(items) >= 1500
    tally = collections.Counter()
    pool.run(warm, items, tally)
    assert tally["fast" if which == "none_irregular" else "irregular"] == len(items) - tally["exotic"], tally


# ---- 4. packed output -------------------------------------------------------------------------------------------------------------

def _packed(engine, pool, items, slot_cap=None, out=None):
    bodies = [pool.bodies[j] for j, _ in items]
    buf, off = rw.pack_bodies(bodies)
    idx = np.array([pool.variants[v][0] for _, v in items], dtype=np.uint32)
    if slot_cap is None:
        slot_cap = (6 * max(len(b) for b in bodies) + pool.table.max_growth() + 64 + 15) & ~15
    return engine.rewrite_packed(buf, off, idx, slot_cap, out=out)


@pytest.mark.parametrize("n", [1023, 1024, 1025, 2047, 2049, 4097])
def test_packed_offsets_across_blocks(warm, pool, n):
    """k_body_offsets carries its sum from one block of 1 024 results to the next: OK and failed bodies on both sides"""
    warm.load_rules(pool.table)
    rng = random.Random(n)
    items = [pool.item(rng.randrange(len(pool.bodies) * 3)) for _ in range(n)]
    out, out_off, res = _packed(warm, pool, items)
    ok = res["status"] == rw.BODY_OK
    lens = np.where(ok, res["out_len"], 0).astype(np.uint64)
    assert np.array_equal(out_off, np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64))
    tally = collections.Counter()
    pool.check(items, [(int(res["status"][i]), bytes(out[int(out_off[i]):int(out_off[i + 1])]) if ok[i] else b"", 0, 0) for i in range(n)], tally)
    assert tally[rw.BODY_OK] > 0.8 * n and 0 < tally[rw.BODY_PARSE_ERROR], tally


@pytest.mark.parametrize("delta", [1, 2, 3])
def test_packed_unaligned_slots(warm, pool, delta):
    """slot_cap not a multiple of 4 (odd, 2 mod 4): k_body_pack reads the slots unaligned; the output is the aligned run's"""
    warm.load_rules(pool.table)
    items = [pool.item(k) for k in range(2049)]
    out, out_off, res = _packed(warm, pool, items)
    base = int((6 * max(len(pool.bodies[j]) for j, _ in items) + pool.table.max_growth() + 64 + 15) & ~15)
    out2, off2, res2 = _packed(warm, pool, items, slot_cap=base + delta)
    assert np.array_equal(res, res2) and np.array_equal(out_off, off2)
    assert bytes(out[:int(out_off[-1])]) == bytes(out2[:int(off2[-1])])


def test_slot_exactly_the_output_length(warm, pool):
    """slot_cap == out_len fits, out_len - 1 is OVERFLOW with the needed length -- for a fast-path body and an irregular one, odd
    and even lengths, in both modes"""
    warm.load_rules(pool.table)
    fast = [it for it in (pool.item(k) for k in range(3000)) if pool.fast(it)]
    irr = [it for it in (pool.item(k) for k in range(3000)) if not pool.fast(it)]
    chosen = []
    for group in (fast, irr):
        got = pool.run(warm, group[:300], collections.Counter())
        oks = [(it, len(g[1])) for it, g in zip(group, got) if g[0] == rw.BODY_OK and len(g[1]) > 40]
        chosen += [next(x for x in oks if x[1] % 2 == 1), next(x for x in oks if x[1] % 4 == 2)]
    for it, L in chosen:
        body, pi = pool.bodies[it[0]], pool.variants[it[1]][0]
        for cap in (L, L - 1):
            got = both_modes(warm, [body] * 3, [pi] * 3, slot_cap=cap)
            for st, out, _, _ in got:
                if cap == L:
                    assert st == rw.BODY_OK and out == pool._want[it][1]
                else:
                    assert st == rw.BODY_OVERFLOW
            _, off, res = _packed(warm, pool, [it] * 3, slot_cap=cap)
            assert list(res["out_len"]) == [L] * 3 and list(res["status"]) == [rw.BODY_OK if cap == L else rw.BODY_OVERFLOW] * 3


def test_caller_buffer_cut_at_body_boundaries(warm, pool):
    warm.load_rules(pool.table)
    items = [pool.item(k) for k in range(1500)]
    full, full_off, res = _packed(warm, pool, items)
    ok = res["status"] == rw.BODY_OK
    oks = np.flatnonzero(ok)
    for k in (int(oks[1]), int(oks[700]), 1023, 1024, 1025, int(oks[-1])):
        for cut in (int(full_off[k]) - 1, int(full_off[k]), int(full_off[k]) + 1):
            small = np.zeros(max(cut, 1), dtype=np.uint8)
            out2, off2, res2 = _packed(warm, pool, items, out=small[:cut] if cut else small[:0])
            assert np.array_equal(off2, full_off)
            for i in range(len(items)):
                if not ok[i]:
                    assert res2["status"][i] == res["status"][i]
                elif int(full_off[i + 1]) <= cut:
                    assert res2["status"][i] == rw.BODY_OK and bytes(out2[int(off2[i]):int(off2[i + 1])]) == bytes(full[int(full_off[i]):int(full_off[i + 1])])
                else:
                    assert res2["status"][i] == rw.BODY_OVERFLOW, (i, cut)


# ---- 5. device entry point ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["production_8192", "blocks_2049_odd_slots"])
def test_device_entry_point(warm, pool, case):
    """lgw_bodies_rewrite_device on torch CUDA tensors == lgw_bodies_rewrite"""
    import torch
    warm.load_rules(pool.table)
    if case == "production_8192":
        items, delta = _layout(pool, [pool.item(k) for k in range(8192)], "interleaved"), 0
    else:
        rng = random.Random(7)
        items, delta = [pool.item(rng.randrange(len(pool.bodies) * 3)) for _ in range(2049)], 1
    bodies = [pool.bodies[j] for j, _ in items]
    buf, off = rw.pack_bodies(bodies)
    idx = np.array([pool.variants[v][0] for _, v in items], dtype=np.uint32)
    slot_cap = ((6 * max(len(b) for b in bodies) + pool.table.max_growth() + 64 + 15) & ~15) + delta
    out, out_off, res = warm.rewrite_packed(buf, off, idx, slot_cap)
    n = len(items)
    dev = torch.device("cuda", warm.device)
    d_buf = torch.from_numpy(buf).to(dev)
    d_off = torch.from_numpy(off.view(np.int64)).to(dev)
    d_idx = torch.from_numpy(idx.view(np.int32)).to(dev)
    d_out = torch.zeros(out.nbytes, dtype=torch.uint8, device=dev)
    d_out_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    d_res = torch.zeros(n * 4, dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = warm._lib.lgw_bodies_rewrite_device(warm._h, p(d_buf), p(d_off), n, int(off[-1]), p(d_idx), slot_cap, p(d_out), out.nbytes, p(d_out_off), p(d_res))
    assert rc == 0, warm._lib.lgw_last_error(warm._h)
    warm.sync()
    g_off = d_out_off.cpu().numpy().view(np.uint64)
    g_res = d_res.cpu().numpy().view(rw.RESULT_DTYPE)
    assert np.array_equal(g_off, out_off) and np.array_equal(g_res, res)
    assert bytes(d_out.cpu().numpy()[:int(g_off[-1])]) == bytes(out[:int(out_off[-1])])


# ---- 6. warm engine, every kind of call --------------------------------------------------------------------------------------------

def _usage_doc(rng, size, usage_first):
    u = b'"usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d,"cost":%s}' % (
        rng.randrange(10 ** 6), rng.randrange(10 ** 5), rng.randrange(10 ** 6), rng.choice([b"0", b"1.5e-05", b"0.25", b"3"]))
    head = b'{"id":"x",' + (u + b"," if usage_first else b"") + b'"choices":[{"message":{"content":"'
    tail = b'"}}]' + (b"" if usage_first else b"," + u) + b',"model":"m","provider":"P"}'
    return head + _pad(size - len(head) - len(tail), rng) + tail


def _pad(k, rng):
    """k bytes of string content with escapes and UTF-8"""
    piece = rng.choice([b"plain text ", b"caf\xc3\xa9 \\n ", b"\\u00e9\\\"q\\\" ", b"\xe4\xb8\xad\xf0\x9f\x98\x80 "])
    return piece * (k // len(piece)) + b"z" * (k % len(piece))       # whole pieces: no escape or UTF-8 sequence is cut


def _error_doc(rng, size):
    msg = _pad(rng.randrange(0, 3000), rng)
    head = b'{"error":{"message":"' + msg + b'","code":1},"pad":"'
    tail = b'"}'
    return head + _pad(max(0, size - len(head) - len(tail)), rng) + tail


def _docs(rng, n, sizes):
    return [(_usage_doc(rng, s, i % 2 == 0) if i % 3 else _error_doc(rng, s)) for i, s in zip(range(n), sizes)]


def _calls(pool):
    rng = random.Random(11)
    small = [pool.item(k) for k in range(64)]
    large = [pool.item(k) for k in range(9000)]
    docs_small = _docs(rng, 40, [rng.randrange(100, 2000) for _ in range(40)])
    docs_large = _docs(rng, 600, [rng.choice([6143, 6144, 6145, 20000, 70000]) for _ in range(600)])
    scan_small = [pool.bodies[j] for j, _ in small]
    scan_large = [pool.bodies[j] for j, _ in large[:5000]]
    return [("rewrite", small), ("scan", scan_large), ("usage", docs_small), ("rewrite", large), ("detail", docs_large), ("scan", scan_small),
            ("rewrite", small), ("usage", docs_large), ("detail", docs_small), ("rewrite", large[:3000])]


def _call(engine, pool, kind, arg):
    if kind == "rewrite":
        engine.load_rules(pool.table)
        out, off, res = _packed(engine, pool, arg)
        return bytes(out[:int(off[-1])]), off.tobytes(), res.tobytes()
    if kind == "scan":
        scans, models = engine.scan_bodies(arg)
        return scans.tobytes(), models
    if kind == "usage":
        return [(canon_rows(r), e) for r, e in engine.documents_usage(arg)]
    return [(bytes(e), t) for e, t in engine.documents_error_detail(arg, 4096)]


def test_warm_engine_interleaved_calls(warm, pool):
    """rewrite, scan and both document calls share b_in / b_off / b_results / the slots, which grow on demand: small, large, small
    calls of every kind on one engine give what a fresh engine gives"""
    for kind, arg in _calls(pool):
        got = _call(warm, pool, kind, arg)
        fresh = new_engine()
        try:
            want = _call(fresh, pool, kind, arg)
        finally:
            fresh.close_engine()
        assert got == want, kind


# ---- 7. scan --------------------------------------------------------------------------------------------------------------------

def test_scan_model_cap(warm):
    U = G.U.decode()
    rng = random.Random(12)
    bodies = []
    for L in (1, 254, 255, 256, 257, 300):
        bodies.append(json.dumps({"model": "a" * L, "stream": True}).encode())
    for pre in range(250, 258):                     # an escape / a multi-byte character across byte 256 of the model text
        bodies += [('{"model":"' + "a" * pre + chr(0xE9) + "b" * 9 + '"}').encode(), ('{"model":"' + "a" * pre + U + '00e9' + "b" * 9 + '","stream":1}').encode(),
                   ('{"model":"' + "a" * pre + U + "d83d" + U + "de00" + "b" + '"}').encode(), ('{"model":"' + "a" * pre + chr(0x1F600) + '"}').encode(),
                   ('{"model":"' + "a" * pre + chr(0x4E2D) + '","stream":"x"}').encode(), ('{"model":"' + "a" * pre + "\\n\\\"" + '"}').encode()]
    for v in ("12", "null", "true", "false", "[]", "{}", '""', "0.0", '["m"]', '{"a":"m"}', "-1"):
        bodies += [('{"model":%s,"stream":%s}' % (v, v)).encode(), ('{"stream":true,"model":%s}' % v).encode()]
    bodies += [bc.spell(rng, bc.rand_body(rng)).encode("utf-8") for _ in range(3000)]
    bodies += chat_bodies(512, 4096, seed=9, stream=True) + chat_bodies(16, 20000, seed=10)
    scans, models = warm.scan_bodies(bodies)
    seen = collections.Counter()
    for raw, sc, model in zip(bodies, scans, models):
        ost, body, omodel, ostream = bo.parse_body(raw)
        assert int(sc["status"]) == ost, raw[:300]
        seen[ost] += 1
        if ost == 1:
            continue
        assert bool(sc["model_truthy"]) == bool(omodel) and bool(sc["stream_truthy"]) == bool(ostream), raw[:300]
        if isinstance(omodel, str):
            m = omodel.encode("utf-8", "surrogatepass")
            assert model == m[:256] and int(sc["model_len"]) == len(m), raw[:300]
    assert seen[0] > 2500 and seen[2] > 20, seen


# ---- 8. documents --------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def documents():
    """more than 8 x SMs x 4 documents (every warp makes more than one grid-stride lap), staged and unstaged ones alternating"""
    rng = random.Random(13)
    sizes = []
    for i in range(4800):
        sizes.append(rng.choice([6143, 6144, 300, 6000]) if i % 2 == 0 else rng.choice([6145, 6200, 9000, 30000]))
    for k, s in enumerate((65536, 200000, 1 << 20)):
        sizes[100 + 977 * k] = s
    return _docs(rng, len(sizes), sizes)


def test_documents_usage(warm, documents):
    from oracle.sse_oracle import tap_nonstream
    import torch
    assert len(documents) > 8 * torch.cuda.get_device_properties(warm.device).multi_processor_count * 4
    got = warm.documents_usage(documents)
    n = 0
    for t, (rows, exotic) in zip(documents, got):
        assert not exotic, t[:200]
        assert canon_rows(rows) == canon_rows(tap_nonstream([t]).rows), t[:200]
        n += 1
    assert n == len(documents)


def test_documents_error_detail(warm, documents):
    from llmapigateway_b200.responses import _error_detail
    got = warm.documents_error_detail(documents, 4096)
    n_text = 0
    for raw, (e, text) in zip(documents, got):
        doc = json.loads(raw)
        try:
            want = doc.get("error", {}).get("message") or doc.get("detail")
        except Exception as ex:
            want = f"Unexpected error during request to u: {str(ex)}"

        class One:
            def documents_error_detail(self, _docs, text_stride=4096):
                return [(e, text)]

        mapped, exotic = _error_detail(One(), raw, "u", rw.KIND_OBJ)
        assert exotic is None, raw[:200]
        assert type(mapped) is type(want) and mapped == want, raw[:200]
        n_text += isinstance(want, str)
    assert n_text > 1000


def test_normalise_responses_large(warm, tables, documents):
    from llmapigateway_b200.responses import normalise_responses
    from oracle import response_oracle as ro
    table = tables["httpx028"]
    warm.load_rules(table)
    rng = random.Random(14)
    docs = documents[:1500]
    sts = [rng.choice([200, 200, 201, 500]) for _ in docs]
    got = normalise_responses(warm, table, docs, sts, "u", strict=False)
    n_ok = n_big = 0
    for raw, st, (body, detail) in zip(docs, sts, got):
        kind, val = ro.normalise(st, raw, "u")
        assert body != "exotic", raw[:200]
        if kind == "ok":
            assert (body, detail) == (val, None), raw[:200]
            n_ok += 1
            n_big += len(raw) > G.MAXB
        else:
            assert body is None and detail == val, raw[:200]
    assert n_ok > 400 and n_big > 100, (n_ok, n_big)
