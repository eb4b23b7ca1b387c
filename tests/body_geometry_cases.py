"""Request bodies at the limits and per-thread chunk edges of the data-parallel rewrite (csrc/body_fast.cuh), shared by
tests/test_body_geometry_cpu.py (the host build of the kernel source) and tests/test_body_geometry_gpu.py (k_body_fast and the
kernels around it on the device).

k_body_fast gives each body one block of 384 threads; thread t owns the bytes [t * chunk, (t + 1) * chunk) with
chunk = roundup8(ceil(n / 384)).  An escape, a surrogate pair or a UTF-8 sequence that crosses such an edge is where
fj_swallowed, the chunk-start escape state of the quote and token passes and fph_utf8's continuation check do their work, so
`chunk_edge_bodies` puts every hard piece at every offset from edge - 6 to edge + 6 (further back for pieces longer than 6
bytes) of several edges.  `ladder_bodies` builds bodies one below, at and one above each limit of the data-parallel path."""
from __future__ import annotations

import json

import numpy as np

import body_cases as bc
from llmapigateway_b200 import rewrite as rw
from oracle import body_oracle as bo

THREADS = 384            # LGW_FAST_THREADS
MAXB = 6144              # LGW_FAST_MAXB: bytes
MAXT = 1536              # LGW_FAST_MAXT: tokens
MAXBR = 512              # LGW_FAST_MAXBR: brackets
MAXKEYS = 24             # LGW_BODY_MAXKEYS: keys per object
MAXD = 16                # LGW_BODY_MAXD: nesting depth
KEYCAP = 128             # LGW_BODY_KEYCAP: bytes per key
NUMCAP = 48              # LGW_BODY_NUMCAP: bytes per number
MODE_NAMES = ["httpx028", "httpx027", "json5"]
FAST_IRREGULAR = 0xFFFFFFFF

# every attempt chat.py walks for "gw/chain", the fifth rule (unicode keys and values), and the fallback-provider plan (None)
ATTEMPTS = bc.CHAIN_ATTEMPTS + [(4, -1, False), None]


def chunk_of(n: int) -> int:
    return ((n + THREADS - 1) // THREADS + 7) & ~7


def tokens(raw: bytes) -> int:
    """The token count of body_fast.cuh's token pass: structural characters, strings and scalars (valid JSON only)."""
    n, i, L = 0, 0, len(raw)
    while i < L:
        c = raw[i]
        if c == 0x22:
            n += 1
            i += 1
            while raw[i] != 0x22:
                i += 2 if raw[i] == 0x5C else 1
            i += 1
        elif c in b"{}[],:":
            n += 1
            i += 1
        elif c in b" \t\r\n":
            i += 1
        else:
            n += 1
            while i < L and raw[i] not in b' \t\r\n{}[],:"':
                i += 1
    return n


def brackets(raw: bytes) -> int:
    n, in_str, esc = 0, False, False
    for c in raw:
        if in_str:
            if esc:
                esc = False
            elif c == 0x5C:
                esc = True
            elif c == 0x22:
                in_str = False
        elif c == 0x22:
            in_str = True
        elif c in b"{}[]":
            n += 1
    return n


# ---- plans and the reference ----------------------------------------------------------------------------------------------------

def plan_tables():
    """The two plan tables an engine can hold: stream plans render like httpx 0.28 or 0.27, non-stream plans like json5."""
    return {m: rw.RulePlans(bc.RULES, fallback_provider="fb", stream_mode=m) for m in ("httpx028", "httpx027")}


def plan_variants(plans):
    """[(plan index, render mode name, oracle ops)] for every attempt of ATTEMPTS, stream and non-stream."""
    out = []
    for att in ATTEMPTS:
        for stream in (True, False):
            mode = plans.stream_mode if stream else "json5"
            if att is None:
                out.append((plans.plan_index("not-in-rules", stream=stream), mode, []))
            else:
                rule, prov, sp, rt = bc.attempt_for_oracle(*att)
                out.append((plans.plan_index("gw/chain", *att, stream=stream), mode, bo.rule_ops(rule, prov, sp, rt)))
    return out


def mode_plans(tables):
    """[[(table, plan index, mode name, ops)] per attempt] for the three render modes: httpx028 and httpx027 stream plans, json5 non-stream"""
    out = []
    for name, stream in (("httpx028", True), ("httpx027", True), ("httpx028", False)):
        t = tables[name]
        out.append([(t, pi, mode, ops) for pi, mode, ops in plan_variants(t)[(0 if stream else 1)::2]])
    return out


def want(raw: bytes, ops, mode_name: str):
    """(status, bytes) of the reference for one attempt; status None: not an object root (the engine may call it exotic)."""
    try:
        body = json.loads(raw.decode("utf-8"))
    except Exception:
        return rw.BODY_PARSE_ERROR, b""
    if not isinstance(body, dict):
        return None, b""
    payload = bo.rewrite_payload(body, ops)
    try:
        return rw.BODY_OK, bo.RENDERERS[mode_name](payload)
    except (ValueError, UnicodeEncodeError):
        return rw.BODY_ENCODE_ERROR, b""


def check_against_reference(raw, st, out, ops, mode_name, tally):
    """One engine answer against the reference; EXOTIC is counted (callers cap it) and only accepted where the reference renders."""
    wst, w = want(raw, ops, mode_name)
    out = out if st == rw.BODY_OK else b""
    if st == rw.BODY_EXOTIC:
        assert wst in (None, rw.BODY_OK, rw.BODY_ENCODE_ERROR), (raw[:200], mode_name, wst)
        tally["exotic"] = tally.get("exotic", 0) + 1
        return
    assert st == wst, (raw[:200], mode_name, st, wst)
    assert out == w, (raw[:200], mode_name)
    tally[st] = tally.get(st, 0) + 1


def host_fast(raw, packed, pi, cap=1 << 17):
    """(status | FAST_IRREGULAR, bytes, needed) of the host build of fast_rewrite()"""
    import host_machine as hm
    plans, ops, blob = packed
    return hm.rewrite_body_fast(raw, plans, ops, blob, pi, cap=cap)


def is_fast(raw, packed, pi) -> bool:
    return host_fast(raw, packed, pi)[0] != FAST_IRREGULAR


# ---- chunk edges ------------------------------------------------------------------------------------------------------------------

CHUNK_LENGTHS = [383, 384, 385, 3071, 3072, 4096, 6143, 6144]
HEAD, TAIL = b'{"p":"', b'"}'
BS = b"\\"                       # one backslash
U = BS + b"u"                    # the start of a \uXXXX escape


def _str_pieces():
    """(name, bytes, focus): string content that stays inside the string (or closes it and opens the next member's string)."""
    p = [("esc_quote", BS + b'"', 0), ("esc_slash", BS + b"/", 0), ("u00e9", U + b"00e9", 0), ("u4e2d", U + b"4E2D", 0), ("u2028", U + b"2028", 0),
         ("pair", U + b"d83d" + U + b"de00", 0), ("lone_high", U + b"d800x", 0), ("lone_low", U + b"dc00", 0), ("high_then_bmp", U + b"d83d" + U + b"0041", 0),
         ("bs_u0041", BS + U + b"0041", 0), ("utf8_2", chr(0xE9).encode(), 0), ("utf8_3", chr(0x4E2D).encode(), 0), ("utf8_4", chr(0x1F600).encode(), 0),
         ("utf8_2028", chr(0x2028).encode(), 0), ("del", b"\x7f", 0), ("ctl_u0001", U + b"0001", 0), ("ctl_b", BS + b"b", 0), ("ctl_u001f", U + b"001f", 0),
         ("ctl_u0000", U + b"0000", 0), ("ctl_vt", U + b"000b", 0)]
    for k in range(1, 6):          # a run of k backslashes, then a quote: escaped (k odd) or closing the string (k even)
        p.append(("bs%d_quote" % k, b"\\" * k + b'"' + (b',"q":"' if k % 2 == 0 else b""), 0))
    return p


def _bad_pieces():
    """invalid UTF-8 around an edge: the reference answers PARSE_ERROR"""
    return [("stray_cont", b"\x80", 0), ("stray_cont_bf", b"\xbf", 0), ("extra_cont", b"\xc3\xa9\xa9", 0),
            ("cut_3", b"\xe4\xb8a", 0), ("cut_4", b"\xf0\x9f\x98a", 0), ("surrogate_utf8", b"\xed\xa0\x80", 0), ("five_cont", b"\xe4\xb8\xad\x80\x80", 0)]


def _struct_pieces():
    """members between two strings; focus = the byte put at the target offset"""
    def f(name, text, at):
        return (name, text, text.index(at))
    return [f("number", b'","n":-12.5e+3,"q":"', b"-"), f("integer", b'","n":1234567,"q":"', b"1"),
            f("float_repr", b'","n":[1e15,0.10,-0.0],"q":"', b"1e15"),
            f("key_colon", b'","key":"', b":"), f("key_comma", b'",  "key" :"', b","),
            f("model_end", b'","model":"old-model","q":"', b'","q'), f("temperature_end", b'","temperature":0.25,"q":"', b'5,'),
            f("messages_end", b'","messages":[{"role":"user","content":"hi"}],"q":"', b"],"),
            f("provider_end", b'","provider":{"order":["x"]},"q":"', b"},")]


def chunk_pieces():
    return [(n, t, f, "str") for n, t, f in _str_pieces()] + [(n, t, f, "bad") for n, t, f in _bad_pieces()] + \
           [(n, t, f, "struct") for n, t, f in _struct_pieces()]


def body_at(n: int, off: int, piece: bytes, focus: int = 0):
    """A body of exactly n bytes with piece[focus] at byte `off` (None when it does not fit)."""
    x = off - len(HEAD) - focus
    y = n - len(HEAD) - x - len(piece) - len(TAIL)
    if x < 0 or y < 0:
        return None
    return HEAD + b"a" * x + piece + b"b" * y + TAIL


def chunk_edges(n: int):
    c = chunk_of(n)
    last = (n - 1) // c * c
    return sorted({c, 2 * c, (n // 2) // c * c, last})


def chunk_edge_bodies(lengths=CHUNK_LENGTHS):
    """[(family tag, body)] for every length, edge, piece and offset; family tag = (piece kind, piece name)"""
    out = []
    for n in lengths:
        for edge in chunk_edges(n):
            for name, text, focus, kind in chunk_pieces():
                back = max(6, len(text) - 1) if focus == 0 else 6
                for off in range(edge - back, edge + 7):
                    raw = body_at(n, off, text, focus)
                    if raw is not None:
                        out.append(((kind, name), raw))
    return out


# ---- the limit ladder ---------------------------------------------------------------------------------------------------------------

def _obj(members) -> bytes:
    return b"{" + b",".join(members) + b"}"


def _fill_to(n: int, head: bytes = b'{"model":"gw/chain","messages":[{"role":"user","content":"', tail: bytes = b'"}]}', ch: bytes = b"x"):
    k = n - len(head) - len(tail)
    assert k >= 0
    return head + ch * k + tail


def _token_body(t: int) -> bytes:
    """a body of exactly t tokens (an array of ones, plus an empty array member for even counts)"""
    for extra in (b"", b',"b":[]'):
        for m in range(1, 2000):
            raw = b'{"model":"gw/chain","a":[' + b",".join([b"1"] * m) + b"]" + extra + b"}"
            if tokens(raw) == t:
                return raw
            if tokens(raw) > t:
                break
    raise AssertionError(t)


def _bracket_body(nbr: int) -> bytes:
    k = (nbr - 4) // 2
    raw = b'{"model":"gw/chain","a":[' + b",".join([b"[]"] * k) + b"]}"
    assert brackets(raw) == nbr
    return raw


def _keys_body(total: int) -> bytes:
    """`total` keys spread over objects of 23 keys each (every key needs its value and a comma: 4 tokens a key)"""
    members, left, o = [b'"model":"gw/chain"'], total - 1, 0
    while left > 0:
        inner = min(23, left - 1)
        members.append(b'"o%d":' % o + _obj([b'"k%d":%d' % (j, j % 10) for j in range(inner)]))
        left -= inner + 1
        o += 1
    raw = _obj(members)
    assert raw.count(b":") == total
    return raw


def _depth_body(d: int) -> bytes:
    return b'{"model":"gw/chain","a":' + b"[" * (d - 1) + b"1" + b"]" * (d - 1) + b"}"


NUMBERS = [b"0", b"-0", b"-0.0", b"0.0", b"1e15", b"1E15", b"1e16", b"1e5", b"1E+5", b"123456789012345", b"1234567890123456",
           b"0.123456789012345", b"0.1234567890123456", b"123456789012345.6", b"9007199254740993", b"-9223372036854775809",
           b"1.5e-7", b"0.0001", b"0.00001", b"100.000", b"2.5E-3", b"NaN", b"Infinity", b"-Infinity"]


def _number_of_len(L: int, neg: bool, flt: bool) -> bytes:
    s = (b"-" if neg else b"")
    if flt:
        s += b"1."
        return s + b"0" * (L - len(s))
    s += b"1"
    return s + b"0" * (L - len(s))


def ladder_bodies():
    """[(name, body, fast, exotic)] around every limit.  fast: what the data-parallel path must decide for an httpx028 stream plan;
    exotic: True when the exact machine must hand the body back under every plan (one past its own limits: keys per object,
    depth, key and number length), False when it must never.  None: no claim."""
    L = []
    for n, fast in ((MAXB - 1, True), (MAXB, True), (MAXB + 1, False)):
        L.append(("bytes_%d" % n, _fill_to(n), fast, False))
    for t, fast in ((MAXT - 1, True), (MAXT, True), (MAXT + 1, False)):
        raw = _token_body(t)
        assert tokens(raw) == t
        L.append(("tokens_%d" % t, raw, fast, False))
    for nbr, fast in ((MAXBR - 2, True), (MAXBR, True), (MAXBR + 2, False)):
        L.append(("brackets_%d" % nbr, _bracket_body(nbr), fast, False))
    # 1 536 tokens hold at most 383 keys (4 tokens a key), so the token limit answers before the hash table's 512: both sides of it
    for k, fast in ((382, True), (383, True), (384, False)):
        raw = _keys_body(k)
        assert tokens(raw) == 4 * k + 1
        L.append(("keys_total_%d" % k, raw, fast, False))
    for k, fast in ((MAXKEYS - 1, True), (MAXKEYS, True), (MAXKEYS + 1, False)):
        L.append(("keys_root_%d" % k, _obj([b'"model":"gw/chain"'] + [b'"k%02d":%d' % (j, j) for j in range(k - 1)]), fast, not fast))
        L.append(("keys_inner_%d" % k, _obj([b'"model":"gw/chain"', b'"o":' + _obj([b'"k%02d":"v"' % j for j in range(k)])]), fast, not fast))
    for d, fast in ((MAXD - 1, True), (MAXD, True), (MAXD + 1, False)):
        L.append(("depth_%d" % d, _depth_body(d), fast, not fast))
        L.append(("depth_obj_%d" % d, b'{"model":"gw/chain","a":' + b'{"a":' * (d - 1) + b"1" + b"}" * (d - 1) + b"}", fast, not fast))
    for k, fast in ((KEYCAP - 1, True), (KEYCAP, True), (KEYCAP + 1, False)):
        L.append(("keylen_%d" % k, b'{"model":"gw/chain","' + b"k" * k + b'":1}', fast, not fast))
        L.append(("keylen_inner_%d" % k, b'{"model":"gw/chain","o":{"' + b"k" * k + b'":"v"}}', fast, not fast))
        # (json5 hands non-ASCII keys back: exotic there at every length)
        L.append(("keylen_utf8_%d" % k, b'{"model":"gw/chain","' + b"k" * (k - 2) + chr(0xE9).encode() + b'":1}', fast, True if not fast else None))
    for ln, fast in ((NUMCAP - 1, True), (NUMCAP, True), (NUMCAP + 1, False)):
        for neg in (False, True):
            for flt in (False, True):
                num = _number_of_len(ln, neg, flt)
                assert len(num) == ln
                L.append(("number_%d%s%s" % (ln, "_neg" if neg else "", "_float" if flt else ""), b'{"model":"gw/chain","t":' + num + b"}", fast, not fast))
    for num in NUMBERS:
        L.append(("number_" + num.decode(), b'{"model":"gw/chain","t":' + num + b',"u":[' + num + b"]}", None, None))
    L.append(("numbers_all", b'{"model":"gw/chain","t":[' + b",".join(NUMBERS) + b"]}", None, None))
    # 6 144 bytes of string content that renders six times as long in the ASCII modes (DEL -> \u007f): the output-slot bound
    head = b'{"model":"gw/chain","c":"'
    L.append(("del_6144", _fill_to(MAXB, head, b'"}', b"\x7f"), True, False))
    L.append(("del_6145", _fill_to(MAXB + 1, head, b'"}', b"\x7f"), False, False))
    room = MAXB - len(head) - 2
    L.append(("ctl_6144", head + (U + b"0001") * (room // 6) + b"x" * (room % 6) + b'"}', True, False))
    L.append(("utf8_6144", head + chr(0x4E2D).encode() * (room // 3) + b"x" * (room % 3) + b'"}', True, False))
    L.append(("utf8_4_6144", head + chr(0x1F600).encode() * (room // 4) + b"x" * (room % 4) + b'"}', True, False))
    for name, raw, _, _ in L:
        if name.startswith(("del_", "ctl_", "utf8_", "bytes_")):
            assert len(raw) == int(name.rsplit("_", 1)[1]), name
    return L


# ---- production pools ----------------------------------------------------------------------------------------------------------------

def damaged(raw: bytes, rng) -> bytes:
    b = bytearray(raw)
    k = int(rng.integers(0, len(b)))
    op = int(rng.integers(0, 3))
    if op == 0:
        return bytes(b[:k])                       # cut short
    if op == 1:
        b[k] = int(rng.choice(np.frombuffer(b'{}[]",:\\\x80\xff', dtype=np.uint8)))
        return bytes(b)
    return bytes(b[:k]) + b"\xc3" + bytes(b[k:])  # a lead byte without its continuation
