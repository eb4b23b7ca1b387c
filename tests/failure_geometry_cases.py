"""Failed streaming attempts built by construction: every shape of a failing first event (and the near misses that commit), at
sizes around `detail_cap`, with UTF-8 characters across byte `detail_cap`, cut at every byte, over two and three steps, among
empty and undecodable chunks.  Each attempt knows the event it fails on (the bytes the engine keeps, then the whole text the
client's 503 carries), and `oracle.sse_oracle.run_stream` confirms the verdict: `check_against_oracle`.

Shared by tests/test_failures_geometry_cpu.py (oracle and host build) and tests/test_failures_geometry_gpu.py (the engine)."""
from __future__ import annotations

import json
import random
from dataclasses import dataclass, field

from llmapigateway_b200 import _abi
from llmapigateway_b200.synth import DELTA_HEAD, DELTA_TAIL

DETAIL_CAP = 4096
SEP = b"\n\n"
DONE = b"data: [DONE]\n\n"
KiB = 1024


@dataclass
class Attempt:
    name: str
    chunks: list                       # every network chunk of the attempt
    event: bytes | None                # the failing first event (no separator); None: the attempt commits
    verdict: int                       # _abi.VERDICT_*
    steps: list = field(default_factory=lambda: [0])      # chunk indices where a step begins (the first is 0)

    def step_chunks(self):
        """the chunks of every step"""
        b = list(self.steps) + [len(self.chunks)]
        return [self.chunks[b[k]:b[k + 1]] for k in range(len(self.steps))]

    def detail(self, cap: int = DETAIL_CAP) -> bytes:
        """what the engine keeps of the event"""
        return b"" if self.event is None else self.event[:cap]

    def truncated(self, cap: int = DETAIL_CAP) -> bool:
        return self.event is not None and len(self.event) > cap

    def counted(self):
        """(n_chunks_in, bytes_in) at the end of the attempt: the non-empty chunks up to the one the verdict falls in (an
        undecodable chunk counts, an empty one does not; after a failure nothing counts)"""
        if self.event is None:
            return sum(1 for c in self.chunks if c), sum(len(c) for c in self.chunks)
        n = b = 0
        carry = b""
        for c in self.chunks:
            if not c:
                continue
            n += 1; b += len(c)
            try:
                c.decode("utf-8")
            except UnicodeDecodeError:
                continue
            carry += c
            if self.event + SEP in carry:
                return n, b
        raise AssertionError(self.name)


# ---- failing events of an exact length ---------------------------------------------------------------------------------------------

SHAPES = {   # name: (head, tail, verdict); the event is head + padding + tail.  The padding is the text of a JSON string.
    "error_obj": (b'data: {"error":{"message":"', b'","code":503}}', _abi.VERDICT_FAIL_EVENT),
    "error_null": (b'data: {"error":null,"note":"', b'"}', _abi.VERDICT_FAIL_EVENT),
    "detail": (b'data: {"detail":"', b'"}', _abi.VERDICT_FAIL_EVENT),
    "escaped_key": (b'data: {"\\u0065rror":1,"note":"', b'"}', _abi.VERDICT_FAIL_EVENT),
    "invalid_json": (b'data: {"error":{"message":"', b'",}}', _abi.VERDICT_FAIL_PARSE),
    "template_error": (DELTA_HEAD + b'abcdefgh"}}],"error":{"message":"', b'"}}', _abi.VERDICT_FAIL_EVENT),
    "template_detail": (DELTA_HEAD + b'abcdefgh"}}],"x":"', b'","detail":"late"}', _abi.VERDICT_FAIL_EVENT),
    "choices_error": (b'data: {"choices":[{"index":0,"error":{"message":"', b'"}}]}', _abi.VERDICT_OK),
}
WIDE = ["é", "中", "\U0001F600"]          # 2-, 3- and 4-byte UTF-8


def padding(n: int, seed: int, wide: str | None = None, at: int | None = None) -> bytes:
    """n bytes of JSON string text (letters, escapes, spaces); with `wide`, that character starts at byte `at` of it"""
    if wide is not None:
        w = wide.encode("utf-8")
        return padding(at, seed) + w + b"q" * (n - at - len(w))
    rng = random.Random(seed)
    words = [b"overloaded ", b"prompt ", b"\\\"quoted\\\" ", b"tab\\t", b"line\\n", b"\\u00e9t\\u00e9 ", b"x"]
    out = b""
    while len(out) < n:
        out += rng.choice(words)
    out = out[:n]
    while True:                                                   # never end inside an escape
        try:
            json.loads(b'"' + out + b'"')
            break
        except ValueError:
            out = out[:-1]
    return out + b"z" * (n - len(out))


def event(shape: str, size: int, seed: int = 0, wide: str | None = None, straddle: int = 1, cap: int = DETAIL_CAP) -> bytes:
    """a `shape` event of exactly `size` bytes; with `wide`, that character covers byte `cap` of the event, `straddle` (1 ..
    width - 1) of its bytes before it"""
    head, tail, _ = SHAPES[shape]
    n = size - len(head) - len(tail)
    at = None if wide is None else cap - straddle - len(head)
    ev = head + padding(n, seed, wide, at) + tail
    assert len(ev) == size
    if wide is not None:
        w = wide.encode("utf-8")
        assert ev[cap - straddle:cap - straddle + len(w)] == w
    return ev


def delta(text: str) -> bytes:
    return DELTA_HEAD + text.encode("utf-8") + DELTA_TAIL


# ---- attempts -------------------------------------------------------------------------------------------------------------------

LEADS = {   # what comes before the first real event
    "none": [],
    "comment": [b": keep-alive\n\n", b": ping\n\n"],
    "done": [DONE],
    "event_line": [b"event: message\n\n", b"id: 7\n\n"],
}


def attempt(name: str, shape: str, ev: bytes, lead="none", cuts=None, same_chunk_lead=False, steps=None, extra=()) -> Attempt:
    """`lead` parts, the event and its separator, then a delta and [DONE] (never reached when it fails); `cuts` = byte offsets
    into the event+separator where the chunks break (default: one chunk); `same_chunk_lead`: the lead parts share the event's
    first chunk (the event is then not the chunk's first part)"""
    _, _, verdict = SHAPES[shape]
    body = ev + SEP
    pieces = [body[a:b] for a, b in zip([0] + sorted(cuts or []), sorted(cuts or []) + [len(body)])]
    lead_parts = list(LEADS[lead])
    if same_chunk_lead and lead_parts:
        pieces[0] = b"".join(lead_parts) + pieces[0]
        lead_parts = []
    chunks = lead_parts + pieces + list(extra) + [delta("after"), DONE]
    return Attempt(name, chunks, None if verdict == _abi.VERDICT_OK else ev, verdict, steps or [0])


def sized_attempts(cap: int = DETAIL_CAP) -> list[Attempt]:
    """every shape at every size around `cap` and far beyond it, behind every lead, in one chunk or cut in two / four"""
    out = []
    sizes = [cap - 1, cap, cap + 1, 3 * cap, 60 * KiB]
    for si, shape in enumerate(SHAPES):
        for zi, size in enumerate(sizes):
            for li, lead in enumerate(LEADS):
                seed = si * 100 + zi * 10 + li
                ev = event(shape, size, seed)
                k = (si + zi + li) % 3
                cuts = [] if k == 0 else ([size // 2] if k == 1 else [7, cap - 1, cap + 3, size + 1])
                cuts = [c for c in cuts if 0 < c < size + 2]
                out.append(attempt(f"{shape}-{size}-{lead}-cut{k}", shape, ev, lead, cuts, same_chunk_lead=(li % 2 == 1)))
    return out


def straddling_attempts(cap: int = DETAIL_CAP) -> list[Attempt]:
    """a 2-, 3- or 4-byte character across byte `cap`, every split of it, events of cap + 1 .. 3 * cap bytes"""
    out = []
    for shape in ("error_obj", "detail", "error_null", "invalid_json", "template_error"):
        for wide in WIDE:
            w = len(wide.encode("utf-8"))
            for straddle in range(1, w):
                for size in (cap + 1 + straddle, cap + 40, 3 * cap):
                    if size - cap < w - straddle + len(SHAPES[shape][1]):
                        continue
                    ev = event(shape, size, size + straddle, wide, straddle, cap)
                    out.append(attempt(f"{shape}-wide{w}-{straddle}-{size}", shape, ev, "comment", [cap // 2]))
    return out


def short_event_cuts() -> list[Attempt]:
    """a ~120-byte failing event cut into two chunks at every byte, the separator included (a cut between its two newlines)"""
    out = []
    for shape, size in (("error_obj", 120), ("detail", 118), ("template_error", 131)):
        ev = event(shape, size, size)
        for c in range(1, len(ev) + 2):
            out.append(attempt(f"{shape}-cut-at-{c}", shape, ev, "none", [c]))
    return out


def multi_step_attempts(cap: int = DETAIL_CAP) -> list[Attempt]:
    """events held in the carry between steps: cut over two and three steps, long ones included, behind other parts"""
    out = []
    for shape in ("error_obj", "detail", "escaped_key", "invalid_json", "template_error", "choices_error"):
        for size in (120, cap + 1, 3 * cap, 40 * KiB):
            ev = event(shape, size, size ^ 5)
            for n_steps in (2, 3):
                cuts = [size * j // n_steps for j in range(1, n_steps)]
                a = attempt(f"{shape}-{size}-{n_steps}steps", shape, ev, "comment", cuts)
                first = len(LEADS["comment"])
                a.steps = [0] + [first + j for j in range(1, n_steps)]
                out.append(a)
            a = attempt(f"{shape}-{size}-sep-across-steps", shape, ev, "event_line", [size + 1])     # "\n" | "\n"
            a.steps = [0, len(LEADS["event_line"]) + 1]
            out.append(a)
    return out


def dropped_chunk_attempts(cap: int = DETAIL_CAP) -> list[Attempt]:
    """empty and undecodable chunks inside the event (both dropped by the reference, the undecodable ones counted), and a
    character cut across two chunks, which drops both halves"""
    out = []
    for shape in ("error_obj", "detail", "template_error"):
        for size in (150, cap + 2, 3 * cap):
            ev = event(shape, size, size + 1)
            head, rest = ev[:size // 3], ev[size // 3:] + SEP
            chunks = [b": c\n\n", head, b"", b"\xff\xfe", b"", rest[:5], b"\xc3", rest[5:], b"", delta("x"), DONE]
            out.append(Attempt(f"{shape}-{size}-empty-and-bad", chunks, ev, SHAPES[shape][2]))
            # "é" split across two chunks: both are undecodable on their own and both are dropped
            a, b = ev[:size // 2], ev[size // 2:]
            chunks = [a, b"pre\xc3", b"\xa9post", b + SEP, delta("x"), DONE]
            out.append(Attempt(f"{shape}-{size}-split-char", chunks, ev, SHAPES[shape][2]))
    return out


def all_attempts(cap: int = DETAIL_CAP) -> list[Attempt]:
    return sized_attempts(cap) + straddling_attempts(cap) + short_event_cuts() + dropped_chunk_attempts(cap)


def single_step(attempts) -> list[Attempt]:
    return [a for a in attempts if len(a.steps) == 1]


def check_against_oracle(a: Attempt):
    """the oracle agrees with what the attempt was built to do"""
    from oracle.sse_oracle import run_stream
    relay, _ = run_stream(list(a.chunks))
    assert relay.failed == (a.verdict != _abi.VERDICT_OK), a.name
    if a.verdict == _abi.VERDICT_FAIL_EVENT:
        assert relay.error_detail == a.event.decode("utf-8"), a.name
    elif a.verdict == _abi.VERDICT_FAIL_PARSE:
        assert relay.error_detail.startswith("Unexpected error during request to "), a.name
    return relay


# ---- the provider side of the chain walker, failing with these events ------------------------------------------------------------

def chain_upstream(n_streams: int, n_events: int, seed: int, p_fail: float, cap: int = DETAIL_CAP):
    """synth.ChainUpstream whose failing attempts stream the cases' VERDICT_FAIL_EVENT attempts (long, split, UTF-8 across byte
    `cap`, behind comments, among dropped chunks) instead of its one-chunk events; HTTP 500 failures are kept"""
    from llmapigateway_b200 import synth
    fails = [a for a in all_attempts(cap) + multi_step_attempts(cap) if a.verdict == _abi.VERDICT_FAIL_EVENT]
    pool = [a for a in fails if a.truncated(cap)] + [a for a in fails if not a.truncated(cap)][::4]      # mostly long ones

    class LongFailures(synth.ChainUpstream):
        def failure_chunks(self, sid: int, attempt: int, kind: int):
            if kind == synth.FAIL_HTTP500:
                return super().failure_chunks(sid, attempt, kind)
            return list(pool[(sid * 31 + attempt * 7 + kind) % len(pool)].chunks)

    return LongFailures(n_streams, n_events, seed=seed, p_fail=p_fail)
