"""Stream generators of the bulk-kernel fuzz campaign (tools/fuzz_relay2_cpu.py), shared with the GPU geometry tests
(tests/test_sse_geometry_gpu.py) so that both run the same content.  Each returns a list of streams, a stream being its list
of network chunks.  `make_streams(gen, n, seed)` picks one by name:

    random, template    tests/test_sse_gpu.py: mostly well-formed streams with a share of odd ones; near-identical events
                        (the template shortcut)
    usage               one usage skeleton, the values of its eight fields in every spelling JSON allows
    skeleton            usage events of odd shapes, each repeated so that it becomes a template
    openai, c3          realistic OpenAI chunks; the benchmark's 64-byte deltas -- both recut at arbitrary bytes
"""
from __future__ import annotations

import random

GENERATORS = ["random", "template", "usage", "openai", "c3", "skeleton"]

NUMBERS = ["0", "7", "12", "123456", "2147483647", "2147483648", "4294967296", "9007199254740993", "18446744073709551616",
           "-1", "-0", "0.0", "0.5", "1.25", "1e3", "1E3", "1e+3", "1e-3", "12.5e-2", "0.000001", "1.7976931348623157e308", "1e400",
           "123456789012345678901234567890", "0.1234567890123456789", "3.0", "5e0", "100000000000000000000.0", "4.9e-324", "1e-400"]
BAD_NUMBERS = ["01", "1.", ".5", "+1", "1e", "1e+", "--1", "0x10", "1_000", "NaN", "Infinity", "1.2.3", "1e1.5", ""]
STRINGS = ["m", "gpt-4o", "openai/gpt-4o-mini", "", "x" * 63, "x" * 64, "x" * 65, "x" * 200, "café", "中文", "\U0001F600",
           "a\\\"b", "tab\\there", "nl\\nx", "\\u0041\\u00e9", "\\ud83d\\ude00", "\\ud83d", "\\ude00x", "back\\\\slash", "sl\\/ash", "\\b\\f\\r"]
BAD_STRINGS = ["a\\qb", "\\u12", "\\u12G4", "ctl\x01x", 'q"q']


def usage_variant_streams(n_streams: int, seed: int):
    """Streams whose usage events share ONE skeleton (so that after the first few the kernel holds a usage template) while the
    values of the eight fields run through every number and string spelling; some events break the skeleton on purpose."""
    import sse_cases as sc
    rng = random.Random(seed)
    out = []
    for s in range(n_streams):
        evs = [sc.delta(rng.choice(["a", "hello", "x" * rng.randrange(1, 90)])) for _ in range(rng.randrange(1, 24))]
        n_usage = 1 if rng.random() < 0.8 else rng.randrange(0, 4)
        for _ in range(n_usage):
            def num():
                r = rng.random()
                return rng.choice(NUMBERS) if r < 0.85 else (rng.choice(BAD_NUMBERS) if r < 0.93 else rng.choice(["null", "true", '"7"', "[1]", "{}"]))

            def text():
                r = rng.random()
                return '"' + (rng.choice(STRINGS) if r < 0.9 else rng.choice(BAD_STRINGS)) + '"' if r < 0.96 else rng.choice(["null", "12", "[]"])
            shape = rng.random()
            if shape < 0.75:         # the C3 skeleton (SURVEY 8(d)): every field present
                ev = ('{"choices":[],"usage":{"prompt_tokens":%s,"completion_tokens":%s,"total_tokens":%s,"cost":%s,'
                      '"completion_tokens_details":{"reasoning_tokens":%s},"prompt_tokens_details":{"cached_tokens":%s}},"model":%s,"provider":%s}'
                      % (num(), num(), num(), num(), num(), num(), text(), text()))
            elif shape < 0.85:       # a second skeleton: no details, no provider
                ev = '{"id":"u","choices":[],"usage":{"prompt_tokens":%s,"completion_tokens":%s,"total_tokens":%s},"model":%s}' % (num(), num(), num(), text())
            elif shape < 0.92:       # usage beside a delta (the choices walk meets value spans)
                ev = '{"choices":[{"index":0,"delta":{"content":%s}}],"usage":{"prompt_tokens":%s,"completion_tokens":%s,"total_tokens":%s,"cost":%s}}' % (text(), num(), num(), num(), num())
            else:                    # details present but null / not objects
                ev = '{"choices":[],"usage":{"prompt_tokens":%s,"completion_tokens":%s,"total_tokens":%s,"completion_tokens_details":%s,"prompt_tokens_details":%s},"model":%s}' % (
                    num(), num(), num(), rng.choice(["null", "{}", '{"reasoning_tokens":3}', "5"]), rng.choice(["null", "{}", '{"cached_tokens":4}', '"x"']), text())
            if rng.random() < 0.04:
                i = rng.randrange(len(ev)); ev = ev[:i] + rng.choice(['"', "\\", "}", " ", "\n", ","]) + ev[i + 1:]
            evs.append(("data: " + ev + "\n\n").encode("utf-8", errors="surrogatepass") if rng.random() < 0.97 else (ev + "\n\n").encode("utf-8", errors="surrogatepass"))
            if rng.random() < 0.3:
                evs.append(sc.delta("more"))
        if rng.random() < 0.8:
            evs.append(sc.DONE)
        blob = b"".join(evs)
        m = rng.random()
        if m < 0.55:
            chunks = evs
        elif m < 0.8:
            step = rng.randrange(5, 300)
            chunks = sc.rechunk(blob, list(range(step, len(blob), step)))
        else:
            chunks = sc.rechunk(blob, [rng.randrange(1, max(2, len(blob))) for _ in range(rng.randrange(0, 9))])
        out.append([c for c in chunks if c])
    return out


def _recut(rng, chunks):
    """the same bytes in other network chunks: whole events, a fixed stride, or a few arbitrary cuts"""
    import sse_cases as sc
    m = rng.random()
    if m < 0.5:
        return chunks
    blob = b"".join(chunks)
    if m < 0.75:
        step = rng.randrange(7, 700)
        return [c for c in sc.rechunk(blob, list(range(step, len(blob), step))) if c]
    return [c for c in sc.rechunk(blob, [rng.randrange(1, max(2, len(blob))) for _ in range(rng.randrange(1, 9))]) if c]


def shaped_streams(gen: str, n: int, seed: int):
    """`openai`: realistic OpenAI chunks (synth.openai_stream: id / created / model on every event, role and finish chunks, pieces
    of varying length with escapes and raw UTF-8); `c3`: the benchmark's own 64-byte deltas (synth.sse_batch).  Both with the
    usage event and [DONE], 1..k events per chunk or recut at arbitrary bytes."""
    import numpy as np
    from llmapigateway_b200 import synth
    rng = random.Random(seed)
    if gen == "openai":
        nrng = np.random.default_rng(seed)
        truths = synth._usage_truths(n, seed)
        out = []
        for s_ in range(n):
            epc = rng.choice([(1, 1), (1, 4), (2, 2), (1, 9)])
            out.append(_recut(rng, synth.openai_stream(nrng, rng.randrange(1, 60), truths[s_], "chatcmpl-%08x" % rng.randrange(2**32), epc)))
        return out
    n_events = rng.choice([8, 16, 48, 96])
    b = synth.sse_batch(n_streams=n, n_events=n_events, seed=seed, events_per_chunk=rng.choice([1, 1, 2, 8]),
                        with_usage=rng.random() < 0.9, with_done=rng.random() < 0.9)
    return [_recut(rng, b.stream_chunks(s_)) for s_ in range(n)]


SKELETONS = [   # %n = a number spelling, %s = a string value; every batch repeats a few of these so that they become templates
    '{"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n},"model":%s,"provider":%s}',
    '{"choices": [], "usage": {"prompt_tokens": %n, "completion_tokens": %n, "total_tokens": %n, "cost": %n}, "model": %s}',
    '{"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n,"cost":%n},"choices":[{"index":0,"delta":{"content":%s},"finish_reason":null}]}',
    '{"id":%s,"choices":[{"index":0,"delta":{},"finish_reason":"stop","usage":{"prompt_tokens":%n}}],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n}}',
    '{"x":{"usage":{"prompt_tokens":%n,"completion_tokens":%n}},"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n},"model":%s}',
    '{"choices":[],"usage":{"prompt_tokens":%n,"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n},"model":%s}',
    '{"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n},"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n},"model":%s}',
    '{"choices":[],"model":%s,"model":%s,"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n}}',
    '{"choices":[],"usage":{"completion_tokens_details":{"reasoning_tokens":%n,"prompt_tokens":%n},"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n,"prompt_tokens_details":{"cached_tokens":%n,"cost":%n}},"model":%s}',
    '{"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n,"completion_tokens_details":null,"prompt_tokens_details":{"cached_tokens":%n}},"provider":%s}',
    '{"choices":[],"usage":null,"model":%s,"provider":%s,"cost":%n}',
    '{"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n,"cost":%n,"cost_details":{"upstream_inference_cost":%n},"is_byok":false},"model":%s,"provider":%s}',
    '{"choices":[{"index":0,"message":{"role":"assistant","content":%s}}],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n}}',
    '{"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n,"reasoning_tokens":%n,"cached_tokens":%n},"model":%s}',
    '{"choices":[],"usage":{"total_tokens":%n,"completion_tokens":%n,"prompt_tokens":%n,"cost":%n},"provider":%s,"model":%s}',
    '{"model":%s,"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n,"completion_tokens_details":{"reasoning_tokens":%n,"accepted_prediction_tokens":%n},"prompt_tokens_details":{"cached_tokens":%n,"audio_tokens":%n}},"choices":[],"provider":%s}',
    '{"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n},"model":{"name":%s},"provider":[%s]}',
    '{"choices":[],"usage":[{"prompt_tokens":%n}],"model":%s}',
    '{"choices":[],"usage":{"prompt_tokens":{"v":%n},"completion_tokens":[%n,%n],"total_tokens":%n},"model":%s}',
    '{"error":{"message":%s,"code":%n},"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n}}',
    '{"choices":[],"usage":{"prompt_tokens":%n,"completion_tokens":%n,"total_tokens":%n},"code":%n,"model":%s}',
]


def skeleton_streams(n_streams: int, seed: int):
    """Usage events of odd shapes, each shape repeated across the batch with other values (so that it is learnt as a template and
    then FOLLOWED): keys in other places and orders, repeated keys, usage-like keys where get_token_usage does not look, containers
    and null where numbers go, spaces inside the event."""
    import re
    import sse_cases as sc
    rng = random.Random(seed)
    shapes = rng.sample(SKELETONS, rng.randrange(2, 5))
    out = []
    for s_ in range(n_streams):
        evs = [sc.delta(rng.choice(["a", "hello", "x" * rng.randrange(1, 70)])) for _ in range(rng.randrange(1, 16))]
        for _ in range(1 if rng.random() < 0.85 else 2):
            shape = rng.choice(shapes) if rng.random() < 0.93 else rng.choice(SKELETONS)

            def fill(m):
                r = rng.random()
                if m.group(0) == "%n":
                    return rng.choice(NUMBERS) if r < 0.9 else (rng.choice(BAD_NUMBERS) if r < 0.94 else rng.choice(["null", "true", '"7"', "[1]", "{}"]))
                return '"' + (rng.choice(STRINGS) if r < 0.93 else rng.choice(BAD_STRINGS)) + '"' if r < 0.97 else rng.choice(["null", "12", "[]"])
            ev = re.sub(r"%[ns]", fill, shape)
            evs.append(("data: " + ev + "\n\n").encode("utf-8", errors="surrogatepass"))
            if rng.random() < 0.25:
                evs.append(sc.delta("more"))
        if rng.random() < 0.8:
            evs.append(sc.DONE)
        out.append(_recut(rng, evs))
    return out


def make_streams(gen: str, n: int, seed: int):
    """`gen` = one of GENERATORS"""
    import test_sse_gpu as G
    if gen in ("openai", "c3"):
        return shaped_streams(gen, n, seed)
    if gen == "skeleton":
        return skeleton_streams(n, seed)
    if gen == "random":
        return G._random_streams(n, seed)
    if gen == "template":
        return G._template_variant_streams(n, seed)
    return usage_variant_streams(n, seed)
