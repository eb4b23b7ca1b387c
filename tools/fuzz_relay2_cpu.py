"""Differential fuzz campaign of the bulk SSE kernels on the CPU box (test aid, not a product path).

The kernels of csrc/relay2.cuh are run through the SIMT emulator (tests/host_relay.py) in their bulk mode (mode 0) and in the
exact sequential mode (mode 1) on streams from the generators of tests/sse_generators.py (the two of tests/test_sse_gpu.py with
fresh seeds, usage events whose numbers and strings take every spelling JSON allows, odd usage skeletons, OpenAI- and C3-shaped
streams), and both are compared with the oracle (oracle/sse_oracle.py, the restatement of request_handler.py:21-150 and
chat_logging.py:87-150,233-272).  Engine geometries (blocks, tiles per warp) and step counts vary per round; with --slices
every round also cuts its bulk steps into 1..14 slices the way lgw_sse_step cuts a host-buffer step.

    python tools/fuzz_relay2_cpu.py --rounds 40 --procs 6 --seed 1000 [--slices]

Prints one line per round; a divergence is reported with the generator, seed and stream so that it can be replayed
(`--replay gen:seed:n_steps:geometry:cold[:slices]`).
"""
from __future__ import annotations

import argparse
import json
import multiprocessing as mp
import os
import random
import sys
import traceback
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

GEOMETRIES = [(2, 0), (3, 1), (1, 0), (5, 2), (4, 1)]
GENERATORS = ["random", "template", "usage", "usage", "openai", "c3", "skeleton", "skeleton"]

from sse_generators import make_streams  # noqa: E402


def one_round(job):
    gen, seed, n_steps, geo, n_streams, cold, n_slices = job
    import test_sse_gpu as G
    from golden_io import canon_rows
    from host_relay_sliced import SlicedHostBulkEngine
    from llmapigateway_b200 import _abi
    from oracle.sse_oracle import run_stream
    tag = f"{gen}:{seed}:{n_steps}:{geo}:{int(cold)}:{n_slices}"
    try:
        nb, tpw = GEOMETRIES[geo]
        cap = int(os.environ.get("LGW_FUZZ_CARRY_CAP", "4096"))     # a small carry capacity stresses the overflow paths (bulk vs sequential only)
        eng = SlicedHostBulkEngine(max_streams=2048, carry_cap=cap, n_blocks=nb, tiles_per_warp=tpw, n_slices=n_slices)
        try:
            streams = make_streams(gen, n_streams, seed)
            if not cold:                      # warm templates: a first batch of the same generator, other seed
                G._run_all(eng, make_streams(gen, 64, seed + 1), 0, 1, seed=3)
            s_fast, r_fast, e_fast = G._run_all(eng, streams, 0, n_steps, seed=seed)
            counters = eng.counters()
            s_seq, r_seq, e_seq = G._run_all(eng, streams, 1, n_steps, seed=seed)
            n_ok = 0
            for i, (a, b) in enumerate(zip(s_fast, s_seq)):
                where = f"{tag} stream {i}"
                assert e_fast[i] == e_seq[i], where + " emitted bytes: bulk != sequential"
                assert bytes(a)[:64] == bytes(b)[:64], where + " state header: bulk != sequential"
                if a.flags & _abi.SF_REC_VALID:
                    assert a.rec.exotic == b.rec.exotic, where + " exotic flag"
                    if not a.rec.exotic:
                        assert canon_rows([_abi.usage_rec_to_dict(a.rec)]) == canon_rows([_abi.usage_rec_to_dict(b.rec)]), where + " usage record: bulk != sequential"
                if (a.flags | b.flags) & _abi.SF_CARRY_OVERFLOW:      # an event outgrew the engine's carry capacity: the reference buffers without
                    continue                                           #   bound, so only bulk == sequential is checked for such a stream
                relay, tap = run_stream(streams[i])
                assert e_fast[i] == relay.emitted, where + " emitted bytes != oracle"
                assert (a.phase == _abi.PHASE_FAILED) == relay.failed, where + " verdict != oracle"
                if not relay.failed and not a.n_exotic:
                    got = [json.loads(r[2])[0] for r in r_fast if r[0] == i]
                    if a.flags & _abi.SF_EMITTED_ANY:
                        got.append(json.loads(canon_rows([_abi.usage_rec_to_dict(a.rec)]))[0])
                    assert canon_rows(got) == canon_rows(tap.rows), where + " usage rows != oracle"
                    assert (not (a.flags & _abi.SF_A_USAGE_BOUND)) == relay.end_raises, where + " end_raises != oracle"
                    n_ok += 1
            assert r_fast == r_seq, tag + " mid-stream rows: bulk != sequential"
            return tag, True, f"{n_ok}/{n_streams} compared with the oracle; {counters}"
        finally:
            eng.close_engine()
    except Exception:
        return tag, False, traceback.format_exc(limit=3)


def transcript_round(job):
    """The same generators through the transcript tap (k_text_extract / scan / pack on the emulator, TranscriptBook on the host)
    against the oracle's llm_response_accum at every write_log call."""
    gen, seed, n_steps, geo, n_streams, cold, _ = job
    import test_transcript_gpu as T
    from host_relay import HostBulkEngine
    from llmapigateway_b200 import _abi
    from llmapigateway_b200.transcripts import decode_text
    from oracle.sse_oracle import run_stream
    tag = f"{gen}:{seed}:{n_steps}:{geo}:{int(cold)}"
    try:
        nb, tpw = GEOMETRIES[geo]
        eng = HostBulkEngine(max_streams=2048, carry_cap=8192, n_blocks=nb, tiles_per_warp=tpw)
        eng.enable_transcripts()
        try:
            streams = make_streams(gen, n_streams, seed)
            rng = random.Random(seed)
            scheds = [[0] + sorted(set(rng.randrange(1, max(2, len(c))) for _ in range(n_steps - 1))) if len(c) > 1 else [0] for c in streams]
            res = T.run_streams(eng, streams, scheds)
            n_cmp = 0
            for i, (chunks, (snaps, flags, emitted_any, seq_steps)) in enumerate(zip(streams, res)):
                relay, tap = run_stream(chunks)
                where = f"{tag} stream {i}"
                if relay.failed:
                    assert snaps == [], where + " transcript of a failed stream"
                    continue
                if flags & _abi.TF_EXOTIC:
                    continue
                assert [decode_text(t) for t in snaps] == tap.transcripts, where + " transcripts != oracle"
                n_cmp += 1
            return tag, True, f"{n_cmp}/{n_streams} transcripts compared with the oracle"
        finally:
            eng.close_engine()
    except Exception:
        return tag, False, traceback.format_exc(limit=3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--procs", type=int, default=4)
    ap.add_argument("--seed", type=int, default=1000)
    ap.add_argument("--streams", type=int, default=300)
    ap.add_argument("--replay", default=None)
    ap.add_argument("--gens", default=None, help="comma-separated subset of the generators")
    ap.add_argument("--transcripts", action="store_true", help="check the transcript tap instead of the relay / usage results")
    ap.add_argument("--slices", action="store_true", help="cut every bulk step into 1..14 slices (drawn per round), as lgw_sse_step does")
    args = ap.parse_args()
    if args.replay:
        gen, seed, n_steps, geo, *rest = args.replay.split(":")
        fn = transcript_round if args.transcripts else one_round
        cold, n_slices = (rest + ["0", "1"][len(rest):])[:2]
        print(*fn((gen, int(seed), int(n_steps), int(geo), args.streams, bool(int(cold)), int(n_slices))), sep="\n")
        return 0
    if args.gens:
        GENERATORS[:] = args.gens.split(",")
    rng = random.Random(args.seed)
    jobs = []
    for r in range(args.rounds):
        jobs.append((rng.choice(GENERATORS), args.seed * 1000 + r, rng.choice([1, 1, 2, 3, 5]), rng.randrange(len(GEOMETRIES)), args.streams, rng.random() < 0.25,
                     rng.randrange(1, 15) if args.slices else 1))
    from host_relay_sliced import lib
    lib()                                   # build the emulator libraries once, before the workers start
    # every round in a process of its own: the emulator ABORTS on a divergent collective or a deadlock (a finding, not a crash of
    # the campaign), and a pool worker that dies takes its job with it
    import subprocess
    from concurrent.futures import ThreadPoolExecutor

    def spawn(job):
        gen, seed, n_steps, geo, n_streams, cold, n_slices = job
        tag = f"{gen}:{seed}:{n_steps}:{geo}:{int(cold)}:{n_slices}"
        r = subprocess.run([sys.executable, __file__, "--replay", tag, "--streams", str(n_streams)] + (["--transcripts"] if args.transcripts else []),
                           capture_output=True, text=True)
        lines = [l for l in r.stdout.splitlines() if l.strip()]
        if r.returncode != 0 or len(lines) < 3:
            return tag, False, "process ended with status %d: %s" % (r.returncode, (r.stderr or r.stdout)[-400:])
        return tag, lines[1] == "True", "\n".join(lines[2:])
    bad = 0
    with ThreadPoolExecutor(args.procs) as pool:
        for tag, ok, msg in pool.map(spawn, jobs):
            print(("ok   " if ok else "FAIL ") + tag + "  " + msg, flush=True)
            bad += 0 if ok else 1
    print(f"{len(jobs) - bad}/{len(jobs)} rounds clean")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
