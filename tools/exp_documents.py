"""Times the two document calls of the engine, which no benchmark covers: Engine.documents_usage and
Engine.documents_error_detail on a few thousand seeded non-streaming responses.  One JSON line: the library that was loaded
(LGW_NATIVE_LIB selects another build of it), the GPU's name and power limit, and per call the median and minimum wall time of
the Engine method and of the C call alone (both end in a stream synchronise).
    python tools/exp_documents.py [--docs 4096] [--reps 30]
"""
import argparse
import json
import random
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def seeded_docs(n, seed):
    rng = random.Random(seed)
    docs = []
    for i in range(n):
        if i % 4 == 3:
            docs.append(json.dumps({"error": {"message": "upstream failed " + "x" * rng.randrange(8, 200), "code": rng.choice([429, 500, 503])}}).encode())
        else:
            p, c = rng.randrange(1, 9000), rng.randrange(1, 4000)
            docs.append(json.dumps({"id": f"gen-{i}", "choices": [{"message": {"role": "assistant", "content": "w " * rng.randrange(16, 700)}}],
                                    "usage": {"prompt_tokens": p, "completion_tokens": c, "total_tokens": p + c, "cost": rng.random() / 100}}).encode())
    return docs


def wall_ms(fn, reps, warmup=3):
    out = []
    for it in range(reps + warmup):
        t0 = time.perf_counter()
        fn()
        if it >= warmup:
            out.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": round(float(np.median(out)), 4), "min_ms": round(float(min(out)), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    import llmapigateway_b200 as L
    from llmapigateway_b200 import _abi, _native, rewrite as rw
    from llmapigateway_b200.engine import _ptr
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    eng = L.Engine(max_streams=64, max_step_chunks=1024, max_step_bytes=1 << 20)
    docs = seeded_docs(args.docs, seed=7)
    buf, off = rw.pack_bodies(docs)
    n, stride, lib = len(docs), 4096, eng._lib
    usage, err = (_abi.DocUsage * n)(), (_abi.DocError * n)()
    text = np.zeros(n * stride, dtype=np.uint8)
    launches0 = eng.launch_count()
    res = {"library": str(_native.LIB_PATH), "gpu": q.stdout.strip(), "docs": n, "bytes": int(off[-1]), "reps": args.reps,
           "documents_usage": wall_ms(lambda: eng.documents_usage(docs), args.reps),
           "documents_usage_c_call": wall_ms(lambda: eng._ck(lib.lgw_documents_usage(eng._h, _ptr(buf), _ptr(off), n, usage), "documents_usage"), args.reps),
           "documents_error_detail": wall_ms(lambda: eng.documents_error_detail(docs, stride), args.reps),
           "documents_error_detail_c_call": wall_ms(lambda: eng._ck(lib.lgw_documents_error_detail(eng._h, _ptr(buf), _ptr(off), n, err, _ptr(text), stride),
                                                                    "documents_error_detail"), args.reps)}
    res["launches"] = eng.launch_count() - launches0
    res["rows_with_usage"] = sum(1 for rows, _ in eng.documents_usage(docs) if rows[-1].get("total_tokens"))
    print(json.dumps(res))
    eng.close_engine()


if __name__ == "__main__":
    main()
