"""Time Engine.documents_text (lgw_documents_text: k_docs_text -> k_text_scan -> k_docs_text_pack) against the host doing what the
reference's tap thread does for the same documents: json.loads plus the choices walk (chat_logging.py:123-139).

    python tools/bench_documents_text.py [--reps 20]

Two workloads: 1 024 OpenAI-shaped completion documents of about 4 KiB, and 64 documents of 256 KiB.  Prints one JSON line per
workload with the GPU's name and power limit (device time from CUDA events, wall time of the whole call incl. copies)."""
from __future__ import annotations

import argparse
import json
import random
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def documents(n: int, size: int, seed: int) -> list[bytes]:
    rng = random.Random(seed)
    words = ["the ", "model ", "answer ", "é ", "中文 ", "\\n", "\\\"q\\\" ", "😀 ", "\\u00e9 ", "tokens "]
    out = []
    for i in range(n):
        head = {"id": "chatcmpl-%d" % i, "object": "chat.completion", "created": 1700000000 + i, "model": "openai/gpt-4o-mini"}
        tail = {"usage": {"prompt_tokens": rng.randint(10, 5000), "completion_tokens": rng.randint(10, 2000), "total_tokens": 9999,
                          "prompt_tokens_details": {"cached_tokens": 0}, "completion_tokens_details": {"reasoning_tokens": 0}, "cost": 0.0012}}
        skeleton = json.dumps({**head, "choices": [{"index": 0, "message": {"role": "assistant", "content": ""}, "finish_reason": "stop"}], **tail},
                              ensure_ascii=False)
        room = max(0, size - len(skeleton.encode()))
        content = []
        used = 0
        while used < room:
            w = rng.choice(words)
            content.append(w)
            used += len(w.encode())
        doc = skeleton.replace('"content": ""', '"content": "%s"' % "".join(content), 1)
        out.append(doc.encode())
    return out


def host_walk(docs):
    out = []
    for d in docs:
        doc = json.loads(d.decode("utf-8"))
        accum = ""
        for choice in doc.get("choices", []):
            if "delta" in choice and "content" in choice["delta"]:
                if choice["delta"]["content"]:
                    accum += choice["delta"]["content"]
            elif "message" in choice and "content" in choice["message"]:
                if choice["message"]["content"]:
                    accum += choice["message"]["content"]
        if "error" in doc:
            accum += d.decode("utf-8")
        out.append(accum.encode("utf-8", "surrogatepass"))
    return out


def gpu_info():
    try:
        import torch
        name = torch.cuda.get_device_name(0)
    except Exception:
        name = "unknown"
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import llmapigateway_b200 as L
    name, power = gpu_info()
    eng = L.Engine(max_streams=4)
    for label, n, size in (("1024 x 4 KiB", 1024, 4096), ("64 x 256 KiB", 64, 256 << 10)):
        docs = documents(n, size, seed=n)
        got = eng.documents_text(docs)                           # warm-up: grows the scratch once
        want = host_walk(docs)
        assert [t for t, _ in got] == want, "device text differs from the host walk"
        dev, wall = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            eng.documents_text(docs)
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(eng.documents_text_last_ms())
        host = []
        for _ in range(max(3, args.reps // 4)):
            t0 = time.perf_counter()
            host_walk(docs)
            host.append((time.perf_counter() - t0) * 1e3)
        med = lambda xs: sorted(xs)[len(xs) // 2]
        print(json.dumps(dict(workload=label, bytes=sum(map(len, docs)), text_bytes=sum(map(len, want)), device_ms=round(med(dev), 4),
                              wall_ms=round(med(wall), 4), host_json_walk_ms=round(med(host), 4), reps=args.reps, gpu=name, power_limit=power)))
    eng.close_engine()


if __name__ == "__main__":
    main()
