"""Cost of sampled decoding: the step tail's device sampler against greedy decoding and the host sampler.

    python tools/sample_bench.py                 # both parts
    python tools/sample_bench.py --part step     # device ms per step, cl_decode_greedy_batch vs cl_decode_sample_batch
    python tools/sample_bench.py --part req      # scheduler: concurrent cl_generate_ids clients, CL_DEVICE_SAMPLE 1 / 0 / greedy

Llama-3-8B shapes with synthetic weights.  Sampled requests use Ollama's defaults (temperature 0.8, top-k 40, top-p 0.9,
repeat penalty 1.1 over 64 tokens) with fixed seeds.  The request part runs every configuration in its own process,
alternating them, because CL_DEVICE_SAMPLE is read when the engine is created.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402

KV_TOKEN_BYTES = 2 * 32 * 8 * 128 * 2          # Llama-3-8B: K and V, 32 layers, 8 kv heads x 128 dims, bf16


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                      # the numbers stay valid; say that the card could not be read
        return f"unknown ({ex})"


def step_part(batches, ctx, steps):
    mb = max(batches)
    with eng.Engine(preset="llama3-8b", seed=1234, max_batch=mb, max_seqs=mb,
                    kv_pool_bytes=mb * (ctx + 4 * steps + 64) * KV_TOKEN_BYTES) as e:
        for B in batches:
            seqs = [e.seq_create() for _ in range(B)]
            for s in seqs:
                e.seq_fake_fill(s, ctx)
            firsts = [17 + b for b in range(B)]
            sps = [eng.ollama_default_sampling(seed=1000 + b) for b in range(B)]
            e.decode_greedy_batch(seqs, firsts, 4)
            e.decode_sample_batch(seqs, firsts, sps, 4)
            res = {}
            for rep in range(2):                 # alternate the two, twice
                _, g = e.decode_greedy_batch(seqs, firsts, steps)
                _, s = e.decode_sample_batch(seqs, firsts, sps, steps)
                res.setdefault("greedy", []).append(g / steps)
                res.setdefault("sampled", []).append(s / steps)
            g, s = min(res["greedy"]), min(res["sampled"])
            print(json.dumps({"part": "step", "B": B, "ctx": ctx, "greedy_ms": round(g, 4), "sampled_ms": round(s, 4),
                              "sampler_ms": round(s - g, 4), "runs": {k: [round(x, 4) for x in v] for k, v in res.items()}}),
                  flush=True)
            for s_ in seqs:
                e.seq_free(s_)


def req_child(mode, clients_list, prompt_len, new_tokens):
    """One process: one engine, each concurrency level once after a warm-up wave."""
    mb = 128
    e = eng.Engine(preset="llama3-8b", seed=1234, max_batch=mb, max_seqs=mb, start_scheduler=True,
                   kv_pool_bytes=mb * (prompt_len + new_tokens + 64) * KV_TOKEN_BYTES)
    V = e.cfg["vocab_size"]

    def sampling(i):
        s = eng.greedy(new_tokens, ignore_eos=True) if mode == "greedy" else eng.ollama_default_sampling(seed=7 + i,
                                                                                                        max_new_tokens=new_tokens)
        s.ignore_eos = 1
        return s

    def wave(n):
        out = [None] * n

        def run(i):
            p = [(i * 7919 + j * 104729 + 13) % V for j in range(prompt_len)]
            out[i] = e.generate_ids(p, sampling(i))

        th = [threading.Thread(target=run, args=(i,)) for i in range(n)]
        t0 = time.perf_counter()
        for t in th:
            t.start()
        for t in th:
            t.join()
        return time.perf_counter() - t0, out

    wave(8)
    for n in clients_list:
        st0 = e.stats()
        wall, out = wave(n)
        st1 = e.stats()
        toks = sum(r.n_generated for r in out)
        steps = st1["sched_decode_steps"] - st0["sched_decode_steps"]
        print(json.dumps({"part": "req", "mode": mode, "clients": n, "req_s": round(n / wall, 3), "tok_s": round(toks / wall, 1),
                          "mean_batch": round((st1["tokens_generated"] - st0["tokens_generated"]) / max(steps, 1), 2),
                          "mean_step_ms": round((st1["sched_decode_ns"] - st0["sched_decode_ns"]) / max(steps, 1) / 1e6, 3),
                          "wall_s": round(wall, 3)}), flush=True)
    e.close()


def req_part(clients_list, prompt_len, new_tokens, runs):
    modes = [("device", "1"), ("host", "0"), ("greedy", "1")]
    for rep in range(runs):
        for mode, flag in modes:
            env = dict(os.environ, CL_DEVICE_SAMPLE=flag)
            cmd = [sys.executable, __file__, "--child", mode, "--clients", ",".join(map(str, clients_list)),
                   "--prompt", str(prompt_len), "--tokens", str(new_tokens)]
            r = subprocess.run(cmd, env=env, capture_output=True, text=True)
            for line in r.stdout.splitlines():
                if line.startswith("{"):
                    d = json.loads(line)
                    d["run"] = rep
                    print(json.dumps(d), flush=True)
            if r.returncode:
                print(r.stderr[-2000:], file=sys.stderr)
                raise SystemExit(f"{mode} run failed ({r.returncode})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", default="all", choices=["all", "step", "req"])
    ap.add_argument("--batches", default="1,8,32,64,128")
    ap.add_argument("--ctx", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--clients", default="64,128")
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    clients = [int(x) for x in a.clients.split(",")]
    if a.child:
        req_child(a.child, clients, a.prompt, a.tokens)
        return
    print(json.dumps({"card": card()}), flush=True)
    if a.part in ("all", "step"):
        step_part([int(x) for x in a.batches.split(",")], a.ctx, a.steps)
    if a.part in ("all", "req"):
        req_part(clients, a.prompt, a.tokens, a.runs)


if __name__ == "__main__":
    main()
