"""Speculative decoding over several sequences on Llama-3-8B (synthetic weights): one verify pass (cl_decode_verify_batch)
for B = 2, 4, 8, 16 sequences with k = 1, 3, 7, 15 drafts each, against one batched decode step (cl_decode_greedy_batch) at
the same B, at contexts 512 and 4096.  The card's name, power limit and clocks are read in the same run.

  - break-even: how many drafted tokens per sequence a pass must accept to beat single batched steps in time,
    pass / step - 1
  - tokens/s with always-right drafts, B (k + 1) / pass, and with always-wrong drafts, where each rejected pass is
    followed by the back-off's 8 batched steps, B (1 + 8) / (pass + 8 step).  Both follow from the measured pass and step
    times: a pass does the same work whatever it accepts.

Times are host wall clock around calls that end in a device synchronise, the mean of --reps calls after two warm-up calls.
Acceptance on real text is not measured here: the weights are synthetic.

    python tools/spec_batch_bench.py [--out profiles/h100_spec_batch.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from crowdllama_b200 import engine as eng  # noqa: E402

BACKOFF = 8        # engine.h kSpecBackoff
BS = (2, 4, 8, 16)
KS = (1, 3, 7, 15)
CTXS = (512, 4096)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def seqs(e, B, ctx):
    ss = [e.seq_create() for _ in range(B)]
    for s in ss:
        e.seq_fake_fill(s, ctx)
    return ss


def step_ms(e, B, ctx, n):
    ss = seqs(e, B, ctx)
    e.decode_greedy_batch(ss, [17] * B, 4)
    t0 = time.perf_counter()
    e.decode_greedy_batch(ss, [17] * B, n)
    t = time.perf_counter() - t0
    for s in ss:
        e.seq_free(s)
    return 1e3 * t / n


def pass_ms(e, B, ctx, k, reps):
    V = e.cfg["vocab_size"]
    rng = np.random.default_rng(B * 100 + k)
    ss = seqs(e, B, ctx)
    ts = []
    for i in range(reps + 2):
        ds = [rng.integers(0, V, k) for _ in range(B)]
        t0 = time.perf_counter()
        e.decode_verify_batch(ss, [17] * B, ds)
        if i >= 2:
            ts.append(time.perf_counter() - t0)
    for s in ss:
        e.seq_free(s)
    return 1e3 * float(np.mean(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_spec_batch.json")
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--steps", type=int, default=32)
    a = ap.parse_args()
    res = dict(metric="multi-sequence verify pass vs batched decode step, Llama-3-8B bf16 synthetic weights", card_before=card(),
               results={})
    e = eng.Engine(preset="llama3-8b", seed=1234, max_batch=max(BS), max_seqs=max(BS))
    for ctx in CTXS:
        for B in BS:
            st = step_ms(e, B, ctx, a.steps)
            pm = {k: pass_ms(e, B, ctx, k, a.reps) for k in KS if B * (k + 1) <= 128}   # one pass holds 128 rows
            r = dict(step_ms=st, pass_ms=pm,
                     break_even_accepted={k: max(0.0, pm[k] / st - 1.0) for k in pm},
                     step_tok_s=1e3 * B / st,
                     right_tok_s_derived={k: 1e3 * B * (k + 1) / pm[k] for k in pm},
                     wrong_tok_s_derived={k: 1e3 * B * (1 + BACKOFF) / (pm[k] + BACKOFF * st) for k in pm})
            res["results"][f"ctx{ctx}_B{B}"] = r
            print(json.dumps({"ctx": ctx, "B": B, **r}), flush=True)
    e.close()
    res["card_after"] = card()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
