"""Speculative decoding on Llama-3-8B (synthetic weights) at contexts 512 and 4096, with the card's name, power limit and
clocks read in the same run.  Speculation on and off alternate twice; every number is the mean of the two rounds.

  1. verify pass (cl_decode_verify) for k = 1, 3, 7, 15 against one B = 1 decode step: the break-even acceptance, i.e.
     how many drafted tokens a pass must accept to beat k + 1 single steps in time
  2. token level, against cl_decode_greedy: always-right drafts (the upper bound: the sequence's own greedy continuation)
     and always-wrong drafts (the lower bound: each rejected pass is followed by the back-off's single steps)
  3. request level: cl_generate_ids at B = 1, speculation off vs on, on a repetitive prompt, with the acceptance from
     cl_engine_spec_stats

Times are host wall clock around calls that end in a device synchronise (a verify pass's ~11 launches per layer are
enqueued eagerly, so their enqueue time counts), per pass or per token.  Acceptance on real text is not measured here:
the weights are synthetic.

    python tools/spec_bench.py [--out profiles/h100_spec.json] [--tokens 96]
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

BACKOFF = 8        # engine.h kSpecBackoff: single steps after a pass that accepted nothing
KS = (1, 3, 7, 15)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def wall(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def fresh(e, ctx):
    s = e.seq_create()
    e.seq_fake_fill(s, ctx)
    return s


def step_ms(e, ctx, n):
    s = fresh(e, ctx)
    e.decode_greedy(s, 17, 4)
    t, _ = wall(lambda: e.decode_greedy(s, 17, n))
    e.seq_free(s)
    return 1e3 * t / n


def verify_ms(e, ctx, k, n):
    s = fresh(e, ctx)
    V = e.cfg["vocab_size"]
    rng = np.random.default_rng(k)
    x = 17
    e.decode_verify(s, x, rng.integers(0, V, k), None, 0)
    ts = []
    for _ in range(n):
        t, (ids, _) = wall(lambda: e.decode_verify(s, x, rng.integers(0, V, k), None, 0))
        ts.append(t)
        x = int(ids[-1])
    e.seq_free(s)
    return 1e3 * float(np.mean(ts))


def token_rates(e, ctx, k, n_tokens):
    """tokens/s: cl_decode_greedy, always-right drafts, always-wrong drafts with the back-off (and acceptance seen)."""
    V = e.cfg["vocab_size"]
    s = fresh(e, ctx)
    cont, _ = e.decode_greedy(s, 17, n_tokens + 16)            # the sequence's own continuation: the right drafts
    e.seq_free(s)
    s = fresh(e, ctx)
    t_base, _ = wall(lambda: e.decode_greedy(s, 17, n_tokens))
    e.seq_free(s)
    # always right: x0 = 17, then the continuation; drafts are the next k ids of it
    s = fresh(e, ctx)
    chain = [17] + [int(i) for i in cont]
    pos, emitted, acc, passes, t0 = 0, 0, 0, 0, time.perf_counter()
    while emitted < n_tokens:
        d = chain[pos + 1:pos + 1 + k]
        ids, _ = e.decode_verify(s, chain[pos], d, None, 0)
        acc += len(ids) - 1
        passes += 1
        emitted += len(ids)
        if ids.tolist() != chain[pos + 1:pos + 1 + len(ids)]:  # a near-tie flip between the two paths: stop following
            break
        pos += len(ids)
    t_right = time.perf_counter() - t0
    right_emitted = emitted
    e.seq_free(s)
    # always wrong: a rejected pass, then BACKOFF single steps
    s = fresh(e, ctx)
    x, emitted, t0 = 17, 0, time.perf_counter()
    rng = np.random.default_rng(3)
    while emitted < n_tokens:
        ids, _ = e.decode_verify(s, x, (rng.integers(1, V, k) + x) % V, None, 0)
        ids2, _ = e.decode_greedy(s, int(ids[-1]), BACKOFF)
        emitted += len(ids) + BACKOFF
        x = int(ids2[-1])
    t_wrong = time.perf_counter() - t0
    e.seq_free(s)
    return dict(greedy_tok_s=n_tokens / t_base, right_tok_s=right_emitted / t_right, right_accept=acc / (passes * k),
                wrong_tok_s=emitted / t_wrong)


def repetitive_prompt(n, V):
    block = np.array([(i * 7919 + 101) % (V - 3) + 3 for i in range(64)], np.int32)
    return np.resize(block, n)


def request_rate(e, ctx, n_tokens):
    p = repetitive_prompt(ctx, e.cfg["vocab_size"])
    e.generate_ids(p[:64], eng.greedy(4, ignore_eos=True))
    before = e.spec_stats()
    t, r = wall(lambda: e.generate_ids(p, eng.greedy(n_tokens, ignore_eos=True)))
    after = e.spec_stats()
    d = {k: after[k] - before[k] for k in ("verify_passes", "tokens_drafted", "tokens_accepted", "tokens_emitted")}
    return dict(decode_tok_s=r.n_generated / (r.decode_ns * 1e-9), request_s=t, **d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_spec.json")
    ap.add_argument("--tokens", type=int, default=96)
    ap.add_argument("--passes", type=int, default=24)
    a = ap.parse_args()
    res = dict(metric="speculative decoding, Llama-3-8B bf16 synthetic weights, B = 1", card_before=card(), rounds=[])
    engines = {"off": eng.Engine(preset="llama3-8b", seed=1234, max_batch=2, max_seqs=2, start_scheduler=True),
               "on": eng.Engine(preset="llama3-8b", seed=1234, max_batch=2, max_seqs=2, start_scheduler=True, speculate=7)}
    for rnd in range(2):
        for mode in ("off", "on"):
            e = engines[mode]
            row = dict(round=rnd, speculate=mode, ctx={})
            for ctx in (512, 4096):
                c = dict(step_ms=step_ms(e, ctx, 64))
                if mode == "on":
                    c["verify_ms"] = {k: verify_ms(e, ctx, k, a.passes) for k in KS}
                    c["token_level"] = {k: token_rates(e, ctx, k, a.tokens) for k in (3, 7, 15)}
                c["request"] = request_rate(e, ctx, a.tokens)
                row["ctx"][ctx] = c
                print(json.dumps({"round": rnd, "mode": mode, "ctx": ctx, **c}), flush=True)
            res["rounds"].append(row)
    res["card_after"] = card()
    summ = {}
    for ctx in (512, 4096):
        on = [r["ctx"][ctx] for r in res["rounds"] if r["speculate"] == "on"]
        off = [r["ctx"][ctx] for r in res["rounds"] if r["speculate"] == "off"]
        st = float(np.mean([c["step_ms"] for c in on + off]))
        vm = {k: float(np.mean([c["verify_ms"][k] for c in on])) for k in KS}
        summ[ctx] = dict(
            step_ms=st,
            verify_ms=vm,
            verify_over_step={k: vm[k] / st for k in KS},
            # a pass emits a + 1 tokens; it beats single steps when (a + 1) * step > verify time
            break_even_accepted={k: max(0.0, vm[k] / st - 1.0) for k in KS},
            token_level={k: {m: float(np.mean([c["token_level"][k][m] for c in on])) for m in on[0]["token_level"][k]} for k in (3, 7, 15)},
            request_off_tok_s=float(np.mean([c["request"]["decode_tok_s"] for c in off])),
            request_on_tok_s=float(np.mean([c["request"]["decode_tok_s"] for c in on])),
            request_on_acceptance=float(sum(c["request"]["tokens_accepted"] for c in on) / max(1, sum(c["request"]["tokens_drafted"] for c in on))),
        )
    res["summary"] = summ
    for e in engines.values():
        e.close()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps(summ, indent=1))


if __name__ == "__main__":
    main()
