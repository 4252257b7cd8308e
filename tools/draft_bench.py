"""Speculative decoding with a draft model: Llama-3-8B target, Llama-3.2-1B draft, synthetic weights, contexts 512 and 4096,
with the card's name, power limit and SM clocks read in the same run.

  1. the draft step at B = 1, 8 and 32 (a standalone engine of the draft's shape running the same step the drafter runs),
     against its bytes bound: weights + the K/V it reads, over the data sheet's 3.35 TB/s
  2. the draft's catch-up pass of 1, 2 and 512 rows (cl_draft_model with k = 1 on a mirror that holds the rest)
  3. the whole round, cl_draft_model plus cl_decode_verify, for k = 1, 3, 5, 7, 15, and the target's B = 1 step; break-even
     accepted tokens per round = round / step - 1, and the derived tokens/s of always-right and always-wrong drafts
  4. end to end: cl_generate_ids of a self-draft (the 8B target drafting for itself) against the same request without a
     draft; it is not expected to be faster

Times are host wall clock around calls that end in a device synchronise.  Acceptance on real text is not measured: the
weights are synthetic.

    python tools/draft_bench.py [--out profiles/h100_draft.json]
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

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
BACKOFF = 8                 # engine.h kSpecBackoff
CTXS = (512, 4096)
KS = (1, 3, 5, 7, 15)
WINDOW = 8192


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def wall(fn):
    t0 = time.perf_counter()
    r = fn()
    return time.perf_counter() - t0, r


def ids(n, salt):
    return [(i * 7919 + 13 + salt * 104729) % 128000 + 3 for i in range(n)]


def weight_bytes(c):
    q, kv = c["n_heads"] * c["head_dim"], c["n_kv_heads"] * c["head_dim"]
    return 2 * (2 * c["vocab_size"] * c["d_model"]) + c["n_layers"] * 2 * ((q + 2 * kv) * c["d_model"] + c["d_model"] * q + 3 * c["d_ff"] * c["d_model"])


def kv_bytes_per_token(c):
    return 2 * c["n_layers"] * c["n_kv_heads"] * c["head_dim"] * 2


def draft_steps(res, n_steps):
    with eng.Engine(preset="llama3.2-1b", seed=2, max_batch=32, max_seqs=32, context_length=WINDOW,
                    kv_pool_bytes=32 * WINDOW * 32768) as d:
        c = d.cfg
        for ctx in CTXS:
            for B in (1, 8, 32):
                ss = [d.seq_create() for _ in range(B)]
                for s in ss:
                    d.seq_fake_fill(s, ctx)
                first = [17 + b for b in range(B)]
                run = (lambda: d.decode_greedy(ss[0], first[0], n_steps)) if B == 1 else (lambda: d.decode_greedy_batch(ss, first, n_steps))
                run()
                t, _ = wall(run)
                ms = 1e3 * t / n_steps
                bound = 1e3 * (weight_bytes(c) + B * (ctx + n_steps) * kv_bytes_per_token(c)) / HBM_BYTES_PER_S
                row = dict(ctx=ctx, B=B, step_ms=ms, bytes_bound_ms=bound, share_of_bound=bound / ms)
                res["draft_step"].append(row)
                print(json.dumps(row), flush=True)
                for s in ss:
                    d.seq_free(s)


def rounds(res, reps):
    with eng.Engine(preset="llama3-8b", seed=1, max_batch=4, max_seqs=4, speculate=15, context_length=WINDOW,
                    kv_pool_bytes=4 * WINDOW * 131072, draft_preset="llama3.2-1b", draft_seed=2) as e:
        for ctx in CTXS:
            # the target's step at this context
            s = e.seq_create()
            e.seq_fake_fill(s, ctx)
            e.decode_greedy(s, 17, 4)
            t, _ = wall(lambda: e.decode_greedy(s, 17, 64))
            step = 1e3 * t / 64
            e.seq_free(s)
            # catch-up passes: a mirror that holds the window takes r new rows, drafting d1 only
            s = e.seq_create()
            hist = ids(ctx, 1)
            e.draft_model([s], [hist], [1])
            catch = {}
            for r in (1, 2, 512):
                ts = []
                for rep in range(reps if r < 512 else min(reps, 3)):
                    hist = hist + ids(r, 100 + rep + r)
                    dt, _ = wall(lambda: e.draft_model([s], [hist], [1]))
                    ts.append(dt)
                catch[r] = 1e3 * float(np.median(ts))
            e.seq_free(s)
            # whole rounds behind ctx cached tokens
            for k in KS:
                s = e.seq_create()
                e.seq_fake_fill(s, ctx)
                hist = ids(ctx + 1, 3)
                e.draft_model([s], [hist], [k])   # the mirror's first catch-up is the whole window: not timed
                td, tv = [], []
                for _ in range(reps):
                    a, d = wall(lambda: e.draft_model([s], [hist], [k]))
                    b, (out, _) = wall(lambda: e.decode_verify(s, hist[-1], d[0]))
                    td.append(a)
                    tv.append(b)
                    hist = hist + [int(i) for i in out]
                e.seq_free(s)
                draft_ms, verify_ms = 1e3 * float(np.median(td)), 1e3 * float(np.median(tv))
                rnd = draft_ms + verify_ms
                row = dict(ctx=ctx, k=k, draft_ms=draft_ms, verify_ms=verify_ms, round_ms=rnd, target_step_ms=step,
                           break_even_accepted=rnd / step - 1,
                           derived_always_right_tok_s=(k + 1) / rnd * 1e3,
                           derived_always_wrong_tok_s=(1 + BACKOFF) / (rnd + BACKOFF * step) * 1e3,
                           target_alone_tok_s=1e3 / step)
                res["round"].append(row)
                print(json.dumps(row), flush=True)
            res["catch_up"].append(dict(ctx=ctx, rows_ms={str(r): v for r, v in catch.items()}))
            print(json.dumps(res["catch_up"][-1]), flush=True)
        res["spec_stats"] = e.spec_stats()
        res["draft_stats"] = e.draft_stats()


def end_to_end(res, n_new):
    prompt = ids(512, 7)
    sp = eng.greedy(n_new, ignore_eos=True)
    for mode in ("plain", "self_draft", "plain", "self_draft"):
        kw = dict(speculate=7, draft_preset="llama3-8b", draft_seed=1) if mode == "self_draft" else {}
        with eng.Engine(preset="llama3-8b", seed=1, max_batch=4, max_seqs=4, context_length=WINDOW,
                        kv_pool_bytes=4 * WINDOW * 131072, **kw) as e:
            e.generate_ids(prompt, eng.greedy(16, ignore_eos=True))
            t, g = wall(lambda: e.generate_ids(prompt, sp))
            row = dict(mode=mode, tokens=int(g.n_generated), wall_s=t, tok_s=g.n_generated / t, spec=e.spec_stats(),
                       draft=e.draft_stats())
            res["end_to_end"].append(row)
            print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_draft.json")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--tokens", type=int, default=128)
    a = ap.parse_args()
    res = dict(card=card(), target="llama3-8b (synthetic)", draft="llama3.2-1b (synthetic)", contexts=list(CTXS),
               timing="host wall clock around calls that end in a device synchronise; medians",
               hbm_bytes_per_s_datasheet=HBM_BYTES_PER_S, acceptance_on_real_text="not measured: no real weights",
               draft_step=[], catch_up=[], round=[], end_to_end=[])
    draft_steps(res, a.steps)
    rounds(res, a.reps)
    end_to_end(res, a.tokens)
    res["card_after"] = card()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
