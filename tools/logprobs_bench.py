"""Cost of per-token log-probabilities in the decode step, on Llama-3-8B (synthetic weights) at contexts 512 and 4096.

For B = 1, 8 and 64 sequences, cl_decode_greedy_batch runs `--steps` steps with no sequence armed, one armed and every
one armed, at top_n 0 and 20.  Every call starts from fresh sequences at exactly the context under test (seq_fake_fill),
so no configuration runs at a longer context than another, and the configurations run in a new random order in each of
`--rounds` rounds.  A number is the mean over rounds of the host wall clock around the call (which ends in a device
synchronise and includes the record ring's copy back) and of the device time between the events around the steps, per
step; `delta_wall_ms` and `delta_device_ms` compare each configuration with the unarmed one.  The card's name, power limit and
clocks are read in the same run.  --bench-lines DIR adds the JSON lines of bench.py runs made in the same session
(files DIR/*.json, e.g. the parent and this tree alternating) to the profile as they are.

Estimate from bytes, not measured: an armed row reads its 513 KB logits row once more (V = 128 256 fp32), at most about
66 MB per step at B = 128: tens of microseconds against a step of several milliseconds.

    python tools/logprobs_bench.py [--out profiles/h100_logprobs.json] [--steps 64] [--rounds 5]
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

CONFIGS = [("none", -1), ("one", 0), ("one", 20), ("all", 0), ("all", 20)]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--bench-lines", default="")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--ctxs", default="512,4096")
    args = ap.parse_args()
    batches = [int(b) for b in args.batches.split(",")]
    ctxs = [int(c) for c in args.ctxs.split(",")]
    bmax = max(batches)
    rng = np.random.default_rng(0)
    cfg = eng.model_preset("llama3-8b")
    kv_tok = 2 * cfg["n_layers"] * cfg["n_kv_heads"] * cfg["head_dim"] * 2
    need = bmax * (max(ctxs) + args.steps + 64)
    res = {"card_before": card(), "model": "llama3-8b (synthetic weights)", "steps_per_call": args.steps, "rounds": args.rounds,
           "times": "ms per decode step: wall = host clock around cl_decode_greedy_batch, device = CUDA events around its steps",
           "results": []}
    with eng.Engine(preset="llama3-8b", seed=1, max_batch=bmax, max_seqs=bmax, kv_pool_bytes=need * kv_tok) as e:
        for ctx in ctxs:
            for B in batches:
                first = [17 + b for b in range(B)]

                def call(who, top_n, steps):
                    seqs = [e.seq_create() for _ in range(B)]
                    for b, s in enumerate(seqs):
                        e.seq_fake_fill(s, ctx)
                        e.set_logprobs(s, top_n if (who == "all" or (who == "one" and b == 0)) else -1)
                    t0 = time.perf_counter()
                    _, dev_ms = e.decode_greedy_batch(seqs, first, steps)
                    wall = time.perf_counter() - t0
                    for s in seqs:
                        e.seq_free(s)
                    return 1e3 * wall / steps, dev_ms / steps

                call("all", 20, 4)                          # warm-up: graphs, modules, the record ring copy
                acc = {c: ([], []) for c in CONFIGS}
                for _ in range(args.rounds):
                    for i in rng.permutation(len(CONFIGS)):
                        w, d = call(*CONFIGS[i], args.steps)
                        acc[CONFIGS[i]][0].append(w)
                        acc[CONFIGS[i]][1].append(d)
                none_w, none_d = float(np.mean(acc[("none", -1)][0])), float(np.mean(acc[("none", -1)][1]))
                for (who, top_n), (w, d) in acc.items():
                    row = {"ctx": ctx, "B": B, "armed": who, "top_n": top_n, "wall_ms": float(np.mean(w)), "device_ms": float(np.mean(d)),
                           "delta_wall_ms": float(np.mean(w)) - none_w, "delta_device_ms": float(np.mean(d)) - none_d,
                           "wall_ms_rounds": [round(x, 4) for x in w]}
                    res["results"].append(row)
                    print(json.dumps(row), flush=True)
    res["card_after"] = card()
    if args.bench_lines:
        res["bench_py"] = {p.name: json.loads(p.read_text().strip().splitlines()[-1]) for p in sorted(Path(args.bench_lines).glob("*.json"))}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
