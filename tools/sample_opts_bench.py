"""Cost of min_p and the presence / frequency penalties in the decode step's device draw, on Llama-3-8B (synthetic weights)
at contexts 512 and 4096.

For B = 1, 8 and 64 sequences, cl_decode_sample_batch runs `--steps` steps with Ollama's default sampler (temperature 0.8,
top_k 40, top_p 0.9, repeat_penalty 1.1 over 64 ids) and with those defaults plus min_p 0.05, presence_penalty 0.5 and
frequency_penalty 0.5 (cl_seq_set_sampling_ext).  Every call starts from fresh sequences at exactly the context under test
(seq_fake_fill, whose history ids are placeholders; the window fills with the drawn ids as the steps go), and the two
configurations alternate, in a new random order, over `--rounds` rounds.  A number is the mean over rounds of the device
time between the events around the steps and of the host wall clock around the call, per step; `delta_device_ms` compares
the options with the defaults.  The card's name, power limit and clocks are read in the same run.

    python tools/sample_opts_bench.py [--out profiles/h100_sample_opts.json] [--steps 64] [--rounds 6]
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

CONFIGS = ["defaults", "defaults+min_p+penalties"]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.splitlines()[0].split(",")])) if out else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=6)
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
    ext = eng.sampling_ext(min_p=0.05, presence_penalty=0.5, frequency_penalty=0.5)
    res = {"card_before": card(), "model": "llama3-8b (synthetic weights)", "steps_per_call": args.steps, "rounds": args.rounds,
           "sampler": "Ollama defaults: temperature 0.8, top_k 40, top_p 0.9, repeat_penalty 1.1, repeat_last_n 64",
           "options": "min_p 0.05, presence_penalty 0.5, frequency_penalty 0.5",
           "times": "ms per decode step: device = CUDA events around the steps of cl_decode_sample_batch, wall = host clock around it",
           "results": []}
    with eng.Engine(preset="llama3-8b", seed=1, max_batch=bmax, max_seqs=bmax, kv_pool_bytes=need * kv_tok) as e:
        for ctx in ctxs:
            for B in batches:
                first = [17 + b for b in range(B)]
                sps = [eng.ollama_default_sampling(seed=100 + b) for b in range(B)]

                def call(conf, steps):
                    seqs = [e.seq_create() for _ in range(B)]
                    for s in seqs:
                        e.seq_fake_fill(s, ctx)
                        if conf != "defaults":
                            e.set_sampling_ext(s, ext)
                    t0 = time.perf_counter()
                    _, dev_ms = e.decode_sample_batch(seqs, first, sps, steps)
                    wall = time.perf_counter() - t0
                    for s in seqs:
                        e.seq_free(s)
                    return dev_ms / steps, 1e3 * wall / steps

                for c in CONFIGS:                          # warm-up: graphs and modules
                    call(c, 4)
                acc = {c: ([], []) for c in CONFIGS}
                for _ in range(args.rounds):
                    for i in rng.permutation(len(CONFIGS)):
                        d, w = call(CONFIGS[i], args.steps)
                        acc[CONFIGS[i]][0].append(d)
                        acc[CONFIGS[i]][1].append(w)
                base_d = float(np.mean(acc["defaults"][0]))
                for conf, (d, w) in acc.items():
                    row = {"ctx": ctx, "B": B, "config": conf, "device_ms": float(np.mean(d)), "wall_ms": float(np.mean(w)),
                           "delta_device_ms": float(np.mean(d)) - base_d, "device_ms_rounds": [round(x, 4) for x in d]}
                    res["results"].append(row)
                    print(json.dumps(row), flush=True)
    res["card_after"] = card()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
