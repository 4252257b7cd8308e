"""Deterministic mode against the default paths on one GPU, 32-layer Llama-3-8B with synthetic weights.

Per round, one engine of each mode in turn (default first, then deterministic), so that the two alternate:
  - step time: cl_decode_greedy_batch over `--steps` steps at B = 1, 8 and 64 behind 512 and 4096 cached tokens
    (cl_seq_fake_fill), device-event time of the loop divided by the steps;
  - prefill wall time of a 128, 512 and 4096-token prompt into an empty sequence (the call ends in a synchronise);
  - the deterministic step again with CL_VERIFY_ONE_ROW=0, so that its one-row segments run the 4-warp instantiation of
    the multi-row attention instead of the one-warp one.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON document (and writes it to --out)."""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402
from oracle import oracle as oc  # noqa: E402

BATCHES = [1, 8, 64]
CONTEXTS = [512, 4096]
PROMPTS = [128, 512, 4096]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.splitlines()[0].split(",")])) if out else {}


def ids(n, vocab, salt):
    return np.array([(i * 7919 + 13 + salt * 104729) % (vocab - 3) + 3 for i in range(n)], np.int32)


def measure(deterministic, steps, one_row=True, prefill=True):
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["max_seq_len"] = 4096 + steps + 64
    res = {"step_ms": {}, "prefill_ms": {}}
    os.environ["CL_VERIFY_ONE_ROW"] = "1" if one_row else "0"
    with eng.Engine(model=cfg, seed=1, max_batch=64, max_seqs=64, deterministic=deterministic) as e:
        V = e.cfg["vocab_size"]
        for ctx in CONTEXTS:
            for B in BATCHES:
                ss = [e.seq_create() for _ in range(B)]
                for s in ss:
                    e.seq_fake_fill(s, ctx)
                e.decode_greedy_batch(ss, [5] * B, 2)   # warm-up
                _, ms = e.decode_greedy_batch(ss, [7] * B, steps)
                res["step_ms"][f"B{B}_ctx{ctx}"] = ms / steps
                for s in ss:
                    e.seq_free(s)
        for n in PROMPTS if prefill else []:
            s = e.seq_create()
            e.prefill(s, ids(n, V, 1), want_logits=False)   # warm-up of this length's shapes
            e.seq_free(s)
            s = e.seq_create()
            t0 = time.perf_counter()
            e.prefill(s, ids(n, V, 2), want_logits=False)
            res["prefill_ms"][str(n)] = (time.perf_counter() - t0) * 1e3
            e.seq_free(s)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    doc = {"model": "llama3-8b synthetic, 32 layers", "card": card(), "rounds": []}
    for r in range(a.rounds):
        doc["rounds"].append({"default": measure(False, a.steps), "deterministic": measure(True, a.steps),
                              "deterministic_4warp": measure(True, a.steps, one_row=False, prefill=False)})
    doc["card_after"] = card()
    summary = {}
    for kind in ("step_ms", "prefill_ms"):
        for key in doc["rounds"][0]["default"][kind]:
            d = [r["default"][kind][key] for r in doc["rounds"]]
            t = [r["deterministic"][kind][key] for r in doc["rounds"]]
            summary[f"{kind}/{key}"] = {"default": min(d), "deterministic": min(t), "ratio": min(t) / min(d)}
            if kind == "step_ms":
                w = [r["deterministic_4warp"][kind][key] for r in doc["rounds"]]
                summary[f"{kind}/{key}"].update(deterministic_4warp=min(w), one_row_over_4warp=min(t) / min(w))
    doc["summary_min_over_rounds"] = summary
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
