"""Context shift (cl_seq_shift) at Llama-3-8B sizes on one GPU, against recomputing the kept tokens.

Configurations, alternated and repeated (--rounds):
  in_place  prefix cache off: a sequence of 8192 cached tokens (cl_seq_fake_fill) discards 4064 after the first 4; every
            kept page holds private K, which kv_shift_kernel rotates in place (V moves only in the partial page).
  cow       prefix cache on: the same after a real 8192-token prefill, so every page is indexed and the shift first copies
            each page it writes (copy-on-write): K and V of every kept row are read and written.
  prefill   the alternative: cl_prefill of the 4128 kept tokens on a fresh sequence.
Each call is timed on the host around the call, which ends in a stream synchronise.  The kernel alone is timed with CUDA
events over repeated launches (cl_op_kv_shift) at the same per-layer shape on --kernel-layers layers, in place.

Algorithmic bytes are the K (and V) rows the shift must read and write, from the shapes; GB/s is set against the
3039.7 GB/s copy rate measured on the same card (profiles/h100_bench.json, roofline.peak).

    python tools/shift_bench.py [--rounds 3] [--out profiles/h100_context_shift.json]

The card's name, power limit and SM clock are read in the same run and written beside the numbers.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402

COPY_GBS = 3039.7           # measured HBM copy rate (profiles/h100_bench.json roofline.peak, NVIDIA H100 80GB HBM3)
LEN, KEEP, DELTA, P = 8192, 4, 4064, 32


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def shift_bytes(n_layers, n_kv, hd, cow):
    """Bytes the shift reads and writes: every kept row after KEEP moves (K rotated; V too when its page is copied, else only
    the rows of the partial page), plus the unrotated rows [0, KEEP % P) of a copied first page."""
    row = n_layers * n_kv * hd * 2
    moved = LEN - KEEP - DELTA
    partial = min(P, LEN - DELTA - KEEP // P * P) - KEEP % P if KEEP % P else 0
    if cow:
        return 2 * (2 * moved + 2 * (KEEP % P)) * row
    return 2 * (moved + partial) * row


def ids(n, salt, vocab):
    return ((np.arange(n, dtype=np.int64) * 7919 + 13 + salt * 104729) % (vocab - 3) + 3).astype(np.int32)


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-layers", type=int, default=8)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_context_shift.json"))
    a = ap.parse_args()
    res = {"card": card(), "shape": {"preset": "llama3-8b", "len": LEN, "num_keep": KEEP, "discard": DELTA, "page_size": P,
                                      "kept_tokens": LEN - DELTA}, "copy_gbs": COPY_GBS, "runs": []}
    kw = dict(preset="llama3-8b", seed=1234, max_batch=2, max_seqs=3, page_size=P)
    off = eng.Engine(**kw)
    on = eng.Engine(prefix_cache=True, **kw)
    cfg = off.cfg
    V, L, KV, D = cfg["vocab_size"], cfg["n_layers"], cfg["n_kv_heads"], cfg["head_dim"]

    def in_place():
        s = off.seq_create()
        off.seq_fake_fill(s, LEN)
        ms = timed(lambda: off.seq_shift(s, KEEP, DELTA))
        off.seq_free(s)
        return ms

    def cow(salt):
        s = on.seq_create()
        on.prefill(s, ids(LEN, salt, V), want_logits=False)   # new ids every time: all 256 pages indexed
        ms = timed(lambda: on.seq_shift(s, KEEP, DELTA))
        on.seq_free(s)
        return ms

    def prefill(salt):
        s = off.seq_create()
        ms = timed(lambda: off.prefill(s, ids(LEN - DELTA, salt, V), want_logits=False))
        off.seq_free(s)
        return ms

    in_place(), cow(1000), prefill(1000)   # warm-up: workspaces, first launches
    for r in range(a.rounds):
        for name, fn in (("in_place", in_place), ("cow", lambda: cow(r)), ("prefill", lambda: prefill(r))):
            ms = fn()
            row = {"round": r, "config": name, "ms": round(ms, 4)}
            if name != "prefill":
                nbytes = shift_bytes(L, KV, D, name == "cow")
                row.update(algorithmic_bytes=nbytes, gbs=round(nbytes / ms * 1e-6, 1), frac_of_copy=round(nbytes / ms * 1e-6 / COPY_GBS, 4))
            res["runs"].append(row)
            print(json.dumps(row), flush=True)
    off.close()
    on.close()
    # the kernel alone, in place, at the same per-layer shape
    rng = np.random.default_rng(0)
    kl = a.kernel_layers
    k = (rng.standard_normal((kl, LEN, KV, D)).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    v = (rng.standard_normal((kl, LEN, KV, D)).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    ang = DELTA * np.power(5e5, -2.0 * np.arange(D // 2) / D)
    row_cs = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)
    _, _, kms = eng.op_kv_shift(k, v, P, KEEP, DELTA, row_cs, iters=a.kernel_iters)
    nbytes = shift_bytes(kl, KV, D, False)
    res["kernel"] = {"layers": kl, "iters": a.kernel_iters, "ms": round(kms, 5), "algorithmic_bytes": nbytes,
                     "gbs": round(nbytes / kms * 1e-6, 1), "frac_of_copy": round(nbytes / kms * 1e-6 / COPY_GBS, 4),
                     "ms_scaled_to_32_layers": round(kms * L / kl, 4)}
    print(json.dumps(res["kernel"]), flush=True)
    for name in ("in_place", "cow", "prefill"):
        ms = [x["ms"] for x in res["runs"] if x["config"] == name]
        res[name + "_ms_median"] = float(np.median(ms))
    res["card"] = res["card"] or card()
    Path(a.out).write_text(json.dumps(res, indent=1) + "\n")
    print(json.dumps({k_: res[k_] for k_ in ("card", "in_place_ms_median", "cow_ms_median", "prefill_ms_median")}))


if __name__ == "__main__":
    main()
