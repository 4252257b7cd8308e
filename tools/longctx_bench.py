"""Long-context measurements -> profiles/h100_longctx.json (or --out).

kernel: the split-KV wgmma prefill attention (variant 2) against the mma.sync kernel (variant 0) at pos0 + T in
        {16384, 32768, 65536, 131072} x T in {16, 300, 4096}, Llama-3-8B attention (32 q heads, 8 kv heads, d 128),
        alternating rounds; ms per launch (CUDA events over `iters` launches) and TFLOP/s of the causal flops.
engine: the 32-layer Llama-3.1-8B synthetic model with context_length 131072: decode step time (B = 1 and 4) behind
        fake-filled caches of 32K / 64K / 128K tokens, a single-sequence verify pass (k = 7) against a step at 128K, and
        the wall time of prefilling a 32K / 64K / 128K-token prompt as the scheduler chunks it (cl_generate_ids, 1 token).
The card's name, power limit and SM clocks are read in the same run.

    python tools/longctx_bench.py [--rounds 3] [--iters 5] [--skip-engine] [--out PATH]
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
from oracle import oracle as oc  # noqa: E402

H, KV, D = 32, 8, 128


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    vals = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else []
    return dict(zip(q.split(","), vals))


def causal_flops(pos0, T):
    """4 H D per (query, visible key): S = Q K^T and O = P V"""
    keys = T * pos0 + T * (T + 1) / 2
    return 4.0 * H * D * keys


def kernel_bench(rounds, iters):
    rng = np.random.default_rng(0)
    out = []
    for n_tok in (16384, 32768, 65536, 131072):
        k = oc.np_bf16_from_f32(rng.standard_normal((n_tok, KV, D), dtype=np.float32))
        v = oc.np_bf16_from_f32(rng.standard_normal((n_tok, KV, D), dtype=np.float32))
        for T in (16, 300, 4096):
            q = oc.np_bf16_from_f32(rng.standard_normal((T, H * D), dtype=np.float32))
            pos0 = n_tok - T
            ms = {0: [], 2: []}
            ns = 1
            for _ in range(rounds):
                for variant in (2, 0):
                    _, used, _, t = eng.op_attn_prefill_long(q, k, v, pos0, H, KV, D, variant=variant, iters=iters)
                    ms[variant].append(t)
                    if variant == 2:
                        ns = used
            fl = causal_flops(pos0, T)
            row = dict(n_tok=n_tok, T=T, nsplit=ns, flops=fl)
            for variant, name in ((2, "split_kv"), (0, "mma_sync")):
                m = float(np.median(ms[variant]))
                row[name] = dict(ms_median=round(m, 4), ms_min=round(min(ms[variant]), 4), ms_max=round(max(ms[variant]), 4),
                                 tflops=round(fl / (m * 1e-3) / 1e12, 1))
            row["speedup"] = round(row["mma_sync"]["ms_median"] / row["split_kv"]["ms_median"], 2)
            print(json.dumps(row), flush=True)
            out.append(row)
    return out


def engine_bench(iters):
    cfg = dict(oc.PRESETS["llama3.1-8b"])
    res = {"model": "llama3.1-8b synthetic, 32 layers, context_length 131072", "decode": [], "verify": None, "prefill": []}
    with eng.Engine(model=cfg, seed=1, max_batch=4, context_length=131072) as e:
        res["kv_pool_pages"] = e.stats()["kv_pages_total"]
        for ctx in (32768, 65536, 131072 - 64):
            for B in (1, 4):
                seqs = [e.seq_create() for _ in range(B)]
                try:
                    for s in seqs:
                        e.seq_fake_fill(s, ctx - 2 * iters - 32)
                    toks = [1] * B
                    if B == 1:
                        e.decode_step(seqs[0], 1)
                    else:
                        e.decode_step_batch(seqs, toks)
                    t0 = time.perf_counter()
                    for _ in range(iters):
                        if B == 1:
                            e.decode_step(seqs[0], 1)
                        else:
                            e.decode_step_batch(seqs, toks)
                    ms = (time.perf_counter() - t0) * 1e3 / iters
                    res["decode"].append(dict(ctx=ctx, B=B, ms_per_step=round(ms, 3)))
                    print(json.dumps(res["decode"][-1]), flush=True)
                except eng.EngineError as ex:
                    res["decode"].append(dict(ctx=ctx, B=B, error=str(ex)))
                    print(json.dumps(res["decode"][-1]), flush=True)
                finally:
                    for s in seqs:
                        e.seq_free(s)
        s = e.seq_create()
        e.seq_fake_fill(s, 131072 - 64)
        e.decode_step(s, 1)
        ids = np.array([5, 6, 7, 8, 9, 10, 11], np.int32)
        t0 = time.perf_counter()
        e.decode_step(s, 2)
        step_ms = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        e.decode_verify(s, 3, ids)
        ver_ms = (time.perf_counter() - t0) * 1e3
        res["verify"] = dict(ctx=131072 - 64, k=7, verify_ms=round(ver_ms, 3), step_ms=round(step_ms, 3))
        print(json.dumps(res["verify"]), flush=True)
        e.seq_free(s)
    with eng.Engine(model=cfg, seed=1, max_batch=1, context_length=131072, start_scheduler=True) as e:
        rng = np.random.default_rng(1)
        for n in (32768, 65536, 131072 - 8):
            ids = rng.integers(0, cfg["vocab_size"], n).astype(np.int32)
            t0 = time.perf_counter()
            r = e.generate_ids(ids, eng.greedy(1, ignore_eos=True))
            res["prefill"].append(dict(tokens=n, wall_s=round(time.perf_counter() - t0, 3), generated=int(r.n_generated)))
            print(json.dumps(res["prefill"][-1]), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--skip-engine", action="store_true")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_longctx.json"))
    a = ap.parse_args()
    res = {"card": card(), "kernel": kernel_bench(a.rounds, a.iters)}
    res["engine"] = "not measured" if a.skip_engine else engine_bench(10)
    res["card_after"] = card()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(res, indent=1))
    print("wrote", a.out)


if __name__ == "__main__":
    main()
