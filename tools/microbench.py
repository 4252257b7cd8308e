"""GPU microbenchmarks (run on the box through gpurun): per-kernel GEMV bandwidth for both
variants at the Llama-3-8B shapes, then whole-step decode tok/s across engine switches.
Writes JSON lines to gpurun_out/microbench.jsonl."""
import json
import os
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402

OUT = ROOT / "gpurun_out"
OUT.mkdir(exist_ok=True)
HBM = 3350.0   # H100 SXM data sheet, GB/s


def emit(f, **kw):
    line = json.dumps(kw)
    print(line, flush=True)
    f.write(line + "\n")
    f.flush()


def gemv_sweep(f):
    rng = np.random.default_rng(0)
    for name, n, k in [("qkv", 6144, 4096), ("o", 4096, 4096), ("gateup", 28672, 4096), ("down", 4096, 14336),
                       ("lm_head", 128256, 4096)]:
        w = rng.integers(0, 1 << 16, size=(n, k), dtype=np.uint16) & 0xBFFF
        x = rng.standard_normal(k).astype(np.float32)
        for variant in (0, 1):
            try:
                y, ms = eng.op_gemv(w, x, variant=variant, iters=50)
                gbs = n * k * 2 / (ms * 1e-3) / 1e9
                emit(f, bench="gemv", shape=name, n=n, k=k, variant=variant, ms=round(ms, 5), gbs=round(gbs, 1),
                     frac=round(gbs / HBM, 4))
            except Exception as ex:  # noqa: BLE001
                emit(f, bench="gemv", shape=name, variant=variant, error=str(ex))


def decode_sweep(f, preset="llama3-8b", ctx=4096, steps=128):
    bytes_per_tok = None
    # (decode_path, environment): decode_path 2 = TMA-ring GEMV, 1 = LDG GEMV (per-op path)
    runs = [(2, dict(CL_PDL="1")), (2, dict(CL_PDL="0"))]
    if "full" in sys.argv:
        runs += [(1, dict(CL_PDL="0")), (1, dict(CL_PDL="1")), (2, dict(CL_PDL="1", CL_GRAPH="0"))]
    for spec in sys.argv:
        if "=" in spec and spec.startswith("CL_"):
            runs = [(2, dict(kv.split("=") for kv in spec.split(",")))] + runs[:1]
    for decode_path, env in runs:
        for k in ("CL_PDL", "CL_GRAPH"):
            os.environ.pop(k, None)
        os.environ.update(env)
        try:
            t0 = time.time()
            with eng.Engine(preset=preset, seed=1234, max_batch=1, decode_path=decode_path) as e:
                t_init = time.time() - t0
                c = e.cfg
                p_read = c["n_layers"] * ((c["n_heads"] + 2 * c["n_kv_heads"]) * c["head_dim"] * c["d_model"] +
                                          c["d_model"] * c["n_heads"] * c["head_dim"] + 3 * c["d_ff"] * c["d_model"] +
                                          2 * c["d_model"]) + c["d_model"] + c["vocab_size"] * c["d_model"]
                kv_tok = 2 * c["n_layers"] * c["n_kv_heads"] * c["head_dim"] * 2
                s = e.seq_create()
                prompt = np.array([(i * 7919 + 13) % c["vocab_size"] for i in range(ctx)], np.int32)
                t0 = time.time()
                # fill the cache cheaply: the prompt goes through the (slow, exact) token-wise path only
                # for a short prefix; the rest of the context is decode steps on device
                lg = e.prefill(s, prompt[:ctx - 64])          # tensor-core prefill
                t_prefill = time.time() - t0
                ids, ms_fill = e.decode_greedy(s, int(lg.argmax()), 64)
                t_fill = time.time() - t0
                ids, ms = e.decode_greedy(s, int(ids[-1]), steps)
                mean_ctx = ctx + steps / 2
                bytes_per_tok = 2 * p_read + kv_tok * (mean_ctx + 1)
                tps = steps / (ms * 1e-3)
                emit(f, bench="decode", preset=preset, ctx=ctx, steps=steps, decode_path=decode_path, env=env, ms_per_tok=round(ms / steps, 4),
                     tok_s=round(tps, 2), gbs=round(bytes_per_tok * tps / 1e9, 1),
                     frac=round(bytes_per_tok * tps / 1e9 / HBM, 4), init_s=round(t_init, 1), fill_s=round(t_fill, 1),
                     prefill_s=round(t_prefill, 3), fill_ms_per_tok=round(ms_fill / 64, 4), launches=e.stats()["kernel_launches"])
        except Exception as ex:  # noqa: BLE001
            emit(f, bench="decode", decode_path=decode_path, env=env, error=str(ex))


def gemm_sweep(f):
    """Prefill projections on wgmma (cl_op_gemm_bf16, T = 4096 tokens)."""
    rng = np.random.default_rng(0)
    T = 4096
    for name, n, k in [("qkv", 6144, 4096), ("o", 4096, 4096), ("gateup", 28672, 4096), ("down", 4096, 14336)]:
        x = (rng.integers(0, 1 << 16, size=(T, k), dtype=np.uint16) & 0xBF7F)
        w = (rng.integers(0, 1 << 16, size=(n, k), dtype=np.uint16) & 0xBF7F)
        try:
            _, ms = eng.op_gemm_bf16(x, w, iters=10)
            tf = 2.0 * T * n * k / (ms * 1e-3) / 1e12
            emit(f, bench="gemm_wgmma", shape=name, t=T, n=n, k=k, ms=round(ms, 4), tflops=round(tf, 1), frac_of_peak=round(tf / 989.0, 3))
        except Exception as ex:  # noqa: BLE001
            emit(f, bench="gemm_wgmma", shape=name, error=str(ex))


def batch_sweep(f, preset="llama3-8b", ctx=1024, steps=64):
    """Continuous-batching inner loop: B sequences advance together (cl_decode_greedy_batch)."""
    for B in [int(x) for x in os.environ.get("CL_BATCH_LIST", "1,2,4,8").split(",")]:
        try:
            with eng.Engine(preset=preset, seed=1234, max_batch=B) as e:
                V = e.cfg["vocab_size"]
                seqs, firsts = [], []
                for b in range(B):
                    s = e.seq_create()
                    lg = e.prefill(s, np.array([(i * 7919 + 13 + b) % V for i in range(ctx)], np.int32))
                    seqs.append(s)
                    firsts.append(int(lg.argmax()))
                ids, _ = e.decode_greedy_batch(seqs, firsts, 8)
                ids, ms = e.decode_greedy_batch(seqs, ids[-1], steps)
                emit(f, bench="batch_decode", preset=preset, batch=B, ctx=ctx, steps=steps, ms_per_step=round(ms / steps, 4),
                     tok_s=round(B * steps / (ms * 1e-3), 1))
        except Exception as ex:  # noqa: BLE001
            emit(f, bench="batch_decode", batch=B, error=str(ex))


if __name__ == "__main__":
    with open(OUT / "microbench.jsonl", "a") as f:
        if "gemv" in sys.argv or len(sys.argv) == 1:
            gemv_sweep(f)
        if "decode" in sys.argv or len(sys.argv) == 1:
            decode_sweep(f)
        if "batch" in sys.argv:
            batch_sweep(f)
        if "gemm" in sys.argv:
            gemm_sweep(f)
