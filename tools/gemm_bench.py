"""wgmma GEMM microbenchmark at the Llama-3-8B prefill shapes (T tokens): ms and TFLOP/s per projection.
    python tools/gemm_bench.py [T] [iters]"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402

T = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
ITERS = int(sys.argv[2]) if len(sys.argv) > 2 else 10        # a few hundred = sustained (power-limited) clocks
rng = np.random.default_rng(0)
tot_ms = tot_fl = 0.0
for name, n, k in (("qkv", 6144, 4096), ("o", 4096, 4096), ("gate|up", 28672, 4096), ("down", 4096, 14336)):
    x = rng.integers(0, 1 << 16, size=(T, k), dtype=np.uint16) & 0xBF7F
    w = rng.integers(0, 1 << 16, size=(n, k), dtype=np.uint16) & 0xBF7F
    _, ms = eng.op_gemm_bf16(x, w, iters=ITERS)
    fl = 2.0 * T * n * k
    tot_ms += ms; tot_fl += fl
    print(json.dumps({"T": T, "iters": ITERS, "proj": name, "n": n, "k": k, "ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1)}), flush=True)
print(json.dumps({"T": T, "layer_ms": round(tot_ms, 4), "tflops": round(tot_fl / tot_ms / 1e9, 1)}), flush=True)
