"""Prefill attention microbenchmark: both kernels (0 = mma.sync, 1 = wgmma) at Llama-3-8B head geometry.
    python tools/attn_bench.py [T ...]      -> one JSON line per (T, variant): ms per launch, causal TFLOP/s"""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402

H, KV, HD = 32, 8, 128
rng = np.random.default_rng(0)
for T in [int(a) for a in sys.argv[1:]] or [1024, 4096]:
    bf = lambda shape, sc: ((rng.standard_normal(shape) * sc).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)  # noqa: E731
    q, k, v = bf((T, H * HD), 1.0), bf((T, KV, HD), 1.0), bf((T, KV, HD), 1.0)
    outs = {}
    for variant in (0, 1):
        try:
            out, ms = eng.op_attn_prefill_variant(q, k, v, H, KV, HD, variant, iters=5)
            flops = 4.0 * H * HD * T * (T + 1) / 2
            outs[variant] = out
            print(json.dumps({"T": T, "variant": variant, "ms": round(ms, 4), "tflops": round(flops / (ms * 1e-3) / 1e12, 1),
                              "finite": bool(np.isfinite(out).all())}), flush=True)
        except Exception as ex:  # noqa: BLE001
            print(json.dumps({"T": T, "variant": variant, "error": str(ex)}), flush=True)
    if len(outs) == 2:
        d = np.abs(outs[0] - outs[1])
        print(json.dumps({"T": T, "max_abs_diff_between_kernels": float(d.max()), "mean": float(d.mean())}), flush=True)
