"""Measure the GPU's practical peaks and write MEASURED_PEAKS.json, which bench.py reads for its roofline fractions.

    python tools/measure_peaks.py [out.json]        (default: MEASURED_PEAKS.json at the repository root)

hbm_gbs: device-to-device copy of 1 Gi bf16 elements (read + write bytes), best of 10.
bf16_tflops_burst / _sustained: 8192^3 bf16 matmul, best of 10 / mean over 4 s back to back.
The card's name, power limit and SM clock limit are stored beside the numbers.
"""
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    best = float("inf")
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        best = min(best, ev[0].elapsed_time(ev[1]) * 1e-3)
    return best


def main(out):
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    a = torch.empty(1 << 30, dtype=torch.bfloat16, device="cuda")
    b = torch.empty_like(a)
    b.copy_(a)
    hbm = 2 * a.numel() * 2 / timed(lambda: b.copy_(a), 10) / 1e9
    del a, b
    n = 8192
    x = torch.randn(n, n, dtype=torch.bfloat16, device="cuda")
    y = torch.randn(n, n, dtype=torch.bfloat16, device="cuda")
    flop = 2.0 * n ** 3
    for _ in range(3):
        x @ y
    burst = flop / timed(lambda: x @ y, 10) / 1e12
    torch.cuda.synchronize()
    k, t0 = 0, time.time()
    while time.time() - t0 < 4.0:
        for _ in range(10):
            x @ y
        torch.cuda.synchronize()
        k += 10
    sustained = flop * k / (time.time() - t0) / 1e12
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    d = {"hbm_gbs": round(hbm, 1), "bf16_tflops_burst": round(burst, 1), "bf16_tflops_sustained": round(sustained, 1),
         "gpu": q[0] if q else torch.cuda.get_device_name()}
    Path(out).write_text(json.dumps(d) + "\n")
    print(json.dumps(d))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else str(ROOT / "MEASURED_PEAKS.json"))
