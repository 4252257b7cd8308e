"""Host tier of the prefix cache (CL_PREFIX_CACHE_HOST_MIB) on one GPU.

1. Transfer rates: kv_spill_kernel / kv_fill_kernel (cl_op_kv_host_roundtrip) moving 1 / 16 / 256 Llama-3-8B / Mistral-7B
   pages (32 layers, 8 kv heads, head_dim 128, page 32: 4 MiB each), next to cudaMemcpyAsync of the same bytes between
   pinned host memory and HBM on the same card.
2. BASELINE config 5 (tools/evict_bench.py with the prefix cache on), tier off and on, alternated twice.
3. The same load with few enough clients that no request is preempted: no prompt is ever reused, so every spill is
   pure cost.

    python tools/host_tier_bench.py [--seconds 30] [--host-gib 16] [--out profiles/h100_prefix_host.json]

The card's name, power limit and SM clock are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def transfer_rates(iters):
    import torch
    L, KV, D, P = 32, 8, 128, 32
    page_bytes = 2 * L * KV * P * D * 2
    rows = []
    for n in (1, 16, 256):
        spill_ms, fill_ms = eng.op_kv_host_roundtrip(L, KV, D, P, n, iters=iters)
        nbytes = n * page_bytes
        h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        for _ in range(2):
            h.copy_(d, non_blocking=True)
            d.copy_(h, non_blocking=True)
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(iters):
            h.copy_(d, non_blocking=True)
        ev[1].record()
        for _ in range(iters):
            d.copy_(h, non_blocking=True)
        ev[2].record()
        torch.cuda.synchronize()
        d2h, h2d = ev[0].elapsed_time(ev[1]) / iters, ev[1].elapsed_time(ev[2]) / iters
        del h, d
        gbs = lambda ms: round(nbytes / (ms * 1e-3) / 1e9, 2)  # noqa: E731
        rows.append(dict(pages=n, bytes=nbytes, spill_kernel_ms=round(spill_ms, 4), spill_kernel_gb_s=gbs(spill_ms),
                         fill_kernel_ms=round(fill_ms, 4), fill_kernel_gb_s=gbs(fill_ms), memcpy_d2h_ms=round(d2h, 4),
                         memcpy_d2h_gb_s=gbs(d2h), memcpy_h2d_ms=round(h2d, 4), memcpy_h2d_gb_s=gbs(h2d)))
        print(json.dumps(rows[-1]), flush=True)
    return dict(shape=dict(n_layers=L, n_kv=KV, head_dim=D, page=P, page_bytes=page_bytes), iters=iters, rows=rows)


def evict_run(tier_mib, seconds, clients, check):
    env = dict(os.environ, CL_PREFIX_CACHE="1")
    env.pop("CL_PREFIX_CACHE_HOST_MIB", None)
    if tier_mib:
        env["CL_PREFIX_CACHE_HOST_MIB"] = str(tier_mib)
    cmd = [sys.executable, str(ROOT / "tools" / "evict_bench.py"), "--seconds", str(seconds), "--clients", str(clients),
           "--check", str(check)]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode:
        raise RuntimeError(f"evict_bench failed:\n{r.stdout}\n{r.stderr[-4000:]}")
    out = json.loads(r.stdout.strip().splitlines()[-1])
    out["host_tier_mib"] = tier_mib
    print(json.dumps({k: out[k] for k in ("host_tier_mib", "clients", "requests_per_s", "gen_tokens_per_s", "preemptions",
                                          "prefill_tokens")} | {"prefix_cache": out["prefix_cache"]}), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--host-gib", type=float, default=16.0)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--check", type=int, default=4)
    ap.add_argument("--quiet-clients", type=int, default=6, help="clients of the load in which nothing is preempted")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "h100_prefix_host.json"))
    a = ap.parse_args()
    mib = int(a.host_gib * 1024)
    res = dict(bench="host_tier_bench", card_before=card())
    res["transfer"] = transfer_rates(a.iters)
    res["config5"] = [evict_run(t, a.seconds, 64, a.check) for t in (0, mib, 0, mib)]
    res["never_reused"] = [evict_run(t, a.seconds, a.quiet_clients, a.check) for t in (0, mib)]
    res["card_after"] = card()
    Path(a.out).parent.mkdir(parents=True, exist_ok=True)
    Path(a.out).write_text(json.dumps(res, indent=1) + "\n")
    print(f"wrote {a.out}")


if __name__ == "__main__":
    main()
