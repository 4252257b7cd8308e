"""Prefix cache: time to first token of a request whose prompt starts with a long prefix an earlier request already
prefilled, with the cache on and off, and how much of the remaining suffix prefill is attention.

    python tools/prefix_bench.py [--preset llama3-8b] [--prefix 4096] [--suffix 64] [--reps 5]

Each round sends one request with the prefix and a fresh suffix (greedy, one token) through the synchronous request
path; `prefill_ns` of its result is the time to first token.  The first request of an engine fills the cache and is not
counted.  Rounds alternate between an engine with the cache off and one with it on.  The suffix prefill's kernel
breakdown comes from CL_PREFILL_PROFILE=1 in a child process (the library prints it to stderr).  Prints one JSON line,
with the GPU's name and power limit beside the numbers.
"""
import argparse
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402


def _prompt(n, vocab, salt):
    return np.array([(i * 7919 + 13 + salt * 104729) % (vocab - 3) + 3 for i in range(n)], np.int32)


def _ttft(preset, prefix_cache, prefix, suffix, reps, salt0):
    c = eng.model_preset(preset)
    V = c["vocab_size"]
    base = _prompt(prefix, V, 1)
    out = []
    with eng.Engine(preset=preset, seed=1234, max_batch=1, prefix_cache=prefix_cache) as e:
        sp = eng.greedy(1, ignore_eos=True)
        e.generate_ids(np.concatenate([base, _prompt(suffix, V, salt0)]), sp)       # fills the cache
        for r in range(reps):
            res = e.generate_ids(np.concatenate([base, _prompt(suffix, V, salt0 + 1 + r)]), sp)
            out.append(res.prefill_ns / 1e6)
        ps = e.prefix_stats()
    return out, ps


def _profile_child(a):
    _ttft(a.preset, True, a.prefix, a.suffix, 1, 500)


def _suffix_profile(a):
    env = dict(os.environ, CL_PREFILL_PROFILE="1")
    r = subprocess.run([sys.executable, __file__, "--profile-child", "--preset", a.preset, "--prefix", str(a.prefix), "--suffix", str(a.suffix)],
                       env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[prefill profile]")]
    heads = [i for i, ln in enumerate(lines) if "on the device" in ln]
    if r.returncode or not heads:
        return dict(error=r.stderr[-2000:])
    block = lines[heads[-1]:]                       # the last prefill: the measured request's suffix
    total = float(re.search(r"([\d.]+) ms on the device", block[0]).group(1))
    kinds = {}
    for ln in block[1:]:
        m = re.match(r"\[prefill profile\]\s+(\S+)\s+n=\s*(\d+) total\s+([\d.]+) ms", ln)
        if m:
            kinds[m.group(1)] = round(float(m.group(3)), 4)
    attn = sum(v for k, v in kinds.items() if k.startswith("launch_attn_prefill"))
    return dict(path=block[0].split("] ", 1)[1].split(",")[0], device_ms=total, attention_ms=round(attn, 4),
                attention_share=round(attn / total, 4) if total else None, kernels_ms=kinds)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="llama3-8b")
    ap.add_argument("--prefix", type=int, default=4096)
    ap.add_argument("--suffix", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile-child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    os.environ.pop("CL_PREFIX_CACHE", None)         # the engines below choose explicitly
    if a.profile_child:
        _profile_child(a)
        return
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    runs = {"off": [], "on": []}
    stats = None
    for rnd in range(2):                            # two alternating rounds per setting
        for name in ("off", "on"):
            t, ps = _ttft(a.preset, name == "on", a.prefix, a.suffix, a.reps, 10 * rnd + (0 if name == "off" else 100))
            runs[name].append([round(x, 3) for x in t])
            if name == "on":
                stats = ps
    med = {k: round(float(np.median(sum(v, []))), 3) for k, v in runs.items()}
    out = dict(bench="prefix_bench", gpu=gpu, preset=a.preset, prefix_tokens=a.prefix, suffix_tokens=a.suffix,
               ttft_ms_median=med, speedup=round(med["off"] / med["on"], 2) if med["on"] else None, ttft_ms_runs=runs,
               prefix_stats_cache_on=stats, suffix_prefill_profile=_suffix_profile(a))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
