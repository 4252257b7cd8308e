"""Workload for ncu: Llama-3-8B, 4096-token prefill, then a few eager (non-graph) decode steps.
Usage (Nsight Compute on the GPU machine):
  CL_GRAPH=0 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:'gemv|attn_decode|step_|embed_kernel' \
      -s 164 -c 330 --csv --log-file gpurun_out/launches.csv python tools/step_profile.py 3
"""
import os
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from crowdllama_b200 import engine as eng  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
ctx = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
preset = sys.argv[3] if len(sys.argv) > 3 else "llama3-8b"
os.environ.setdefault("CL_GRAPH", "0")
with eng.Engine(preset=preset, seed=1234, max_batch=1) as e:
    V = e.cfg["vocab_size"]
    ids = np.array([(i * 7919 + 13) % V for i in range(ctx)], np.int32)
    s = e.seq_create()
    lg = e.prefill(s, ids)
    out, ms = e.decode_greedy(s, int(lg.argmax()), steps)
    print("decoded", out.tolist(), "ms/step", ms / steps)
