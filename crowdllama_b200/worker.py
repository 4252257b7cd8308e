"""Worker peer stand-in: one process per GPU serving the reference's two stream protocols over TCP.

The reference's worker is a libp2p host (pkg/peer/peer.go); Go and libp2p are absent here, so this harness
keeps the *application* protocols and replaces the transport by plain TCP with a multistream-style first
line naming the protocol:
    "/crowdllama/inference/1.0.0\\n"  then one length-prefixed BaseMessage each way   (peer.go:190-256)
    "/crowdllama/metadata/1.0.0\\n"   then the worker writes its Resource JSON and closes (peer.go:284-316)
The handler behind the inference protocol is `handler.worker_api_handler(engine)` — the same closure shape
the Go cgo shim installs into Peer.APIHandler.

    python -m crowdllama_b200.worker --device 0 --port 9101 --preset llama3-8b --model-name llama3:8b
"""
from __future__ import annotations

import argparse
import os
import socketserver
import threading

from . import engine as eng
from . import handler as H
from .router import resource_from_engine

INFERENCE_PROTOCOL = "/crowdllama/inference/1.0.0"     # pkg/crowdllama/types.go:20
METADATA_PROTOCOL = "/crowdllama/metadata/1.0.0"       # pkg/crowdllama/types.go:16
STOP_PROTOCOL = "/crowdllama-b200/bench-stop/1.0.0"    # harness only: the load generator tells the worker peers it is done
STATS_PROTOCOL = "/crowdllama-b200/bench-stats/1.0.0"  # harness only: raw cl_engine_stats as JSON (preemptions, KV pages ...)


class _Stream:
    def __init__(self, sock):
        self.r = sock.makefile("rb")
        self.w = sock.makefile("wb")

    def read(self, n):
        return self.r.read(n)

    def write(self, b):
        n = self.w.write(b)
        self.w.flush()
        return n


class WorkerServer(socketserver.ThreadingTCPServer):
    allow_reuse_address = True
    daemon_threads = True
    request_queue_size = 256

    def __init__(self, addr, engine: "eng.Engine", peer_id: str, sampling=None):
        self.engine, self.peer_id = engine, peer_id
        self.api_handler = H.worker_api_handler(engine, sampling)
        self.served = 0
        self.stop_event = threading.Event()
        self._lock = threading.Lock()
        super().__init__(addr, _Conn)


class _Conn(socketserver.BaseRequestHandler):
    def handle(self):
        srv: WorkerServer = self.server
        s = _Stream(self.request)
        proto = s.r.readline().decode(errors="replace").strip()
        if proto == METADATA_PROTOCOL:
            s.write(resource_from_engine(srv.peer_id, srv.engine).to_json())
        elif proto == STOP_PROTOCOL:
            srv.stop_event.set()
        elif proto == STATS_PROTOCOL:
            import json
            s.write(json.dumps(srv.engine.stats()).encode())
        elif proto == INFERENCE_PROTOCOL:
            if H.handle_inference_stream(srv.api_handler, s, worker_mode=True):
                with srv._lock:
                    srv.served += 1


def draft_kwargs(draft_model: str | None, draft_seed: int | None) -> dict:
    """Engine keywords of --draft-model PRESET|DIR and --draft-seed: a directory is a checkpoint, anything else a preset."""
    if not draft_model:
        return {}
    kw = dict(draft_weights_path=draft_model) if os.path.isdir(draft_model) else dict(draft_preset=draft_model)
    if draft_seed is not None:
        kw["draft_seed"] = draft_seed
    return kw


def serve(device: int, port: int, preset: str, model_name: str, max_batch: int = 8, greedy_tokens: int = 0, host="127.0.0.1",
          ready_event=None, seed: int = 1234, tokenizer: str | None = None, chat_family: str | None = None, prefix_cache: bool = False,
          speculate: int = 0, speculate_batch: int = 1, prefix_cache_host_bytes: int = 0, context_shift: bool = False,
          num_keep: int = 4, context_length: int = 0, draft_model: str | None = None, draft_seed: int | None = None,
          deterministic: bool = False):
    e = eng.Engine(preset=preset, model_name=model_name, device=device, seed=seed, max_batch=max_batch, start_scheduler=True,
                   prefix_cache=prefix_cache, speculate=speculate, speculate_batch=speculate_batch,
                   prefix_cache_host_bytes=prefix_cache_host_bytes, context_shift=context_shift, num_keep=num_keep,
                   context_length=context_length, deterministic=deterministic, **draft_kwargs(draft_model, draft_seed))
    if tokenizer:
        e.load_tokenizer(tokenizer, chat_family)      # HF tokenizer.json instead of the byte-level fallback
    sampling = eng.greedy(greedy_tokens, ignore_eos=True) if greedy_tokens > 0 else None   # None = Ollama defaults
    srv = WorkerServer((host, port), e, peer_id=f"b200-worker-{device}", sampling=sampling)
    if ready_event is not None:
        ready_event.set()
    try:
        srv.serve_forever(poll_interval=0.2)
    finally:
        srv.server_close()
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--port", type=int, default=9101)
    ap.add_argument("--preset", default="llama3-8b")
    ap.add_argument("--model-name", default="llama3:8b")
    ap.add_argument("--max-batch", type=int, default=8)
    ap.add_argument("--greedy-tokens", type=int, default=0, help="> 0: force greedy with this num_predict (benchmarks)")
    ap.add_argument("--tokenizer", default=None, help="path of an HF tokenizer.json (default: byte-level fallback)")
    ap.add_argument("--chat-family", default=None, help="llama3 | mistral | zephyr | chatml (default: auto-detect)")
    ap.add_argument("--prefix-cache", action="store_true",
                    help="reuse the cached KV pages of earlier requests that share a prompt prefix (env CL_PREFIX_CACHE overrides)")
    ap.add_argument("--speculate", type=int, default=0,
                    help="1..15: a request decoding alone drafts up to this many ids from its own history and verifies them in "
                         "one pass (0 = off; env CL_SPECULATE overrides)")
    ap.add_argument("--speculate-batch", type=int, default=1,
                    help="1..min(max_batch, 32): with --speculate, up to this many running requests verify their drafts in one "
                         "pass (1 = only a request running alone; env CL_SPECULATE_BATCH overrides)")
    ap.add_argument("--prefix-cache-host-gib", type=float, default=0.0,
                    help="with --prefix-cache: GiB of pinned host memory that keeps evicted cached KV pages for reuse "
                         "(0 = off; env CL_PREFIX_CACHE_HOST_MIB overrides)")
    ap.add_argument("--context-shift", action="store_true",
                    help="a request that fills the context window discards half of its tokens after the first --num-keep and goes "
                         "on generating, instead of ending with done_reason \"length\" (env CL_CONTEXT_SHIFT overrides)")
    ap.add_argument("--num-keep", type=int, default=None,
                    help="with --context-shift: leading tokens a shift never discards (default 4; env CL_NUM_KEEP overrides)")
    ap.add_argument("--context-length", type=int, default=0,
                    help="the context window in tokens, up to 131072 (Ollama's num_ctx / OLLAMA_CONTEXT_LENGTH for the whole "
                         "worker; 0 = the model's default; env CL_CONTEXT_LENGTH overrides)")
    ap.add_argument("--draft-model", default=None,
                    help="with --speculate: a preset name or a model directory of the same vocabulary whose drafts the served "
                         "model verifies, in place of drafting from the request's own history (env CL_DRAFT_MODEL)")
    ap.add_argument("--draft-seed", type=int, default=None,
                    help="synthetic-weight seed of a preset --draft-model (default: the served model's seed)")
    ap.add_argument("--deterministic", action="store_true",
                    help="a request's output depends only on its prompt, settings and seed, not on what else the worker runs "
                         "(Llama-3-8B / Mistral-7B shapes; env CL_DETERMINISTIC overrides)")
    a = ap.parse_args()
    if a.prefix_cache_host_gib and not a.prefix_cache:
        ap.error("--prefix-cache-host-gib requires --prefix-cache")
    if a.draft_model and not a.speculate:
        ap.error("--draft-model requires --speculate")
    if a.num_keep is not None and not a.context_shift:
        ap.error("--num-keep requires --context-shift")
    print(f"worker on cuda:{a.device} port {a.port} serving {a.model_name}", flush=True)
    serve(a.device, a.port, a.preset, a.model_name, a.max_batch, a.greedy_tokens, tokenizer=a.tokenizer, chat_family=a.chat_family,
          prefix_cache=a.prefix_cache, speculate=a.speculate, speculate_batch=a.speculate_batch,
          prefix_cache_host_bytes=int(a.prefix_cache_host_gib * 2**30), context_shift=a.context_shift,
          num_keep=4 if a.num_keep is None else a.num_keep, context_length=a.context_length, draft_model=a.draft_model,
          draft_seed=a.draft_seed, deterministic=a.deterministic)


if __name__ == "__main__":
    main()
