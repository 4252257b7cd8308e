"""CPU tests of the request-level harness: gateway stand-in + worker protocol servers with a MOCK engine
(mirrors /root/reference/test/integration_test.go:139-191, where the only faked piece is the model server)."""
import json
import socket
import threading
import urllib.error
import urllib.request

import pytest

from crowdllama_b200 import gateway, worker
from crowdllama_b200 import handler as H
from crowdllama_b200.router import Resource


class _MockEngine:
    def __init__(self, name, tput=150.0):
        self.model_name, self.tput = name, tput

    def generate(self, model, prompt, sampling=None):
        class R:
            text, done_reason = f"This is a mock response. You asked: {prompt}", "stop"
        if model != self.model_name:
            raise RuntimeError("unknown model")
        return R()

    def generate_stream(self, model, prompt, sampling=None, on_text=None):
        r = self.generate(model, prompt, sampling)
        self.last_sampling = sampling
        for w in r.text.split(" "):
            on_text(w + " ", [0])
        return r

    def stats(self):
        return dict(tokens_per_sec=self.tput, load=0.3, vram_gb=79, gpu_model="mock H100")


def _spawn_worker(port, name):
    srv = worker.WorkerServer(("127.0.0.1", port), _MockEngine(name), peer_id=f"w{port}")
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    return srv


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _post(url, obj):
    req = urllib.request.Request(url, json.dumps(obj).encode(), {"Content-Type": "application/json"})
    with urllib.request.urlopen(req, timeout=10) as r:
        return r.status, json.loads(r.read())


def test_gateway_to_worker_round_trip_and_errors():
    p1, p2, gp = _free_port(), _free_port(), _free_port()
    w1, w2 = _spawn_worker(p1, "llama3.2"), _spawn_worker(p2, "llama3.2")
    gw = gateway.make_server([("127.0.0.1", p1), ("127.0.0.1", p2)], port=gp)
    threading.Thread(target=gw.serve_forever, daemon=True).start()
    try:
        base = f"http://127.0.0.1:{gp}"
        # metadata protocol feeds the peer table (truthful Resource from engine stats)
        with urllib.request.urlopen(base + "/api/health", timeout=5) as r:
            health = json.loads(r.read())
        assert set(health["peers"]) == {f"w{p1}", f"w{p2}"}
        assert health["peers"][f"w{p1}"]["supported_models"] == ["llama3.2"]
        # integration_test.go:490-553: 200, model echo, non-empty content, done
        st, out = _post(base + "/api/chat", {"model": "llama3.2", "messages": [{"role": "user", "content": "Hello"},
                                                                               {"role": "user", "content": "dropped"}], "stream": False})
        assert st == 200 and out["model"] == "llama3.2" and out["done"] and out["done_reason"] == "stop"
        assert out["message"] == {"role": "assistant", "content": "This is a mock response. You asked: Hello"}   # only messages[0]
        # requests spread over both tied workers (random among ties)
        for i in range(30):
            _post(base + "/api/chat", {"model": "llama3.2", "messages": [{"role": "user", "content": str(i)}]})
        assert len(gw.counts) == 2 and sum(gw.counts.values()) == 31
        # unknown model -> 503; missing fields -> 400 (gateway.go:175-199)
        for body, code in [({"model": "nope", "messages": [{"role": "user", "content": "x"}]}, 503), ({"model": "llama3.2"}, 400),
                           ({"messages": [{"role": "user", "content": "x"}]}, 400)]:
            with pytest.raises(urllib.error.HTTPError) as ei:
                _post(base + "/api/chat", body)
            assert ei.value.code == code
    finally:
        gw.shutdown(); w1.shutdown(); w2.shutdown()


def test_worker_handler_error_becomes_assistant_text():
    """A handler error travels as Response="Error: ..." (peer.go:232-243) and the gateway still answers 200."""
    p, gp = _free_port(), _free_port()
    srv = worker.WorkerServer(("127.0.0.1", p), _MockEngine("m"), peer_id="w")

    def boom(ctx, req):
        raise RuntimeError("engine exploded")
    srv.api_handler = boom
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    gw = gateway.make_server([("127.0.0.1", p)], port=gp)
    threading.Thread(target=gw.serve_forever, daemon=True).start()
    try:
        st, out = _post(f"http://127.0.0.1:{gp}/api/chat", {"model": "m", "messages": [{"role": "user", "content": "x"}]})
        assert st == 200 and out["message"]["content"] == "Error: engine exploded" and out["done"]
    finally:
        gw.shutdown(); srv.shutdown()


def test_metadata_protocol_returns_resource_json():
    p = _free_port()
    srv = _spawn_worker(p, "tinyllama")
    try:
        with socket.create_connection(("127.0.0.1", p), timeout=5) as s:
            s.sendall((worker.METADATA_PROTOCOL + "\n").encode())
            data = b""
            while chunk := s.recv(4096):
                data += chunk
        r = Resource.from_json(data)
        assert r.worker_mode and r.supported_models == ["tinyllama"] and r.tokens_throughput == pytest.approx(128.0) and r.gpu_model == "mock H100"   # 150 tok/s -> half-octave bucket 2^7
    finally:
        srv.shutdown()


def test_generate_endpoint_options_and_streaming():
    """SURVEY.md §8f rows 3-4: POST /api/generate, `options` passed through to the worker, NDJSON streaming."""
    wp, gp = _free_port(), _free_port()
    w = _spawn_worker(wp, "tinyllama")
    seen = {}
    orig = w.engine.generate

    def rec(model, prompt, sampling=None):
        seen["sampling"] = sampling
        return orig(model, prompt, sampling)
    w.engine.generate = rec
    g = gateway.make_server([("127.0.0.1", wp)], port=gp)
    threading.Thread(target=g.serve_forever, daemon=True).start()
    try:
        base = f"http://127.0.0.1:{gp}"
        _, r = _post(base + "/api/generate", {"model": "tinyllama", "prompt": "why?", "stream": False,
                                              "options": {"temperature": 0, "seed": 42, "num_predict": 32, "mirostat": 2}})
        assert r["response"] == "This is a mock response. You asked: why?" and r["done"] and r["done_reason"] == "stop"
        assert "message" not in r and r["stream"] is False
        s = seen["sampling"]
        assert (s.temperature, s.seed, s.max_new_tokens) == (0.0, 42, 32) and s.top_k == 40      # unset fields: Ollama defaults
        _, r = _post(base + "/api/chat", {"model": "tinyllama", "messages": [{"role": "user", "content": "hi"}],
                                          "options": {"top_k": 1}})
        assert r["message"]["content"].endswith("You asked: hi") and seen["sampling"].top_k == 1
        with pytest.raises(urllib.error.HTTPError) as ei:
            _post(base + "/api/generate", {"model": "tinyllama"})
        assert ei.value.code == 400
        # streaming: one NDJSON line per worker frame, done only on the last
        req = urllib.request.Request(base + "/api/generate", data=json.dumps({"model": "tinyllama", "prompt": "a b", "stream": True}).encode(),
                                     headers={"Content-Type": "application/json"})
        with urllib.request.urlopen(req, timeout=10) as resp:
            assert resp.headers["Content-Type"] == "application/x-ndjson"
            lines = [json.loads(x) for x in resp.read().decode().splitlines() if x.strip()]
        assert len(lines) >= 3 and [x["done"] for x in lines] == [False] * (len(lines) - 1) + [True]
        assert "".join(x["response"] for x in lines).strip() == "This is a mock response. You asked: a b"
        assert lines[-1]["done_reason"] == "stop"
        req = urllib.request.Request(base + "/api/chat", data=json.dumps({"model": "tinyllama", "stream": True,
                                     "messages": [{"role": "user", "content": "x"}]}).encode(), headers={"Content-Type": "application/json"})
        with urllib.request.urlopen(req, timeout=10) as resp:
            lines = [json.loads(x) for x in resp.read().decode().splitlines() if x.strip()]
        assert "".join(x["message"]["content"] for x in lines).strip().endswith("You asked: x") and lines[-1]["done"]
    finally:
        g.shutdown(); g.server_close(); w.shutdown(); w.server_close()


def test_bench_box_load_generator_against_two_mock_peers():
    """bench.py's request-level leg (BASELINE.json configs[3]) without a GPU: two worker peers with mock engines play the
    two ranks of `bench.py --gpus 2`; the load generator (its own process, as in the benchmark) routes 64 concurrent
    chats through the gateway stand-in, reports req/s and per-worker counts, and tells every peer to stop."""
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parents[1]
    base = _free_port() + 1
    srvs = [_spawn_worker(base + i, "llama3:8b") for i in range(2)]
    try:
        out = subprocess.run([sys.executable, str(root / "bench.py"), "--box-client", "--workers", "2", "--base-port", str(base)],
                             capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        res = json.loads(out.stdout.strip().splitlines()[-1])
        assert "error" not in res, res
        import bench
        for key, conc in (("config4", 64), ("saturated", 2 * bench.BOX_MAX_BATCH)):
            sc = res[key]
            assert sc["concurrency"] == conc and sc["ok"] == sc["requests"] and not sc["errors"] and sc["req_per_s"] > 0
            assert sum(sc["per_worker_requests"].values()) == sc["requests"] and len(sc["per_worker_requests"]) == 2
        assert all(s.stop_event.wait(5) for s in srvs)          # the ranks leave their serving loop
    finally:
        for s in srvs:
            s.shutdown()


def test_peer_table_survives_a_peer_that_answers_garbage():
    """ADVICE r1: a worker that accepts the metadata stream and closes without (valid) JSON must be dropped from the
    table, not kill the refresh thread — the healthy peer stays routable."""
    import socketserver

    class _Bad(socketserver.BaseRequestHandler):
        def handle(self):
            self.request.recv(64)
            self.request.sendall(b'{"peer_id": "half')          # partial JSON, then close

    bad_port, good_port = _free_port(), _free_port()
    bad = socketserver.ThreadingTCPServer(("127.0.0.1", bad_port), _Bad)
    threading.Thread(target=bad.serve_forever, daemon=True).start()
    good = _spawn_worker(good_port, "m")
    try:
        t = gateway.PeerTable([("127.0.0.1", bad_port), ("127.0.0.1", good_port), ("127.0.0.1", _free_port())])
        t.probe()                                                 # must not raise
        t.probe()
        assert list(t.peers) == [("127.0.0.1", good_port)]
        addr, w = t.best("m")
        assert addr == ("127.0.0.1", good_port) and w.peer_id == f"w{good_port}"
    finally:
        bad.shutdown(); good.shutdown()


def test_pb_rejects_truncated_fixed_width_fields():
    from crowdllama_b200 import pb
    with pytest.raises(ValueError):
        list(pb._fields(bytes([0x0d, 1, 2])))                     # field 1, wire type 5 (fixed32), only 2 bytes
    with pytest.raises(ValueError):
        list(pb._fields(bytes([0x09, 1, 2, 3, 4])))               # field 1, wire type 1 (fixed64), only 4 bytes
    assert [(f, wt) for f, wt, _ in pb._fields(bytes([0x0d, 0, 0, 0x80, 0x3f]))] == [(1, 5)]


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the CPU arm the driver runs beside ours): one JSON line with the contract's keys, the
    same metric / unit / config as our arm, `impl: reference`, a cpu_baseline describing this run and an e2e that repeats
    the value with zero host<->device bytes.  Runs the CPU oracle port on Llama-3-8B shapes for 3 steps (~25 s)."""
    import subprocess
    import sys
    from pathlib import Path
    import bench
    root = Path(__file__).resolve().parents[1]
    out = subprocess.run([sys.executable, str(root / "bench.py"), "--impl", "reference", "--steps", "3", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.strip().splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == bench.METRIC and d["unit"] == "tokens/s" and d["higher_is_better"] is True
    assert d["n_gpus"] == 1 and d["steps"] == 3 and d["value"] > 0 and abs(d["ms_per_step"] * d["value"] - 1000.0) < 1.0
    assert d["dtype"] == "bf16" and d["data"] == "synthetic" and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["config"]["preset"] == bench.PRESET and d["config"]["ctx"] == bench.CTX and "workload" in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert d["e2e"] == {"value": d["value"], "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["gpu_launches"] == 0


def test_committed_bench_line_carries_every_contract_key():
    """The bench line the README's numbers come from (profiles/h100_bench.json, produced by `python bench.py --gpus 1
    --steps 256 --warmup 8` on one H100 SXM after tools/measure_peaks.py): every key of the bench contract is present
    and internally consistent — a reader of profiles/ and a consumer of bench.py parse the same structure."""
    from pathlib import Path
    import bench
    p = Path(__file__).resolve().parents[1] / "profiles" / "h100_bench.json"
    d = json.loads(p.read_text().strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "roofline", "cpu_baseline", "e2e", "gpu_launches", "clocks", "box", "configs"):
        assert k in d, k
    assert d["metric"] == bench.METRIC and d["n_gpus"] == 1 and d["warmup"] >= 3 and d["gpu_launches"] > 0
    assert abs(d["value"] * d["ms_per_step"] - 1000.0) < 1.0                       # tokens/s x ms/token, one replica
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and r["kernel"] == "decode_mega_kernel"
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3 and 0.5 < r["frac"] < 1.0
    assert "traffic" in r                                                          # ncu DRAM bytes, when a capture of this build is committed
    if r["traffic"] is not None:
        assert 0.98 < r["traffic"] / r["detail"]["algorithmic_bytes"] < 1.02        # = algorithmic bytes
    assert r["prefill"]["bound"] == "tensor" and 0.5 < r["prefill"]["frac"] < 1.0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] > 0
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and 0.9 < e["value"] / d["value"] <= 1.0
    assert d["clocks"]["reasons"] == [] and d["clocks"]["sm_mhz"] > 0.9 * d["clocks"]["sm_max_mhz"]
    assert "l2" in d["config"] and "workload" in d["config"]
    for sc in ("config4", "saturated"):
        b = d["box"][sc]
        assert b["ok"] == b["requests"] and not b["errors"] and b["req_per_s"] > 0 and sum(b["per_worker_requests"].values()) == b["requests"]
