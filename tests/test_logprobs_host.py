"""CPU-only checks of the log-probability C-ABI: the new symbols are exported, the ABI version and existing structs are
unchanged, cl_token_logprob is 172 bytes with the header's layout, and without a GPU the calls fail loudly."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

from crowdllama_b200 import engine as eng

ROOT = Path(__file__).resolve().parents[1]
NEW = ("cl_seq_set_logprobs", "cl_seq_take_logprobs", "cl_generate_ids_logprobs", "cl_op_sample_logprobs")


def test_new_symbols_are_exported_and_abi_unchanged():
    L = eng.lib()
    for name in NEW:
        assert hasattr(L, name) and name in eng.EXPORTS
    assert L.cl_abi_version() == 2
    header = (ROOT / "include" / "clengine.h").read_text()
    assert re.search(r"#define CL_MAX_TOP_LOGPROBS 20\b", header)
    assert re.search(r"#define CL_ABI_VERSION 2\b", header)


def test_token_logprob_layout():
    assert eng.TOKEN_LOGPROB.itemsize == 172
    assert [eng.TOKEN_LOGPROB.fields[f][1] for f in ("id", "logprob", "n_top", "top_ids", "top_logprobs")] == [0, 4, 8, 12, 92]


def test_calls_without_a_device():
    if eng.device_count() > 0:
        pytest.skip("GPU present")
    lg = np.zeros((1, 512), np.float32)
    sp = eng.greedy(1)
    with pytest.raises(eng.EngineError) as ei:
        eng.op_sample_logprobs(lg, [sp], [[]], [0], 5)
    assert ei.value.status == eng.CL_ERR_NO_DEVICE
    L = eng.lib()
    n = C.c_int32()
    # the engine-level calls reject a missing engine before touching a device
    assert L.cl_seq_set_logprobs(None, 0, 5) == eng.CL_ERR_INVALID_ARG
    assert L.cl_seq_take_logprobs(None, 0, None, 0, C.byref(n)) == eng.CL_ERR_INVALID_ARG
    out, lp = eng.Result(), C.c_void_p()
    ids = np.arange(4, dtype=np.int32)
    assert L.cl_generate_ids_logprobs(None, ids.ctypes.data, 4, C.byref(sp), 5, C.byref(out), C.byref(lp)) == eng.CL_ERR_INVALID_ARG


def test_top_n_range_is_checked_before_the_device():
    lg = np.zeros((1, 512), np.float32)
    for bad in (-1, 21):
        with pytest.raises(eng.EngineError) as ei:
            eng.op_sample_logprobs(lg, [eng.greedy(1)], [[]], [0], bad)
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
    big = np.zeros((1, 64 * 2560 + 1), np.float32)          # above the device sampler's vocabulary limit
    with pytest.raises(eng.EngineError) as ei:
        eng.op_sample_logprobs(big, [eng.greedy(1)], [[]], [0], 5)
    assert ei.value.status == eng.CL_ERR_INVALID_ARG


# ---- wire: the protobuf extension -------------------------------------------------------------------------------
def _descriptor_pool_classes():
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fd = descriptor_pb2.FileDescriptorProto(name="llama_v1_lp_test.proto", package="llama.v1lp", syntax="proto3")
    T = descriptor_pb2.FieldDescriptorProto
    go = fd.message_type.add(name="GenerateOptions")
    for i, (nm, no, ty) in enumerate([("temperature", 2, T.TYPE_FLOAT), ("logprobs", 9, T.TYPE_BOOL), ("top_logprobs", 10, T.TYPE_INT32)]):
        go.oneof_decl.add(name=f"_{nm}")
        go.field.add(name=nm, number=no, type=ty, label=T.LABEL_OPTIONAL, oneof_index=i, proto3_optional=True)
    gr = fd.message_type.add(name="GenerateRequest")
    gr.field.add(name="model", number=1, type=T.TYPE_STRING, label=T.LABEL_OPTIONAL)
    gr.field.add(name="options", number=4, type=T.TYPE_MESSAGE, type_name=".llama.v1lp.GenerateOptions", label=T.LABEL_OPTIONAL)
    tl = fd.message_type.add(name="TokenLogprob")
    tl.field.add(name="token", number=1, type=T.TYPE_STRING, label=T.LABEL_OPTIONAL)
    tl.field.add(name="logprob", number=2, type=T.TYPE_FLOAT, label=T.LABEL_OPTIONAL)
    tl.field.add(name="bytes", number=3, type=T.TYPE_BYTES, label=T.LABEL_OPTIONAL)
    tl.field.add(name="top_logprobs", number=4, type=T.TYPE_MESSAGE, type_name=".llama.v1lp.TokenLogprob", label=T.LABEL_REPEATED)
    gp = fd.message_type.add(name="GenerateResponse")
    gp.field.add(name="model", number=1, type=T.TYPE_STRING, label=T.LABEL_OPTIONAL)
    gp.field.add(name="response", number=3, type=T.TYPE_STRING, label=T.LABEL_OPTIONAL)
    gp.field.add(name="done", number=4, type=T.TYPE_BOOL, label=T.LABEL_OPTIONAL)
    gp.field.add(name="logprobs", number=8, type=T.TYPE_MESSAGE, type_name=".llama.v1lp.TokenLogprob", label=T.LABEL_REPEATED)
    pool = descriptor_pool.Default()
    try:
        pool.Add(fd)
    except TypeError:
        pass
    get = lambda n: message_factory.GetMessageClass(pool.FindMessageTypeByName(f"llama.v1lp.{n}"))   # noqa: E731
    return get("GenerateRequest"), get("GenerateResponse")


def test_protobuf_fields_round_trip():
    from crowdllama_b200.pb import GenerateOptions, GenerateRequest, GenerateResponse, TokenLogprob
    Req, Resp = _descriptor_pool_classes()
    # our request -> the runtime's parser
    ours = GenerateRequest(model="m", options=GenerateOptions(temperature=0.0, logprobs=True, top_logprobs=0)).encode()
    g = Req.FromString(ours)
    assert g.options.HasField("logprobs") and g.options.logprobs and g.options.HasField("top_logprobs") and g.options.top_logprobs == 0
    # the runtime's request -> ours
    g2 = Req(model="m")
    g2.options.logprobs = True
    g2.options.top_logprobs = 7
    back = GenerateRequest.decode(g2.SerializeToString())
    assert back.options.logprobs is True and back.options.top_logprobs == 7 and back.options.temperature is None
    # responses both ways, nested alternatives and exact bytes included
    r = GenerateResponse(model="m", response="hi", done=True, logprobs=[
        TokenLogprob("h", -0.25, b"h", [TokenLogprob("h", -0.25, b"h"), TokenLogprob("�", -3.5, b"\xe2\x98")]),
        TokenLogprob("i", 0.0, b"i", [])])
    gr = Resp.FromString(r.encode())
    assert [t.token for t in gr.logprobs] == ["h", "i"] and gr.logprobs[0].top_logprobs[1].bytes == b"\xe2\x98"
    assert gr.logprobs[0].logprob == -0.25 and gr.logprobs[1].logprob == 0.0
    assert GenerateResponse.decode(gr.SerializeToString()) == r
    # old messages decode exactly as before: no logprobs fields, defaults
    old = Resp(model="m", response="x", done=True).SerializeToString()
    assert GenerateResponse.decode(old) == GenerateResponse(model="m", response="x", done=True)
    assert GenerateRequest.decode(Req(model="m").SerializeToString()).options is None


# ---- gateway stand-in in front of a mock worker -------------------------------------------------------------------
class _LpEngine:
    """Byte-level mock: answers a request for logprobs with one record per character of the reply."""
    model_name = "lp-model"

    def __init__(self):
        self.seen = []

    def stats(self):
        return dict(tokens_per_sec=100.0, load=0.1, vram_gb=80, gpu_model="mock")

    def _frames(self, req_bytes, stream):
        from crowdllama_b200.pb import BaseMessage, GenerateResponse, TokenLogprob
        g = BaseMessage.decode(req_bytes).generate_request
        self.seen.append(g.options)
        text = "ab"
        o = g.options
        n_top = o.top_logprobs or 0 if o and o.logprobs else None

        def recs(chars):
            if n_top is None:
                return []
            return [TokenLogprob(c, -0.5, c.encode(), [TokenLogprob(c, -0.5, c.encode())] * n_top) for c in chars]
        if not stream:
            return [GenerateResponse(model=g.model, response=text, done=True, done_reason="stop", logprobs=recs(text))]
        return [GenerateResponse(model=g.model, response=c, logprobs=recs(c)) for c in text] + \
               [GenerateResponse(model=g.model, done=True, done_reason="stop")]

    def handle_message(self, req, sampling=None):
        from crowdllama_b200.pb import BaseMessage
        return BaseMessage(generate_response=self._frames(req, False)[0]).encode()

    def handle_message_stream(self, req, sampling=None, on_frame=None):
        from crowdllama_b200.pb import BaseMessage
        fr = self._frames(req, True)
        for f in fr:
            on_frame(BaseMessage(generate_response=f).encode())
        return len(fr)

    def generate(self, model, prompt, sampling=None):
        raise AssertionError("logprobs requests must take the byte-level path")


def test_gateway_logprobs_shape_and_validation():
    import json
    import socket
    import threading
    import urllib.error
    import urllib.request
    from crowdllama_b200 import gateway, worker

    def free_port():
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            return s.getsockname()[1]
    wp, gp = free_port(), free_port()
    engine = _LpEngine()
    w = worker.WorkerServer(("127.0.0.1", wp), engine, peer_id="w")
    threading.Thread(target=w.serve_forever, daemon=True).start()
    g = gateway.make_server([("127.0.0.1", wp)], port=gp)
    threading.Thread(target=g.serve_forever, daemon=True).start()

    def post(path, obj):
        req = urllib.request.Request(f"http://127.0.0.1:{gp}{path}", json.dumps(obj).encode(), {"Content-Type": "application/json"})
        with urllib.request.urlopen(req, timeout=10) as r:
            body = r.read().decode()
        return [json.loads(x) for x in body.splitlines() if x.strip()]
    try:
        for path, base in (("/api/generate", {"model": "lp-model", "prompt": "q"}),
                           ("/api/chat", {"model": "lp-model", "messages": [{"role": "user", "content": "q"}]})):
            (one,) = post(path, {**base, "stream": False, "logprobs": True, "top_logprobs": 2})
            assert [t["token"] for t in one["logprobs"]] == ["a", "b"]
            t = one["logprobs"][0]
            assert set(t) == {"token", "logprob", "bytes", "top_logprobs"} and t["bytes"] == [97] and t["logprob"] == -0.5
            assert len(t["top_logprobs"]) == 2 and set(t["top_logprobs"][0]) == {"token", "logprob", "bytes"}
            lines = post(path, {**base, "stream": True, "logprobs": True})
            assert [x["token"] for ln in lines for x in ln["logprobs"]] == ["a", "b"]
            assert all(x["top_logprobs"] == [] for ln in lines for x in ln["logprobs"]) and lines[-1]["done"]
            assert engine.seen[-1].logprobs is True and engine.seen[-1].top_logprobs == 0
            (plain,) = post(path, {**base, "stream": False})
            assert "logprobs" not in plain
            for bad in ({"top_logprobs": 21, "logprobs": True}, {"top_logprobs": -1, "logprobs": True}, {"top_logprobs": 3},
                        {"top_logprobs": 2, "logprobs": False}):
                with pytest.raises(urllib.error.HTTPError) as ei:
                    post(path, {**base, **bad})
                assert ei.value.code == 400 and "error" in json.loads(ei.value.read())
    finally:
        g.shutdown()
        w.shutdown()
