"""Host reference of Ollama's remaining sampler options (cl_sample_token_ext: min_p, presence / frequency penalties) against
independent statements of each stage, and the wire / handler plumbing of stop, min_p and the penalties.  No GPU needed."""
import ctypes as C
import zlib

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from crowdllama_b200 import handler as H
from crowdllama_b200.pb import BaseMessage, GenerateOptions


def _sp(temperature, top_k, top_p, penalty, last_n=64, seed=4242):
    sp = eng.ollama_default_sampling(seed=seed)
    sp.temperature, sp.top_k, sp.top_p, sp.repeat_penalty, sp.repeat_last_n = temperature, top_k, top_p, penalty, last_n
    return sp


def _rng(case):
    return np.random.default_rng(zlib.crc32(repr(sorted(case.items())).encode()))


def _hf_probs(logits, temperature, top_k, top_p, min_p):
    """HF transformers' processors in the engine's order: top-k -> temperature -> top-p -> min-p, then softmax."""
    import torch
    from transformers.generation.logits_process import MinPLogitsWarper, TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    sc = torch.tensor(np.asarray(logits, np.float32))[None, :].double()
    ids = torch.zeros((1, 0), dtype=torch.long)
    if top_k > 0:
        sc = TopKLogitsWarper(top_k)(ids, sc)
    sc = TemperatureLogitsWarper(temperature)(ids, sc)
    if 0.0 < top_p < 1.0:
        sc = TopPLogitsWarper(top_p)(ids, sc)
    if min_p > 0.0:
        sc = MinPLogitsWarper(min_p)(ids, sc)
    return torch.softmax(sc, dim=-1)[0].numpy()


def _np_penalised(logits, history, last_n, repeat, presence, frequency):
    """llama.cpp's penalty formula in fp32: an id occurring c > 0 times in the window takes the repeat penalty, then
    v -= c * frequency + presence.  Ids outside the vocabulary are skipped."""
    v = np.asarray(logits, np.float32).copy()
    win = list(history)[-last_n:] if last_n > 0 else list(history)
    counts = {}
    for t in win:
        if 0 <= t < len(v):
            counts[t] = counts.get(t, 0) + 1
    for t, c in counts.items():
        x = v[t]
        if repeat != 1.0:
            x = np.float32(x / np.float32(repeat)) if x > 0 else np.float32(x * np.float32(repeat))
        v[t] = np.float32(x - np.float32(np.float32(c) * np.float32(frequency) + np.float32(presence)))
    return v


def _check_freq(draws, p, n):
    assert draws[p == 0].sum() == 0, "a token outside the reference's support set was drawn"
    sigma = np.sqrt(n * p * (1 - p)) + 1e-9
    assert (np.abs(draws - n * p) <= 5 * sigma + 1).all(), (draws, n * p)
    assert (p > 0).sum() >= 2


@pytest.mark.parametrize("case", [
    dict(temperature=0.8, top_k=40, top_p=0.9, penalty=1.1, hist=24),     # Ollama's defaults
    dict(temperature=1.3, top_k=0, top_p=0.7, penalty=1.0, hist=0),
    dict(temperature=0.5, top_k=5, top_p=1.0, penalty=1.6, hist=10),
    dict(temperature=1.0, top_k=12, top_p=0.5, penalty=1.3, hist=40),
    dict(temperature=0.0, top_k=40, top_p=0.9, penalty=1.1, hist=8),      # greedy
])
def test_zero_ext_draws_exactly_what_cl_sample_token_draws(case):
    rng = _rng(case)
    V = 64
    lg = (rng.standard_normal(V) * 2.0).astype(np.float32)
    hist = [int(x) for x in rng.integers(0, V, size=case["hist"])]
    sp = _sp(case["temperature"], case["top_k"], case["top_p"], case["penalty"])
    for ext in (None, eng.sampling_ext()):
        a = [eng.sample_token(lg, sp, hist, step=i) for i in range(2000)]
        b = [eng.sample_token_ext(lg, sp, ext, hist, step=i) for i in range(2000)]
        assert a == b


@pytest.mark.parametrize("case", [
    dict(temperature=0.8, top_k=40, top_p=0.9, min_p=0.1, cuts=True),
    dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.2, cuts=True),
    dict(temperature=1.5, top_k=20, top_p=0.95, min_p=0.3, cuts=True),
    dict(temperature=1.2, top_k=64, top_p=0.8, min_p=0.01, cuts=False),    # top-p already cut below what min_p would
])
def test_min_p_matches_hf_min_p_warper_after_top_p(case):
    rng = _rng(case)
    V, n = 64, 8000
    lg = (rng.standard_normal(V) * 2.0).astype(np.float32)
    p = _hf_probs(lg, case["temperature"], case["top_k"], case["top_p"], case["min_p"])
    sp = _sp(case["temperature"], case["top_k"], case["top_p"], 1.0)
    ext = eng.sampling_ext(min_p=case["min_p"])
    draws = np.bincount([eng.sample_token_ext(lg, sp, ext, (), step=i) for i in range(n)], minlength=V)
    assert set(np.flatnonzero(draws)) <= set(np.flatnonzero(p))
    _check_freq(draws, p, n)
    without = _hf_probs(lg, case["temperature"], case["top_k"], case["top_p"], 0.0) > 0
    assert ((p > 0).sum() < without.sum()) == case["cuts"]


@pytest.mark.parametrize("case", [
    dict(temperature=0.8, top_k=40, top_p=0.9, penalty=1.1, presence=0.5, frequency=0.5, last_n=64),
    dict(temperature=1.0, top_k=20, top_p=1.0, penalty=1.0, presence=1.5, frequency=0.0, last_n=32),
    dict(temperature=1.2, top_k=0, top_p=0.8, penalty=1.0, presence=0.0, frequency=0.8, last_n=64),
    dict(temperature=0.9, top_k=30, top_p=0.95, penalty=1.3, presence=-0.7, frequency=-0.4, last_n=16),
])
def test_penalties_match_numpy_formula_through_hf_chain(case):
    rng = _rng(case)
    V, n = 64, 8000
    lg = (rng.standard_normal(V) * 2.0).astype(np.float32)
    lg[:8] = -np.abs(lg[:8])                                     # negative logits in the window
    hist = [int(x) for x in rng.integers(0, 12, size=48)]        # many duplicates
    hist[5:5] = [-3, V, V + 100]                                 # out-of-range ids are skipped
    pen = _np_penalised(lg, hist, case["last_n"], case["penalty"], case["presence"], case["frequency"])
    p = _hf_probs(pen, case["temperature"], case["top_k"], case["top_p"], 0.0)
    sp = _sp(case["temperature"], case["top_k"], case["top_p"], case["penalty"], case["last_n"])
    ext = eng.sampling_ext(presence_penalty=case["presence"], frequency_penalty=case["frequency"])
    draws = np.bincount([eng.sample_token_ext(lg, sp, ext, hist, step=i) for i in range(n)], minlength=V)
    _check_freq(draws, p, n)


def test_frequency_penalty_scales_with_the_count():
    """Only the count-dependent term drops id 0 out of top-k: an implementation that applied it once per id would keep it."""
    V, n = 16, 2000
    lg = np.full(V, -5.0, np.float32)
    lg[:4] = [5.0, 4.0, 3.5, 3.2]
    hist = [0, 0, 0, 9]
    sp = _sp(1.0, 3, 1.0, 1.0)
    ext = eng.sampling_ext(frequency_penalty=0.7)
    draws = np.bincount([eng.sample_token_ext(lg, sp, ext, hist, step=i) for i in range(n)], minlength=V)
    assert draws[0] == 0 and draws[3] > 0 and draws[1:4].sum() == n
    once = _np_penalised(lg, [0, 9], 64, 1.0, 0.0, 0.7)          # what a presence-like (c = 1) rule would leave
    assert once[0] > lg[3]


@pytest.mark.parametrize("field,value", [("min_p", -0.01), ("min_p", 1.01), ("min_p", float("nan")),
                                         ("presence_penalty", float("nan")), ("presence_penalty", float("inf")),
                                         ("frequency_penalty", float("-inf"))])
def test_invalid_ext_is_rejected(field, value):
    lg = np.zeros(16, np.float32)
    x = eng.sampling_ext(**{field: value})
    with pytest.raises(eng.EngineError):
        eng.sample_token_ext(lg, _sp(0.8, 4, 0.9, 1.0), x)
    ok = eng.sampling_ext(min_p=1.0, presence_penalty=-2.0, frequency_penalty=3.0)
    assert 0 <= eng.sample_token_ext(lg, _sp(0.8, 4, 0.9, 1.0), ok) < 16


def test_sampling_ext_layout():
    assert C.sizeof(eng.SamplingExt) == 56
    assert eng.SamplingExt.stop.offset == 16


def test_options_11_to_14_are_wire_compatible_with_google_protobuf():
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    fd = descriptor_pb2.FileDescriptorProto(name="llama_v1_opts_test.proto", package="llama.v1o", syntax="proto3")
    T = descriptor_pb2.FieldDescriptorProto
    go = fd.message_type.add(name="GenerateOptions")
    go.field.add(name="top_k", number=3, type=T.TYPE_INT32, label=T.LABEL_OPTIONAL)
    go.field.add(name="stop", number=11, type=T.TYPE_STRING, label=T.LABEL_REPEATED)
    for i, nm in enumerate(["min_p", "presence_penalty", "frequency_penalty"]):
        go.oneof_decl.add(name=f"_{nm}")
        go.field.add(name=nm, number=12 + i, type=T.TYPE_FLOAT, label=T.LABEL_OPTIONAL, oneof_index=i, proto3_optional=True)
    pool = descriptor_pool.Default()
    try:
        pool.Add(fd)
    except TypeError:
        pass
    M = message_factory.GetMessageClass(pool.FindMessageTypeByName("llama.v1o.GenerateOptions"))
    ours = GenerateOptions(top_k=7, stop=["\n\n", "User:", "☃"], min_p=0.05, presence_penalty=0.0, frequency_penalty=-0.5)
    g = M.FromString(ours.encode())
    assert list(g.stop) == ["\n\n", "User:", "☃"] and g.top_k == 7
    assert abs(g.min_p - 0.05) < 1e-7 and g.HasField("presence_penalty") and g.presence_penalty == 0.0 and g.frequency_penalty == -0.5
    back = GenerateOptions.decode(g.SerializeToString())
    assert back.stop == ["\n\n", "User:", "☃"] and back.presence_penalty == 0.0 and back.frequency_penalty == -0.5
    g2 = M(stop=["x"])
    assert GenerateOptions.decode(g2.SerializeToString()) == GenerateOptions(stop=["x"])


def test_from_json_and_handler_routing():
    o = GenerateOptions.from_json({"stop": ["\n", "###"], "min_p": 0.1, "presence_penalty": 0.5, "frequency_penalty": 0.25,
                                   "typical_p": 0.7, "mirostat": 2})
    assert o.stop == ["\n", "###"] and o.min_p == pytest.approx(0.1) and o.presence_penalty == 0.5 and o.frequency_penalty == 0.25
    assert GenerateOptions.from_json({"stop": "END"}).stop == ["END"]
    assert GenerateOptions.from_json({"typical_p": 0.7}).is_empty()
    base = eng.Sampling()
    base.temperature, base.top_k = 0.8, 40
    # merge_sampling carries only cl_sampling fields; the new options travel to libclengine over the byte-level path
    assert H.merge_sampling(base, GenerateOptions(stop=["a"])).top_k == 40
    assert H.merge_sampling(base, GenerateOptions(top_k=3, min_p=0.2)).top_k == 3
    seen = []

    class Bytes:
        model_name = "m"

        def generate(self, model, prompt, sampling=None):
            raise AssertionError("stop / min_p / penalties must take the byte-level path")

        def handle_message(self, req, sampling=None):
            seen.append(BaseMessage.decode(req).generate_request.options)
            return H._response("m", "cut", True, "stop").encode()

        def handle_message_stream(self, req, sampling=None, on_frame=None):
            raise AssertionError

    h = H.worker_api_handler(Bytes())
    for opts in (GenerateOptions(stop=["\n"]), GenerateOptions(min_p=0.1), GenerateOptions(presence_penalty=0.5),
                 GenerateOptions(frequency_penalty=0.5)):
        g = h(None, H.create_generate_request("m", "p", False, opts)).generate_response
        assert g.response == "cut" and g.done_reason == "stop"
    assert seen[0].stop == ["\n"] and seen[1].min_p == pytest.approx(0.1)
