"""min_p, presence / frequency penalties and stop strings on the GPU: the step tail's draw against cl_sample_token_ext id
for id, every token path that draws for an armed sequence, and the stop rule through every request path."""
import itertools
import threading

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from crowdllama_b200.pb import BaseMessage, GenerateOptions, GenerateRequest

pytestmark = pytest.mark.gpu

TOPK_CAP, HIST_CAP = 128, 256          # kSampleTopKMax, kSampleHistMax (csrc/kernels.h)


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    for k in ("CL_SPECULATE", "CL_SPECULATE_BATCH", "CL_PREFIX_CACHE", "CL_DEVICE_SAMPLE", "CL_CONTEXT_SHIFT", "CL_NUM_KEEP"):
        monkeypatch.delenv(k, raising=False)


def _sp(temperature, top_k, top_p, penalty, last_n, seed, max_new=-1):
    s = eng.ollama_default_sampling(seed=seed, max_new_tokens=max_new)
    s.temperature, s.top_k, s.top_p, s.repeat_penalty, s.repeat_last_n = temperature, top_k, top_p, penalty, last_n
    return s


def _logits(kind, V, rng):
    x = rng.normal(0.0, 2.5, V).astype(np.float32)
    if kind == "ties":
        x = (np.round(x * 2) / 2).astype(np.float32)
    elif kind == "inf":
        x[rng.random(V) < 0.6] = -np.inf
    elif kind == "neg":
        x = -np.abs(x) - np.float32(0.01)
    return x


def _history(logits, window, V, rng, kind):
    top = np.argsort(-logits, kind="stable")[:48]
    n = window + 9
    if kind == "same":                                   # one id repeated over the whole window
        return np.full(n, int(top[0]), np.int32)
    h = rng.choice(top, n).astype(np.int64)
    h[rng.random(n) < 0.2] = int(top[int(rng.integers(0, 8))])
    h[rng.random(n) < 0.1] = -1 - rng.integers(0, 5)
    h[rng.random(n) < 0.1] = V + rng.integers(0, 5)
    return h.astype(np.int32)


MINP = [0.0, 0.02, 0.3]
PEN = [(0.0, 0.0), (0.5, 0.5), (-0.6, 0.0), (0.0, 0.9), (1.5, -0.4)]       # (presence, frequency)


@pytest.mark.parametrize("V", [512, 32000, 128256])
def test_op_sample_ext_matches_host_sampler(V):
    rng = np.random.default_rng(V + 7)
    grid = list(itertools.product([1, 5, 40, TOPK_CAP], [0.5, 0.9, 1.0], [0.3, 0.9, 1.5], [1.0, 1.1, 1.6], [1, 17, 64, HIST_CAP],
                                  ["gauss", "ties", "neg", "inf"], MINP, PEN, ["mix", "same"]))
    rng.shuffle(grid)
    grid = grid[:2048]
    rows, mism = 64, []
    for c0 in range(0, len(grid), rows):
        chunk = grid[c0:c0 + rows]
        lg = np.stack([_logits(g[5], V, rng) for g in chunk])
        sps = [_sp(g[2], g[0], g[1], g[3], g[4], int(rng.integers(0, 2**63))) for g in chunk]
        exts = [eng.sampling_ext(min_p=g[6], presence_penalty=g[7][0], frequency_penalty=g[7][1]) for g in chunk]
        hists = [_history(lg[i], g[4], V, rng, g[8]) for i, g in enumerate(chunk)]
        steps = rng.integers(0, 2**40, len(chunk)).astype(np.uint64)
        dev = eng.op_sample_ext(lg, sps, exts, hists, steps)
        for i in range(len(chunk)):
            host = eng.sample_token_ext(lg[i], sps[i], exts[i], hists[i], int(steps[i]))
            if host != dev[i]:
                mism.append((chunk[i], int(host), int(dev[i])))
    assert not mism, mism[:10]


def test_op_sample_ext_validates_and_zero_ext_is_op_sample():
    rng = np.random.default_rng(3)
    lg = np.stack([_logits("gauss", 512, rng) for _ in range(8)])
    sps = [_sp(0.8, 40, 0.9, 1.1, 64, i) for i in range(8)]
    hists = [_history(lg[i], 64, 512, rng, "mix") for i in range(8)]
    np.testing.assert_array_equal(eng.op_sample_ext(lg, sps, [None] * 8, hists, range(8)), eng.op_sample(lg, sps, hists, range(8)))
    for bad in (eng.sampling_ext(min_p=1.5), eng.sampling_ext(presence_penalty=float("nan")),
                eng.sampling_ext(frequency_penalty=float("inf"))):
        with pytest.raises(eng.EngineError) as ei:
            eng.op_sample_ext(lg[:1], sps[:1], [bad], hists[:1], [0])
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
    # a penalty over repeat_last_n -1 needs the host sampler; with every penalty off any window is fine
    with pytest.raises(eng.EngineError):
        eng.op_sample_ext(lg[:1], [_sp(0.8, 40, 0.9, 1.0, -1, 1)], [eng.sampling_ext(presence_penalty=0.5)], [[]], [0])
    eng.op_sample_ext(lg[:1], [_sp(0.8, 40, 0.9, 1.0, -1, 1)], [eng.sampling_ext(min_p=0.5)], [[]], [0])


# ---- token paths -----------------------------------------------------------------------------------------------------
def _prompt(n, V, k=0):
    return np.array([(i * 7919 + 13 + 101 * k) % V for i in range(n)], np.int32)


EXT = eng.sampling_ext(min_p=0.05, presence_penalty=0.5, frequency_penalty=0.5)
EXT2 = eng.sampling_ext(min_p=0.3, presence_penalty=-0.4, frequency_penalty=1.2)


def _run_sample_batch(e, B, kinds, n_steps=32):
    """kinds[b]: 'g' greedy, 'p' plain-sampled, 'x' sampled with EXT / EXT2 armed.  The loop's ids against a step replay."""
    V = e.cfg["vocab_size"]
    rng = np.random.default_rng(B * 1000 + V)
    prompts = [_prompt(20 + 13 * b, V, b) for b in range(B)]
    pool = [_sp(0.8, 40, 0.9, 1.1, 64, 11), _sp(1.5, TOPK_CAP, 1.0, 1.0, HIST_CAP, 12), _sp(0.9, 20, 0.95, 1.3, 8, 14)]
    sps = [eng.greedy(0) if k == "g" else pool[b % len(pool)] for b, k in enumerate(kinds)]
    exts = [(EXT if b % 2 == 0 else EXT2) if k == "x" else None for b, k in enumerate(kinds)]
    firsts = [int(p[-1] * 3 % V) for p in prompts]
    step0 = rng.integers(0, 1000, B).astype(np.uint64)
    seqs = [e.seq_create() for _ in range(B)]
    for s, p, x in zip(seqs, prompts, exts):
        e.prefill(s, p, want_logits=False)
        if x is not None:
            e.set_sampling_ext(s, x)
    ids, _ = e.decode_sample_batch(seqs, firsts, sps, n_steps, step0)
    for s in seqs:
        e.seq_free(s)
    rep = [e.seq_create() for _ in range(B)]
    for s, p in zip(rep, prompts):
        e.prefill(s, p, want_logits=False)
    hist = [list(p) for p in prompts]
    feed = list(firsts)
    for i in range(n_steps):
        lg, _ = e.decode_step_batch(rep, feed)
        for b in range(B):
            hist[b].append(feed[b])
            want = eng.sample_token_ext(lg[b], sps[b], exts[b], hist[b], int(step0[b]) + i)
            assert want == ids[i, b], (i, b, kinds[b], want, ids[i, b])
        feed = [int(x) for x in ids[i]]
    for s in rep:
        e.seq_free(s)
    assert e.stats()["kv_pages_used"] == 0


@pytest.mark.parametrize("mega", ["1", "0"])
def test_decode_sample_batch_single_sequence_ext(monkeypatch, mega):
    monkeypatch.setenv("CL_MEGA", mega)
    cfg = eng.model_preset("llama3-8b")
    cfg.update(n_layers=2, max_seq_len=256)
    with eng.Engine(model=cfg, seed=5, max_batch=8) as e:
        _run_sample_batch(e, 1, "x")


@pytest.mark.parametrize("B", [3, 8])
def test_decode_sample_batch_mixed_ext(B):
    with eng.Engine(preset="tiny-test", seed=6, max_batch=8) as e:
        _run_sample_batch(e, B, ("gpx" * 3)[:B])


def test_verify_passes_count_their_own_inputs():
    with eng.Engine(preset="tiny-test", seed=9, max_batch=8, max_seqs=16) as e:
        V = e.cfg["vocab_size"]
        sp = _sp(0.9, 40, 0.95, 1.1, 64, 21)
        p = _prompt(40, V, 2)
        x0 = 77

        def fresh(x=EXT):
            s = e.seq_create()
            e.prefill(s, p, want_logits=False)
            e.set_sampling_ext(s, x)
            return s

        def check(ids, lg, drafts, x, sp_, step0):
            hist = list(p) + [x0]
            for j in range(len(ids)):
                want = eng.sample_token_ext(lg[j], sp_, x, hist + list(drafts[:j]), step0 + j)
                assert want == ids[j], (j, want, ids[j])

        # the drafts repeat x0, so the penalty counts of later rows depend on the pass's own inputs
        y1 = e.decode_verify(fresh(), x0, [x0, x0, 5], sp, 3)[0][0]
        y2 = e.decode_verify(fresh(), x0, [int(y1), x0, x0], sp, 3)[0][1]
        drafts = [int(y1), int(y2), x0, x0, x0]
        ids, lg = e.decode_verify(fresh(), x0, drafts, sp, 3, want_logits=True)
        assert len(ids) >= 3
        check(ids, lg, drafts, EXT, sp, 3)
        # batched verify: ext, plain and greedy sequences in one pass
        seqs = [fresh(EXT2), fresh(eng.sampling_ext()), fresh(EXT)]
        sps = [sp, _sp(0.7, 10, 0.9, 1.0, 0, 4), None]
        dr = [[x0, x0, 9], [x0], [int(y1), 3]]
        out, lg = e.decode_verify_batch(seqs, [x0] * 3, dr, samplings=sps, step0=[5, 6, 0], want_logits=True)
        row0 = 0
        for i in range(3):
            if sps[i] is not None:
                check(out[i], lg[row0:], dr[i], (EXT2, None, EXT)[i], sps[i], [5, 6, 0][i])
            row0 += len(dr[i]) + 1


# ---- request level ---------------------------------------------------------------------------------------------------
def _reqs(V):
    out = []
    for i, n in enumerate([7, 40, 150]):
        sp = _sp(0.8, 40, 0.9, 1.1, 64, 100 + i, 48)
        sp.ignore_eos = 1
        out.append((_prompt(n, V, i), sp, eng.sampling_ext(min_p=0.05 * i, presence_penalty=0.5, frequency_penalty=0.3 * i)))
    sp = _sp(0.8, 0, 0.9, 1.1, 64, 7, 24)                      # top-k 0: the host sampler, ext on the host too
    sp.ignore_eos = 1
    out.append((_prompt(12, V, 9), sp, EXT))
    return out


@pytest.mark.parametrize("scheduler", [False, True])
def test_requests_device_and_host_sampling_agree(monkeypatch, scheduler):
    out, zero = {}, {}
    for dev in ("1", "0"):
        monkeypatch.setenv("CL_DEVICE_SAMPLE", dev)
        with eng.Engine(preset="tiny-test", seed=31, max_batch=4, start_scheduler=scheduler) as e:
            out[dev] = [e.generate_ids_ext(p, sp, x)[0].token_ids for p, sp, x in _reqs(512)]
            if dev == "1":
                zero = [(e.generate_ids_ext(p, sp, eng.sampling_ext())[0].token_ids, e.generate_ids(p, sp).token_ids)
                        for p, sp, _ in _reqs(512)]
            assert e.stats()["kv_pages_used"] == 0
    for a, b in zip(out["1"], out["0"]):
        np.testing.assert_array_equal(a, b)
    for a, b in zero:
        np.testing.assert_array_equal(a, b)
    assert any(not np.array_equal(a, b) for a, (b, _) in zip(out["1"], zero))      # the options change the draws


# ---- stop strings ----------------------------------------------------------------------------------------------------
def _piece(i):
    return b"" if i < 3 else bytes([i - 3]) if i < 259 else b"<%d>" % i


def _raw(ids):
    return b"".join(_piece(int(i)) for i in ids)


def _sanitize(raw: bytes) -> str:
    """Tokenizer::sanitize (csrc/host_util.cpp): invalid UTF-8 and control bytes other than \\n \\t \\r -> U+FFFD."""
    out, i = [], 0
    while i < len(raw):
        c = raw[i]
        n = 1 if c < 0x80 else 2 if c >> 5 == 6 else 3 if c >> 4 == 14 else 4 if c >> 3 == 30 else 0
        ok = n > 0 and i + n <= len(raw) and all(raw[i + k] >> 6 == 2 for k in range(1, n))
        if ok and n == 1 and c < 0x20 and c not in (10, 9, 13):
            ok = False
        if ok:
            out.append(raw[i:i + n].decode("utf-8", "surrogatepass"))
            i += n
        else:
            out.append("�")
            i += 1
    return "".join(out)


def _expect(ids, stops):
    """(text, ids) the stop rule gives for a run that produced ids: ids through the first one whose text contains a stop,
    text cut before the earliest occurrence; None when no stop occurs."""
    for k in range(len(ids)):
        r = _raw(ids[:k + 1])
        hits = [r.find(s) for s in stops if s in r]
        if hits:
            return _sanitize(r[:min(hits)]), np.asarray(ids[:k + 1])
    return None


def _pick_stops(ids):
    """Stop strings taken from a stop-free run's text: inside one token, across tokens and an <id> surface, at the first
    byte, never occurring, and two where the later-listed one matches first."""
    pieces = [_piece(int(i)) for i in ids]
    raw = b"".join(pieces)
    starts = np.cumsum([0] + [len(p) for p in pieces])
    cases = []
    long_tok = [k for k, p in enumerate(pieces) if len(p) >= 4]
    if long_tok:
        k = long_tok[len(long_tok) // 2]
        cases.append([pieces[k][1:-1]])                                      # inside one token's bytes
    surf = [k for k in range(1, len(pieces) - 2) if len(pieces[k]) >= 4]
    if surf:
        k = surf[len(surf) // 2]
        cases.append([raw[starts[k] - 1:starts[k + 2] + 1]])                 # spanning an <id> surface and its neighbours
    mid = len(raw) // 2
    cases.append([raw[mid:mid + 6]])                                         # several tokens
    cases.append([raw[:1]])                                                  # the very first generated byte
    cases.append([b"\x01never\x02"])                                         # never occurs
    cases.append([raw[2 * len(raw) // 3:2 * len(raw) // 3 + 3], raw[len(raw) // 4:len(raw) // 4 + 3]])   # later-listed first
    return [c for c in cases if all(c)]


def _check_stop(res, stops, base_ids, base_text, deltas=None):
    exp = _expect(base_ids, stops)
    if exp is None:
        assert res.done_reason != "stop" and res.text == base_text
        np.testing.assert_array_equal(res.token_ids, base_ids)
    else:
        text, ids = exp
        assert (res.done_reason, res.text) == ("stop", text), (stops, res.text, text)
        np.testing.assert_array_equal(res.token_ids, ids)
    if deltas is not None:
        assert "".join(deltas) == res.text
        for d in deltas:                                                      # no delta carries a stop string
            for s in stops:
                if all(0x20 <= c < 0x7F for c in s):
                    assert s.decode() not in d


def _stop_runs(e, prompts, sps, check_stream=True):
    for p, sp in zip(prompts, sps):
        base = e.generate_ids(p, sp)
        assert base.n_generated > 10
        cases = _pick_stops(base.token_ids)
        assert len(cases) >= 5
        for stops in cases:
            x = eng.sampling_ext(stop=stops)
            res, _ = e.generate_ids_ext(p, sp, x)
            _check_stop(res, stops, base.token_ids, base.text)
            if check_stream:
                deltas = []
                res2, _ = e.generate_ids_ext(p, sp, x, on_text=lambda d, i: deltas.append(d) and False)
                _check_stop(res2, stops, base.token_ids, base.text, deltas)
    assert e.stats()["kv_pages_used"] == 0


def _stop_setup():
    greedy = eng.greedy(120, ignore_eos=True)
    dev = _sp(1.2, 128, 1.0, 1.0, 0, 77, 120)                  # device-sampled, wide: many <id> surfaces
    dev.ignore_eos = 1
    return [_prompt(30, 512, 1), _prompt(50, 512, 4)], [greedy, dev]


@pytest.mark.parametrize("scheduler", [False, True])
def test_stop_strings_sync_and_scheduler(scheduler):
    prompts, sps = _stop_setup()
    with eng.Engine(preset="tiny-test", seed=41, max_batch=4, start_scheduler=scheduler) as e:
        _stop_runs(e, prompts, sps)


def test_stop_strings_with_speculation():
    prompts, sps = _stop_setup()
    with eng.Engine(preset="tiny-test", seed=41, max_batch=4, speculate=6) as e:
        _stop_runs(e, prompts, sps, check_stream=False)
        assert e.spec_stats()["tokens_accepted"] > 0


def test_stop_strings_with_context_shift():
    cfg = eng.model_preset("tiny-test")
    cfg["max_seq_len"] = 160
    with eng.Engine(model=cfg, seed=43, max_batch=4, context_shift=True, num_keep=4, page_size=16) as e:
        sp = eng.greedy(300, ignore_eos=True)
        p = _prompt(40, 512, 3)
        base = e.generate_ids(p, sp)
        assert base.n_generated == 300
        raw = _raw(base.token_ids)
        late = _raw(base.token_ids[:250])
        for stops in ([raw[len(late):len(late) + 4]], [raw[-3:]]):            # matched after the window has shifted
            res, _ = e.generate_ids_ext(p, sp, eng.sampling_ext(stop=stops))
            _check_stop(res, stops, base.token_ids, base.text)
        assert e.stats()["kv_pages_used"] == 0


def test_stop_strings_under_preemption():
    cfg = eng.model_preset("tiny-test")
    cfg["max_seq_len"] = 512
    kv_bytes = 2 * cfg["n_layers"] * cfg["n_kv_heads"] * cfg["head_dim"] * 2 * 16 * 40
    with eng.Engine(model=cfg, seed=7, max_batch=4, max_seqs=4, page_size=16, kv_pool_bytes=kv_bytes, start_scheduler=True) as e:
        sp = eng.greedy(200, ignore_eos=True)
        out = {}

        def run(i):
            p = _prompt(100, 512, i)
            base = e.generate_ids(p, sp)
            stops = [_raw(base.token_ids)[150:154]]
            out[i] = (e.generate_ids_ext(p, sp, eng.sampling_ext(stop=stops))[0], stops)

        ts = [threading.Thread(target=run, args=(i,)) for i in range(4)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert sum(out[i][0].n_preempted for i in range(4)) > 0
        stopped = 0
        for i in range(4):
            res, stops = out[i]
            # the run's own ids: the match completes on the last one, and the text is cut before it
            exp = _expect(res.token_ids, stops)
            if exp is None:                     # recomputation after a preemption may move a near tie: no match at all
                assert res.done_reason == "length" and res.n_generated == 200
                continue
            stopped += 1
            assert res.done_reason == "stop" and res.text == exp[0] and len(exp[1]) == res.n_generated
        assert stopped >= 2
        assert e.stats()["kv_pages_used"] == 0


def test_stop_strings_over_the_wire():
    with eng.Engine(preset="tiny-test", seed=47, max_batch=4) as e:
        for temp in (0.0, 1.1):
            opts = dict(temperature=temp, top_k=64, seed=3, num_predict=80, logprobs=True, top_logprobs=2)

            def ask(stream, **kw):
                req = BaseMessage(generate_request=GenerateRequest(model=e.model_name, prompt="stop me ☃", stream=stream,
                                                                   options=GenerateOptions(**opts, **kw))).encode()
                if not stream:
                    return [BaseMessage.decode(e.handle_message(req)).generate_response]
                frames = []
                e.handle_message_stream(req, None, lambda f: frames.append(BaseMessage.decode(f).generate_response) and False)
                return frames

            base = ask(False)[0]
            raw = b"".join(t.bytes for t in base.logprobs)
            assert len(raw) > 20

            def text_at(i, n):                  # the first printable ASCII window at or after i (the wire carries strings)
                while i + n <= len(raw) and not all(0x20 <= c < 0x7F for c in raw[i:i + n]):
                    i += 1
                return raw[i:i + n] if i + n <= len(raw) else b""

            cases = [c for c in ([text_at(10, 3)], [text_at(0, 1)], [text_at(len(raw) // 2, 3), text_at(5, 3)]) if all(c)]
            assert len(cases) >= 2
            for stops in cases:
                ids_like = [t.bytes for t in base.logprobs]
                k = next(j for j in range(len(ids_like)) if any(s in b"".join(ids_like[:j + 1]) for s in stops))
                r = b"".join(ids_like[:k + 1])
                want = _sanitize(r[:min(r.find(s) for s in stops if s in r)])
                one = ask(False, stop=[s.decode() for s in stops])[0]
                assert (one.done_reason, one.response) == ("stop", want)
                assert len(one.logprobs) == k + 1 and one.logprobs == base.logprobs[:k + 1]
                frames = ask(True, stop=[s.decode() for s in stops])
                assert frames[-1].done and frames[-1].done_reason == "stop"
                assert "".join(f.response for f in frames) == want
                assert sum(len(f.logprobs) for f in frames) == k + 1
        assert e.stats()["kv_pages_used"] == 0


def test_stop_and_ext_inputs_over_the_limits_are_rejected():
    with eng.Engine(preset="tiny-test", seed=1) as e:
        p, sp = _prompt(10, 512), eng.greedy(8)
        for bad in (eng.sampling_ext(stop=["x"] * 17), eng.sampling_ext(stop=["y" * 257]), eng.sampling_ext(min_p=-0.5),
                    eng.sampling_ext(presence_penalty=float("nan"))):
            with pytest.raises(eng.EngineError) as ei:
                e.generate_ids_ext(p, sp, bad)
            assert ei.value.status == eng.CL_ERR_INVALID_ARG and ei.value.detail
        ok, _ = e.generate_ids_ext(p, sp, eng.sampling_ext(stop=["", "z" * 256] + ["q"] * 15))   # empty strings are dropped
        assert ok.n_generated == 8
        s = e.seq_create()
        with pytest.raises(eng.EngineError):
            e.set_sampling_ext(s, eng.sampling_ext(min_p=2.0))
        e.set_sampling_ext(s, eng.sampling_ext(stop=["ignored"], min_p=0.1))
        e.seq_free(s)
        assert e.stats()["kv_pages_used"] == 0
