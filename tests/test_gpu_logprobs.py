"""Per-token log-probabilities of the step tail (cl_seq_set_logprobs, cl_op_sample_logprobs, cl_generate_ids_logprobs).

A record is {chosen id, its logprob, the top n ids and logprobs} of log_softmax over the raw fp32 logits row the tail
chose from.  The kernel is checked against float64 log_softmax of the same fp32 rows; every engine path against float64
log_softmax of that call's own logits_out; the request level against the same request without logprobs (same ids) and
a teacher-forced replay.  Turning logprobs on never changes an id."""
import threading

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    for k in ("CL_SPECULATE", "CL_SPECULATE_BATCH", "CL_PREFIX_CACHE"):
        monkeypatch.delenv(k, raising=False)


def _bound(ref):
    """|kernel - float64| allowed for one logprob: fp32 slice sums, expf and the final fp32 subtraction."""
    return 2e-5 + np.abs(ref) * 2.0 ** -20


def _ref(row):
    x = np.asarray(row, np.float64)
    m = x.max()
    lse = m + np.log(np.exp(x - m).sum())
    return x - lse


def _top_ref(row, n):
    # value descending, id ascending
    order = np.lexsort((np.arange(len(row)), -np.asarray(row, np.float64)))
    return order[:n]


def _check_record(rec, row, top_n, chosen=None):
    ref = _ref(row)
    n = min(top_n, len(row))
    assert rec["n_top"] == n
    want = _top_ref(row, n)
    assert np.array_equal(rec["top_ids"][:n], want), (rec["top_ids"][:n], want)
    got = rec["top_logprobs"][:n].astype(np.float64)
    assert np.all(np.abs(got - ref[want]) <= _bound(ref[want])), np.abs(got - ref[want]).max()
    idx = int(rec["id"]) if chosen is None else int(chosen)
    assert rec["id"] == idx
    assert abs(float(rec["logprob"]) - ref[idx]) <= _bound(ref[idx]), (float(rec["logprob"]), ref[idx])
    assert rec["logprob"] <= 0.0


def _sp(temp, top_k, top_p, pen, last_n, seed):
    s = eng.Sampling()
    s.temperature, s.top_k, s.top_p, s.repeat_penalty, s.repeat_last_n, s.seed = temp, top_k, top_p, pen, last_n, seed
    s.max_new_tokens = -1
    return s


def _bf16(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def _row(kind, V, rng):
    if kind == "equal":
        return np.full(V, 1.25, np.float32)
    x = rng.normal(0.0, 3.0, V).astype(np.float32)
    if kind == "bf16":
        x = _bf16(x)
    elif kind == "wide":
        x = rng.uniform(-1e4, 1e4, V).astype(np.float32)
    return x


SAMPLERS = [None, _sp(0.8, 40, 0.9, 1.1, 64, 7), _sp(1.0, 5, 1.0, 1.0, 0, 11), _sp(1.3, 128, 0.5, 1.3, 16, 13),
            _sp(0.6, 1, 1.0, 1.0, 0, 3)]


def _greedy_sp():
    return _sp(0.0, 40, 0.9, 1.0, 0, 0)


@pytest.mark.parametrize("V", [512, 32000, 32003, 128256, 163840])
def test_op_logprobs_against_float64(V):
    rng = np.random.default_rng(V)
    kinds = ["gauss", "bf16", "equal", "wide"]
    for top_n in (0, 1, 5, 20):
        rows, sps, hists = [], [], []
        for kind in kinds:
            for sp in SAMPLERS:
                rows.append(_row(kind, V, rng))
                sps.append(sp if sp is not None else _greedy_sp())
                hists.append(rng.integers(0, V, 20).astype(np.int32))
        lg = np.stack(rows)
        steps = rng.integers(0, 2**40, len(rows)).astype(np.uint64)
        ids, recs = eng.op_sample_logprobs(lg, sps, hists, steps, top_n)
        ids2, recs2 = eng.op_sample_logprobs(lg, sps, hists, steps, top_n)
        assert np.array_equal(ids, ids2) and recs.tobytes() == recs2.tobytes()   # bit-identical launches
        for i in range(len(rows)):
            _check_record(recs[i], lg[i], top_n, ids[i])
            if sps[i].temperature <= 0:
                assert ids[i] == _top_ref(lg[i], 1)[0]
                if top_n > 0:
                    assert recs[i]["top_ids"][0] == ids[i] and recs[i]["top_logprobs"][0] == recs[i]["logprob"]
        # the draws equal cl_op_sample's
        drawn = [i for i in range(len(rows)) if sps[i].temperature > 0]
        plain = eng.op_sample(lg[drawn], [sps[i] for i in drawn], [hists[i] for i in drawn], steps[drawn])
        assert np.array_equal(plain, ids[drawn])


def test_op_logprobs_bound_has_teeth():
    """A wrong lse (one slice's mass dropped, or the max alone) lands outside the bound on these rows."""
    rng = np.random.default_rng(5)
    for V in (512, 32000, 128256):
        for kind in ("gauss", "bf16", "equal"):
            row = _row(kind, V, rng).astype(np.float64)
            ref = _ref(row)
            slice_ = (V + 63) // 64
            m = row.max()
            dropped = m + np.log(np.exp(row[slice_:] - m).sum())
            max_only = m
            for wrong in (dropped, max_only):
                bad = row - wrong
                assert np.any(np.abs(bad - ref) > _bound(ref))


def test_op_logprobs_row_independent_of_neighbours():
    V = 32000
    rng = np.random.default_rng(9)
    lg = np.stack([_row("gauss", V, rng) for _ in range(8)])
    sps = [_greedy_sp() if i % 2 else SAMPLERS[1 + i % 4] for i in range(8)]
    hists = [rng.integers(0, V, 10).astype(np.int32) for _ in range(8)]
    steps = np.arange(8, dtype=np.uint64)
    _, together = eng.op_sample_logprobs(lg, sps, hists, steps, 20)
    for i in range(8):
        _, alone = eng.op_sample_logprobs(lg[i:i + 1], [sps[i]], [hists[i]], steps[i:i + 1], 20)
        assert alone.tobytes() == together[i:i + 1].tobytes()
    with pytest.raises(eng.EngineError) as ei:
        eng.op_sample_logprobs(lg[:1], [sps[0]], [hists[0]], steps[:1], 21)
    assert ei.value.status == eng.CL_ERR_INVALID_ARG


def _cfg(name, max_seq_len=2048):
    cfg = dict(oc.PRESETS["llama3-8b" if name == "llama3-8b-2l" else name])
    if name == "llama3-8b-2l":
        cfg["n_layers"] = 2
    cfg["max_seq_len"] = max_seq_len
    return cfg


def _ids(n, vocab, salt):
    return np.array([(i * 7919 + 13 + salt * 104729) % (vocab - 3) + 3 for i in range(n)], np.int32)


@pytest.mark.parametrize("shape,page,mega,graph", [("tiny-test", 16, True, True), ("tiny-test", 64, False, False),
                                                   ("tiny-test", 32, True, False), ("llama3-8b-2l", 32, True, True),
                                                   ("llama3-8b-2l", 32, False, True), ("llama3-8b-2l", 16, True, True),
                                                   ("llama3-8b-2l", 64, False, True)])
def test_engine_paths_record_their_logits(shape, page, mega, graph, monkeypatch):
    monkeypatch.setenv("CL_MEGA", "1" if mega else "0")
    cfg = _cfg(shape)
    V = cfg["vocab_size"]
    with eng.Engine(model=cfg, seed=17, max_batch=8, max_seqs=32, page_size=page, use_cuda_graph=graph) as e:
        if not mega:
            assert not e.runs_mega_kernel()
        def armed(top_n=20):
            s = e.seq_create()
            e.set_logprobs(s, top_n)
            return s

        # prefill: token-wise, split-K and tile paths
        for n in (1, 40, 300):
            s = armed(5)
            lg = e.prefill(s, _ids(n, V, n))
            rec = e.take_logprobs(s)
            assert len(rec) == 1
            _check_record(rec[0], lg, 5)
            # decode_step, with an unarmed twin giving the same ids
            t = e.seq_create()
            e.prefill(t, _ids(n, V, n), want_logits=False)
            tok = int(rec[0]["id"])
            for _ in range(3):
                lg, am = e.decode_step(s, tok)
                _, am2 = e.decode_step(t, tok, want_logits=False)
                assert am == am2
                r = e.take_logprobs(s)
                assert len(r) == 1 and r[0]["id"] == am
                _check_record(r[0], lg, 5)
                tok = am
            assert len(e.take_logprobs(t)) == 0
            e.seq_free(s)
            e.seq_free(t)
        # batched step mixing armed and unarmed sequences, against an all-armed twin batch and an unarmed one: the same
        # ids, and an armed row's record the same bits whatever its neighbours' arming
        for B in (3, 8):
            def batch(arm):
                seqs = [e.seq_create() for _ in range(B)]
                for b, s in enumerate(seqs):
                    e.prefill(s, _ids(10 + 7 * b, V, b), want_logits=False)
                    if arm(b):
                        e.set_logprobs(s, 20)
                    e.take_logprobs(s)
                return seqs
            toks = [int(x) for x in _ids(B, V, 99)]
            mixed, full, none = batch(lambda b: b % 2 == 0), batch(lambda b: True), batch(lambda b: False)
            lg, am = e.decode_step_batch(mixed, toks)
            _, am_full = e.decode_step_batch(full, toks, want_logits=False)
            _, am_none = e.decode_step_batch(none, toks, want_logits=False)
            assert np.array_equal(am, am_full) and np.array_equal(am, am_none)
            for b, s in enumerate(mixed):
                r, rf = e.take_logprobs(s), e.take_logprobs(full[b])
                assert len(e.take_logprobs(none[b])) == 0
                if b % 2:
                    assert len(r) == 0
                else:
                    assert len(r) == 1 and r[0]["id"] == am[b]
                    _check_record(r[0], lg[b], 20)
                    assert r.tobytes() == rf.tobytes()
            for s in mixed + full + none:
                e.seq_free(s)
        # multi-prompt prefill
        seqs = [armed(3) for _ in range(3)]
        lg = e.prefill_batch(seqs, [_ids(20 + 30 * i, V, i) for i in range(3)])
        for i, s in enumerate(seqs):
            r = e.take_logprobs(s)
            assert len(r) == 1
            _check_record(r[0], lg[i], 3)
            e.seq_free(s)


@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_device_loops_match_step_replay(shape):
    cfg = _cfg(shape)
    V = cfg["vocab_size"]
    n_steps = 1030 if shape == "tiny-test" else 40      # past the 1024-step ring at tiny-test
    prompts = [_ids(12 + 5 * b, V, b) for b in range(3)]
    sps = [_sp(0.9, 40, 0.9, 1.1, 32, 5), None, _sp(1.1, 8, 1.0, 1.0, 0, 9)]
    with eng.Engine(model=cfg, seed=23, max_batch=4, max_seqs=16) as e:
        def fresh(arm):
            seqs = [e.seq_create() for _ in prompts]
            for s, p in zip(seqs, prompts):
                e.prefill(s, p, want_logits=False)
                if arm:
                    e.set_logprobs(s, 20)
            return seqs
        firsts = [int(p[-1]) for p in prompts]
        samplings = [s if s is not None else _sp(0.0, 40, 0.9, 1.0, 0, 0) for s in sps]
        seqs = fresh(True)
        for s in seqs:
            e.take_logprobs(s)
        ids, _ = e.decode_sample_batch(seqs, firsts, samplings, n_steps)
        recs = [e.take_logprobs(s) for s in seqs]
        twin = fresh(False)
        ids2, _ = e.decode_sample_batch(twin, firsts, samplings, n_steps)
        assert np.array_equal(ids, ids2)
        for b in range(3):
            assert len(recs[b]) == n_steps and np.array_equal(recs[b]["id"], ids[:, b])
        # replay the same ids through cl_decode_step_batch (armed): records within the bound of the replay's logits
        rep = fresh(True)
        for s in rep:
            e.take_logprobs(s)
        feed = firsts
        check = range(n_steps) if n_steps <= 64 else list(range(8)) + list(range(1016, 1030))
        for i in range(n_steps):
            lg, _ = e.decode_step_batch(rep, feed, want_logits=i in check)
            for b, s in enumerate(rep):
                r = e.take_logprobs(s)[0]
                if i in check:                  # the loop's record of step i against the replay's logits of step i
                    _check_record(recs[b][i], lg[b], 20, ids[i, b])
                    _check_record(r, lg[b], 20)
                    np.testing.assert_array_equal(r["top_ids"], recs[b][i]["top_ids"])
            feed = [int(x) for x in ids[i]]
        # greedy device loop
        g = fresh(True)
        for s in g:
            e.take_logprobs(s)
        gids = e.decode_greedy_batch(g, firsts, 16)[0]
        for b, s in enumerate(g):
            r = e.take_logprobs(s)
            assert len(r) == 16 and np.array_equal(r["id"], gids[:, b])
            assert np.array_equal(r["top_ids"][:, 0], gids[:, b])


@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_verify_records_of_emitted_rows(shape):
    cfg = _cfg(shape)
    V = cfg["vocab_size"]
    with eng.Engine(model=cfg, seed=29, max_batch=8, max_seqs=8) as e:
        s = e.seq_create()
        p = _ids(30, V, 1)
        e.prefill(s, p, want_logits=False)
        e.set_logprobs(s, 20)
        x0 = int(p[-1])
        twin = e.seq_create()
        e.prefill(twin, p, want_logits=False)
        ids, lg = e.decode_verify(s, x0, [int(v) for v in p[:5]], want_logits=True)
        ids_twin, _ = e.decode_verify(twin, x0, [int(v) for v in p[:5]])
        assert np.array_equal(ids, ids_twin)
        r = e.take_logprobs(s)
        assert len(r) == len(ids)
        for j in range(len(ids)):
            _check_record(r[j], lg[j], 20, ids[j])
        # several sequences, mixed arming and samplers
        seqs = [e.seq_create() for _ in range(3)]
        for i, q in enumerate(seqs):
            e.prefill(q, _ids(20 + i, V, i + 3), want_logits=False)
            if i != 1:
                e.set_logprobs(q, 7)
        drafts = [[3, 4, 5], [], [7, 8]]
        out, lg = e.decode_verify_batch(seqs, [11, 12, 13], drafts, samplings=[None, _sp(0.8, 40, 0.9, 1.0, 0, 1), None],
                                        want_logits=True)
        row0 = 0
        for i, q in enumerate(seqs):
            r = e.take_logprobs(q)
            if i == 1:
                assert len(r) == 0
            else:
                assert len(r) == len(out[i])
                for j in range(len(out[i])):
                    _check_record(r[j], lg[row0 + j], 7, out[i][j])
            row0 += len(drafts[i]) + 1


def _req_checks(res, recs, top_n):
    assert len(recs) == res.n_generated
    assert np.array_equal(recs["id"], res.token_ids)
    assert np.all(recs["logprob"] <= 0)
    assert np.all(recs["n_top"] == top_n)
    for r in recs:
        t = r["top_logprobs"][:top_n]
        assert np.all(np.diff(t) <= 0)
        assert np.exp(t.astype(np.float64)).sum() <= 1 + 1e-6


@pytest.mark.parametrize("scheduler", [False, True])
def test_request_level_logprobs(scheduler):
    cfg = _cfg("tiny-test")
    V = cfg["vocab_size"]
    greedy = eng.greedy(40, ignore_eos=True)
    dev = eng.ollama_default_sampling(seed=5, max_new_tokens=40)
    dev.ignore_eos = 1
    host = eng.ollama_default_sampling(seed=3, max_new_tokens=40)
    host.top_k, host.ignore_eos = 0, 1
    prompts = {k: _ids(30 + 11 * i, V, i) for i, k in enumerate(("g", "d", "h"))}
    sps = {"g": greedy, "d": dev, "h": host}
    for spec in (0, 4):
        with eng.Engine(model=cfg, seed=31, max_batch=4, max_seqs=4, speculate=spec, speculate_batch=4 if spec else 1,
                        start_scheduler=scheduler) as e:
            plain, withlp = {}, {}
            for k in sps:                       # one request at a time: the same steps with and without logprobs
                plain[k] = e.generate_ids(prompts[k], sps[k])
                withlp[k] = e.generate_ids_logprobs(prompts[k], sps[k], 5)
                assert np.array_equal(withlp[k][0].token_ids, plain[k].token_ids), k
                _req_checks(*withlp[k], 5)
            if scheduler:                       # concurrent: batch composition varies, so only the records' own rules
                out = {}
                ts = [threading.Thread(target=lambda k=k: out.__setitem__(k, e.generate_ids_logprobs(prompts[k], sps[k], 5)))
                      for k in sps]
                for t in ts:
                    t.start()
                for t in ts:
                    t.join()
                for k in sps:
                    _req_checks(*out[k], 5)
                assert e.stats()["kv_pages_used"] == 0
        # teacher-forced replay of every request (greedy, device-sampled, host-sampled) on an engine of the same weights: the
        # chosen id's logprob within twice the logit tolerance of float64 log_softmax of the replay's logits
        tol = 2 * (0.05 + 0.03 * np.sqrt(cfg["n_layers"]))
        with eng.Engine(model=cfg, seed=31, max_batch=4, max_seqs=4) as ref:
            for k in sps:
                res, recs = withlp[k]
                s = ref.seq_create()
                seen = [ref.prefill(s, prompts[k])]
                for t in res.token_ids[:-1]:
                    seen.append(ref.decode_step(s, int(t))[0])
                for i, lgi in enumerate(seen):
                    want = _ref(lgi)[res.token_ids[i]]
                    assert abs(float(recs[i]["logprob"]) - want) <= tol, (k, i, float(recs[i]["logprob"]), want)
                ref.seq_free(s)


def test_stream_frames_concatenate_to_the_single_response():
    from crowdllama_b200.pb import BaseMessage, GenerateOptions, GenerateRequest
    cfg = _cfg("tiny-test")
    with eng.Engine(model=cfg, seed=31, max_batch=4, max_seqs=4) as e:
        for opts in (GenerateOptions(temperature=0.0, num_predict=24, logprobs=True, top_logprobs=4),
                     GenerateOptions(temperature=0.7, top_k=40, seed=9, num_predict=24, logprobs=True, top_logprobs=0),
                     GenerateOptions(temperature=0.7, top_k=0, seed=9, num_predict=24, logprobs=True, top_logprobs=2)):
            req = BaseMessage(generate_request=GenerateRequest(model=e.model_name, prompt="héllo wörld ☃", stream=True, options=opts))
            one = BaseMessage.decode(e.handle_message(req.encode())).generate_response
            frames = []
            e.handle_message_stream(req.encode(), None, lambda f: frames.append(BaseMessage.decode(f).generate_response) and False)
            assert frames[-1].done and sum(len(f.logprobs) for f in frames) == len(one.logprobs) > 0
            assert [t for f in frames for t in f.logprobs] == one.logprobs        # bit for bit: floats compare exactly
            assert "".join(f.response for f in frames) == one.response
            for t in one.logprobs:
                assert len(t.top_logprobs) == opts.top_logprobs and t.logprob <= 0
                assert t.token == t.bytes.decode("utf-8", "replace") or "\ufffd" in t.token
        # without logprobs: no records; top_logprobs without logprobs or above 20: refused
        plain = BaseMessage(generate_request=GenerateRequest(model=e.model_name, prompt="x", options=GenerateOptions(num_predict=4)))
        assert BaseMessage.decode(e.handle_message(plain.encode())).generate_response.logprobs == []
        for bad in (GenerateOptions(top_logprobs=3), GenerateOptions(logprobs=True, top_logprobs=21)):
            with pytest.raises(eng.EngineError) as ei:
                e.handle_message(BaseMessage(generate_request=GenerateRequest(model=e.model_name, prompt="x", options=bad)).encode())
            assert ei.value.status == eng.CL_ERR_INVALID_ARG


def test_request_logprobs_under_preemption():
    cfg = _cfg("tiny-test", 512)
    V = cfg["vocab_size"]
    kv_bytes = 2 * cfg["n_layers"] * cfg["n_kv_heads"] * cfg["head_dim"] * 2 * 16 * 40   # 40 pages of 16 tokens
    with eng.Engine(model=cfg, seed=7, max_batch=4, max_seqs=4, page_size=16, kv_pool_bytes=kv_bytes, start_scheduler=True) as e:
        out = {}
        ts = [threading.Thread(target=lambda i=i: out.__setitem__(i, e.generate_ids_logprobs(_ids(100, V, i),
                                                                                              eng.greedy(200, ignore_eos=True), 3)))
              for i in range(4)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert sum(out[i][0].n_preempted for i in range(4)) > 0
        for i in range(4):
            res, recs = out[i]
            assert res.n_generated == 200
            _req_checks(res, recs, 3)
            assert np.array_equal(recs["top_ids"][:, 0], res.token_ids)   # greedy: the chosen id is the top one
        assert e.stats()["kv_pages_used"] == 0
