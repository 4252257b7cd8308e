"""Speculative decoding (cl_decode_verify, cl_engine_config.speculate): a verify pass runs x0, d1 .. dk through every layer
at once, and row r makes the decode step tail's choice.  Acceptance must equal a host replay on the returned logits id for
id, the logits must match the CPU oracle teacher-forced, rejected rows must leave no trace, the state after a pass must be
that of a + 1 single steps, attached prefix-cache pages must stay untouched, and the scheduler must emit what sequential
decoding emits."""
import threading
import time

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    for k in ("CL_SPECULATE", "CL_PREFIX_CACHE"):
        monkeypatch.delenv(k, raising=False)


def _cfg(name, max_seq_len):
    cfg = dict(oc.PRESETS["llama3-8b" if name == "llama3-8b-2l" else name])
    if name == "llama3-8b-2l":
        cfg["n_layers"] = 2
    cfg["max_seq_len"] = max_seq_len
    return cfg


def _tol(n_layers):
    return 0.05 + 0.03 * float(np.sqrt(n_layers))


def _ids(n, vocab, salt):
    return np.array([(i * 7919 + 13 + salt * 104729) % (vocab - 3) + 3 for i in range(n)], np.int32)


def _sp(temp, top_k, top_p, pen, last_n, seed):
    s = eng.Sampling()
    s.temperature, s.top_k, s.top_p, s.repeat_penalty, s.repeat_last_n, s.seed = temp, top_k, top_p, pen, last_n, seed
    s.max_new_tokens = -1
    return s


SAMPLINGS = {
    "greedy": None,
    "ollama": _sp(0.8, 40, 0.9, 1.1, 64, 7),
    "topk5": _sp(1.0, 5, 1.0, 1.0, 0, 11),
    "wide": _sp(1.3, 128, 0.5, 1.3, 16, 13),
}


def _choice(lg, sp, hist, step):
    return int(np.argmax(lg)) if sp is None else eng.sample_token(lg, sp, hist, step)


def _replay(logits, sp, hist, x0, draft, step0):
    """Host replay of a verify pass: row r's choice with history hist + x0, d1 .. dr at step step0 + r; then the rule."""
    inputs = [int(x0)] + [int(d) for d in draft]
    y = [_choice(logits[r], sp, list(hist) + inputs[:r + 1], step0 + r) for r in range(len(inputs))]
    a = 0
    while a < len(draft) and y[a] == int(draft[a]):
        a += 1
    return y[:a + 1]


def _fresh(e, prompt):
    s = e.seq_create()
    lg = e.prefill(s, prompt)
    return s, int(lg.argmax())


def _continuation(e, prompt, x0, sp, step0, n):
    """The ids sequential decoding draws after x0 (a twin sequence)."""
    s, _ = _fresh(e, prompt)
    if sp is None:
        ids, _ = e.decode_greedy(s, x0, n)
    else:
        ids, _ = e.decode_sample_batch([s], [x0], [sp], n, step0=[step0])
        ids = ids[:, 0]
    e.seq_free(s)
    return [int(i) for i in ids]


# ---- 1. acceptance is exact ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("page", [16, 32, 64])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_acceptance_equals_host_replay(shape, page):
    cfg = _cfg(shape, 1024)
    V = cfg["vocab_size"]
    rng = np.random.default_rng(page)
    prompt = _ids(2 * page + page // 2 + 3, V, 1)          # the 16 verify rows cross a page boundary
    step0 = 5
    accepted = 0
    with eng.Engine(model=cfg, seed=77, max_batch=2, max_seqs=4, page_size=page) as e:
        for name, sp in SAMPLINGS.items():
            s, x0 = _fresh(e, prompt)
            e.seq_free(s)
            right = _continuation(e, prompt, x0, sp, step0, 15)
            for k in (1, 4, 15):
                drafts = [right[:k]]                                        # all right (up to near-tie flips)
                for j in range(k):                                          # first wrong at d_{j+1}
                    d = list(right[:k])
                    d[j] = (d[j] + 1 + int(rng.integers(0, V - 1))) % V
                    drafts.append(d)
                drafts.append([int(v) for v in rng.integers(0, V, k)])      # random
                for d in drafts:
                    s, x = _fresh(e, prompt)
                    assert x == x0
                    len0 = e.seq_len(s)
                    ids, lg = e.decode_verify(s, x0, d, sp, step0, want_logits=True)
                    assert lg.shape == (k + 1, V) and np.isfinite(lg).all()
                    want = _replay(lg, sp, prompt, x0, d, step0)
                    assert ids.tolist() == want, (name, k, d, ids, want)
                    assert e.seq_len(s) == len0 + len(ids)
                    accepted += len(ids) - 1
                    e.seq_free(s)
        st = e.spec_stats()
        assert st["enabled"] == 0 and st["verify_passes"] > 0
        assert st["tokens_emitted"] == st["tokens_accepted"] + st["verify_passes"] and st["tokens_accepted"] == accepted
        assert e.stats()["kv_pages_used"] == 0
    print(f"{shape}/page {page}: {accepted} drafted tokens accepted")


# ---- 2. verify logits match the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("page", [16, 32, 64])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_verify_logits_match_the_oracle(shape, page):
    cfg = _cfg(shape, 512)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    prompt = _ids(page + 5, V, 2)
    m = oc.Model(cfg, seed=4242)
    with eng.Engine(model=cfg, seed=4242, max_batch=2, max_seqs=2, page_size=page) as e:
        so = m.new_seq(256)
        so.forward(prompt)
        s, x0 = _fresh(e, prompt)
        worst = 0.0
        for k in (1, 7, 15):
            d = _ids(k, V, 30 + k)
            ids, lg = e.decode_verify(s, x0, d, None, 0, want_logits=True)
            ref = so.forward(np.concatenate([[x0], d]), all_logits=True)
            err = float(np.abs(lg - ref).max())
            worst = max(worst, err)
            assert err < _tol(L), (k, err)
            n = len(ids)
            so.truncate(len(so) - (k + 1) + n)             # the oracle keeps x0, d1 .. da, like the engine
            assert len(so) == e.seq_len(s)
            x0 = int(ids[-1])
        so.close()
    m.close()
    print(f"{shape}/page {page}: max |dlogit| {worst:.4f} (tolerance {_tol(L):.3f})")


@pytest.mark.parametrize("shape,n_layers", [("llama3-8b", 2), ("llama3-8b", 32)])
def test_verify_logits_match_the_oracle_behind_a_long_cache(shape, n_layers):
    cfg = _cfg(shape, 4096 + 64)
    cfg["n_layers"] = n_layers
    V = cfg["vocab_size"]
    m = oc.Model(cfg, seed=1234)
    with eng.Engine(model=cfg, seed=1234, max_batch=2, max_seqs=2) as e:
        s = e.seq_create()
        e.seq_fake_fill(s, 4096)
        so = m.new_seq(4096 + 32)
        so.fake_fill(4096)
        d = _ids(15, V, 5)
        _, lg = e.decode_verify(s, 17, d, None, 0, want_logits=True)
        ref = so.forward(np.concatenate([[17], d]), all_logits=True)
        err = float(np.abs(lg - ref).max())
        so.close()
    m.close()
    print(f"{shape}/{n_layers}L behind 4096 cached tokens: max |dlogit| {err:.4f} (tolerance {_tol(n_layers):.3f})")
    assert err < _tol(n_layers)


# ---- 3. rejected drafts leave no trace -------------------------------------------------------------------------------------
@pytest.mark.parametrize("page", [16, 64])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_rejected_drafts_leave_no_trace(shape, page):
    cfg = _cfg(shape, 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    prompt = _ids(page + page // 2 + 7, V, 3)
    with eng.Engine(model=cfg, seed=5, max_batch=2, max_seqs=4, page_size=page) as e:
        s, x0 = _fresh(e, prompt)
        e.seq_free(s)
        right = _continuation(e, prompt, x0, None, 0, 8)
        for keep in (0, 2):                                    # a = 0, and a pass that accepts a right prefix first
            da = right[:keep] + [(right[keep] + 1 + i) % V for i in range(7 - keep)]
            db = right[:keep] + [(right[keep] + 101 + 3 * i) % V for i in range(7 - keep)]
            sa, _ = _fresh(e, prompt)
            sb, _ = _fresh(e, prompt)
            ia, _ = e.decode_verify(sa, x0, da, None, 0)
            ib, _ = e.decode_verify(sb, x0, db, None, 0)
            assert ia.tolist() == ib.tolist()
            n = e.seq_len(sa)
            assert n == e.seq_len(sb) == len(prompt) + len(ia)
            for l in range(L):
                for w in (0, 1):
                    assert np.array_equal(e.debug_kv(sa, l, w, 0, n), e.debug_kv(sb, l, w, 0, n))
            tok = int(ia[-1])
            for _ in range(6):                                 # the next decode steps, bit for bit
                la, am = e.decode_step(sa, tok)
                lb, _ = e.decode_step(sb, tok)
                assert np.array_equal(la, lb)
                tok = am
            e.seq_free(sa)
            e.seq_free(sb)
        assert e.stats()["kv_pages_used"] == 0


# ---- 4. the state after a pass equals a + 1 steps --------------------------------------------------------------------------
@pytest.mark.parametrize("mega", ["1", "0"])
def test_state_after_a_pass_equals_single_steps(monkeypatch, mega):
    monkeypatch.setenv("CL_MEGA", mega)
    cfg = _cfg("llama3-8b-2l", 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = _tol(L)
    prompt = _ids(45, V, 4)
    with eng.Engine(model=cfg, seed=21, max_batch=2, max_seqs=4) as e:
        # greedy: continue with single steps after a partially accepted pass; a twin stepped x0, d1 .. da one at a time
        s, x0 = _fresh(e, prompt)
        e.seq_free(s)
        right = _continuation(e, prompt, x0, None, 0, 8)
        d = right[:3] + [(right[3] + 9) % V] + right[4:7]
        s, _ = _fresh(e, prompt)
        ids, _ = e.decode_verify(s, x0, d, None, 0)
        n = len(ids)
        t, _ = _fresh(e, prompt)
        for tok in [x0] + d[:n - 1]:
            e.decode_step(t, tok)
        assert e.seq_len(s) == e.seq_len(t)
        tok = int(ids[-1])
        for _ in range(8):
            ls, am = e.decode_step(s, tok)
            lt, _ = e.decode_step(t, tok)
            assert float(np.abs(ls - lt).max()) < tol
            tok = am
        g_s, _ = e.decode_greedy(s, tok, 16)                    # B = 1: persistent kernel (CL_MEGA=1) or per-op
        g_t, _ = e.decode_greedy(t, tok, 16)
        assert len(g_s) == len(g_t) == 16
        e.seq_free(s)
        e.seq_free(t)
        # sampled: the next draws are the host sampler's at step step0 + n, with the accepted tokens in the history
        sp, step0 = SAMPLINGS["ollama"], 3
        right = _continuation(e, prompt, x0, sp, step0, 8)
        d = right[:2] + [(right[2] + 5) % V] + right[3:6]
        s, _ = _fresh(e, prompt)
        c, _ = _fresh(e, prompt)
        ids, _ = e.decode_verify(s, x0, d, sp, step0)
        ids_c, _ = e.decode_verify(c, x0, d, sp, step0)
        assert ids.tolist() == ids_c.tolist()
        n = len(ids)
        nxt, _ = e.decode_sample_batch([s], [int(ids[-1])], [sp], 8, step0=[step0 + n])
        hist = list(prompt) + [x0] + d[:n - 1]
        tok = int(ids[-1])
        for i in range(8):                                      # replay on the twin: its logits are the same bit for bit
            lg, _ = e.decode_step(c, tok)
            hist.append(tok)
            tok = eng.sample_token(lg, sp, hist, step0 + n + i)
            assert tok == int(nxt[i, 0]), i
        e.seq_free(s)
        e.seq_free(c)
        assert e.stats()["kv_pages_used"] == 0


# ---- 5. prefix cache -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("page", [16, 32])
def test_prefix_cache_pages_stay_untouched(page):
    cfg = _cfg("llama3-8b-2l", 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    P = _ids(3 * page + 5, V, 6)
    with eng.Engine(model=cfg, seed=8, max_batch=2, max_seqs=4, page_size=page, prefix_cache=True) as e:
        x = e.seq_create()
        e.prefill(x, P, want_logits=False)
        e.seq_free(x)
        y = e.seq_create()
        shared = e.attach_prefix(y, P)
        assert shared == 3 * page
        before = [e.debug_kv(y, l, w, 0, shared) for l in range(L) for w in (0, 1)]
        x0 = int(e.prefill(y, P[shared:]).argmax())
        hist = list(P)
        rng = np.random.default_rng(page)
        last = None
        for i in range(12):                                     # mostly rejected drafts, some passes accept a run
            d = [int(v) for v in rng.integers(0, V, 15)]
            ids, _ = e.decode_verify(y, x0, d, None, 0)
            hist += [x0] + d[:len(ids) - 1]
            last = d[len(ids) - 1:]
            x0 = int(ids[-1])
        n = e.seq_len(y)
        assert n == len(hist)
        for a, b in zip(before, [e.debug_kv(y, l, w, 0, shared) for l in range(L) for w in (0, 1)]):
            assert np.array_equal(a, b)
        z = e.seq_create()                                      # history + the rejected drafts of the last pass
        reused = e.attach_prefix(z, np.array(hist + [x0] + last, np.int32))
        assert reused == page * (n // page), (reused, n)
        e.seq_free(z)
        e.seq_free(y)
        assert e.stats()["kv_pages_used"] == 0


# ---- 6. scheduler and synchronous path ----------------------------------------------------------------------------------
def _teacher_forced_gaps(ref, prompt, ids):
    """Top logit minus the logit of every produced id, replaying prompt + ids through a speculation-off engine."""
    s = ref.seq_create()
    lg = ref.prefill(s, prompt)
    gaps = []
    for i, tok in enumerate(ids):
        gaps.append(float(lg.max() - lg[tok]))
        if i + 1 < len(ids):
            lg, _ = ref.decode_step(s, int(tok))
    ref.seq_free(s)
    return np.array(gaps)


def _spec_prompt(V, salt):
    """Every id follows one marker id somewhere: whatever x0 is, the history's last bigram has an earlier occurrence.
    Then a repeated run, so that a right draft is likely too."""
    c = 3 + salt
    pairs = np.stack([np.full(V, c), np.arange(V)], 1).reshape(-1)
    run = _ids(40, V, salt)
    return np.concatenate([run, pairs, run, run, [c]]).astype(np.int32)


def _token_level_replay(e, prompt, sp, k_spec, max_new):
    """What a speculating request does, through cl_decode_verify and single steps (scheduler.cpp Engine::spec_round with one request)."""
    s = e.seq_create()
    lg = e.prefill(s, prompt)
    out = [eng.sample_token(lg, sp, list(prompt), 0)]
    backoff = 0
    while len(out) < max_new:
        n = 0
        k_max = min(k_spec, max_new - len(out) - 1, e.cfg["max_seq_len"] - e.seq_len(s) - 1)
        if backoff == 0 and k_max >= 1:
            d = eng.draft_ngram(list(prompt) + out, k_max)
            if len(d):
                ids, _ = e.decode_verify(s, out[-1], d, sp, len(out))
                n = len(ids)
                backoff = 8 if n == 1 else 0
                out += [int(i) for i in ids]
        if n == 0:
            ids, _ = e.decode_sample_batch([s], [out[-1]], [sp], 1, step0=[len(out)])
            out.append(int(ids[0, 0]))
            backoff = max(0, backoff - 1)
    e.seq_free(s)
    return out[:max_new]


@pytest.mark.parametrize("scheduler", [True, False])
def test_requests_with_speculation(scheduler):
    cfg = _cfg("tiny-test", 2048)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = _tol(L)
    prompt = _spec_prompt(V, 1)
    with eng.Engine(model=cfg, seed=31, max_batch=4, max_seqs=4, speculate=7, start_scheduler=scheduler) as e:
        g = e.generate_ids(prompt, eng.greedy(96, ignore_eos=True))
        st = e.spec_stats()
        assert g.n_generated == 96
        assert st["enabled"] == 1 and st["max_draft"] == 7 and st["tokens_drafted"] > 0 and st["verify_passes"] > 0
        assert st["tokens_emitted"] == st["tokens_accepted"] + st["verify_passes"]
        sp = eng.ollama_default_sampling(seed=5, max_new_tokens=64)
        sp.ignore_eos = 1
        smp = e.generate_ids(prompt, sp)
        assert smp.n_generated == 64
        five = e.generate_ids(prompt, eng.greedy(5, ignore_eos=True))
        assert five.n_generated == 5
        assert e.stats()["kv_pages_used"] == 0
        print(f"scheduler={scheduler}: spec stats {e.spec_stats()}")
    with eng.Engine(model=cfg, seed=31, max_batch=4, max_seqs=4) as ref:
        assert ref.spec_stats()["verify_passes"] == 0
        gaps = _teacher_forced_gaps(ref, prompt, g.token_ids)
        assert gaps.max() <= tol, gaps.max()
        assert five.token_ids.tolist() == g.token_ids[:5].tolist() or _teacher_forced_gaps(ref, prompt, five.token_ids).max() <= tol
        assert smp.token_ids.tolist() == _token_level_replay(ref, prompt, sp, 7, 64)


def test_second_request_switches_to_batched_steps():
    cfg = _cfg("tiny-test", 2048)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = _tol(L)
    pa, pb = _spec_prompt(V, 2), _spec_prompt(V, 4)[-300:]
    with eng.Engine(model=cfg, seed=41, max_batch=4, max_seqs=4, speculate=15, start_scheduler=True) as e:
        out = {}
        ta = threading.Thread(target=lambda: out.__setitem__("a", e.generate_ids(pa, eng.greedy(400, ignore_eos=True))))
        ta.start()
        while e.stats()["tokens_generated"] < 40 and ta.is_alive():     # request a is decoding alone, speculating
            time.sleep(0.001)
        before = e.stats()["sched_decode_steps"]
        out["b"] = e.generate_ids(pb, eng.greedy(48, ignore_eos=True))
        ta.join()
        st = e.stats()
        assert st["sched_decode_steps"] > before and st["kv_pages_used"] == 0 and st["requests_completed"] == 2
        assert st["preemptions"] == out["a"].n_preempted + out["b"].n_preempted
        assert e.spec_stats()["verify_passes"] > 0
    with eng.Engine(model=cfg, seed=41, max_batch=4, max_seqs=4) as ref:
        for p, r, n in ((pa, out["a"], 400), (pb, out["b"], 48)):
            assert r.n_generated == n
            assert _teacher_forced_gaps(ref, p, r.token_ids).max() <= tol


# ---- 7. default off, switches and errors -----------------------------------------------------------------------------------
def test_default_off_env_override_and_errors(monkeypatch):
    cfg = _cfg("tiny-test", 2048)
    prompt = _spec_prompt(cfg["vocab_size"], 3)
    with eng.Engine(model=cfg, seed=1, start_scheduler=True) as e:
        e.generate_ids(prompt, eng.greedy(32, ignore_eos=True))
        st = e.spec_stats()
        assert st == dict(enabled=0, max_draft=0, verify_passes=0, tokens_drafted=0, tokens_accepted=0, tokens_emitted=0)
        s = e.seq_create()
        x0 = int(e.prefill(s, prompt[:40]).argmax())
        for k in (0, 16):
            with pytest.raises(eng.EngineError) as ei:
                e.decode_verify(s, x0, [1] * k, None, 0)
            assert ei.value.status == eng.CL_ERR_INVALID_ARG
        with pytest.raises(eng.EngineError) as ei:
            e.decode_verify(s, x0, [1, 2], _sp(0.8, 0, 0.9, 1.1, 64, 1), 0)     # top_k 0: host sampler only
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
        with pytest.raises(eng.EngineError) as ei:
            e.decode_verify(s, V_OUT, [1, 2], None, 0)
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
        assert e.seq_len(s) == 40                                              # nothing ran
        e.seq_fake_fill(s, e.cfg["max_seq_len"] - 3)
        with pytest.raises(eng.EngineError) as ei:
            e.decode_verify(s, x0, [1, 2, 3], None, 0)
        assert ei.value.status == eng.CL_ERR_TOO_LONG
        ids, _ = e.decode_verify(s, x0, [1, 2], None, 0)                       # len + 3 == max_seq_len fits
        assert 1 <= len(ids) <= 3
        e.seq_free(s)
    for bad in (16, -1):
        with pytest.raises(eng.EngineError) as ei:
            eng.Engine(preset="tiny-test", seed=1, speculate=bad)
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
    monkeypatch.setenv("CL_SPECULATE", "15")
    with eng.Engine(model=cfg, seed=1, start_scheduler=True) as e:
        r = e.generate_ids(prompt, eng.greedy(5, ignore_eos=True))
        assert r.n_generated == 5
        st = e.spec_stats()
        assert st["enabled"] == 1 and st["max_draft"] == 15 and st["verify_passes"] > 0
        assert st["tokens_drafted"] <= 3 * st["verify_passes"]                  # clipped: never past max_new_tokens
        assert e.stats()["kv_pages_used"] == 0
    monkeypatch.setenv("CL_SPECULATE", "0")
    with eng.Engine(preset="tiny-test", seed=1, speculate=7) as e:
        assert e.spec_stats()["enabled"] == 0


V_OUT = 512     # tiny-test's vocabulary size: the first id out of range
