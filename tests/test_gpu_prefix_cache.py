"""Prefix cache (cl_engine_config.prefix_cache / CL_PREFIX_CACHE): full KV pages of earlier sequences are attached
read-only by later sequences that share the prefix.  Reuse must be bit-identical to computing the prefix, shared pages
must never change, unknown history must never be shared, and the scheduler must reuse across requests and after a
preemption without leaking pages."""
import threading

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu


def _cfg(name, max_seq_len):
    cfg = dict(oc.PRESETS["llama3-8b" if name == "llama3-8b-2l" else name])
    if name == "llama3-8b-2l":
        cfg["n_layers"] = 2
    cfg["max_seq_len"] = max_seq_len
    return cfg


def _ids(n, vocab, salt):
    return np.array([(i * 7919 + 13 + salt * 104729) % (vocab - 3) + 3 for i in range(n)], np.int32)


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    monkeypatch.delenv("CL_PREFIX_CACHE", raising=False)


def _kv(e, s, n, layers):
    return [e.debug_kv(s, l, w, 0, n) for l in range(layers) for w in (0, 1)]


@pytest.mark.parametrize("page", [16, 32, 64])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_reused_prefix_is_bit_identical_to_computing_it(shape, page):
    cfg = _cfg(shape, 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    A = _ids(256, V, 1)
    with eng.Engine(model=cfg, seed=4321, max_batch=2, max_seqs=4, page_size=page, prefix_cache=True) as e:
        x = e.seq_create()
        e.prefill(x, A, want_logits=False)
        e.seq_free(x)
        assert e.prefix_stats()["cached_pages"] == 256 // page
        for nq in (1, 40, 300):                          # token-wise, split-K and tile paths for the suffix
            Q = _ids(nq, V, 2 + nq)
            y = e.seq_create()
            assert e.attach_prefix(y, np.concatenate([A, Q])) == 256
            assert e.seq_len(y) == 256
            lg_y = e.prefill(y, Q)
            r = e.seq_create()
            e.prefill(r, A, want_logits=False)
            lg_r = e.prefill(r, Q)
            assert np.array_equal(lg_y, lg_r), (nq, float(np.abs(lg_y - lg_r).max()))
            for a, b in zip(_kv(e, y, 256 + nq, L), _kv(e, r, 256 + nq, L)):
                assert np.array_equal(a, b)
            e.seq_free(y)
            e.seq_free(r)
        # full hit: the same prompt again reuses all but its last page (at least one token is computed).  A fresh prompt:
        # one that started with A would chain onto the pages of A computed by the short-prompt path above, while the
        # reference below computes all of its rows in one tile-path call
        P = _ids(333, V, 9)
        s = e.seq_create()
        e.prefill(s, P, want_logits=False)
        e.seq_free(s)
        s = e.seq_create()
        k = e.attach_prefix(s, P)
        assert k == page * ((len(P) - 1) // page)
        lg_s = e.prefill(s, P[k:])
        r = e.seq_create()
        e.prefill(r, P[:k], want_logits=False)
        assert np.array_equal(lg_s, e.prefill(r, P[k:]))
        e.seq_free(s)
        e.seq_free(r)
        st = e.prefix_stats()
        assert st["enabled"] == 1 and st["lookups"] == 4 and st["tokens_reused"] == 3 * 256 + k
        assert e.stats()["kv_pages_used"] == 0


@pytest.mark.parametrize("shape,page,mega", [("llama3-8b-2l", 32, "1"), ("llama3-8b-2l", 32, "0"), ("llama3-8b-2l", 64, "0"),
                                             ("tiny-test", 16, "1")])
def test_shared_pages_stay_read_only(monkeypatch, shape, page, mega):
    """Two sequences attach one prefix and decode with different suffixes; they must produce exactly what two
    sequences holding private copies produce, on the batched, persistent and per-op paths, and the shared K/V must
    be unchanged afterwards."""
    monkeypatch.setenv("CL_MEGA", mega)
    cfg = _cfg(shape, 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    A = _ids(256, V, 3)
    Q = [_ids(40, V, 4), _ids(40, V, 5)]
    with eng.Engine(model=cfg, seed=99, max_batch=2, max_seqs=6, page_size=page, prefix_cache=True) as e:
        x = e.seq_create()
        e.prefill(x, A, want_logits=False)
        e.seq_free(x)
        shared, private, first = [], [], []
        for q in Q:
            s = e.seq_create()
            assert e.attach_prefix(s, np.concatenate([A, q])) == 256
            first.append(int(e.prefill(s, q).argmax()))
            shared.append(s)
        for q in Q:
            p = e.seq_create()
            e.prefill(p, A, want_logits=False)
            assert int(e.prefill(p, q).argmax()) == first[len(private)]
            private.append(p)
        before = _kv(e, shared[0], 256, L)
        ids_s, _ = e.decode_greedy_batch(shared, first, 64)
        ids_p, _ = e.decode_greedy_batch(private, first, 64)
        assert np.array_equal(ids_s, ids_p)
        toks = ids_s[-1]
        for _ in range(8):                                   # teacher-forced batched steps, logits bit for bit
            lg_s, am = e.decode_step_batch(shared, toks)
            lg_p, _ = e.decode_step_batch(private, toks)
            assert np.array_equal(lg_s, lg_p)
            toks = am
        for b in range(2):                                   # B = 1: persistent kernel (CL_MEGA=1 where supported) / per-op
            g_s, _ = e.decode_greedy(shared[b], int(toks[b]), 32)
            g_p, _ = e.decode_greedy(private[b], int(toks[b]), 32)
            assert np.array_equal(g_s, g_p)
        for a, b in zip(before, _kv(e, shared[0], 256, L)):
            assert np.array_equal(a, b)
        for a, b in zip(_kv(e, shared[1], 256, L), _kv(e, private[0], 256, L)):
            assert np.array_equal(a, b)
        for s in shared + private:
            e.seq_free(s)
        assert e.stats()["kv_pages_used"] == 0


def test_unknown_history_is_never_shared():
    cfg = _cfg("llama3-8b-2l", 2048)
    V = cfg["vocab_size"]
    page = 16
    with eng.Engine(model=cfg, seed=5, max_batch=1, max_seqs=2, page_size=page, prefix_cache=True) as e:
        # seq_fake_fill: a synthetic cache under a history of zeros, then real tokens on top
        s = e.seq_create()
        e.seq_fake_fill(s, 256)
        tail = _ids(40, V, 6)
        e.prefill(s, tail, want_logits=False)
        e.seq_free(s)
        assert e.prefix_stats()["cached_pages"] == 0
        t = e.seq_create()
        assert e.attach_prefix(t, np.concatenate([np.zeros(256, np.int32), tail, [7]])) == 0
        e.seq_free(t)
        # more eager steps than the id ring holds (1024): only the prompt and the first fed token are known
        prompt = _ids(40, V, 7)
        s = e.seq_create()
        first = int(e.prefill(s, prompt).argmax())
        e.time_dominant_kernel(s, first, 1100)
        e.seq_free(s)
        t = e.seq_create()
        hist = np.concatenate([prompt, [first], np.zeros(1100, np.int32)])
        assert e.attach_prefix(t, hist) == page * (41 // page)
        e.seq_free(t)
        # decode_greedy reads every id back, ring or not: a run longer than the ring is shared in full
        s = e.seq_create()
        first = int(e.prefill(s, prompt).argmax())
        ids, _ = e.decode_greedy(s, first, 1100)
        e.seq_free(s)
        t = e.seq_create()
        hist = np.concatenate([prompt, [first], ids])                # 40 + 1101 tokens, 40 + 1100 of them cached
        assert e.attach_prefix(t, hist) == page * ((len(hist) - 1) // page)
        e.seq_free(t)
        assert e.stats()["kv_pages_used"] == 0


def _teacher_forced_gaps(ref, prompt, ids):
    """Top logit minus the logit of every produced id, replaying prompt + ids through a cache-off engine."""
    s = ref.seq_create()
    lg = ref.prefill(s, prompt)
    gaps = []
    for i, tok in enumerate(ids):
        gaps.append(float(lg.max() - lg[tok]))
        if i + 1 < len(ids):
            lg, _ = ref.decode_step(s, int(tok))
    ref.seq_free(s)
    return np.array(gaps)


def test_scheduler_reuses_a_shared_prefix():
    cfg = _cfg("tiny-test", 2048)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = 0.05 + 0.03 * np.sqrt(L)
    prefix = _ids(1024, V, 11)
    prompts = [np.concatenate([prefix, _ids(20 + 7 * i, V, 100 + i)]) for i in range(16)]
    sps = [eng.greedy(24, ignore_eos=True) if i % 3 else eng.ollama_default_sampling(seed=i, max_new_tokens=24) for i in range(16)]
    for sp in sps:
        sp.ignore_eos = 1
    with eng.Engine(model=cfg, seed=31, max_batch=8, max_seqs=8, start_scheduler=True, prefix_cache=True) as e:
        out = [None] * 16
        out[0] = e.generate_ids(prompts[0], sps[0])

        def run(i):
            out[i] = e.generate_ids(prompts[i], sps[i])
        th = [threading.Thread(target=run, args=(i,)) for i in range(1, 16)]
        [t.start() for t in th]
        [t.join() for t in th]
        ps, st = e.prefix_stats(), e.stats()
        assert ps["lookups"] == 16 and ps["tokens_reused"] >= 15 * 1024, ps
        assert st["kv_pages_used"] == 0 and st["active_seqs"] == 0 and st["requests_completed"] == 16
        assert st["preemptions"] == sum(o.n_preempted for o in out)
    with eng.Engine(model=cfg, seed=31, max_batch=1, max_seqs=1) as ref:
        assert ref.prefix_stats()["lookups"] == 0
        for i in range(16):
            assert out[i].n_generated == 24
            if sps[i].temperature == 0:
                gaps = _teacher_forced_gaps(ref, prompts[i], out[i].token_ids)
                assert gaps.max() <= tol, (i, gaps.max())


def test_preempted_requests_reattach_their_pages():
    cfg = _cfg("tiny-test", 2048)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = 0.05 + 0.03 * np.sqrt(L)
    kv_tok = 2 * L * cfg["n_kv_heads"] * cfg["head_dim"] * 2
    prompts = [_ids(500 + 13 * i, V, 200 + i) for i in range(6)]
    sp = eng.greedy(160, ignore_eos=True)
    with eng.Engine(model=cfg, seed=8, max_batch=4, max_seqs=4, page_size=16, kv_pool_bytes=1600 * kv_tok,
                    start_scheduler=True, prefix_cache=True) as e:
        out = [None] * len(prompts)

        def run(i):
            out[i] = e.generate_ids(prompts[i], sp)
        th = [threading.Thread(target=run, args=(i,)) for i in range(len(prompts))]
        [t.start() for t in th]
        [t.join() for t in th]
        ps, st = e.prefix_stats(), e.stats()
        print(f"preemptions {st['preemptions']}, prefix stats {ps}")
        assert st["preemptions"] > 0 and ps["tokens_reused"] > 0 and ps["pages_evicted"] > 0
        assert st["kv_pages_used"] == 0 and st["active_seqs"] == 0 and st["requests_completed"] == len(prompts)
        assert st["preemptions"] == sum(o.n_preempted for o in out)
    with eng.Engine(model=cfg, seed=8, max_batch=1, max_seqs=1) as ref:
        for i, p in enumerate(prompts):
            assert out[i].n_generated == 160
            assert _teacher_forced_gaps(ref, p, out[i].token_ids).max() <= tol, i


def test_prefix_cache_is_off_by_default():
    with eng.Engine(preset="tiny-test", seed=1, start_scheduler=True) as e:
        p = _ids(100, 512, 3)
        for _ in range(2):
            e.generate_ids(p, eng.greedy(4, ignore_eos=True))
        s = e.seq_create()
        assert e.attach_prefix(s, p) == 0 and e.seq_len(s) == 0
        e.seq_free(s)
        ps = e.prefix_stats()
        assert ps == dict(enabled=0, cached_pages=0, lookups=0, tokens_looked_up=0, tokens_reused=0, pages_evicted=0)
