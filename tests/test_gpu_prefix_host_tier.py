"""Host tier of the prefix cache (cl_engine_set_prefix_host_cache / CL_PREFIX_CACHE_HOST_MIB): cached KV pages the pool
evicts are copied to pinned host pages and copied back when a prompt reaches them.  A restored page must hold exactly
the evicted bytes, so reuse from the host is bit-identical to computing the prefix, and no copy may touch a page it does
not name.  Pinned memory stays at a few hundred MiB at most."""
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


def _kv(e, s, n, layers):
    return [e.debug_kv(s, l, w, 0, n) for l in range(layers) for w in (0, 1)]


def _kv_tok(cfg):
    return 2 * cfg["n_layers"] * cfg["n_kv_heads"] * cfg["head_dim"] * 2


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    monkeypatch.delenv("CL_PREFIX_CACHE", raising=False)
    monkeypatch.delenv("CL_PREFIX_CACHE_HOST_MIB", raising=False)


@pytest.mark.parametrize("n_moves", [1, 5])
@pytest.mark.parametrize("page", [16, 32, 64])
@pytest.mark.parametrize("head_dim,n_kv", [(64, 2), (128, 8)])
def test_kernel_round_trip_is_bit_exact(head_dim, n_kv, page, n_moves):
    eng.op_kv_host_roundtrip(3, n_kv, head_dim, page, n_moves)   # raises unless exact and every other page untouched


def _evict_all(e, tokens):
    """A sequence of placeholder K/V over the whole pool: every cached page is evicted; none of its pages is published."""
    f = e.seq_create()
    e.seq_fake_fill(f, tokens)
    e.seq_free(f)


@pytest.mark.parametrize("page", [16, 32, 64])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_reuse_from_host_is_bit_identical_to_computing_it(shape, page):
    cfg = _cfg(shape, 2048)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    A = _ids(256, V, 1)
    n_a = 256 // page
    page_bytes = page * _kv_tok(cfg)
    for tier in (True, False):
        with eng.Engine(model=cfg, seed=4321, max_batch=2, max_seqs=4, page_size=page, kv_pool_bytes=2048 * _kv_tok(cfg),
                        prefix_cache=True, prefix_cache_host_bytes=(n_a + 3) * page_bytes if tier else 0) as e:
            assert e.prefix_stats(host=True)["host_pages"] == (n_a + 3 if tier else 0)
            x = e.seq_create()
            e.prefill(x, A, want_logits=False)
            e.seq_free(x)
            to_host = 0
            for i, nq in enumerate((1, 40, 300)):          # token-wise, split-K and tile paths for the suffix
                _evict_all(e, 2048)
                st = e.prefix_stats(host=True)
                assert st["cached_pages"] == 0
                if tier:                                    # A's pages, and the full pages of the last suffix
                    assert st["pages_to_host"] >= to_host + n_a and st["host_pages_cached"] >= n_a, st
                    to_host = st["pages_to_host"]
                else:
                    assert st["pages_to_host"] == 0 and st["host_pages_cached"] == 0
                Q = _ids(nq, V, 2 + nq)
                y = e.seq_create()
                got = e.attach_prefix(y, np.concatenate([A, Q]))
                if not tier:
                    assert got == 0
                    e.seq_free(y)
                    continue
                assert got == 256 and e.prefix_stats(host=True)["pages_from_host"] == n_a * (i + 1)
                lg_y = e.prefill(y, Q)
                r = e.seq_create()
                e.prefill(r, A, want_logits=False)
                lg_r = e.prefill(r, Q)
                assert np.array_equal(lg_y, lg_r), (nq, float(np.abs(lg_y - lg_r).max()))
                for a, b in zip(_kv(e, y, 256 + nq, L), _kv(e, r, 256 + nq, L)):
                    assert np.array_equal(a, b)
                e.seq_free(y)
                e.seq_free(r)
            assert e.stats()["kv_pages_used"] == 0


@pytest.mark.parametrize("mega", ["1", "0"])
def test_decoding_on_restored_pages(monkeypatch, mega):
    """Sequences on pages restored from the host decode exactly as sequences on pages that never left HBM: batched
    (B = 2) and B = 1 on the persistent kernel (CL_MEGA=1) or the per-op kernels."""
    monkeypatch.setenv("CL_MEGA", mega)
    cfg = _cfg("llama3-8b-2l", 2048)
    V, L, page = cfg["vocab_size"], cfg["n_layers"], 32
    A = _ids(256, V, 3)
    Q = [_ids(40, V, 4), _ids(40, V, 5)]
    with eng.Engine(model=cfg, seed=99, max_batch=2, max_seqs=6, page_size=page, kv_pool_bytes=2048 * _kv_tok(cfg),
                    prefix_cache=True, prefix_cache_host_bytes=16 * page * _kv_tok(cfg)) as e:
        x = e.seq_create()
        e.prefill(x, A, want_logits=False)
        e.seq_free(x)
        _evict_all(e, 2048)
        restored, private, first = [], [], []
        for q in Q:
            s = e.seq_create()
            assert e.attach_prefix(s, np.concatenate([A, q])) == 256
            first.append(int(e.prefill(s, q).argmax()))
            restored.append(s)
        assert e.prefix_stats(host=True)["pages_from_host"] == 256 // page
        for q in Q:
            p = e.seq_create()
            e.prefill(p, A, want_logits=False)
            assert int(e.prefill(p, q).argmax()) == first[len(private)]
            private.append(p)
        ids_r, _ = e.decode_greedy_batch(restored, first, 32)
        ids_p, _ = e.decode_greedy_batch(private, first, 32)
        assert np.array_equal(ids_r, ids_p)
        toks = ids_r[-1]
        for _ in range(8):                                   # teacher-forced batched steps, logits bit for bit
            lg_r, am = e.decode_step_batch(restored, toks)
            lg_p, _ = e.decode_step_batch(private, toks)
            assert np.array_equal(lg_r, lg_p)
            toks = am
        for b in range(2):
            lg_r, am_r = e.decode_step(restored[b], int(toks[b]))
            lg_p, am_p = e.decode_step(private[b], int(toks[b]))
            assert np.array_equal(lg_r, lg_p)
            g_r, _ = e.decode_greedy(restored[b], am_r, 24)
            g_p, _ = e.decode_greedy(private[b], am_p, 24)
            assert np.array_equal(g_r, g_p)
        for s in restored + private:
            e.seq_free(s)
        assert e.stats()["kv_pages_used"] == 0


def test_spill_and_fill_in_one_attach_leave_other_pages_alone():
    """The host tier holds exactly A's four pages and the pool is full of B's cached pages and a live sequence's.  Attaching
    A fills its first page into the free page, then evicts B's deepest page to the host page that fill freed and fills A's
    second page into that device page, and so on: spill and fill of one device page, and a host page freed by a fill
    reused by a spill, in one call.  A's K/V must come back exact, the live sequence's must not change, and what is left
    of B must still be B's."""
    cfg = _cfg("tiny-test", 512)
    V, L, page = cfg["vocab_size"], cfg["n_layers"], 16
    with eng.Engine(model=cfg, seed=7, max_batch=2, max_seqs=4, page_size=page, kv_pool_bytes=12 * page * _kv_tok(cfg),
                    prefix_cache=True, prefix_cache_host_bytes=4 * page * _kv_tok(cfg)) as e:
        live = e.seq_create()
        e.prefill(live, _ids(32, V, 1), want_logits=False)            # 2 pages
        kv_live = _kv(e, live, 32, L)
        A, B = _ids(65, V, 2), _ids(145, V, 3)
        a = e.seq_create()
        e.prefill(a, A, want_logits=False)                             # 4 full pages published, 1 private
        kv_a = _kv(e, a, 64, L)
        e.seq_free(a)
        _evict_all(e, 10 * page)                                       # 6 free pages, then A's 4 to the host
        st = e.prefix_stats(host=True)
        assert st["pages_to_host"] == 4 and st["host_pages_cached"] == 4
        b = e.seq_create()
        e.prefill(b, B, want_logits=False)                             # 9 full pages published, 1 private
        kv_b = _kv(e, b, 144, L)
        e.seq_free(b)
        assert e.prefix_stats()["cached_pages"] == 9
        y = e.seq_create()
        assert e.attach_prefix(y, A) == 64
        st = e.prefix_stats(host=True)
        assert st["pages_from_host"] == 4 and st["pages_to_host"] == 4 + 3, st
        for u, w in zip(_kv(e, y, 64, L), kv_a):
            assert np.array_equal(u, w)
        for u, w in zip(_kv(e, live, 32, L), kv_live):
            assert np.array_equal(u, w)
        e.seq_free(y)
        z = e.seq_create()
        got = e.attach_prefix(z, B)
        assert got >= 5 * page, got                                    # B's first pages never left the pool
        for u, w in zip(_kv(e, z, got, L), kv_b):
            assert np.array_equal(u, w[:got])
        e.seq_free(z)
        for u, w in zip(_kv(e, live, 32, L), kv_live):
            assert np.array_equal(u, w)
        e.seq_free(live)
        assert e.stats()["kv_pages_used"] == 0


def test_full_host_tier_drops_deepest_pages_first():
    cfg = _cfg("tiny-test", 512)
    V, L, page = cfg["vocab_size"], cfg["n_layers"], 16
    with eng.Engine(model=cfg, seed=7, max_batch=2, max_seqs=4, page_size=page, kv_pool_bytes=8 * page * _kv_tok(cfg),
                    prefix_cache=True, prefix_cache_host_bytes=3 * page * _kv_tok(cfg)) as e:
        A = _ids(65, V, 2)
        a = e.seq_create()
        e.prefill(a, A, want_logits=False)
        kv_a = _kv(e, a, 64, L)
        e.seq_free(a)
        _evict_all(e, 8 * page)                         # A's four pages, deepest first, into three host pages
        st = e.prefix_stats(host=True)
        assert st["pages_to_host"] == 4 and st["host_pages_cached"] == 3
        assert st["pages_to_host"] - st["pages_from_host"] - st["host_pages_cached"] == 1     # one dropped
        y = e.seq_create()
        assert e.attach_prefix(y, A) == 48              # the root and the next two pages came back, the deepest did not
        for u, w in zip(_kv(e, y, 48, L), kv_a):
            assert np.array_equal(u, w[:48])
        e.seq_free(y)
        assert e.stats()["kv_pages_used"] == 0


def test_chain_whose_root_was_dropped_is_not_attached():
    """A's root page is indexed on W's pages, the rest of A on X's (X's root page stays private).  W is freed first, so
    the root reaches the host first and is the first entry the full tier drops: the rest of A stays on the host,
    unreachable."""
    cfg = _cfg("tiny-test", 512)
    V, page = cfg["vocab_size"], 16
    with eng.Engine(model=cfg, seed=7, max_batch=2, max_seqs=4, page_size=page, kv_pool_bytes=8 * page * _kv_tok(cfg),
                    prefix_cache=True, prefix_cache_host_bytes=3 * page * _kv_tok(cfg)) as e:
        A = _ids(65, V, 5)
        w, x = e.seq_create(), e.seq_create()
        e.prefill(w, A[:17], want_logits=False)
        e.prefill(x, A, want_logits=False)
        e.seq_free(w)
        e.seq_free(x)
        assert e.prefix_stats()["cached_pages"] == 4
        _evict_all(e, 8 * page)                         # root, then pages 3, 2, 1: page 1 drops the root
        st = e.prefix_stats(host=True)
        assert st["pages_to_host"] == 4 and st["host_pages_cached"] == 3
        y = e.seq_create()
        assert e.attach_prefix(y, A) == 0
        e.seq_free(y)
        assert e.prefix_stats(host=True)["pages_from_host"] == 0
        assert e.stats()["kv_pages_used"] == 0


def _teacher_forced_gaps(ref, prompt, ids):
    s = ref.seq_create()
    lg = ref.prefill(s, prompt)
    gaps = []
    for i, tok in enumerate(ids):
        gaps.append(float(lg.max() - lg[tok]))
        if i + 1 < len(ids):
            lg, _ = ref.decode_step(s, int(tok))
    ref.seq_free(s)
    return np.array(gaps)


def test_scheduler_brings_preempted_requests_back_from_the_host():
    cfg = _cfg("tiny-test", 2048)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = 0.05 + 0.03 * np.sqrt(L)
    prompts = [_ids(500 + 13 * i, V, 200 + i) for i in range(6)]
    sp = eng.greedy(160, ignore_eos=True)
    with eng.Engine(model=cfg, seed=8, max_batch=4, max_seqs=4, page_size=16, kv_pool_bytes=1600 * _kv_tok(cfg),
                    start_scheduler=True, prefix_cache=True, prefix_cache_host_bytes=4000 * _kv_tok(cfg)) as e:
        out = [None] * len(prompts)

        def run(i):
            out[i] = e.generate_ids(prompts[i], sp)
        th = [threading.Thread(target=run, args=(i,)) for i in range(len(prompts))]
        [t.start() for t in th]
        [t.join() for t in th]
        ps, st = e.prefix_stats(host=True), e.stats()
        print(f"preemptions {st['preemptions']}, prefix stats {ps}")
        assert st["preemptions"] > 0 and ps["pages_from_host"] > 0 and ps["tokens_reused"] > 0
        assert st["kv_pages_used"] == 0 and st["active_seqs"] == 0 and st["requests_completed"] == len(prompts)
        assert st["preemptions"] == sum(o.n_preempted for o in out)
        assert ps["pages_to_host"] - ps["pages_from_host"] - ps["host_pages_cached"] >= 0
        assert ps["host_pages_cached"] <= ps["host_pages"] == 250
    with eng.Engine(model=cfg, seed=8, max_batch=1, max_seqs=1) as ref:
        for i, p in enumerate(prompts):
            assert out[i].n_generated == 160
            assert _teacher_forced_gaps(ref, p, out[i].token_ids).max() <= tol, i


def test_setter_error_codes(monkeypatch):
    cfg = _cfg("tiny-test", 512)
    page_bytes = 32 * _kv_tok(cfg)
    with eng.Engine(model=cfg, seed=1) as off:
        with pytest.raises(eng.EngineError) as ex:
            off.set_prefix_host_cache(1 << 20)                         # the prefix cache is off
        assert ex.value.status == eng.CL_ERR_INVALID_ARG
    with eng.Engine(model=cfg, seed=1, prefix_cache=True) as e:
        for bad in (-1, 1, page_bytes - 1):
            with pytest.raises(eng.EngineError) as ex:
                e.set_prefix_host_cache(bad)
            assert ex.value.status == eng.CL_ERR_INVALID_ARG
        e.set_prefix_host_cache(5 * page_bytes + 7)                   # rounds down to whole pages
        assert e.prefix_stats(host=True)["host_pages"] == 5
        s = e.seq_create()
        with pytest.raises(eng.EngineError) as ex:
            e.set_prefix_host_cache(page_bytes)                        # a sequence is live
        assert ex.value.status == eng.CL_ERR_INVALID_ARG
        e.seq_free(s)
        with pytest.raises(eng.EngineError) as ex:
            e.set_prefix_host_cache(1 << 50)                           # cannot be pinned
        assert ex.value.status == eng.CL_ERR_OOM
        assert e.prefix_stats(host=True)["host_pages"] == 0
        e.set_prefix_host_cache(page_bytes)
        e.set_prefix_host_cache(0)
        assert e.prefix_stats(host=True)["host_pages"] == 0
    monkeypatch.setenv("CL_PREFIX_CACHE_HOST_MIB", "1")                # the environment wins over the argument
    with eng.Engine(model=cfg, seed=1, prefix_cache=True, prefix_cache_host_bytes=3 * page_bytes) as e:
        assert e.prefix_stats(host=True)["host_pages"] == (1 << 20) // page_bytes
