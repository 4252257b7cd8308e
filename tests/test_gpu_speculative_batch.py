"""Speculative decoding over several sequences (cl_decode_verify_batch, cl_engine_set_speculate_batch): one pass verifies
the drafts of every sequence.  Acceptance must equal a host replay per sequence, each sequence's ids, logits and K/V must
equal verifying it alone, the logits must match the CPU oracle teacher-forced, the state after a pass must be that of
a + 1 single steps, errors must leave every sequence as it was, and the scheduler must emit what decoding without
speculation emits."""
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


SAMPLINGS = [None, _sp(0.8, 40, 0.9, 1.1, 64, 7), _sp(1.0, 5, 1.0, 1.0, 0, 11), _sp(1.3, 128, 0.5, 1.3, 16, 13)]


def _replay(logits, sp, hist, x0, draft, step0):
    """Host replay of one sequence's verify: row r's choice with history hist + x0, d1 .. dr at step step0 + r; then the rule."""
    inputs = [int(x0)] + [int(d) for d in draft]
    y = [int(np.argmax(logits[r])) if sp is None else eng.sample_token(logits[r], sp, list(hist) + inputs[:r + 1], step0 + r)
         for r in range(len(inputs))]
    a = 0
    while a < len(draft) and y[a] == int(draft[a]):
        a += 1
    return y[:a + 1]


def _fresh(e, prompt):
    s = e.seq_create()
    lg = e.prefill(s, prompt)
    return s, int(lg.argmax())


def _continuation(e, prompt, x0, sp, step0, n):
    s, _ = _fresh(e, prompt)
    if sp is None:
        ids, _ = e.decode_greedy(s, x0, n)
    else:
        ids, _ = e.decode_sample_batch([s], [x0], [sp], n, step0=[step0])
        ids = ids[:, 0]
    e.seq_free(s)
    return [int(i) for i in ids]


def _drafts(right, k, kind, rng, V):
    if kind == "right":
        return list(right[:k])
    if kind == "random":
        return [int(v) for v in rng.integers(0, V, k)]
    d = list(right[:k])                                   # first wrong at d_{kind + 1}
    d[kind] = (d[kind] + 1 + int(rng.integers(0, V - 1))) % V
    return d


# ---- 0. the multi-row attention kernel against float64 (cl_op_attn_verify) ----------------------------------------------
# Bound per element as for the decode kernel (DESIGN.md §2): one bf16 ulp of the reference + 2^-14 sum_t p_t |v_t|, since the
# kernel feeds P.V an fp32-accurate hi + lo pair.
ATTN_C = 2.0 ** -14
TC = dict(n_heads=32, n_kv=8, hd=128)


def _bf16(x):
    return oc.np_bf16_from_f32(np.asarray(x, dtype=np.float32))


def _f32(h):
    return oc.np_f32_from_bf16(np.asarray(h, dtype=np.uint16))


def _attn64(q, k, v, len0, n_heads, n_kv, hd):
    """Float64 causal attention of rows len0 .. len0 + R - 1: row r sees keys 0 .. len0 + r.  Returns (out, sum_t p_t |v_t|)."""
    R, n, rep = q.shape[0], k.shape[0], n_heads // n_kv
    q = np.asarray(q, np.float64).reshape(R, n_kv, rep, hd)
    k, v = np.asarray(k, np.float64), np.asarray(v, np.float64)
    vis = np.arange(n)[None, :] <= (len0 + np.arange(R))[:, None]
    out, pv = np.empty((R, n_kv, rep, hd)), np.empty((R, n_kv, rep, hd))
    for g in range(n_kv):
        s = np.einsum("rhd,nd->rhn", q[:, g], k[:, g]) / np.sqrt(hd)
        s = np.where(vis[:, None, :], s, -np.inf)
        p = np.exp(s - s.max(-1, keepdims=True))
        p /= p.sum(-1, keepdims=True)
        out[:, g] = p @ v[:, g]
        pv[:, g] = p @ np.abs(v[:, g])
    return out.reshape(R, -1), pv.reshape(R, -1)


def _verify_case(seed, lens, rows, nsplit):
    rng = np.random.default_rng(seed)
    H, KV, D = TC["n_heads"], TC["n_kv"], TC["hd"]
    qs, ks, vs, refs = [], [], [], []
    for L, R in zip(lens, rows):
        q = _bf16(rng.standard_normal((R, H * D)))
        k = rng.standard_normal((L + R, KV, D)) * 2.0
        v = rng.standard_normal((L + R, KV, D))
        # every row's own key gets a larger score on the first head of its group: a dropped current token shows
        qf = _f32(q).reshape(R, KV, H // KV, D)[:, :, 0].astype(np.float64)
        k[L + np.arange(R)] += 10.0 * np.sqrt(D) * qf / (qf ** 2).sum(-1, keepdims=True)
        k, v = _bf16(k), _bf16(v)
        qs.append(q); ks.append(k); vs.append(v)
        refs.append(_attn64(_f32(q), _f32(k), _f32(v), L, H, KV, D))
    out, ns = eng.op_attn_verify(np.concatenate(qs), np.concatenate(ks), np.concatenate(vs), lens, rows, H, KV, D, 32, nsplit)
    got = _f32(out).astype(np.float64)
    assert not np.isnan(got).any()                            # every row written
    worst, r0 = 0.0, 0
    for (ref, pv), R in zip(refs, rows):
        e = np.floor(np.log2(np.maximum(np.abs(ref), 2.0 ** -126)))
        worst = max(worst, float((np.abs(got[r0:r0 + R] - ref) / (2.0 ** (e - 7) + ATTN_C * pv)).max()))
        r0 += R
    return worst, ns


@pytest.mark.parametrize("lens,rows,nsplit", [
    ([0], [1], 0),
    ([0], [16], 0),
    ([31, 32, 33, 63, 64, 65, 255, 256, 257], [16, 1, 2, 3, 4, 5, 15, 8, 16], 0),
    ([8192 - 16, 4096, 4095, 1000, 7], [16, 16, 3, 9, 16], 0),
    ([((i * 613) % 3000) for i in range(16)], [1 + (i * 5) % 16 for i in range(16)], 0),
    ([2048, 511, 30], [16, 7, 2], 1),
    ([2048, 511, 30], [16, 7, 2], 7),
    ([4000, 100], [13, 16], 64),
])
def test_attn_verify_kernel_matches_float64(lens, rows, nsplit):
    worst, ns = _verify_case(sum(lens) + len(rows) + nsplit, lens, rows, nsplit)
    print(f"[verify attn] lens {lens[:4]}.. rows {rows[:4]}.. splits {ns}: max err/tol {worst:.3g}")
    assert worst <= 1.0


# ---- 1. acceptance equals a host replay, and each sequence equals its pass alone ------------------------------------------
@pytest.mark.parametrize("page", [16, 32, 64])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_acceptance_and_independence(shape, page):
    cfg = _cfg(shape, 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    rng = np.random.default_rng(page)
    prompts = [_ids(2 * page + page // 2 + 3 + 5 * i, V, 10 + i) for i in range(8)]
    accepted = 0
    with eng.Engine(model=cfg, seed=77, max_batch=8, max_seqs=16, page_size=page) as e:
        x0s, rights = [], []
        for i, p in enumerate(prompts):
            s, x0 = _fresh(e, p)
            e.seq_free(s)
            x0s.append(x0)
            rights.append(_continuation(e, p, x0, SAMPLINGS[i % 4], 5 + i, 15))
        ks_all = [0, 1, 4, 15, 15, 4, 1, 0]
        rounds = [(2, "right"), (3, 0), (8, "random"), (8, "right"), (3, 3)] + [(2, j) for j in range(15)]   # first wrong at every j
        for n_seqs, kind in rounds:
            ks = ks_all[:n_seqs] if n_seqs != 2 else [15, 4]
            ds = []
            for i in range(n_seqs):
                k = ks[i]
                knd = kind if not isinstance(kind, int) else min(kind, k - 1) if k > 0 else "right"
                ds.append(_drafts(rights[i], k, knd, rng, V))
            sps = [SAMPLINGS[i % 4] for i in range(n_seqs)]
            st0 = [5 + i for i in range(n_seqs)]
            ss = [_fresh(e, prompts[i])[0] for i in range(n_seqs)]
            lens = [e.seq_len(s) for s in ss]
            ids, lg = e.decode_verify_batch(ss, x0s[:n_seqs], ds, sps, st0, want_logits=True)
            assert lg.shape == (sum(ks) + n_seqs, V) and np.isfinite(lg).all()
            r0 = 0
            for i in range(n_seqs):
                want = _replay(lg[r0:r0 + ks[i] + 1], sps[i], prompts[i], x0s[i], ds[i], st0[i])
                assert ids[i].tolist() == want, (shape, page, n_seqs, kind, i, ids[i], want)
                assert e.seq_len(ss[i]) == lens[i] + len(ids[i])
                accepted += len(ids[i]) - 1
                # independence: the same sequence verified alone, bit for bit
                t, _ = _fresh(e, prompts[i])
                ids1, lg1 = e.decode_verify_batch([t], [x0s[i]], [ds[i]], [sps[i]], [st0[i]], want_logits=True)
                assert ids1[0].tolist() == ids[i].tolist()
                assert np.array_equal(lg1, lg[r0:r0 + ks[i] + 1]), (shape, page, n_seqs, i)
                n = e.seq_len(t)
                assert n == e.seq_len(ss[i])
                for layer in range(L):
                    for w in (0, 1):
                        assert np.array_equal(e.debug_kv(t, layer, w, 0, n), e.debug_kv(ss[i], layer, w, 0, n))
                e.seq_free(t)
                r0 += ks[i] + 1
            for s in ss:
                e.seq_free(s)
        st = e.spec_stats()
        assert st["tokens_emitted"] == st["tokens_accepted"] + st["verify_passes"]
        assert e.spec_multi_passes() == len(rounds)
        assert e.stats()["kv_pages_used"] == 0
    print(f"{shape}/page {page}: {accepted} drafted tokens accepted in multi-sequence passes")


# ---- 2. logits match the oracle, teacher-forced ----------------------------------------------------------------------------
@pytest.mark.parametrize("shape,n_layers,cached", [("tiny-test", 2, 0), ("llama3-8b", 2, 0), ("llama3-8b", 32, 4096)])
def test_batch_logits_match_the_oracle(shape, n_layers, cached):
    cfg = _cfg(shape, 4096 + 64 if cached else 512)
    cfg["n_layers"] = n_layers
    V = cfg["vocab_size"]
    B, k = 4, 3
    m = oc.Model(cfg, seed=99)
    with eng.Engine(model=cfg, seed=99, max_batch=4, max_seqs=4) as e:
        ss, sos, x0s, ds = [], [], [], []
        for i in range(B):
            s = e.seq_create()
            so = m.new_seq((cached or 64) + 32)
            if cached:
                e.seq_fake_fill(s, cached - 7 * i)
                so.fake_fill(cached - 7 * i)
                x0s.append(17 + i)
            else:
                p = _ids(21 + 9 * i, V, 40 + i)
                x0s.append(int(e.prefill(s, p).argmax()))
                so.forward(p)
            ss.append(s)
            sos.append(so)
            ds.append(_ids(k, V, 50 + i))
        _, lg = e.decode_verify_batch(ss, x0s, ds, want_logits=True)
        worst = 0.0
        for i in range(B):
            ref = sos[i].forward(np.concatenate([[x0s[i]], ds[i]]), all_logits=True)
            worst = max(worst, float(np.abs(lg[i * (k + 1):(i + 1) * (k + 1)] - ref).max()))
            sos[i].close()
    m.close()
    print(f"{shape}/{n_layers}L, {B} sequences behind {cached} cached tokens: max |dlogit| {worst:.4f} (tolerance {_tol(n_layers):.3f})")
    assert worst < _tol(n_layers)


# ---- 3. the state after a pass equals a + 1 steps --------------------------------------------------------------------------
def test_state_after_a_batch_pass_equals_single_steps():
    cfg = _cfg("llama3-8b-2l", 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = _tol(L)
    pa, pb = _ids(45, V, 4), _ids(70, V, 5)
    sp, step0 = SAMPLINGS[1], 3
    with eng.Engine(model=cfg, seed=21, max_batch=4, max_seqs=8, prefix_cache=True, page_size=16) as e:
        x = e.seq_create()
        e.prefill(x, pb, want_logits=False)
        e.seq_free(x)
        sa, xa = _fresh(e, pa)
        e.seq_free(sa)
        sb = e.seq_create()
        shared = e.attach_prefix(sb, pb)
        assert shared == 64
        xb = int(e.prefill(sb, pb[shared:]).argmax())
        before = [e.debug_kv(sb, l, w, 0, shared) for l in range(L) for w in (0, 1)]
        ra = _continuation(e, pa, xa, None, 0, 8)
        rb = _continuation(e, pb, xb, sp, step0, 8)
        da = ra[:3] + [(ra[3] + 9) % V] + ra[4:7]
        db = rb[:2] + [(rb[2] + 5) % V] + rb[3:6]
        sa, _ = _fresh(e, pa)
        ta, _ = _fresh(e, pa)
        tb = e.seq_create()                                            # b's twin, built the same way
        assert e.attach_prefix(tb, pb) == shared
        e.prefill(tb, pb[shared:], want_logits=False)
        ids, _ = e.decode_verify_batch([sa, sb], [xa, xb], [da, db], [None, sp], [0, step0])
        ids_t, _ = e.decode_verify(tb, xb, db, sp, step0)              # the sampled one through cl_decode_verify
        assert ids[1].tolist() == ids_t.tolist()
        for a, b in zip(before, [e.debug_kv(sb, l, w, 0, shared) for l in range(L) for w in (0, 1)]):
            assert np.array_equal(a, b)                                # attached prefix-cache pages untouched
        na, nb = len(ids[0]), len(ids[1])
        for tok in [xa] + da[:na - 1]:
            e.decode_step(ta, tok)
        assert e.seq_len(sa) == e.seq_len(ta)
        tok = int(ids[0][-1])
        for _ in range(6):
            ls, am = e.decode_step(sa, tok)
            lt, _ = e.decode_step(ta, tok)
            assert float(np.abs(ls - lt).max()) < tol
            tok = am
        nxt, _ = e.decode_sample_batch([sb], [int(ids[1][-1])], [sp], 6, step0=[step0 + nb])
        hist = list(pb) + [xb] + db[:nb - 1]
        tok = int(ids[1][-1])
        for i in range(6):                                             # the twin's logits are the same bit for bit
            lg, _ = e.decode_step(tb, tok)
            hist.append(tok)
            tok = eng.sample_token(lg, sp, hist, step0 + nb + i)
            assert tok == int(nxt[i, 0]), i
        for s in (sa, sb, ta, tb):
            e.seq_free(s)
        assert e.stats()["kv_pages_used"] == 0


# ---- 4. errors leave every sequence as it was ------------------------------------------------------------------------------
def test_errors_change_nothing(monkeypatch):
    cfg = _cfg("tiny-test", 2048)
    V = cfg["vocab_size"]
    with eng.Engine(model=cfg, seed=1, max_batch=8, max_seqs=16) as e:
        ss = [_fresh(e, _ids(30 + i, V, i))[0] for i in range(9)]
        lens = [e.seq_len(s) for s in ss]

        def bad(status, seqs, drafts, sps=None, x0=None):
            with pytest.raises(eng.EngineError) as ei:
                e.decode_verify_batch(seqs, x0 or [5] * len(seqs), drafts, sps)
            assert ei.value.status == status
            assert [e.seq_len(s) for s in ss] == lens

        bad(eng.CL_ERR_INVALID_ARG, [ss[0], ss[1], ss[0]], [[1], [2], [3]])                 # duplicate sequence
        bad(eng.CL_ERR_INVALID_ARG, ss[:2], [[1] * 16, [2]])                                 # k = 16
        bad(eng.CL_ERR_INVALID_ARG, ss[:9], [[1] * 15] * 8 + [[1] * 0])                      # 8 x 16 + 1 = 129 rows
        bad(eng.CL_ERR_INVALID_ARG, ss[:2], [[1], [2]], [None, _sp(0.8, 0, 0.9, 1.1, 64, 1)])   # top_k 0: host sampler only
        bad(eng.CL_ERR_INVALID_ARG, ss[:2], [[1], [V]])                                      # id out of range
        ids, _ = e.decode_verify_batch(ss[:9], [5] * 9, [[1] * 15] * 7 + [[1] * 14, []])    # exactly 128 rows fit
        assert len(ids[8]) == 1
        e.seq_fake_fill(ss[1], e.cfg["max_seq_len"] - 2)
        lens = [e.seq_len(s) for s in ss]
        bad(eng.CL_ERR_TOO_LONG, ss[:2], [[1], [2, 3]])                                      # past max_seq_len
        for s in ss:
            e.seq_free(s)
        for n in (0, 9, 33):
            with pytest.raises(eng.EngineError) as ei:
                e.set_speculate_batch(n)
            assert ei.value.status == eng.CL_ERR_INVALID_ARG
        e.set_speculate_batch(8)
    monkeypatch.setenv("CL_SPECULATE_BATCH", "5")
    with pytest.raises(eng.EngineError) as ei:
        eng.Engine(preset="tiny-test", seed=1, max_batch=4)                                # 5 > max_batch
    assert ei.value.status == eng.CL_ERR_INVALID_ARG


# ---- 5. the scheduler -----------------------------------------------------------------------------------------------------
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


def _spec_prompt(V, salt):
    """Every id follows one marker id somewhere, so the history's last bigram always has an earlier occurrence; then a
    repeated run, so that a right draft is likely too."""
    c = 3 + salt
    pairs = np.stack([np.full(V, c), np.arange(V)], 1).reshape(-1)
    run = _ids(40, V, salt)
    return np.concatenate([run, pairs, run, run, [c]]).astype(np.int32)


def _concurrent(e, jobs):
    out = {}
    ts = [threading.Thread(target=lambda n=n, f=f: out.__setitem__(n, f())) for n, f in jobs.items()]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def test_scheduler_verifies_several_requests_in_one_pass():
    cfg = _cfg("tiny-test", 2048)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    tol = _tol(L)
    prompts = {n: _spec_prompt(V, i + 1) for i, n in enumerate(("g1", "g2", "s"))}
    sp = eng.ollama_default_sampling(seed=5, max_new_tokens=64)
    sp.ignore_eos = 1
    streamed = []
    with eng.Engine(model=cfg, seed=31, max_batch=4, max_seqs=4, speculate=7, speculate_batch=4, start_scheduler=True) as e:
        out = _concurrent(e, {
            "g1": lambda: e.generate_ids(prompts["g1"], eng.greedy(96, ignore_eos=True)),
            "g2": lambda: e.generate_ids(prompts["g2"], eng.greedy(80, ignore_eos=True)),
            "s": lambda: e.generate_ids(prompts["s"], sp),
            "stream": lambda: e.generate_stream(e.model_name, "abcabcabcabc " * 20, eng.greedy(48, ignore_eos=True),
                                                on_text=lambda t, ids: streamed.extend(ids)),
        })
        st = e.spec_stats()
        assert e.spec_multi_passes() > 0 and st["verify_passes"] > 0
        assert st["tokens_emitted"] == st["tokens_accepted"] + st["verify_passes"]
        assert e.stats()["kv_pages_used"] == 0
        assert out["g1"].n_generated == 96 and out["g2"].n_generated == 80 and out["s"].n_generated == 64
        assert out["stream"].n_generated == 48 and streamed == out["stream"].token_ids.tolist()
        print(f"spec stats {st}, multi passes {e.spec_multi_passes()}")
        # a host-sampled request (top_k 0) in the batch: plain steps only
        before = e.spec_multi_passes()
        host = eng.ollama_default_sampling(seed=3, max_new_tokens=48)
        host.top_k, host.ignore_eos = 0, 1
        _concurrent(e, {"a": lambda: e.generate_ids(prompts["g1"], eng.greedy(48, ignore_eos=True)),
                        "h": lambda: e.generate_ids(prompts["g2"], host)})
        assert e.spec_multi_passes() == before
        assert e.stats()["kv_pages_used"] == 0
    with eng.Engine(model=cfg, seed=31, max_batch=4, max_seqs=4) as ref:
        for n in ("g1", "g2"):
            assert _teacher_forced_gaps(ref, prompts[n], out[n].token_ids).max() <= tol


def test_default_speculate_batch_keeps_single_request_speculation():
    """The same two overlapping requests: no multi-sequence pass with the default speculate_batch, some with 2."""
    cfg = _cfg("tiny-test", 2048)
    V = cfg["vocab_size"]
    multi = {}
    for n in (1, 2):
        with eng.Engine(model=cfg, seed=41, max_batch=4, max_seqs=4, speculate=15, speculate_batch=n, start_scheduler=True) as e:
            _concurrent(e, {c: (lambda p=_spec_prompt(V, i + 2): e.generate_ids(p, eng.greedy(64, ignore_eos=True)))
                            for i, c in enumerate("ab")})
            multi[n] = e.spec_multi_passes()
            assert e.stats()["kv_pages_used"] == 0
    assert multi[1] == 0 and multi[2] > 0, multi


def test_pass_with_more_rows_than_max_seq_len():
    """128 rows in one pass of an engine whose max_seq_len is 64: each sequence fits, the pass's rows do not."""
    cfg = _cfg("tiny-test", 64)
    V = cfg["vocab_size"]
    with eng.Engine(model=cfg, seed=3, max_batch=8, max_seqs=8) as e:
        prompts = [_ids(10 + i, V, 60 + i) for i in range(8)]
        ss, x0s = zip(*[_fresh(e, p) for p in prompts])
        ds = [_ids(15, V, 70 + i).tolist() for i in range(8)]
        ids, lg = e.decode_verify_batch(list(ss), list(x0s), ds, want_logits=True)
        assert lg.shape == (128, V) and np.isfinite(lg).all()
        for i in range(8):
            assert ids[i].tolist() == _replay(lg[16 * i:16 * (i + 1)], None, prompts[i], x0s[i], ds[i], 0)
            assert e.seq_len(ss[i]) == len(prompts[i]) + len(ids[i])
