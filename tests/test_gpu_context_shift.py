"""Context shift on the GPU: kv_shift_kernel against float64 (cl_op_kv_shift), cl_seq_shift's cache against a fresh prefill
and the shifted oracle, the prefix cache and its host tier around a shifting sequence, and the scheduler's request-level
shift against a token-level replay."""
import threading

import numpy as np
import pytest

import shift_util as su
from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    for v in ("CL_PREFIX_CACHE", "CL_CONTEXT_SHIFT", "CL_NUM_KEEP", "CL_SPECULATE", "CL_MEGA"):
        monkeypatch.delenv(v, raising=False)


def _ids(n, vocab, salt):
    return np.array([(i * 7919 + 13 + salt * 104729) % (vocab - 3) + 3 for i in range(n)], np.int32)


def _cfg(name, max_seq_len, n_layers=None):
    base = {"llama3-8b-2l": "llama3-8b", "llama3.2-1b-2l": "llama3.2-1b"}.get(name, name)
    cfg = dict(oc.PRESETS[base])
    if n_layers or name.endswith("-2l"):
        cfg["n_layers"] = n_layers or 2
    cfg["max_seq_len"] = max_seq_len
    return cfg


def _check_shifted_rows(k_new, v_new, k_old, v_old, keep, delta, cs):
    """[len2][...] rows after, [len][...] before: < keep exact, V moved exactly, K bit-identical to the fp32 restatement
    and within the float64 bound."""
    assert np.array_equal(k_new[:keep], k_old[:keep]) and np.array_equal(v_new[:keep], v_old[:keep])
    assert np.array_equal(v_new[keep:], v_old[keep + delta:])
    old = k_old[keep + delta:]
    err = su.shift_err(k_new[keep:], old, cs)
    assert err <= 1.0, err
    assert np.array_equal(k_new[keep:], su.rotate_back(old, cs))
    return err


# ---- the kernel ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [16, 32, 64])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("n_kv", [1, 8])
def test_kernel_matches_float64(P, hd, n_kv):
    rng = np.random.default_rng(P * 1000 + hd + n_kv)
    cfg = dict(oc.PRESETS["llama3.2-1b" if hd == 64 else "llama3-8b"])   # the 1B's table carries the "llama3" scaling
    tab = su.rope_table(cfg, 8192)
    L, T = 2, 10 * P + 7
    for keep in (0, 4, P - 1, P, P + 3):
        for delta in sorted({P, P * ((T - keep) // (2 * P))}):
            k = oc.np_bf16_from_f32(rng.standard_normal((L, T, n_kv, hd)).astype(np.float32) * 2)
            v = oc.np_bf16_from_f32(rng.standard_normal((L, T, n_kv, hd)).astype(np.float32))
            ko, vo, _ = eng.op_kv_shift(k, v, P, keep, delta, tab[delta])
            for l in range(L):
                _check_shifted_rows(oc.np_f32_from_bf16(ko[l]), oc.np_f32_from_bf16(vo[l]), oc.np_f32_from_bf16(k[l]),
                                    oc.np_f32_from_bf16(v[l]), keep, delta, tab[delta])


@pytest.mark.parametrize("preset,delta", [("llama3-8b", 4064), ("llama3.2-1b", 32), ("llama3.2-1b", 4096)])
def test_kernel_8192_tokens(preset, delta):
    cfg = dict(oc.PRESETS[preset])
    P, T, keep = 32, 8192, 4
    tab = su.rope_table(cfg, 8192)
    rng = np.random.default_rng(delta)
    k = oc.np_bf16_from_f32(rng.standard_normal((2, T, cfg["n_kv_heads"], cfg["head_dim"])).astype(np.float32))
    v = oc.np_bf16_from_f32(rng.standard_normal(k.shape).astype(np.float32))
    ko, vo, ms = eng.op_kv_shift(k, v, P, keep, delta, tab[delta], iters=5)
    assert ms > 0
    for l in range(2):
        _check_shifted_rows(oc.np_f32_from_bf16(ko[l]), oc.np_f32_from_bf16(vo[l]), oc.np_f32_from_bf16(k[l]),
                            oc.np_f32_from_bf16(v[l]), keep, delta, tab[delta])


# ---- cl_seq_shift: the cache --------------------------------------------------------------------------------------------
def _pair_ulp_err(a, b, hd):
    """max |a - b| in bf16 ulps of the rotation pair's magnitude (a rotation moves error between the pair's two dims)."""
    x = a.reshape(a.shape[0], -1, hd)
    y = b.reshape(b.shape[0], -1, hd)
    half = hd // 2
    mag = np.sqrt(y[..., :half].astype(np.float64) ** 2 + y[..., half:].astype(np.float64) ** 2)
    mag = np.concatenate([mag, mag], axis=-1)
    ulp = np.exp2(np.floor(np.log2(np.maximum(mag, 1e-30))) - 7)
    return float((np.abs(x.astype(np.float64) - y) / ulp).max())


@pytest.mark.parametrize("P", [16, 32, 64])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l", "llama3.2-1b-2l"])
def test_seq_shift_cache(shape, P):
    cfg = _cfg(shape, 1024)
    V, L, hd = cfg["vocab_size"], cfg["n_layers"], cfg["head_dim"]
    N = 230
    ids = _ids(N, V, 3)
    with eng.Engine(model=cfg, seed=99, max_batch=2, max_seqs=4, page_size=P) as e:
        m = oc.Model(cfg, seed=None)                                    # the engine's own table, bit for bit
        otab = {d: su.oracle_rope_row(m, d) for d in range(P, 1024, P)}
        m.close()
        for keep in (0, 4, P + 3):
            delta = P * ((N - keep) // (2 * P))
            s = e.seq_create()
            e.prefill(s, ids, want_logits=False)
            before = [[e.debug_kv(s, l, w, 0, N) for w in (0, 1)] for l in range(L)]
            e.seq_shift(s, keep, delta)
            assert e.seq_len(s) == N - delta
            for l in range(L):
                k1, v1 = e.debug_kv(s, l, 0, 0, N - delta), e.debug_kv(s, l, 1, 0, N - delta)
                sh = (-1, cfg["n_kv_heads"], hd)
                _check_shifted_rows(k1.reshape(sh), v1.reshape(sh), before[l][0].reshape(sh), before[l][1].reshape(sh), keep,
                                    delta, otab[delta])
            # layer 0 depends on the id and the position only: a fresh prefill of the kept ids writes nearly the same K
            kept = np.concatenate([ids[:keep], ids[keep + delta:]])
            f = e.seq_create()
            e.prefill(f, kept, want_logits=False)
            k0, v0 = e.debug_kv(s, 0, 0, 0, len(kept)), e.debug_kv(s, 0, 1, 0, len(kept))
            assert np.array_equal(v0, e.debug_kv(f, 0, 1, 0, len(kept)))
            assert _pair_ulp_err(k0, e.debug_kv(f, 0, 0, 0, len(kept)), hd) <= 1.5
            e.seq_free(f)
            e.seq_free(s)
        s = e.seq_create()
        e.prefill(s, ids[:40], want_logits=False)
        for keep, delta in ((4, P + 1), (4, 0), (-1, P), (40 - P + 1, P)):
            with pytest.raises(eng.EngineError):
                e.seq_shift(s, keep, delta)
            assert e.seq_len(s) == 40
        e.seq_free(s)
        assert e.stats()["kv_pages_used"] == 0


# ---- whole model against the shifted oracle ---------------------------------------------------------------------------------
def _tol(L):
    return 0.05 + 0.03 * float(np.sqrt(L))


@pytest.mark.parametrize("shape,P,path", [("tiny-test", 16, "per-op"), ("tiny-test", 64, "per-op"), ("llama3-8b-2l", 32, "mega"),
                                          ("llama3-8b-2l", 32, "per-op"), ("llama3.2-1b-2l", 32, "per-op"),
                                          ("tiny-test", 32, "batch3"), ("llama3-8b-2l", 32, "batch3"),
                                          ("tiny-test", 32, "verify"), ("llama3-8b-2l", 32, "verify")])
def test_shifted_model_matches_shifted_oracle(shape, P, path, monkeypatch):
    if path == "per-op":
        monkeypatch.setenv("CL_MEGA", "0")
    cfg = _cfg(shape, 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    N, keep = 300, 4
    delta = P * ((N - keep) // (2 * P))
    ids = _ids(N, V, 5)
    steps = _ids(8, V, 6)
    m = oc.Model(cfg, seed=77)
    so = m.new_seq()
    so.prefill_block(ids)
    su.oracle_shift(so, keep, delta)
    with eng.Engine(model=cfg, seed=77, max_batch=4, max_seqs=4, page_size=P) as e:
        if path == "mega":
            assert e.runs_mega_kernel()
        s = e.seq_create()
        e.prefill(s, ids, want_logits=False)
        e.seq_shift(s, keep, delta)
        worst = 0.0
        if path == "verify":
            _, lg = e.decode_verify(s, int(steps[0]), steps[1:], want_logits=True)
            ref = so.forward(steps, all_logits=True)
            worst = float(np.abs(lg - ref).max())
        elif path == "batch3":
            others = [e.seq_create() for _ in range(2)]
            for i, o in enumerate(others):
                e.prefill(o, _ids(50 + 30 * i, V, 8 + i), want_logits=False)
            for t in steps:
                lg, _ = e.decode_step_batch([others[0], s, others[1]], [int(t), int(t), int(t)])
                worst = max(worst, float(np.abs(lg[1] - so.forward(np.array([t], np.int32))).max()))
        else:
            for t in steps:
                lg, _ = e.decode_step(s, int(t))
                worst = max(worst, float(np.abs(lg - so.forward(np.array([t], np.int32))).max()))
        assert worst <= _tol(L), worst
        print(f"{shape} P{P} {path}: max|dlogit| {worst:.4f} (tolerance {_tol(L):.3f})")


# ---- prefix cache and host tier ---------------------------------------------------------------------------------------------
def _shared_run(shift_b):
    """a holds a prompt, b shares its first 16 pages (prefix cache, host tier on) and may shift; a's K/V and next logits."""
    cfg = _cfg("tiny-test", 1024)
    V, L, P = cfg["vocab_size"], cfg["n_layers"], 16
    X = _ids(320, V, 9)
    page_bytes = 2 * L * P * cfg["n_kv_heads"] * cfg["head_dim"] * 2
    with eng.Engine(model=cfg, seed=5, max_batch=4, max_seqs=6, page_size=P, prefix_cache=True,
                    prefix_cache_host_bytes=64 * page_bytes) as e:
        a = e.seq_create()
        e.prefill(a, X, want_logits=False)
        b = e.seq_create()
        Y = np.concatenate([X[:256], _ids(100, V, 11)])
        assert e.attach_prefix(b, Y) == 256
        e.prefill(b, Y[256:], want_logits=False)
        if shift_b:
            e.seq_shift(b, 4, 160)                                      # writes pages that a holds and the index keys
            e.decode_step(b, 7)
        kv_a = [e.debug_kv(a, l, w, 0, 320) for l in range(L) for w in (0, 1)]
        lg_a, _ = e.decode_step(a, int(_ids(1, V, 10)[0]))
        e.seq_free(a)
        e.seq_free(b)
        c = e.seq_create()
        assert e.attach_prefix(c, X) == 304                              # a third request takes the original pages
        kv_c = [e.debug_kv(c, l, w, 0, 304) for l in range(L) for w in (0, 1)]
        e.seq_free(c)
        assert e.stats()["kv_pages_used"] == 0
    return kv_a, lg_a, kv_c


def test_shift_leaves_shared_pages_alone():
    kv_ref, lg_ref, kvc_ref = _shared_run(False)
    kv_a, lg_a, kv_c = _shared_run(True)
    assert all(np.array_equal(x, y) for x, y in zip(kv_a, kv_ref))
    assert np.array_equal(lg_a, lg_ref)
    assert all(np.array_equal(x, y[:304]) for x, y in zip(kv_c, kv_ref))
    assert all(np.array_equal(x, y) for x, y in zip(kv_c, kvc_ref))


# ---- request level ------------------------------------------------------------------------------------------------------------
W, PS, KEEP = 256, 16, 4
DELTA = PS * ((W - KEEP) // (2 * PS))


def _replay(e, prompt, n, sp=None):
    """Token-level replay of a request with the switch on: prefill, decode steps, and cl_seq_shift whenever the next step
    would write position W."""
    s = e.seq_create()
    hist = list(prompt)
    lg = e.prefill(s, prompt)
    pick = (lambda lg, step: int(np.argmax(lg))) if sp is None else (lambda lg, step: eng.sample_token(lg, sp, hist, step))
    out = [pick(lg, 0)]
    while len(out) < n:
        if e.seq_len(s) >= W:
            e.seq_shift(s, KEEP, DELTA)
        hist.append(out[-1])
        lg, _ = e.decode_step(s, out[-1])
        out.append(pick(lg, len(out)))
    e.seq_free(s)
    return np.array(out, np.int32)


def _tiny(**kw):
    cfg = _cfg("tiny-test", W)
    return eng.Engine(model=cfg, seed=31, page_size=PS, context_shift=True, num_keep=KEEP, **kw)


@pytest.mark.parametrize("scheduler", [False, True])
def test_requests_match_token_replay(scheduler):
    V = oc.PRESETS["tiny-test"]["vocab_size"]
    prompt = _ids(100, V, 12)
    n = 400                                                              # 100 + 400 tokens: three shifts
    sampled = eng.ollama_default_sampling(seed=3, max_new_tokens=n)
    sampled.ignore_eos = 1
    with _tiny(max_batch=2, max_seqs=4) as ref:
        want_g = _replay(ref, prompt, n)
        want_s = _replay(ref, prompt, n, sampled)
    with _tiny(max_batch=2, max_seqs=4, start_scheduler=scheduler) as e:
        r = e.generate_ids(prompt, eng.greedy(n, ignore_eos=True))
        assert r.done_reason == "length" and r.n_generated == n and r.n_prompt == 100
        assert np.array_equal(r.token_ids, want_g)
        r = e.generate_ids(prompt, sampled)
        assert np.array_equal(r.token_ids, want_s)
        assert e.stats()["kv_pages_used"] == 0


def _teacher_check(e, prompt, out, tol=0.05):
    """Feeds a request's ids back at the token level, shifting at the same lengths: every id must be the step's argmax or
    within a near tie of it (verify passes and decode steps run different kernels)."""
    s = e.seq_create()
    lg = e.prefill(s, prompt)
    for i, t in enumerate(out):
        if i:
            if e.seq_len(s) >= W:
                e.seq_shift(s, KEEP, DELTA)
            lg, _ = e.decode_step(s, int(out[i - 1]))
        assert lg[t] >= lg.max() - tol, (i, int(t), int(np.argmax(lg)), float(lg.max() - lg[t]))
    e.seq_free(s)


def test_speculation_matches_token_replay():
    V = oc.PRESETS["tiny-test"]["vocab_size"]
    prompt = np.tile(_ids(25, V, 13), 4)                                 # repetitive: the drafter finds matches
    for sched in (False, True):
        with _tiny(max_batch=2, max_seqs=4, speculate=4, start_scheduler=sched) as e:
            r = e.generate_ids(prompt, eng.greedy(300, ignore_eos=True))
            assert r.n_generated == 300 and r.done_reason == "length"
            assert e.spec_stats()["verify_passes"] > 0
            assert e.stats()["kv_pages_used"] == 0
        with _tiny(max_batch=2, max_seqs=4) as ref:
            _teacher_check(ref, prompt, r.token_ids)


def _window(prompt, out, shifted):
    """What a request re-admitted with `out` generated prefills: its window after `shifted` discarded ids, shifted once
    more on the host when it would leave no position for the next token (Engine::preempt)."""
    full = list(prompt) + [int(x) for x in out]
    if len(full) - shifted >= W:
        shifted += DELTA
    return full[:KEEP] + full[KEEP + shifted:], shifted


def _run(e, prompt, out, start, shifted, stop, tol):
    """Token-level replay of a request from a (re-)prefill of its window after `start` ids, then decode steps and shifts at
    the lengths the scheduler shifts at.  Returns the first index in [start, stop) whose id is not the replay's argmax or
    within tol of it (stop if none), and the ids discarded so far at each index."""
    w, shifted = _window(prompt, out[:start], shifted)
    s = e.seq_create()
    sh_at = {}
    try:
        lg = e.prefill(s, np.array(w, np.int32))
        for i in range(start, stop):
            if i > start:
                if e.seq_len(s) >= W:
                    e.seq_shift(s, KEEP, DELTA)
                    shifted += DELTA
                lg, _ = e.decode_step(s, int(out[i - 1]))
            sh_at[i] = shifted
            if lg[out[i]] < lg.max() - tol:
                return i, sh_at
        return stop, sh_at
    finally:
        e.seq_free(s)


def _replay_check(e, prompt, out, n_preempted, tol=0.05):
    """Teacher-forces a finished request's ids through a token-level replay.  Where an id cannot be explained, the request
    must have been preempted after some earlier id j and re-admitted by prefilling its window there: the latest such j
    that explains the ids up to this one is taken, at most n_preempted times."""
    pos, shifted, rebuilds = 0, 0, 0
    while True:
        k, sh_at = _run(e, prompt, out, pos, shifted, len(out), tol)
        if k == len(out):
            return rebuilds
        assert rebuilds < n_preempted, f"id {k} of {len(out)} is not the replay's choice (preemptions {n_preempted})"
        for j in range(k, pos, -1):
            if _run(e, prompt, out, j, sh_at[j], k + 1, tol)[0] == k + 1:
                pos, shifted, rebuilds = j, sh_at[j], rebuilds + 1
                break
        else:
            raise AssertionError(f"id {k}: no re-admission window after ids {pos + 1}..{k} explains it")


def test_concurrent_and_preempted_requests_match_token_replay():
    V = oc.PRESETS["tiny-test"]["vocab_size"]
    # a pool of 40 pages: three requests of up to 16 pages each cannot all hold their windows, so some are preempted
    cfg = _cfg("tiny-test", W)
    page_bytes = 2 * cfg["n_layers"] * PS * cfg["n_kv_heads"] * cfg["head_dim"] * 2
    prompts = [_ids(60 + 40 * i, V, 20 + i) for i in range(3)]
    for pool_pages in (200, 40):
        with _tiny(max_batch=4, max_seqs=4, start_scheduler=True, kv_pool_bytes=pool_pages * page_bytes) as e:
            res = [None] * 3

            def run(i):
                res[i] = e.generate_ids(prompts[i], eng.greedy(350, ignore_eos=True))

            th = [threading.Thread(target=run, args=(i,)) for i in range(3)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            assert all(r.n_generated == 350 and r.done_reason == "length" for r in res)
            if pool_pages == 40:
                assert e.stats()["preemptions"] > 0
            else:
                assert all(r.n_preempted == 0 for r in res)
            assert e.stats()["kv_pages_used"] == 0
        with _tiny(max_batch=4, max_seqs=4) as ref:
            rebuilt = [_replay_check(ref, prompts[i], res[i].token_ids, res[i].n_preempted) for i in range(3)]
        print(f"pool {pool_pages}: preemptions {[r.n_preempted for r in res]}, re-admissions the replay needed {rebuilt}")


def test_llama3_8b_32_layers_8192_behind_fake_fill():
    """The production case: 32 layers of attention over the 4128 kept tokens of an 8192-token cache after a 4064-token
    shift, both sides behind the synthetic cache pattern, 8 teacher-forced steps on the persistent kernel."""
    cfg = dict(oc.PRESETS["llama3-8b"])
    L = cfg["n_layers"]
    steps = _ids(8, cfg["vocab_size"], 30)
    m = oc.Model(cfg, seed=1234)
    so = m.new_seq()
    so.fake_fill(8192)
    su.oracle_shift(so, 4, 4064)
    worst = 0.0
    with eng.Engine(model=cfg, seed=1234, max_batch=1, max_seqs=1, page_size=32) as e:
        assert e.runs_mega_kernel()
        s = e.seq_create()
        e.seq_fake_fill(s, 8192)
        e.seq_shift(s, 4, 4064)
        assert e.seq_len(s) == 4128
        for t in steps:
            lg, _ = e.decode_step(s, int(t))
            worst = max(worst, float(np.abs(lg - so.forward(np.array([t], np.int32))).max()))
    m.close()
    print(f"llama3-8b 32 layers, 8192 -> 4128 tokens: max|dlogit| {worst:.4f} (tolerance {_tol(L):.3f})")
    assert worst <= _tol(L), worst


def test_long_prompt_is_truncated():
    V = oc.PRESETS["tiny-test"]["vocab_size"]
    long = _ids(3 * W, V, 14)
    cut = np.concatenate([long[:KEEP], long[-(W - 1 - KEEP):]])
    with _tiny(max_batch=2, max_seqs=4, start_scheduler=True) as e:
        a = e.generate_ids(long, eng.greedy(40, ignore_eos=True))
        b = e.generate_ids(cut, eng.greedy(40, ignore_eos=True))
        assert a.n_prompt == W - 1 == b.n_prompt
        assert np.array_equal(a.token_ids, b.token_ids) and a.n_generated == 40
        c = e.generate_ids(long, eng.greedy(0, ignore_eos=True))      # num_predict <= 0: bounded by the window
        assert c.n_generated == 1


@pytest.mark.parametrize("scheduler", [False, True])
def test_switch_off_keeps_the_window(scheduler):
    V = oc.PRESETS["tiny-test"]["vocab_size"]
    with eng.Engine(model=_cfg("tiny-test", W), seed=31, page_size=PS, max_batch=2, start_scheduler=scheduler) as e:
        r = e.generate_ids(_ids(100, V, 12), eng.greedy(400, ignore_eos=True))
        assert r.done_reason == "length" and r.n_generated == W - 100
        with pytest.raises(eng.EngineError):
            e.generate_ids(_ids(W, V, 15), eng.greedy(4, ignore_eos=True))


def test_create_refuses_num_keep_without_room():
    with pytest.raises(eng.EngineError):
        eng.Engine(model=_cfg("tiny-test", W), seed=1, page_size=PS, context_shift=True, num_keep=W - 2 * PS + 1)
    with pytest.raises(eng.EngineError):
        eng.Engine(model=_cfg("tiny-test", W), seed=1, page_size=PS, context_shift=True, num_keep=-1)
    eng.Engine(model=_cfg("tiny-test", W), seed=1, page_size=PS, num_keep=W).close()   # off: num_keep unused
