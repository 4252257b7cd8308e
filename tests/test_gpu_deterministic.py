"""Deterministic mode (cl_engine_config.deterministic) on the GPU: every token path runs one row-invariant pass, so a
sequence's logits, K/V, ids and logprob records are the same bits whatever shares its steps and passes, however its
prompt is split, and whether its ids come from single steps or verify passes.

1. Kernels: a row of the split-K GEMM (deterministic split counts) and of the LM head is the same bits in launches of
   1 .. 256 rows; a row of the multi-row attention is the same bits in a one-row segment, in a 16-row segment and among
   other segments.
2. Engine (2-layer Llama-3-8B shape, synthetic weights): logits and K/V of a target sequence across batch sizes with
   neighbours of random lengths, prompt cuts, prefill groups, prefix-cache pages, verify passes and a recompute; ids and
   logprob records of greedy and device-sampled loops; logits within the oracle's tolerance.
3. Requests: one greedy and one seeded sampled request give the same ids, text and logprob records alone and amid 30
   concurrent requests with preemptions, chunked and group admission, speculation and the prefix cache's host tier."""
import threading

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu



@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    for k in ("CL_DETERMINISTIC", "CL_SPECULATE", "CL_SPECULATE_BATCH", "CL_PREFIX_CACHE", "CL_PREFIX_CACHE_HOST_MIB",
              "CL_SCHED_PREFILL_CHUNK", "CL_SCHED_MULTI_PREFILL", "CL_CONTEXT_LENGTH", "CL_DRAFT_MODEL"):
        monkeypatch.delenv(k, raising=False)


def _cfg(n_layers=2, max_seq_len=8192):
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["n_layers"], cfg["max_seq_len"] = n_layers, max_seq_len
    return cfg


def _ids(n, vocab, salt):
    return np.array([(i * 7919 + 13 + salt * 104729) % (vocab - 3) + 3 for i in range(n)], np.int32)


def _sp(temp, top_k, top_p, pen, last_n, seed, n=-1):
    s = eng.Sampling()
    s.temperature, s.top_k, s.top_p, s.repeat_penalty, s.repeat_last_n, s.seed = temp, top_k, top_p, pen, last_n, seed
    s.max_new_tokens = n
    return s


def _bf16(rng, shape, scale=1.0):
    return oc.np_bf16_from_f32((rng.standard_normal(shape) * scale).astype(np.float32))


def _kv(e, s, n):
    """K and V of every layer at positions 0 .. n - 1"""
    return np.stack([e.debug_kv(s, l, w, 0, n) for l in range(e.cfg["n_layers"]) for w in (0, 1)])


def _same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, what
    bad = np.flatnonzero(a.view(np.uint32 if a.dtype == np.float32 else a.dtype).ravel() !=
                         b.view(np.uint32 if b.dtype == np.float32 else b.dtype).ravel())
    assert bad.size == 0, f"{what}: {bad.size} elements differ, first at {bad[0]}"


# ---- 1. kernels ------------------------------------------------------------------------------------------------------------
SHAPES = {"qkv": (6144, 4096), "o": (4096, 4096), "gate|up": (28672, 4096), "down": (4096, 14336)}
TS = [1, 2, 31, 32, 33, 64, 65, 127, 128, 256]


def _split(n, k):
    ks = eng.C.c_int32()
    assert eng.lib().cl_gemm_split_plan(n, k, 0, 1, eng.C.byref(ks)) == eng.CL_OK
    return ks.value


@pytest.mark.parametrize("name", list(SHAPES) + ["lm_head"])
def test_gemm_rows_do_not_depend_on_the_launch(name):
    """Rows come from a pool of 4 distinct rows placed at every position of every tile; each must equal that pool row
    launched alone, split partial for split partial."""
    n, k = SHAPES.get(name, (128256, 4096))
    ks = 1 if name == "lm_head" else _split(n, k)
    rng = np.random.default_rng(n + k)
    w = _bf16(rng, (n, k), 0.02)
    pool = _bf16(rng, (4, k))
    alone = [eng.op_gemm_bf16_epi(pool[i:i + 1], w, k_splits=ks)[0] for i in range(4)]
    for t in TS if name != "lm_head" else [1, 2, 33, 65, 128]:
        sel = (np.arange(t) * 3 + t) % 4
        y, used = eng.op_gemm_bf16_epi(pool[sel], w, k_splits=ks)
        assert used == ks
        for r in range(t):
            _same(y[:, r], alone[sel[r]][:, 0], f"{name} T={t} row {r}")


def _segments(rng, lens, rows, D=128, n_kv=8, H=32):
    """q rows and caches of segments (ctx_lens[s] cached tokens + rows[s] new ones), as cl_op_attn_verify takes them"""
    qs = [_bf16(rng, (r, H * D)) for r in rows]
    ks = [_bf16(rng, (c + r, n_kv, D)) for c, r in zip(lens, rows)]
    vs = [_bf16(rng, (c + r, n_kv, D)) for c, r in zip(lens, rows)]
    return qs, ks, vs


def _verify(qs, ks, vs, lens, rows):
    out, _ = eng.op_attn_verify(np.concatenate(qs), np.concatenate(ks), np.concatenate(vs), lens, rows, 32, 8, 128)
    return out


@pytest.mark.parametrize("L", [255, 256, 257, 4095, 4096, 4097, 8191])
def test_attention_rows_do_not_depend_on_the_segment(L):
    rng = np.random.default_rng(L)
    qs, ks, vs = _segments(rng, [L], [16])
    full = _verify(qs, ks, vs, [L], [16])
    for r in (0, 1, 5, 15):   # row r alone: a one-row segment at cached length L + r
        alone = _verify([qs[0][r:r + 1]], [ks[0][:L + r + 1]], [vs[0][:L + r + 1]], [L + r], [1])
        _same(alone[0], full[r], f"L={L} row {r} alone")
    for n_other in (1, 7, 64):   # among other segments, before and after it
        lens = list(rng.integers(1, 4096, n_other))
        rws = list(rng.integers(1, 17, n_other))
        oq, ok, ov = _segments(rng, lens, rws)
        h = n_other // 2
        out = _verify(oq[:h] + qs + oq[h:], ok[:h] + ks + ok[h:], ov[:h] + vs + ov[h:], lens[:h] + [L] + lens[h:],
                      rws[:h] + [16] + rws[h:])
        r0 = int(sum(rws[:h]))
        _same(out[r0:r0 + 16], full, f"L={L} among {n_other} segments")
        # and one-row segments only (the deterministic step's launch): from 8 segments on, the one-warp instantiation,
        # against the 4-warp kernel's 16-row segment
        ones = _verify([qs[0][15:16]] + [q[:1] for q in oq], [ks[0]] + [kk[:c + 1] for kk, c in zip(ok, lens)],
                       [vs[0]] + [vv[:c + 1] for vv, c in zip(ov, lens)], [L + 15] + lens, [1] * (n_other + 1))
        _same(ones[0], full[15], f"L={L} row 15 among {n_other} one-row segments")


# ---- 2. engine ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def det():
    with eng.Engine(model=_cfg(), seed=5, max_batch=100, max_seqs=104, deterministic=True, prefix_cache=True) as e:
        yield e


def _free_all(e, ss):
    for s in ss:
        e.seq_free(s)


PROMPT_LEN = 300
FORCED = 6


def _reference(e, V):
    """the target alone: prompt in one call, then FORCED teacher-forced steps; logits after every input and its K/V"""
    p = _ids(PROMPT_LEN, V, 1)
    f = _ids(FORCED, V, 2)
    s = e.seq_create()
    lg = [e.prefill(s, p)]
    for x in f:
        lg.append(e.decode_step(s, int(x))[0])
    kv = _kv(e, s, PROMPT_LEN + FORCED)
    e.seq_free(s)
    return p, f, np.stack(lg), kv


@pytest.fixture(scope="module")
def ref(det):
    return _reference(det, det.cfg["vocab_size"])


@pytest.mark.parametrize("B", [2, 8, 100])
def test_decode_bits_do_not_depend_on_the_batch(det, ref, B):
    p, f, lg_ref, kv_ref = ref
    V = det.cfg["vocab_size"]
    rng = np.random.default_rng(B)
    s = det.seq_create()
    _same(det.prefill(s, p), lg_ref[0], "prefill")
    nb = [det.seq_create() for _ in range(B - 1)]
    for o in nb:
        det.seq_fake_fill(o, int(rng.integers(1, 4096)))
    seqs = [s] + nb
    order = rng.permutation(B)   # the target at a random position of the batch
    seqs = [seqs[i] for i in order]
    pos = int(np.flatnonzero(order == 0)[0])
    for i, x in enumerate(f):
        toks = rng.integers(3, V, B).astype(np.int32)
        toks[pos] = x
        lg, _ = det.decode_step_batch(seqs, toks)
        _same(lg[pos], lg_ref[i + 1], f"B={B} step {i}")
    _same(_kv(det, s, PROMPT_LEN + FORCED), kv_ref, f"B={B} K/V")
    _free_all(det, seqs)


@pytest.mark.parametrize("cut", ["tokens", 1, 16, 100, 128, 129, "batch"])
def test_prompt_cuts_give_the_same_bits(det, ref, cut):
    p, f, lg_ref, kv_ref = ref
    V = det.cfg["vocab_size"]
    s = det.seq_create()
    if cut == "batch":   # cl_prefill_batch with other prompts, the target in the middle
        a, b = det.seq_create(), det.seq_create()
        lg = det.prefill_batch([a, s, b], [_ids(77, V, 9), p, _ids(190, V, 8)])[1]
        _free_all(det, [a, b])
    else:
        step = 1 if cut == "tokens" else cut
        for c0 in range(0, PROMPT_LEN, step):
            lg = det.prefill(s, p[c0:c0 + step])
    _same(lg, lg_ref[0], f"cut {cut}: last prompt logits")
    for i, x in enumerate(f):
        _same(det.decode_step(s, int(x))[0], lg_ref[i + 1], f"cut {cut}: step {i}")
    _same(_kv(det, s, PROMPT_LEN + FORCED), kv_ref, f"cut {cut}: K/V")
    det.seq_free(s)


def test_prefix_cache_pages(det, ref):
    p, f, lg_ref, kv_ref = ref
    full = np.concatenate([p, f])
    a = det.seq_create()
    det.prefill(a, full)   # publishes the full pages
    det.seq_free(a)
    s = det.seq_create()
    reused = det.attach_prefix(s, full)
    assert reused > 0
    lg = det.prefill(s, full[reused:])
    _same(lg, lg_ref[-1], "suffix behind prefix-cache pages")
    _same(_kv(det, s, len(full)), kv_ref, "K/V behind prefix-cache pages")
    det.seq_free(s)


@pytest.mark.parametrize("j", [1, 3, FORCED - 1])
def test_recompute_replay(det, ref, j):
    """what preemption does: the sequence is freed, its prompt and the j ids it had generated are prefilled again in one
    call, and decoding goes on teacher-forced; every position's logits and K/V equal the uninterrupted run"""
    p, f, lg_ref, kv_ref = ref
    a = det.seq_create()
    det.prefill(a, p)
    for x in f[:j]:
        det.decode_step(a, int(x))
    det.seq_free(a)
    s = det.seq_create()
    _same(det.prefill(s, np.concatenate([p, f[:j]])), lg_ref[j], f"recompute of {j} ids")
    for i in range(j, FORCED):
        _same(det.decode_step(s, int(f[i]))[0], lg_ref[i + 1], f"replay step {i} after recomputing {j} ids")
    _same(_kv(det, s, PROMPT_LEN + FORCED), kv_ref, f"K/V after recomputing {j} ids")
    det.seq_free(s)


def test_host_tier_restore(ref):
    """the target's pages spill to the host tier when a neighbour needs the pool, then come back for a suffix"""
    p, f, lg_ref, kv_ref = ref
    full = np.concatenate([p, f])
    page_bytes = 32 * 2 * 2 * 8 * 128 * 2
    with eng.Engine(model=_cfg(), seed=5, max_batch=2, max_seqs=2, deterministic=True, prefix_cache=True,
                    kv_pool_bytes=24 * page_bytes, prefix_cache_host_bytes=32 * page_bytes) as e:
        a = e.seq_create()
        e.prefill(a, full)                     # 10 pages, 9 of them full and published
        e.seq_free(a)
        b = e.seq_create()
        e.seq_fake_fill(b, 24 * 32)            # the whole pool: every cached page goes to the host
        e.seq_free(b)
        assert e.prefix_stats(host=True)["pages_to_host"] >= 9
        s = e.seq_create()
        reused = e.attach_prefix(s, full)
        st = e.prefix_stats(host=True)
        assert reused == 9 * 32 and st["pages_from_host"] >= 9, st
        _same(e.prefill(s, full[reused:]), lg_ref[-1], "suffix behind pages restored from the host tier")
        _same(_kv(e, s, len(full)), kv_ref, "K/V on pages restored from the host tier")


def test_verify_passes_equal_single_steps(det, ref):
    p, f, lg_ref, kv_ref = ref
    V = det.cfg["vocab_size"]
    s = det.seq_create()
    det.prefill(s, p)
    # a right draft (the forced ids) and a wrong one: accepted rows equal the single steps' logits
    ids, lg = det.decode_verify(s, int(f[0]), f[1:], want_logits=True)
    _same(lg, lg_ref[1:], "verify rows")
    t = det.seq_create()
    det.prefill(t, p)
    wrong = (f[1:] + 1) % V
    other = det.seq_create()
    det.prefill(other, _ids(500, V, 4))
    out, lg2 = det.decode_verify_batch([other, t], [7, int(f[0])], [_ids(5, V, 3), wrong], want_logits=True)
    _same(lg2[6], lg_ref[1], "first row of a wrong draft in a batch pass")
    n = PROMPT_LEN + len(out[1])
    _same(_kv(det, t, n)[:, :n], kv_ref[:, :n], "K/V after a batch verify")
    _free_all(det, [s, t, other])


def test_device_loops_ids_and_logprobs(det):
    V = det.cfg["vocab_size"]
    rng = np.random.default_rng(3)
    sps = [eng.greedy(-1), _sp(0.9, 40, 0.9, 1.1, 64, 7)]

    def run(B):
        ss = [det.seq_create() for _ in range(B)]
        for j, s in enumerate(ss):
            det.prefill(s, _ids(40 + 9 * j, V, 20 + j))
            det.set_logprobs(s, 5)
        first = [int(x) for x in rng.integers(3, V, B)]
        first[0], first[1] = 11, 12
        samp = sps + [sps[j % 2] for j in range(2, B)]
        ids, _ = det.decode_sample_batch(ss, first, samp, 24)
        recs = [det.take_logprobs(s) for s in ss[:2]]
        _free_all(det, ss)
        return ids[:, :2], recs

    ids1, rec1 = run(2)
    for B in (5, 37):
        ids, rec = run(B)
        _same(ids, ids1, f"device loop ids, B={B}")
        for a, b in zip(rec, rec1):
            assert a.tobytes() == b.tobytes(), f"logprob records, B={B}"


@pytest.mark.parametrize("n_layers,cached", [(2, 0), (32, 4096)])
def test_logits_match_the_oracle(n_layers, cached):
    cfg = _cfg(n_layers, 4096 + 64 if cached else 512)
    V = cfg["vocab_size"]
    tol = 0.05 + 0.03 * float(np.sqrt(n_layers))
    m = oc.Model(cfg, seed=99)
    with eng.Engine(model=cfg, seed=99, max_batch=2, max_seqs=2, deterministic=True) as e:
        s = e.seq_create()
        so = m.new_seq((cached or 64) + 32)
        if cached:
            e.seq_fake_fill(s, cached)
            so.fake_fill(cached)
            inputs = _ids(4, V, 5)
            got = np.stack([e.decode_step(s, int(x))[0] for x in inputs])
        else:
            inputs = _ids(21, V, 5)
            got = np.stack([e.prefill(s, inputs[:1])] + [e.decode_step(s, int(x))[0] for x in inputs[1:]])
        want = so.forward(inputs, all_logits=True)
        worst = float(np.abs(got - want).max())
        so.close()
    m.close()
    print(f"{n_layers} layers behind {cached} cached tokens: max |dlogit| {worst:.4f} (tolerance {tol:.3f})")
    assert worst < tol


# ---- 3. requests ----------------------------------------------------------------------------------------------------------
TOKENS = 32 * 2 * 2 * 8 * 128 * 2 // 32   # KV bytes per token of the 2-layer model


def _tied(e):
    """embedding and LM head set to the same rows (sign and 7-bit mantissa random, magnitude in [16, 32), far above what
    the synthetic layers add to the residual stream): token x's final row stays close to row x, so x is by far its own
    largest logit and every request, greedy or sampled, repeats its input.  The n-gram drafter then drafts at every
    round, and its drafts are accepted."""
    V, d = e.cfg["vocab_size"], e.cfg["d_model"]
    rows = np.random.default_rng(4).integers(0, 256, (V, d), dtype=np.uint16)
    w = ((rows & 0x80) << 8) | (131 << 7) | (rows & 0x7F)
    e.set_tensor(0, "EMBED", w)
    e.set_tensor(0, "LM_HEAD", w)


def _concurrent(jobs):
    out = {}
    ts = [threading.Thread(target=lambda n=n, f=f: out.__setitem__(n, f())) for n, f in jobs.items()]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return out


def _requests(e, V, crowd):
    """the greedy and the sampled request, submitted after a crowd of short ones (queued last, so that they run while the
    queue is empty and the scheduler speculates)"""
    greedy = eng.greedy(64, ignore_eos=True)
    sampled = _sp(0.8, 40, 0.9, 1.1, 64, 1234, 64)
    sampled.ignore_eos = 1
    # repeated runs, so that the n-gram drafter finds matches
    pg, ps = np.tile(_ids(30, V, 61), 6), np.tile(_ids(15, V, 62), 3)
    jobs = {}
    rng = np.random.default_rng(17)
    for i in range(crowd):
        n = int(rng.integers(8, 33))
        sp = eng.greedy(int(rng.integers(8, 33)), ignore_eos=True) if i % 2 else _sp(1.0, 20, 0.95, 1.0, 0, i, int(rng.integers(8, 33)))
        sp.ignore_eos = 1
        jobs[i] = (lambda p=np.tile(_ids(5, V, 100 + i), n // 5 + 1)[:n], sp=sp: e.generate_ids(p, sp))
    jobs["g"] = lambda: e.generate_ids_logprobs(pg, greedy, 3)
    jobs["s"] = lambda: e.generate_ids_logprobs(ps, sampled, 3)
    out = _concurrent(jobs)
    return {k: out[k] for k in ("g", "s")}


def _check_same(a, b, what):
    for k in ("g", "s"):
        (ra, la), (rb, lb) = a[k], b[k]
        assert ra.token_ids.tolist() == rb.token_ids.tolist(), f"{what}: {k} ids"
        assert ra.text == rb.text, f"{what}: {k} text"
        assert la.tobytes() == lb.tobytes(), f"{what}: {k} logprob records"


_ALONE = {}


def _alone(tied):
    if tied not in _ALONE:
        with eng.Engine(model=_cfg(max_seq_len=2048), seed=21, max_batch=8, max_seqs=8, deterministic=True,
                        start_scheduler=True) as e:
            if tied:
                _tied(e)
            _ALONE[tied] = _requests(e, e.cfg["vocab_size"], 0)
    return _ALONE[tied]


@pytest.mark.parametrize("variant", ["crowd", "speculate", "draft", "host_tier"])
def test_requests_amid_a_crowd(variant, monkeypatch):
    tied = variant == "speculate"
    alone = _alone(tied)
    monkeypatch.setenv("CL_SCHED_PREFILL_CHUNK", "64")
    kw = dict(model=_cfg(max_seq_len=2048), seed=21, max_batch=8, max_seqs=32, deterministic=True, start_scheduler=True)
    kw["kv_pool_bytes"] = 416 * TOKENS   # 13 pages: 8 running requests do not fit, so some are preempted
    if variant in ("speculate", "draft"):
        kw.update(speculate=7, speculate_batch=8)
    if variant == "draft":
        kw.update(draft_model=dict(_cfg(1, 2048)), draft_seed=3)
    elif variant == "host_tier":
        kw.update(prefix_cache=True, prefix_cache_host_bytes=64 << 20)
    with eng.Engine(**kw) as e:
        if tied:
            _tied(e)
        V = e.cfg["vocab_size"]
        rounds = 2 if variant == "host_tier" else 1   # cold, then warm
        for r in range(rounds):
            _check_same(_requests(e, V, 30), alone, f"{variant} round {r}")
        st = e.stats()
        print(f"{variant}: {st['preemptions']} preemptions, {st['sched_prefill_calls']} prefill calls for "
              f"{st['requests_completed']} requests, spec stats {e.spec_stats()}, prefix {e.prefix_stats(host=True)}")
        assert st["preemptions"] > 0, st
        # every admission of a request (re-admissions after a preemption included) costs at least one prefill call unless
        # group admission takes several in one call
        assert st["sched_prefill_calls"] < st["requests_completed"] + st["preemptions"], st
        if variant in ("speculate", "draft"):
            assert e.spec_stats()["verify_passes"] > 0
        if variant == "host_tier":
            assert e.prefix_stats(host=True)["pages_from_host"] > 0
