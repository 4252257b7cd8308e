"""Speculative decoding with a draft model (cl_engine_create_with_draft, cl_draft_model): a small model of the same vocabulary
drafts, the served model verifies.  Without real weights, acceptance is steered by the choice of draft: a self-draft (the
target's config and seed) is right up to near-tie flips, a draft with another seed is almost always wrong, and a truncated
self-draft (fewer layers; the synthetic generator keys every tensor by layer * 16 + kind) is right part of the time.  The
drafter alone must equal a standalone engine of the draft's config bit for bit; requests must emit what a draft-off engine
emits (greedy: within near ties, teacher-forced; sampled: a token-level replay of the same rounds)."""
import threading

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_env_override(monkeypatch):
    for k in ("CL_SPECULATE", "CL_SPECULATE_BATCH", "CL_PREFIX_CACHE", "CL_DRAFT_MODEL", "CL_DRAFT_SEED", "CL_CONTEXT_SHIFT",
              "CL_NUM_KEEP", "CL_CONTEXT_LENGTH"):
        monkeypatch.delenv(k, raising=False)


def _cfg(name, max_seq_len, n_layers=None):
    base = {"llama3-8b-2l": "llama3-8b", "llama3.2-1b-2l": "llama3.2-1b"}.get(name, name)
    cfg = dict(oc.PRESETS[base])
    if base != name:
        cfg["n_layers"] = 2
    if n_layers is not None:
        cfg["n_layers"] = n_layers
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


OLLAMA = _sp(0.8, 40, 0.9, 1.1, 64, 7)
SEED = 31

# target shape -> {draft kind: (draft model config, draft seed)}
def _drafts(shape, max_seq_len):
    if shape == "tiny-test":
        cfg = _cfg("tiny-test", max_seq_len)
        return cfg, {"self": (cfg, SEED), "wrong": (cfg, 999), "trunc": (_cfg("tiny-test", max_seq_len, 1), SEED)}
    cfg = _cfg("llama3-8b-2l", max_seq_len)
    return cfg, {"1b": (_cfg("llama3.2-1b-2l", max_seq_len), SEED)}


def _engine(cfg, draft, **kw):
    dcfg, dseed = draft
    return eng.Engine(model=cfg, seed=SEED, draft_model=dcfg, draft_seed=dseed, **kw)


def _teacher_forced_gaps(ref, prompt, ids):
    """Top logit minus the logit of every produced id, replaying prompt + ids through ref."""
    s = ref.seq_create()
    lg = ref.prefill(s, prompt)
    gaps = []
    for i, tok in enumerate(ids):
        gaps.append(float(lg.max() - lg[tok]))
        if i + 1 < len(ids):
            lg, _ = ref.decode_step(s, int(tok))
    ref.seq_free(s)
    return np.array(gaps)


def _first(lg, sp, hist, step):
    return int(np.argmax(lg)) if sp is None else eng.sample_token(lg, sp, hist, step)


def _standalone(ref, hists, ks, sps, step0):
    """What the drafter computes, through a standalone engine of the draft's config: one prefill (cl_prefill for one
    window, cl_prefill_batch for several), the first id from its logits, then max(ks) - 1 device steps."""
    ss = [ref.seq_create() for _ in hists]
    lgs = [ref.prefill(ss[0], hists[0])] if len(ss) == 1 else list(ref.prefill_batch(ss, hists))
    d1 = [_first(lg, sp, list(h), st) for lg, sp, h, st in zip(lgs, sps, hists, step0)]
    K = max(ks)
    steps = None
    if K > 1:
        steps, _ = ref.decode_sample_batch(ss, d1, [sp if sp is not None else eng.greedy(-1) for sp in sps], K - 1,
                                           step0=[st + 1 for st in step0])
    out = [[d1[i]] + ([int(t) for t in steps[:ks[i] - 1, i]] if ks[i] > 1 else []) for i in range(len(ss))]
    for s in ss:
        ref.seq_free(s)
    return out


# ---- 1. the drafter alone -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sampled", [False, True])
@pytest.mark.parametrize("shape", ["tiny-test", "llama3-8b-2l"])
def test_drafter_equals_a_standalone_draft_engine(shape, sampled):
    cfg, drafts = _drafts(shape, 1024)
    kind = "trunc" if shape == "tiny-test" else "1b"
    dcfg, dseed = drafts[kind]
    V = cfg["vocab_size"]
    with _engine(cfg, drafts[kind], max_batch=4, max_seqs=4, speculate=7) as e, \
            eng.Engine(model=dcfg, seed=dseed, max_batch=4, max_seqs=4) as ref:
        for n in (1, 3):
            ss = [e.seq_create() for _ in range(n)]
            hists = [_ids(40 + 23 * i, V, i + 1) for i in range(n)]
            ks = [7, 3, 5][:n]
            sps = [OLLAMA if sampled and i != 1 else None for i in range(n)]
            step0 = [5 * i for i in range(n)]
            got = e.draft_model(ss, hists, ks, sps, step0)
            want = _standalone(ref, hists, ks, sps, step0)
            assert [g.tolist() for g in got] == want, (n, got, want)
            # a second call whose window diverges at m: inside the old mirror, at a page boundary, at 0
            tol = _tol(dcfg["n_layers"])
            for m in (17, 32, 0):
                hists2 = [np.concatenate([h[:m], _ids(30, V, 50 + m)]) for h in hists]
                got2 = e.draft_model(ss, hists2, ks, None, None)
                for h2, g, k in zip(hists2, got2, ks):
                    assert len(g) == k
                    assert _teacher_forced_gaps(ref, h2, g).max() <= tol
            st = e.draft_stats()
            assert st["draft_rows"] > 0 and st["draft_pages_used"] > 0
            for s in ss:
                e.seq_free(s)
            assert e.draft_stats()["draft_pages_used"] == 0
        assert e.stats()["kv_pages_used"] == 0


# ---- 2. requests --------------------------------------------------------------------------------------------------------
def _spec_prompt(V, salt):
    run = _ids(40, V, salt)
    return np.concatenate([run, _ids(60, V, salt + 7), run]).astype(np.int32)


def _token_level_replay(e, prompt, sp, k_spec, max_new):
    """What a speculating request does with a draft model, through cl_draft_model, cl_decode_verify and single steps."""
    s = e.seq_create()
    lg = e.prefill(s, prompt)
    out = [eng.sample_token(lg, sp, list(prompt), 0)]
    backoff = 0
    while len(out) < max_new:
        n = 0
        k_max = min(k_spec, max_new - len(out) - 1, e.cfg["max_seq_len"] - e.seq_len(s) - 1)
        if backoff == 0 and k_max >= 1:
            d = e.draft_model([s], [list(prompt) + out], [k_max], [sp], [len(out)])[0]
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
@pytest.mark.parametrize("shape,kind", [("tiny-test", "self"), ("tiny-test", "wrong"), ("tiny-test", "trunc"), ("llama3-8b-2l", "1b")])
def test_requests_with_a_draft_model(shape, kind, scheduler):
    cfg, drafts = _drafts(shape, 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    prompt = _spec_prompt(V, 1)
    sp = _sp(0.8, 40, 0.9, 1.1, 64, 5)
    sp.max_new_tokens, sp.ignore_eos = 64, 1
    with _engine(cfg, drafts[kind], max_batch=4, max_seqs=4, speculate=7, start_scheduler=scheduler) as e:
        g = e.generate_ids(prompt, eng.greedy(64, ignore_eos=True))
        st_g = e.spec_stats()
        smp = e.generate_ids(prompt, sp)
        st = e.spec_stats()
        dst = e.draft_stats()
        assert g.n_generated == 64 and smp.n_generated == 64
        assert st["enabled"] == 1 and st["verify_passes"] > 0
        assert st["tokens_emitted"] == st["tokens_accepted"] + st["verify_passes"]
        assert dst["draft_rows"] >= st["tokens_drafted"] and dst["draft_ns"] > 0 and dst["draft_pages_used"] == 0
        assert e.stats()["kv_pages_used"] == 0
        if kind == "self":   # the coupled draws: right for greedy and for sampled requests
            assert st_g["tokens_accepted"] >= 0.9 * st_g["tokens_drafted"], st_g
            # Sampled: the synthetic model's top-40 at temperature 0.8 is nearly flat, so logit differences between the
            # draft's step kernels and the verify pass reorder near-tied candidates, and the same uniform then picks
            # another id for about a third of the rows.  A draw independent of the target's would match only sum(p^2).
            s_acc, s_dr = st["tokens_accepted"] - st_g["tokens_accepted"], st["tokens_drafted"] - st_g["tokens_drafted"]
            assert s_acc >= 0.6 * s_dr, st
        if kind == "wrong":  # almost every pass accepts nothing, and the request backs off
            assert st["tokens_accepted"] < 0.5 * st["tokens_drafted"] and st["verify_passes"] <= 128 // 4, st
        print(f"{shape}/{kind} scheduler={scheduler}: greedy {st_g}, all {st}, draft {dst}")
    with eng.Engine(model=cfg, seed=SEED, max_batch=4, max_seqs=4) as ref:
        assert _teacher_forced_gaps(ref, prompt, g.token_ids).max() <= _tol(L)
    with _engine(cfg, drafts[kind], max_batch=4, max_seqs=4, speculate=7) as rep:
        assert smp.token_ids.tolist() == _token_level_replay(rep, prompt, sp, 7, 64)


# ---- 3. batches ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_req", [2, 8])
def test_batched_requests_draft_together(n_req):
    cfg, drafts = _drafts("tiny-test", 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    prompts = [_spec_prompt(V, 3 + i)[: 60 + 7 * i] for i in range(n_req)]
    with _engine(cfg, drafts["self"], max_batch=8, max_seqs=8, speculate=5, speculate_batch=8, start_scheduler=True) as e:
        out = {}

        def run(i):
            if i % 2:
                sp = _sp(0.8, 40, 0.9, 1.0, 0, 100 + i)
                sp.max_new_tokens, sp.ignore_eos = 48, 1
            else:
                sp = eng.greedy(48, ignore_eos=True)
            out[i] = e.generate_ids(prompts[i], sp)

        ts = [threading.Thread(target=run, args=(i,)) for i in range(n_req)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        st = e.spec_stats()
        assert all(out[i].n_generated == 48 for i in range(n_req))
        assert st["tokens_emitted"] == st["tokens_accepted"] + st["verify_passes"]
        assert st["tokens_accepted"] >= 0.7 * st["tokens_drafted"], st   # greedy and sampled requests, half each
        assert e.spec_multi_passes() > 0
        assert e.draft_stats()["draft_pages_used"] == 0 and e.stats()["kv_pages_used"] == 0
    with eng.Engine(model=cfg, seed=SEED, max_batch=8, max_seqs=8) as ref:
        for i in range(0, n_req, 2):
            assert _teacher_forced_gaps(ref, prompts[i], out[i].token_ids).max() <= _tol(L)


# ---- 4. context shift and preemption ---------------------------------------------------------------------------------------
def test_a_shifted_request_keeps_drafting():
    cfg, drafts = _drafts("tiny-test", 256)
    V = cfg["vocab_size"]
    prompt = _ids(200, V, 9)
    with _engine(cfg, drafts["self"], max_batch=2, max_seqs=2, speculate=7, context_shift=True, num_keep=4) as e:
        r = e.generate_ids(prompt, eng.greedy(150, ignore_eos=True))
        st = e.spec_stats()
        assert r.n_generated == 150
        # The window fills after about 56 ids; the rest are drafted too.  After the shift the target's kept K/V still carry
        # the discarded context and the mirror's recomputed ones do not, so fewer drafts are right.
        assert st["tokens_drafted"] > 100 and st["tokens_accepted"] > 0, st
        assert e.draft_stats()["draft_pages_used"] == 0 and e.stats()["kv_pages_used"] == 0


def test_a_preempted_request_keeps_drafting():
    cfg, drafts = _drafts("tiny-test", 1024)
    V, L = cfg["vocab_size"], cfg["n_layers"]
    page_bytes = 32 * 2 * L * cfg["n_kv_heads"] * cfg["head_dim"] * 2
    prompts = [_ids(100, V, 11), _ids(100, V, 12)]
    with _engine(cfg, drafts["self"], max_batch=2, max_seqs=2, speculate=5, speculate_batch=2, start_scheduler=True,
                 kv_pool_bytes=10 * page_bytes) as e:
        out = {}
        ts = [threading.Thread(target=lambda i=i: out.__setitem__(i, e.generate_ids(prompts[i], eng.greedy(120, ignore_eos=True))))
              for i in range(2)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        st = e.spec_stats()
        assert all(out[i].n_generated == 120 for i in range(2))
        assert sum(out[i].n_preempted for i in range(2)) > 0 and st["tokens_drafted"] > 0
        assert e.draft_stats()["draft_pages_used"] == 0 and e.stats()["kv_pages_used"] == 0
    with eng.Engine(model=cfg, seed=SEED, max_batch=2, max_seqs=2) as ref:
        for i in range(2):
            assert _teacher_forced_gaps(ref, prompts[i], out[i].token_ids).max() <= _tol(L)


# ---- 5. refusals and the switch ----------------------------------------------------------------------------------------------
def test_refusals(monkeypatch):
    cfg, drafts = _drafts("tiny-test", 1024)
    cases = [
        (cfg, (_cfg("llama3.2-1b-2l", 1024), SEED), 7, "vocabulary"),
        (cfg, drafts["self"], 0, "speculate"),
        (dict(cfg, d_model=8208), drafts["self"], 7, "verify"),   # d_model above 8192: no verify pass
    ]
    for target, draft, k, what in cases:
        with pytest.raises(eng.EngineError) as ei:
            _engine(target, draft, speculate=k)
        assert ei.value.status == eng.CL_ERR_INVALID_ARG and what in ei.value.detail, ei.value.detail
    with eng.Engine(model=cfg, seed=SEED, speculate=7) as e:   # CL_DRAFT_MODEL unset: the n-gram drafter, no draft
        s = e.seq_create()
        with pytest.raises(eng.EngineError) as ei:
            e.draft_model([s], [_ids(10, cfg["vocab_size"], 1)], [3])
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
        assert e.draft_stats() == dict(draft_rows=0, draft_ns=0, draft_pages_used=0)
    monkeypatch.setenv("CL_DRAFT_MODEL", "tiny-test")
    monkeypatch.setenv("CL_SPECULATE", "5")
    with eng.Engine(preset="tiny-test", seed=SEED) as e:      # the env switch alone turns the draft model on
        s = e.seq_create()
        assert len(e.draft_model([s], [_ids(10, cfg["vocab_size"], 1)], [3])[0]) == 3
        r = e.generate_ids(_ids(50, cfg["vocab_size"], 2), eng.greedy(32, ignore_eos=True))
        assert r.n_generated == 32 and e.spec_stats()["tokens_drafted"] > 0
