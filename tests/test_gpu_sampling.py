"""The device sampler of the decode step's tail kernel against the host sampler (cl_sample_token), id for id."""
import itertools
import threading

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu

TOPK_CAP, HIST_CAP = 128, 256          # kSampleTopKMax, kSampleHistMax (csrc/kernels.h)


def _sp(temperature, top_k, top_p, penalty, last_n, seed):
    s = eng.ollama_default_sampling(seed=seed)
    s.temperature, s.top_k, s.top_p, s.repeat_penalty, s.repeat_last_n = temperature, top_k, top_p, penalty, last_n
    return s


def _bf16(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def _logits(kind, V, rng):
    x = rng.normal(0.0, 2.5, V).astype(np.float32)
    if kind == "bf16":          # bf16-rounded: exact ties
        x = _bf16(x)
    elif kind == "ties":        # coarse grid: long runs of ties across the top-k boundary, +0 and -0 among them
        x = (np.round(x * 2) / 2).astype(np.float32)
        z = np.flatnonzero(x == 0)
        x[z[::2]] = np.float32(-0.0)
    elif kind == "neg":         # every logit negative: the penalty multiplies
        x = -np.abs(x) - np.float32(0.01)
    elif kind == "inf":         # -inf entries, enough of them to reach into the top-k at small vocabularies
        x[rng.random(V) < 0.6] = -np.inf
    return x


def _history(logits, window, V, rng):
    """window + 9 ids: top-ranked ids (so the penalty changes the top-k), duplicates and out-of-range ids."""
    top = np.argsort(-logits, kind="stable")[:48]
    n = window + 9
    h = rng.choice(top, n).astype(np.int64)
    h[rng.random(n) < 0.15] = rng.integers(0, V, 1)[0]                  # duplicates of one id
    h[rng.random(n) < 0.1] = -1 - rng.integers(0, 5)                    # out of range, below
    h[rng.random(n) < 0.1] = V + rng.integers(0, 5)                     # out of range, above
    return h.astype(np.int32)


@pytest.mark.parametrize("V", [512, 32000, 128256])
def test_op_sample_matches_host_sampler(V):
    rng = np.random.default_rng(V)
    grid = list(itertools.product([1, 5, 40, TOPK_CAP], [0.5, 0.9, 1.0], [0.3, 0.8, 1.5], [1.0, 1.1, 1.6], [1, 64, HIST_CAP],
                                  ["gauss", "bf16", "ties", "neg", "inf"]))
    rng.shuffle(grid)
    grid = grid[:1200 if V < 100000 else 400]
    # every value of every factor is still present
    for f in range(6):
        assert len({g[f] for g in grid}) == len({g[f] for g in itertools.product([1, 5, 40, TOPK_CAP], [0.5, 0.9, 1.0], [0.3, 0.8, 1.5],
                                                                                 [1.0, 1.1, 1.6], [1, 64, HIST_CAP],
                                                                                 ["gauss", "bf16", "ties", "neg", "inf"])})
    rows = 64
    mism = []
    for c0 in range(0, len(grid), rows):
        chunk = grid[c0:c0 + rows]
        lg = np.stack([_logits(g[5], V, rng) for g in chunk])
        sps = [_sp(g[2], g[0], g[1], g[3], g[4], int(rng.integers(0, 2**63))) for g in chunk]
        hists = [_history(lg[i], g[4], V, rng) for i, g in enumerate(chunk)]
        steps = rng.integers(0, 2**40, len(chunk)).astype(np.uint64)
        dev = eng.op_sample(lg, sps, hists, steps)
        for i in range(len(chunk)):
            host = eng.sample_token(lg[i], sps[i], hists[i], int(steps[i]))
            if host != dev[i]:
                mism.append((chunk[i], int(host), int(dev[i])))
    assert not mism, mism[:10]


def test_op_sample_rejects_host_only_settings():
    lg = np.zeros((1, 512), np.float32)
    for bad in (_sp(0.8, 0, 0.9, 1.1, 64, 1), _sp(0.8, TOPK_CAP + 1, 0.9, 1.1, 64, 1), _sp(0.8, 40, 0.9, 1.1, -1, 1),
                _sp(0.8, 40, 0.9, 1.1, HIST_CAP + 1, 1), _sp(0.0, 40, 0.9, 1.1, 64, 1)):
        with pytest.raises(eng.EngineError) as ei:
            eng.op_sample(lg, [bad], [[]], [0])
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
    eng.op_sample(lg, [_sp(0.8, 40, 0.9, 1.0, -1, 1)], [[]], [0])      # penalty off: any window


def _prompt(n, V, k=0):
    return np.array([(i * 7919 + 13 + 101 * k) % V for i in range(n)], np.int32)


def _replay(e, prompts, firsts, sps, step0, ids):
    """Feed the device's ids through cl_decode_step_batch on fresh sequences and draw each step with the host sampler."""
    seqs = [e.seq_create() for _ in prompts]
    for s, p in zip(seqs, prompts):
        e.prefill(s, p, want_logits=False)
    hist = [list(p) for p in prompts]
    feed = list(firsts)
    for i in range(ids.shape[0]):
        lg, _ = e.decode_step_batch(seqs, feed)
        for b in range(len(seqs)):
            hist[b].append(feed[b])
            want = eng.sample_token(lg[b], sps[b], hist[b], int(step0[b]) + i)
            assert want == ids[i, b], (i, b, want, ids[i, b])
        feed = [int(x) for x in ids[i]]
    for s in seqs:
        e.seq_free(s)


def _run_sample_batch(e, V, B, n_steps, sampled):
    rng = np.random.default_rng(B * 1000 + V)
    prompts = [_prompt(20 + 13 * b, V, b) for b in range(B)]
    seqs = [e.seq_create() for _ in range(B)]
    for s, p in zip(seqs, prompts):
        e.prefill(s, p, want_logits=False)
    firsts = [int(p[-1] * 3 % V) for p in prompts]
    pool = [_sp(0.8, 40, 0.9, 1.1, 64, 11), _sp(1.5, TOPK_CAP, 1.0, 1.6, HIST_CAP, 12), _sp(0.3, 5, 0.5, 1.0, 0, 13),
            _sp(0.8, 1, 0.9, 1.1, 8, 14)]
    sps = [pool[b % len(pool)] if sampled[b] else eng.greedy(0) for b in range(B)]
    step0 = rng.integers(0, 1000, B).astype(np.uint64)
    l0 = e.stats()["kernel_launches"]
    ids, _ = e.decode_sample_batch(seqs, firsts, sps, n_steps, step0)
    launches = e.stats()["kernel_launches"] - l0
    for s in seqs:
        e.seq_free(s)
    _replay(e, prompts, firsts, sps, step0, ids)
    return ids, launches


def _llama_cfg():
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["n_layers"] = 2
    cfg["max_seq_len"] = 256
    return cfg


@pytest.mark.parametrize("mega", ["1", "0"])
@pytest.mark.parametrize("model", ["tiny-test", "llama3-8b-2l"])
def test_decode_sample_batch_single_sequence_replays(monkeypatch, model, mega):
    monkeypatch.setenv("CL_MEGA", mega)           # B = 1: persistent kernel (Llama-3 shape) and per-op path
    kw = dict(preset="tiny-test") if model == "tiny-test" else dict(model=_llama_cfg())
    with eng.Engine(seed=5, max_batch=8, **kw) as e:
        _run_sample_batch(e, e.cfg["vocab_size"], 1, 32, [True])


@pytest.mark.parametrize("B", [3, 8])
@pytest.mark.parametrize("model", ["tiny-test", "llama3-8b-2l"])
def test_decode_sample_batch_mixed_batch_replays(model, B):
    kw = dict(preset="tiny-test") if model == "tiny-test" else dict(model=_llama_cfg())
    with eng.Engine(seed=6, max_batch=8, **kw) as e:
        sampled = [b % 3 != 1 for b in range(B)]      # greedy slots in between
        _run_sample_batch(e, e.cfg["vocab_size"], B, 32, sampled)


@pytest.mark.parametrize("B", [1, 4])
def test_sampled_steps_launch_the_same_kernels_as_greedy(B):
    with eng.Engine(model=_llama_cfg(), seed=7, max_batch=8) as e:
        V = e.cfg["vocab_size"]
        seqs = [e.seq_create() for _ in range(B)]
        for b, s in enumerate(seqs):
            e.prefill(s, _prompt(24, V, b), want_logits=False)
        firsts = [1] * B
        n = 16
        e.decode_greedy_batch(seqs, firsts, 2)                                        # graphs captured before counting
        l0 = e.stats()["kernel_launches"]
        e.decode_greedy_batch(seqs, firsts, n)
        greedy = e.stats()["kernel_launches"] - l0
        l0 = e.stats()["kernel_launches"]
        e.decode_sample_batch(seqs, firsts, [_sp(0.8, 40, 0.9, 1.1, 64, b) for b in range(B)], n)
        sampled = e.stats()["kernel_launches"] - l0
        assert greedy == sampled and greedy % n == 0, (greedy, sampled)


def test_decode_sample_batch_rejects_host_only_settings():
    with eng.Engine(preset="tiny-test", seed=8) as e:
        s = e.seq_create()
        e.prefill(s, _prompt(5, 512), want_logits=False)
        with pytest.raises(eng.EngineError) as ei:
            e.decode_sample_batch([s], [1], [_sp(0.8, 0, 0.9, 1.1, 64, 1)], 4)
        assert ei.value.status == eng.CL_ERR_INVALID_ARG
        assert e.seq_len(s) == 5


def _requests():
    V = 512
    reqs = []
    for i, n in enumerate([7, 40, 150, 23]):          # tokenwise, short-prompt and tile prefill paths
        sp = _sp(0.8, 40, 0.9, 1.1, 64, 100 + i)
        sp.max_new_tokens, sp.ignore_eos = 48, 1
        reqs.append((_prompt(n, V, i), sp))
    sp = _sp(0.8, 0, 0.9, 1.1, 64, 7)                  # top-k 0: the host sampler
    sp.max_new_tokens, sp.ignore_eos = 24, 1
    reqs.append((_prompt(12, V, 9), sp))
    return reqs


@pytest.mark.parametrize("scheduler", [True, False])
def test_requests_match_between_device_and_host_sampling(monkeypatch, scheduler):
    out = {}
    for dev in ("1", "0"):
        monkeypatch.setenv("CL_DEVICE_SAMPLE", dev)
        with eng.Engine(preset="tiny-test", seed=31, max_batch=4, start_scheduler=scheduler) as e:
            out[dev] = [e.generate_ids(p, sp).token_ids for p, sp in _requests()]
            assert e.stats()["kv_pages_used"] == 0
    for a, b in zip(out["1"], out["0"]):
        np.testing.assert_array_equal(a, b)


def test_concurrent_sampled_requests_complete_without_leaks():
    reqs = _requests() * 3
    with eng.Engine(preset="tiny-test", seed=31, max_batch=4, max_seqs=4, start_scheduler=True) as e:
        solo_r = [e.generate_ids(p, sp) for p, sp in reqs]
        solo = [r.token_ids for r in solo_r]
        res = [None] * len(reqs)

        def run(i):
            res[i] = e.generate_ids(*reqs[i])

        th = [threading.Thread(target=run, args=(i,)) for i in range(len(reqs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for i, r in enumerate(res):
            assert r is not None and r.n_generated == reqs[i][1].max_new_tokens
            assert r.token_ids[0] == solo[i][0]
        st = e.stats()
        assert st["kv_pages_used"] == 0 and st["active_seqs"] == 0
        assert st["requests_completed"] == 2 * len(reqs) and st["preemptions"] == sum(r.n_preempted for r in solo_r + res)
