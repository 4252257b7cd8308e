"""End-to-end parity of the CUDA engine (through the C-ABI) against the CPU oracle and the HF golden vectors."""
from pathlib import Path

import numpy as np
import pytest

from st_util import fixture_cfg

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"

LOGIT_TOL = 0.125          # max-abs on logits (SURVEY.md §8c); observed errors are ~1e-3
MARGIN_TOL = 2e-2          # a greedy mismatch is only tolerated where the oracle's top-2 margin is below this


def _prompt(n, vocab):
    return np.array([(i * 7919 + 13) % vocab for i in range(n)], np.int32)


def _compare_greedy(e, m, prompt, n_steps):
    """Teacher-forced comparison: both sides consume the ORACLE's greedy tokens; logits must agree
    within LOGIT_TOL at every step and argmax must be identical unless the oracle's margin is tiny."""
    so = m.new_seq()
    lo = so.forward(prompt)
    s = e.seq_create()
    lg = e.prefill(s, prompt)
    errs, mism = [float(np.abs(lg - lo).max())], 0
    tok = int(lo.argmax())
    for _ in range(n_steps):
        if int(lg.argmax()) != tok:
            top2 = np.sort(lo)[-2:]
            assert top2[1] - top2[0] < MARGIN_TOL, "greedy token differs at a clear margin"
            mism += 1
        lo = so.forward([tok])
        lg, _ = e.decode_step(s, tok)
        errs.append(float(np.abs(lg - lo).max()))
        tok = int(lo.argmax())
    e.seq_free(s)
    assert max(errs) < LOGIT_TOL, max(errs)
    return max(errs), mism


@pytest.mark.parametrize("decode_path", [1, 2])
@pytest.mark.parametrize("graph", [True, False])
def test_tiny_engine_matches_oracle(decode_path, graph):
    cfg = oc.PRESETS["tiny-test"]
    m = oc.Model(cfg, seed=1234)
    with eng.Engine(preset="tiny-test", seed=1234, decode_path=decode_path, use_cuda_graph=graph) as e:
        err, mism = _compare_greedy(e, m, _prompt(12, cfg["vocab_size"]), 40)
        assert mism == 0
        # free-running greedy: device loop vs oracle loop
        prompt = _prompt(9, cfg["vocab_size"])
        so = m.new_seq()
        first = int(so.forward(prompt).argmax())
        ref_ids, margins = so.greedy(first, 48)
        s = e.seq_create()
        lg = e.prefill(s, prompt)
        assert int(lg.argmax()) == first
        ids, ms = e.decode_greedy(s, first, 48)
        if margins.min() > MARGIN_TOL:
            np.testing.assert_array_equal(ids, ref_ids)
        else:
            k = int(np.argmax(margins <= MARGIN_TOL))
            np.testing.assert_array_equal(ids[:k], ref_ids[:k])
        assert e.seq_len(s) == 9 + 48
        assert e.stats()["kernel_launches"] > 0


@pytest.mark.parametrize("fixture", ["hf_tiny_llama.npz", "hf_tiny_mistral.npz", "hf_tiny_llama31rope.npz"])
def test_engine_matches_hf_golden(fixture):
    """The HF transformers logits (tests/golden/make_golden.py) pin the CUDA engine directly."""
    z = np.load(G / fixture)
    cfg = fixture_cfg(z)
    with eng.Engine(model=cfg, decode_path=1) as e:
        e.set_tensor(0, "EMBED", z["embed"])
        e.set_tensor(0, "LM_HEAD", z["lm_head"])
        e.set_tensor(0, "FINAL_NORM", z["final_norm"])
        for l in range(cfg["n_layers"]):
            for k in ("ATTN_NORM", "FFN_NORM", "WQ", "WK", "WV", "WO", "WGATE", "WUP", "WDOWN"):
                e.set_tensor(l, k, z[f"L{l}.{k}"])
        ids, ref = z["ids"], z["logits"]
        s = e.seq_create()
        got = [e.prefill(s, ids[:1])]
        for t in ids[1:]:
            got.append(e.decode_step(s, int(t))[0])
        got = np.stack(got)
        rms = float(np.sqrt((ref ** 2).mean()))
        assert np.abs(got - ref).max() < 5e-2 * rms       # bf16 rounding points vs HF fp32 math
        agree = (got.argmax(-1) == ref.argmax(-1)).mean()
        assert agree >= 0.9


def _ids_match(ids, ref, margins):
    k = len(ref) if margins.min() > MARGIN_TOL else int(np.argmax(margins <= MARGIN_TOL))
    np.testing.assert_array_equal(ids[:k], ref[:k])
    return k


@pytest.mark.parametrize("batch_gemm", ["1", "0"])
def test_batched_decode_matches_single_and_oracle(monkeypatch, batch_gemm):
    """Continuous-batching inner loop: B sequences of different lengths advance together.  CL_BATCH_GEMM=1 is
    the tensor-core path (wgmma split-K projections + glue kernels), 0 the per-sequence GEMV kernels."""
    monkeypatch.setenv("CL_BATCH_GEMM", batch_gemm)
    cfg = oc.PRESETS["tiny-test"]
    m = oc.Model(cfg, seed=5)
    with eng.Engine(preset="tiny-test", seed=5, max_batch=4) as e:
        V = e.cfg["vocab_size"]
        prompts = [(_prompt(5 + 13 * i, V) + i) % V for i in range(3)]
        refs = []
        for p in prompts:
            so = m.new_seq()
            first = int(so.forward(p).argmax())
            refs.append((first,) + so.greedy(first, 40))
        for p, (first, ref, margins) in zip(prompts, refs):      # one at a time
            s = e.seq_create()
            assert int(e.prefill(s, p).argmax()) == first
            ids, _ = e.decode_greedy(s, first, 40)
            _ids_match(ids, ref, margins)
            e.seq_free(s)
        seqs = []
        for p, (first, _, _) in zip(prompts, refs):               # all together (40 steps cross page boundaries)
            s = e.seq_create()
            assert int(e.prefill(s, p).argmax()) == first
            seqs.append(s)
        ids, _ = e.decode_greedy_batch(seqs, [r[0] for r in refs], 40)
        for b, (first, ref, margins) in enumerate(refs):
            _ids_match(ids[:, b], ref, margins)
            assert (ids[:, b] == ref).mean() >= 0.9 or margins.min() < MARGIN_TOL


def test_batched_decode_llama_shapes():
    """Batched tensor-core step at Llama-3-8B layer shapes (2 layers, split-K 3/4/5/9) vs the oracle, teacher-forced."""
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["n_layers"] = 2
    cfg["max_seq_len"] = 256
    m = oc.Model(cfg, seed=9)
    with eng.Engine(model=cfg, seed=9, max_batch=3) as e:
        V = cfg["vocab_size"]
        prompts = [_prompt(20 + 17 * i, V, ) for i in range(3)]
        prompts = [(p + 101 * i) % V for i, p in enumerate(prompts)]
        os_, seqs, firsts = [], [], []
        for p in prompts:
            so = m.new_seq()
            lo = so.forward(p)
            s = e.seq_create()
            lg = e.prefill(s, p)
            assert np.abs(lg - lo).max() < LOGIT_TOL
            os_.append(so); seqs.append(s); firsts.append(int(lo.argmax()))
        ids, _ = e.decode_greedy_batch(seqs, firsts, 6)
        for b, so in enumerate(os_):
            ref, margins = so.greedy(firsts[b], 6)
            _ids_match(ids[:, b], ref, margins)


def test_page_boundaries_and_pool_exhaustion():
    # 4 pages of 16 tokens: a 2-layer tiny model; one sequence may hold at most 64 tokens
    cfg = oc.PRESETS["tiny-test"]
    kv_bytes_per_token = 2 * cfg["n_layers"] * cfg["n_kv_heads"] * cfg["head_dim"] * 2
    with eng.Engine(preset="tiny-test", seed=9, page_size=16, kv_pool_bytes=4 * 16 * kv_bytes_per_token) as e:
        m = oc.Model(cfg, seed=9)
        p = _prompt(15, cfg["vocab_size"])
        so = m.new_seq()
        first = int(so.forward(p).argmax())
        ref, margins = so.greedy(first, 40)           # crosses pages at 16, 32, 48
        s = e.seq_create()
        assert int(e.prefill(s, p).argmax()) == first
        ids, _ = e.decode_greedy(s, first, 40)
        if margins.min() > MARGIN_TOL:
            np.testing.assert_array_equal(ids, ref)
        assert e.stats()["kv_pages_used"] == 4
        with pytest.raises(eng.EngineError) as ei:
            e.decode_greedy(s, int(ids[-1]), 20)       # 55 + 20 > 64 tokens of pool
        assert ei.value.status == eng.CL_ERR_OOM
        e.seq_free(s)
        assert e.stats()["kv_pages_used"] == 0


def test_generate_ids_greedy_and_sampled_match_oracle_sampler():
    cfg = oc.PRESETS["tiny-test"]
    m = oc.Model(cfg, seed=21)
    with eng.Engine(preset="tiny-test", seed=21) as e:
        p = _prompt(7, cfg["vocab_size"])
        r = e.generate_ids(p, eng.greedy(16, ignore_eos=True))
        so = m.new_seq()
        first = int(so.forward(p).argmax())
        ref, margins = so.greedy(first, 15)
        assert r.n_generated == 16 and r.done_reason == "length"
        assert r.token_ids[0] == first
        if margins.min() > MARGIN_TOL:
            np.testing.assert_array_equal(r.token_ids[1:], ref)
        # stochastic path: the engine's host sampler equals the oracle sampler on the engine's own logits
        sp = eng.ollama_default_sampling(seed=77, max_new_tokens=12)
        sp.ignore_eos = 1
        r2 = e.generate_ids(p, sp)
        s = e.seq_create()
        lg = e.prefill(s, p)
        hist = list(p)
        for i in range(12):
            t = oc.sample(lg, 0.8, 40, 0.9, 1.1, 64, seed=77, history=hist, step=i)
            assert t == r2.token_ids[i]
            lg, _ = e.decode_step(s, t)
            hist.append(t)


@pytest.mark.parametrize("scheduler", [False, True])
def test_streaming_options_and_cancel_through_the_c_abi(scheduler):
    """SURVEY.md §8f rows 3-4 at the C-ABI: cl_generate_stream / cl_handle_message_stream deliver exactly the text and
    ids of the one-shot calls; GenerateRequest.options override the worker's sampling; a callback can cancel."""
    from crowdllama_b200 import handler as H
    from crowdllama_b200.pb import BaseMessage, GenerateOptions
    with eng.Engine(preset="tiny-test", seed=33, model_name="tiny", start_scheduler=scheduler) as e:
        g = eng.greedy(24, ignore_eos=True)
        whole = e.generate("tiny", "why is the sky blue? ☃", g)
        deltas, ids = [], []
        r = e.generate_stream("tiny", "why is the sky blue? ☃", g, lambda d, new: (deltas.append(d), ids.extend(new)) and False)
        assert r.text == whole.text and list(r.token_ids) == list(whole.token_ids) and r.done_reason == "length"
        assert "".join(deltas) == whole.text and ids == list(whole.token_ids)
        assert len([d for d in deltas if d]) > 1                                # really incremental
        # byte-level handler: frames
        req = H.create_generate_request("tiny", "hello", True, GenerateOptions(temperature=0.0, num_predict=12, seed=1))
        frames = []
        n = e.handle_message_stream(req.encode(), None, lambda f: frames.append(BaseMessage.decode(f).generate_response) and False)
        assert n == len(frames) >= 2 and [f.done for f in frames] == [False] * (n - 1) + [True]
        assert frames[-1].done_reason == "length" and all(f.model == "tiny" and f.worker_id == "worker" for f in frames)
        one = BaseMessage.decode(e.handle_message(req.encode(), None)).generate_response       # cl_handle_message ignores stream
        assert one.done and one.response == "".join(f.response for f in frames)
        # options decide: without them the default sampler is stochastic and unbounded; with them greedy and 12 tokens
        again = BaseMessage.decode(e.handle_message(req.encode(), eng.ollama_default_sampling(seed=99, max_new_tokens=5))).generate_response
        assert again.response == one.response
        raw = H.create_generate_request("tiny", "hello", False, GenerateOptions(temperature=0.0, num_predict=12, raw=True))
        assert BaseMessage.decode(e.handle_message(raw.encode(), None)).generate_response.response != one.response  # no chat framing
        # cancel after the third callback
        calls = []
        r = e.generate_stream("tiny", "x", eng.greedy(200, ignore_eos=True), lambda d, new: (calls.append(1), len(calls) >= 3)[1])
        assert r.done_reason == "cancelled" and 3 <= r.n_generated < 200
        assert e.generate("tiny", "why is the sky blue? ☃", g).text == whole.text   # the engine is healthy afterwards


@pytest.mark.parametrize("name", ["spm_legacy", "llama3"])
def test_engine_with_a_tokenizer_json(name):
    """SURVEY.md §8f row 2: an HF tokenizer.json replaces the byte-level fallback behind cl_generate / cl_tokenize."""
    from pathlib import Path
    gold = Path(__file__).resolve().parent / "golden" / "tokenizers" / f"{name}.tokenizer.json"
    cfg = dict(oc.PRESETS["tiny-test"])
    cfg["vocab_size"] = 1024
    ref = eng.HfTokenizer(gold)
    with eng.Engine(model=cfg, seed=3, model_name="tiny") as e:
        with pytest.raises(eng.EngineError):
            e.load_tokenizer(gold.parent / "does-not-exist.json")
        e.load_tokenizer(gold)
        text = "Why is the sky blue? It's 12:45 ☃"
        assert list(e.tokenize(text)) == ref.encode(text)
        r = e.generate("tiny", text, eng.greedy(12, ignore_eos=True))
        assert r.n_prompt == len(ref.encode(text, add_bos=True, chat=True)) and r.n_generated == 12
        assert r.text == e.detokenize(r.token_ids)
        deltas = []
        r2 = e.generate_stream("tiny", text, eng.greedy(12, ignore_eos=True), lambda d, ids: deltas.append(d) and False)
        assert list(r2.token_ids) == list(r.token_ids) and "".join(deltas) == r.text
    with eng.Engine(preset="tiny-test", seed=3) as e:                  # 512-entry model vocabulary < 702 tokenizer ids
        with pytest.raises(eng.EngineError):
            e.load_tokenizer(gold)


@pytest.mark.parametrize("preset", ["tinyllama-1.1b", "llama3.2-1b"])
def test_tinyllama_shapes_match_oracle(preset):
    """Model shapes outside the persistent kernels (head_dim 64): per-op decode kernels + wgmma prefill.  llama3.2-1b
    adds the "llama3" rotary frequency scaling and a 128K vocabulary (6 layers of the 16 keep the test short)."""
    cfg = dict(oc.PRESETS[preset])
    cfg["max_seq_len"] = 256
    cfg["n_layers"] = min(cfg["n_layers"], 22 if preset == "tinyllama-1.1b" else 6)
    m = oc.Model(cfg, seed=1234)
    mc = dict(cfg)
    with eng.Engine(model=mc, seed=1234, max_batch=1) as e:
        err, mism = _compare_greedy(e, m, _prompt(16, cfg["vocab_size"]), 16)
        print(f"{preset}: max logit err {err:.4g}, near-tie mismatches {mism}")


def test_llama3_8b_layer_shapes_match_oracle():
    """Full Llama-3-8B shapes with 2 layers: every kernel shape of the 8B model at a short context.  The 32-layer
    model at the benchmarked contexts (4096 / 8192) is compared with the oracle in tests/test_gpu_longctx.py and
    tests/test_gpu_fullsize.py."""
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["n_layers"] = 2
    cfg["max_seq_len"] = 128
    m = oc.Model(cfg, seed=1234)
    with eng.Engine(model=cfg, seed=1234, max_batch=1) as e:
        err, mism = _compare_greedy(e, m, _prompt(8, cfg["vocab_size"]), 8)
        print(f"llama3-8b(2 layers): max logit err {err:.4g}, near-tie mismatches {mism}")
        assert mism == 0


@pytest.mark.parametrize("mega", ["1", "0"])
def test_megakernel_and_per_op_path_match_oracle(monkeypatch, mega):
    """The persistent whole-stack decode kernel (decode_mega.cu, CL_MEGA=1) and the per-op kernel path
    (CL_MEGA=0) against the oracle at Llama-3-8B layer shapes (3 layers): teacher-forced logits over a
    context that spans several KV pages / splits and crosses page boundaries, then the device-side greedy loop."""
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["n_layers"] = 3
    cfg["max_seq_len"] = 512
    monkeypatch.setenv("CL_MEGA", mega)
    m = oc.Model(cfg, seed=77)
    with eng.Engine(model=cfg, seed=77, max_batch=1) as e:
        err, mism = _compare_greedy(e, m, _prompt(90, cfg["vocab_size"]), 44)   # crosses the 96- and 128-token boundaries
        print(f"CL_MEGA={mega}: max logit err {err:.4g}, near-tie mismatches {mism}")
        prompt = _prompt(61, cfg["vocab_size"])
        so = m.new_seq()
        first = int(so.forward(prompt).argmax())
        ref, margins = so.greedy(first, 24)
        s = e.seq_create()
        assert int(e.prefill(s, prompt).argmax()) == first
        ids, _ = e.decode_greedy(s, first, 24)
        k = len(ref) if margins.min() > MARGIN_TOL else int(np.argmax(margins <= MARGIN_TOL))
        np.testing.assert_array_equal(ids[:k], ref[:k])


def test_short_request_admitted_during_a_long_one_does_not_disturb_it():
    """Regression (ADVICE r1, scheduler.cpp): a request that finishes during admission (num_predict = 1) used to leave
    d_slots_[0] pointing at its freed slot; the running request then stopped advancing and repeated one token.  A long
    greedy request must return exactly its solo ids while one-token requests come and go."""
    import threading
    cfg = oc.PRESETS["tiny-test"]
    V = cfg["vocab_size"]
    long_prompt = _prompt(20, V)
    shorts = [np.array([(7 * i + 3 * j + 1) % V for j in range(5 + i % 4)], np.int32) for i in range(24)]
    with eng.Engine(preset="tiny-test", seed=11, max_batch=4, max_seqs=4, start_scheduler=True) as e:
        solo_r = e.generate_ids(long_prompt, eng.greedy(400, ignore_eos=True))
        solo = solo_r.token_ids
        short_r = [e.generate_ids(p, eng.greedy(1, ignore_eos=True)) for p in shorts]
        short_solo = [int(r.token_ids[0]) for r in short_r]
        out = {}

        def run_long():
            out["long"] = e.generate_ids(long_prompt, eng.greedy(400, ignore_eos=True))
        th = threading.Thread(target=run_long)
        th.start()
        got_r = [e.generate_ids(p, eng.greedy(1, ignore_eos=True)) for p in shorts]
        got = [int(r.token_ids[0]) for r in got_r]
        th.join()
        assert out["long"].n_generated == 400
        np.testing.assert_array_equal(out["long"].token_ids, solo)
        assert got == short_solo
        st = e.stats()
        assert st["kv_pages_used"] == 0 and st["active_seqs"] == 0
        results = [solo_r, out["long"], *short_r, *got_r]
        assert st["requests_completed"] == len(results) and st["preemptions"] == sum(r.n_preempted for r in results)


def test_long_prompt_is_admitted_in_chunks_between_decode_steps(monkeypatch):
    """scheduler.cpp admission: with another request decoding, a long prompt is prefilled CL_SCHED_PREFILL_CHUNK tokens
    per scheduler iteration (here 16), so the running request keeps producing tokens while the newcomer is admitted; a
    burst of short prompts shares one iteration's budget.  Results must be those of the requests run alone (chunk
    boundaries only change the order of a few fp32 additions: allow a near-tie flip)."""
    import threading
    import time
    monkeypatch.setenv("CL_SCHED_PREFILL_CHUNK", "16")
    cfg = oc.PRESETS["tiny-test"]
    V = cfg["vocab_size"]
    long_prompt = np.array([(i * 31 + 7) % V for i in range(200)], np.int32)
    a_prompt = _prompt(12, V)
    shorts = [np.array([(11 * i + 5 * j + 2) % V for j in range(6 + i)], np.int32) for i in range(5)]
    with eng.Engine(preset="tiny-test", seed=21, max_batch=8, max_seqs=8, start_scheduler=True) as e:
        solo_r = [e.generate_ids(p, eng.greedy(n, ignore_eos=True)) for p, n in [(a_prompt, 400), (long_prompt, 24)] + [(p, 10) for p in shorts]]
        a_solo, b_solo = solo_r[0].token_ids, solo_r[1].token_ids
        s_solo = [r.token_ids for r in solo_r[2:]]
        out, stamps = {}, []

        def run_a():
            sp = eng.greedy(400, ignore_eos=True)
            out["a"] = e.generate_ids(a_prompt, sp)

        def run(name, p, n):
            out[name] = e.generate_ids(p, eng.greedy(n, ignore_eos=True))
        ta = threading.Thread(target=run_a)
        ta.start()
        time.sleep(0.02)                                            # A is decoding
        th = [threading.Thread(target=run, args=("b", long_prompt, 24))] + \
             [threading.Thread(target=run, args=(f"s{i}", p, 10)) for i, p in enumerate(shorts)]
        [t.start() for t in th]
        [t.join() for t in th]
        ta.join()
        assert out["a"].n_generated == 400 and out["b"].n_generated == 24
        assert (out["a"].token_ids == a_solo).mean() > 0.9          # identical up to a possible near-tie flip late in the run
        assert out["b"].token_ids[0] == b_solo[0] and (out["b"].token_ids == b_solo).mean() > 0.7
        for i in range(len(shorts)):
            assert out[f"s{i}"].n_generated == 10 and out[f"s{i}"].token_ids[0] == s_solo[i][0]
        st = e.stats()
        assert st["kv_pages_used"] == 0 and st["active_seqs"] == 0 and st["requests_completed"] == 7 + 7
        assert st["preemptions"] == sum(r.n_preempted for r in solo_r + list(out.values()))


def test_group_admission_of_a_burst_matches_requests_run_alone(monkeypatch):
    """scheduler.cpp group admission (CL_SCHED_MULTI_PREFILL=1): a burst of prompts waiting at the head of the queue is
    prefilled in ONE pass (Engine::prefill_multi) and joins the batch together.  Every request must return what it
    returns alone (first token exactly; later tokens up to the near-tie flips of batched vs single-sequence kernels),
    nothing may leak, and a long prompt in the middle of the queue still takes the chunked path."""
    import threading
    monkeypatch.setenv("CL_SCHED_MULTI_PREFILL", "1")
    monkeypatch.setenv("CL_SCHED_PREFILL_CHUNK", "256")
    cfg = oc.PRESETS["tiny-test"]
    V = cfg["vocab_size"]
    prompts = [np.array([(13 * i + 7 * j + 3) % V for j in range(20 + 9 * (i % 5))], np.int32) for i in range(14)]
    prompts[6] = np.array([(i * 31 + 7) % V for i in range(400)], np.int32)      # longer than one pass with others running
    with eng.Engine(preset="tiny-test", seed=77, max_batch=8, max_seqs=8, start_scheduler=True) as e:
        solo = [e.generate_ids(p, eng.greedy(24, ignore_eos=True)).token_ids for p in prompts]
        before = e.stats()
        out = [None] * len(prompts)

        def run(i):
            out[i] = e.generate_ids(prompts[i], eng.greedy(24, ignore_eos=True))
        th = [threading.Thread(target=run, args=(i,)) for i in range(len(prompts))]
        [t.start() for t in th]
        [t.join() for t in th]
        st = e.stats()
        for i in range(len(prompts)):
            assert out[i].n_generated == 24 and out[i].token_ids[0] == solo[i][0], i
            assert (out[i].token_ids == solo[i]).mean() > 0.7, i
        assert st["kv_pages_used"] == 0 and st["active_seqs"] == 0 and st["requests_completed"] - before["requests_completed"] == len(prompts)
        assert st["preemptions"] - before["preemptions"] == sum(r.n_preempted for r in out)
        # fewer prefill calls than requests: groups were formed
        assert st["sched_prefill_calls"] - before["sched_prefill_calls"] < len(prompts)
        # sampled requests go through the group path too (host sampler on the pass's logits): deterministic per seed
        sp = eng.ollama_default_sampling(seed=5, max_new_tokens=12)
        a = [None] * 4

        def run_s(i):
            a[i] = e.generate_ids(prompts[i], sp).token_ids
        th = [threading.Thread(target=run_s, args=(i,)) for i in range(4)]
        [t.start() for t in th]
        [t.join() for t in th]
        ref = [e.generate_ids(prompts[i], sp).token_ids for i in range(4)]
        assert all(a[i][0] == ref[i][0] for i in range(4))
