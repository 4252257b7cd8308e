"""Parity of what bench.py measures: the FULL 32-layer models at context 4096 / 8192 on the kernels that actually run
there — decode_mega_kernel (18 KV splits x 8 kv heads, 128+ pages), the per-op path, the batched tensor-core step
(attn_decode_tc_kernel + wgmma projections) at B = 2, 3, 8, 16 with mixed lengths — against the CPU oracle.

How a 4096-deep cache gets there without a 4096-token CPU prefill: both sides fill the sequence's K/V cache with the
oracle's synthetic pattern (oracle/llama_oracle.c oc_seq_fake_fill; engine: cl_seq_fake_fill -> the same integer
expression on the device, values n/128 exact in bf16), then >= 8 decode steps run teacher-forced on both sides and
the logits are compared step by step.  The long prefill itself is checked separately against the oracle's layer-major
prefill (oc_prefill_block): last-position logits AND the cached K/V of the last layer at EVERY position.

Tolerance (DESIGN.md §2): max |dlogit| <= 0.05 + 0.03*sqrt(L) — 0.22 for 32 layers, 0.11 for 4; SURVEY.md §8(c) asked for
0.125, which the bf16 rounding-point cascade does not allow at depth 32 (observed values are printed; run with -s).
Greedy ids: identical unless the ORACLE's own top-2 margin is below that tolerance.
"""
import os
import time

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu
MAXLEN = 8192 + 64
N_STEPS = 8


def tol_for(n_layers):
    return 0.05 + 0.03 * float(np.sqrt(n_layers))


class _Cache:
    """module-level lazily built oracle models / engines (a 32-layer model is 16 GB on both sides)"""
    models, engines, refs = {}, {}, {}

    @classmethod
    def model(cls, key, cfg, seed):
        if key not in cls.models:
            t0 = time.time()
            cls.models[key] = oc.Model(cfg, seed=seed)
            print(f"[oracle] {key}: built in {time.time() - t0:.1f}s with {oc.num_threads()} threads")
        return cls.models[key]

    @classmethod
    def engine(cls, key, cfg, seed, env=None, **kw):
        if key not in cls.engines:
            old = {k: os.environ.get(k) for k in (env or {})}
            os.environ.update(env or {})
            try:
                cls.engines[key] = eng.Engine(model=cfg, seed=seed, **kw)
            finally:
                for k, v in old.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        return cls.engines[key]

    @classmethod
    def drop(cls, prefix):
        for d in (cls.engines, cls.models, cls.refs):
            for k in [k for k in d if str(k[0] if isinstance(k, tuple) else k).startswith(prefix)]:
                v = d.pop(k)
                if hasattr(v, "close"):
                    v.close()


def _cfg(preset, n_layers=None, max_seq_len=MAXLEN):
    cfg = dict(oc.PRESETS[preset])
    if n_layers:
        cfg["n_layers"] = n_layers
    cfg["max_seq_len"] = max_seq_len
    return cfg


def _oracle_steps(m, lens, first_toks, n_steps):
    """Teacher-forced oracle run: per sequence b a cache of lens[b] synthetic tokens, then n_steps greedy tokens.
    Returns toks[step][b] (the inputs of every step) and logits[step][b]."""
    seqs = []
    for n in lens:
        so = m.new_seq(n + n_steps + 8)
        so.fake_fill(n)
        seqs.append(so)
    toks = [list(first_toks)]
    logits = []
    for _ in range(n_steps):
        row = [so.forward([t]) for so, t in zip(seqs, toks[-1])]
        logits.append(row)
        toks.append([int(lo.argmax()) for lo in row])
    for so in seqs:
        so.close()
    return toks, logits


def _compare_steps(name, e, seqs, toks, ref_logits, tol, batched):
    """Feed the oracle's tokens to the engine; every step's logits within tol, argmax identical unless near-tie."""
    worst, mism = 0.0, 0
    for step, ref_row in enumerate(ref_logits):
        if batched:
            lg, am = e.decode_step_batch(seqs, toks[step])
        else:
            l1, a1 = e.decode_step(seqs[0], toks[step][0])
            lg, am = l1[None, :], np.array([a1])
        for b, lo in enumerate(ref_row):
            err = float(np.abs(lg[b] - lo).max())
            assert np.isfinite(lg[b]).all(), f"{name}: non-finite logits (step {step}, seq {b})"
            worst = max(worst, err)
            assert err < tol, f"{name}: step {step} seq {b}: max |dlogit| {err:.4f} >= {tol:.3f}"
            want = int(lo.argmax())
            if int(am[b]) != want:
                top2 = np.sort(lo)[-2:]
                assert top2[1] - top2[0] < tol, f"{name}: step {step} seq {b}: greedy id differs at margin {top2[1] - top2[0]:.3f}"
                mism += 1
            assert int(lg[b].argmax()) == int(am[b])     # device argmax == argmax of the logits it returned
    return worst, mism


def _run_fake_filled(name, e, m, lens, n_layers, batched, ref_key=None, n_steps=None):
    n_steps = n_steps or N_STEPS
    tol = tol_for(n_layers)
    first = [17 + 101 * b for b in range(len(lens))]
    key = ref_key or (name.split("/")[0] + ":" + name,)
    if key not in _Cache.refs:
        _Cache.refs[key] = _oracle_steps(m, lens, first, n_steps)
    toks, ref = _Cache.refs[key]
    seqs = []
    for n in lens:
        s = e.seq_create()
        e.seq_fake_fill(s, n)
        seqs.append(s)
    try:
        worst, mism = _compare_steps(name, e, seqs, toks, ref, tol, batched)
    finally:
        for s in seqs:
            e.seq_free(s)
    print(f"{name}: lens {lens}: max |dlogit| {worst:.4f} (tolerance {tol:.3f}), near-tie id mismatches {mism} over {n_steps} steps")
    return worst


# ---- full 32-layer Llama-3-8B, single sequence: the benchmarked configuration --------------------------------------
@pytest.mark.parametrize("ctx", [4096, 8192])
@pytest.mark.parametrize("path", ["mega", "perop"])
def test_llama3_8b_full_b1_long_context(path, ctx):
    """bench.py's configuration: 32 layers, ctx 4096 (and 8192), batch 1 — decode_mega_kernel (CL_MEGA=1, the default)
    and the per-op kernel path (CL_MEGA=0).  The 8 steps start 4 tokens below the boundary, so they cross a page
    boundary, allocate a fresh page and change the pages-per-split count."""
    cfg = _cfg("llama3-8b")
    m = _Cache.model("l3", cfg, 1234)
    e = _Cache.engine(f"l3-{path}", cfg, 1234, env={"CL_MEGA": "1" if path == "mega" else "0"},
                      max_batch=16 if path == "mega" else 1, max_seqs=16 if path == "mega" else 2)
    _run_fake_filled(f"llama3-8b/32L/B1/{path}/ctx{ctx}", e, m, [ctx - 4], 32, batched=False, ref_key=("l3-b1", ctx))


def test_llama3_8b_full_greedy_256_steps():
    """SURVEY.md §8(c): 256 free-running greedy steps on the full model (device-side loop, persistent kernel) after a
    32-token wgmma prefill.  The oracle follows the ENGINE's tokens; at every step the engine's id must be the oracle's
    argmax, or a documented near-tie: the oracle's logit of the engine's id within the logit tolerance of its top logit."""
    cfg = _cfg("llama3-8b")
    m = _Cache.model("l3", cfg, 1234)
    e = _Cache.engine("l3-mega", cfg, 1234, env={"CL_MEGA": "1"}, max_batch=16, max_seqs=16)
    tol = tol_for(32)
    prompt = np.array([(i * 7919 + 13) % cfg["vocab_size"] for i in range(32)], np.int32)
    s = e.seq_create()
    lg = e.prefill(s, prompt)
    so = m.new_seq(32 + 256 + 8)
    lo = so.prefill_block(prompt)
    assert float(np.abs(lg - lo).max()) < tol
    first = int(lg.argmax())
    ids, _ = e.decode_greedy(s, first, 256)
    ids2 = None
    e.seq_free(s)
    # determinism: the same 256 ids again
    s = e.seq_create()
    assert int(e.prefill(s, prompt).argmax()) == first
    ids2, _ = e.decode_greedy(s, first, 256)
    e.seq_free(s)
    np.testing.assert_array_equal(ids, ids2)
    chain = [first] + [int(x) for x in ids]
    exact, worst_gap = 0, 0.0
    for i in range(257):                               # the prefill's token + 256 decoded ones
        gap = float(lo.max() - lo[chain[i]])           # oracle's view of the token the engine chose
        if int(lo.argmax()) == chain[i]:
            exact += 1
        else:
            worst_gap = max(worst_gap, gap)
            assert gap < tol, f"step {i}: engine id {chain[i]} is {gap:.3f} below the oracle's top logit (tolerance {tol:.3f})"
        if i < 256:
            lo = so.forward([chain[i]])
    so.close()
    print(f"llama3-8b full, 256 free-running greedy steps: {exact}/257 ids = oracle argmax, the rest near-ties "
          f"(largest oracle gap {worst_gap:.4f} < {tol:.3f}); run-to-run bit-identical")
    assert exact >= 160


def test_llama3_8b_full_batched_b8_long_context():
    """The path the box bench runs: B = 8 on the batched step (wgmma projections + attn_decode_tc_kernel), 32 layers,
    mixed lengths incl. 4096-deep, page-boundary (31, 32, 4093 -> crosses 4096) and empty sequences."""
    cfg = _cfg("llama3-8b")
    m = _Cache.model("l3", cfg, 1234)
    e = _Cache.engine("l3-mega", cfg, 1234, env={"CL_MEGA": "1"}, max_batch=16, max_seqs=16)
    _run_fake_filled("llama3-8b/32L/B8/batched", e, m, [4096, 1023, 31, 0, 2048, 4093, 777, 32], 32, batched=True)
    _Cache.drop("l3")          # 32 GB of host + device memory back before the next full-size model


# ---- 4 layers at full width: more batch shapes for the same oracle budget ----------------------------------------
@pytest.mark.parametrize("B", [2, 3, 16])
def test_llama3_8b_layers_batched_long_context(B):
    """B = 2, 3 and 16 (tensor-core path: KV splits 9, 6 and 1 per sequence) at
    Llama-3-8B layer shapes, contexts up to 8188 tokens, 1-token and page-boundary sequences."""
    cfg = _cfg("llama3-8b", n_layers=4)
    m = _Cache.model("l3x4", cfg, 99)
    e = _Cache.engine("l3x4", cfg, 99, max_batch=16, max_seqs=16)
    lens = [8188, 4096, 4095, 31, 32, 33, 0, 1000, 2047, 2048, 6000, 100, 64, 500, 3000, 7][:B]
    _run_fake_filled(f"llama3-8b/4L/B{B}/batched", e, m, lens, 4, batched=True, ref_key=("l3x4-ref", B))
    if B == 16:
        _Cache.drop("l3x4")


@pytest.mark.parametrize("B", [40, 100])
def test_llama3_8b_layers_wide_batch(B):
    """Batched steps beyond 32 sequences: the projections switch to the 64- and 128-row token tile.  Short, mixed
    contexts (0 ... 600 tokens, page boundaries included) keep the CPU checker's share small."""
    cfg = _cfg("llama3-8b", n_layers=4)
    m = _Cache.model("l3x4w", cfg, 99)
    e = _Cache.engine("l3x4-wide", cfg, 99, max_batch=100, max_seqs=100)
    lens = [(i * 97 + 13) % 600 if i % 7 else (31, 32, 33, 0, 64, 95, 96)[(i // 7) % 7] for i in range(B)]
    _run_fake_filled(f"llama3-8b/4L/B{B}/batched-wide", e, m, lens, 4, batched=True, ref_key=("l3x4w-ref", B), n_steps=3)
    if B == 100:
        _Cache.drop("l3x4w")


# ---- Mistral-7B shapes at 8K (BASELINE.json configs[4]) ------------------------------------------------------------
def test_mistral_7b_full_8k_context():
    cfg = _cfg("mistral-7b", max_seq_len=8192 + 256)
    m = _Cache.model("mi", cfg, 4321)
    e = _Cache.engine("mi", cfg, 4321, max_batch=4, max_seqs=4)
    _run_fake_filled("mistral-7b/32L/B1/mega/ctx8192", e, m, [8188], 32, batched=False)
    _run_fake_filled("mistral-7b/32L/B3/batched", e, m, [8190, 4097, 100], 32, batched=True)
    _Cache.drop("mi")


# ---- the 4096-token prefill, checked at every position ---------------------------------------------------------------
@pytest.mark.parametrize("calls", ["4096+300", "4396"])
def test_prefill_4096_tokens_matches_oracle_at_every_position(calls):
    """A 4096-token prompt (one tensor-core chunk) plus a 300-token continuation (attention over cached pages + the new
    chunk) at Llama-3-8B width, 2 layers, against the oracle's layer-major prefill: last-position logits, and the cached
    K/V of layer 1 at EVERY position — they depend on layer 0's attention output at that position, so the whole causal
    attention matrix is covered.  Then 4 teacher-forced decode steps on top.  calls = "4396": the same 4396 tokens in
    one prefill call, which the engine splits into a 4096-row and a 300-row pass."""
    cfg = _cfg("llama3-8b", n_layers=2, max_seq_len=4096 + 512)
    m = _Cache.model("pf", cfg, 7)
    T0, T1 = 4096, 300
    ids = np.array([(i * 7919 + 13) % cfg["vocab_size"] for i in range(T0 + T1)], np.int32)
    tol = tol_for(2)
    with eng.Engine(model=cfg, seed=7, max_batch=1) as e:
        s = e.seq_create()
        so = m.new_seq(T0 + T1 + 16)
        t0 = time.time()
        lo = so.prefill_block(ids[:T0])
        print(f"[oracle] 4096-token prefill, 2 layers: {time.time() - t0:.1f}s")
        e0 = None
        if calls == "4096+300":
            lg = e.prefill(s, ids[:T0])
            e0 = float(np.abs(lg - lo).max())
            assert e0 < tol, e0
        lo = so.prefill_block(ids[T0:])
        lg = e.prefill(s, ids[T0:] if calls == "4096+300" else ids)
        e1 = float(np.abs(lg - lo).max())
        assert e1 < tol, e1
        stats = {}
        for which, nm in ((0, "K"), (1, "V")):
            ref = so.kv(1, which, 0, T0 + T1)
            got = e.debug_kv(s, 1, which, 0, T0 + T1)
            d = np.abs(got - ref)
            scale = float(np.abs(ref).max())
            per_pos = d.max(axis=1)
            # bf16 cache values: a last-bit difference in fp32 flips one rounding = 2^-8 relative; allow 2^-6 of the range
            assert per_pos.max() <= scale / 64, f"{nm}: position {int(per_pos.argmax())} differs by {per_pos.max():.4g} (range {scale:.3g})"
            stats[nm] = {"max": float(per_pos.max()), "mean": float(d.mean()), "range": scale,
                         "frac_elems_differ": float((d > 0).mean())}
        errs = []
        tok = int(lo.argmax())
        for _ in range(4):
            lo = so.forward([tok])
            lg, am = e.decode_step(s, tok)
            errs.append(float(np.abs(lg - lo).max()))
            tok = int(lo.argmax())
        assert max(errs) < tol
        print(f"prefill {calls} @ llama3-8b width x 2 layers: logits err {e0} / {e1:.4f}, decode after {max(errs):.4f} "
              f"(tolerance {tol:.3f}); layer-1 cache at all {T0 + T1} positions: {stats}")
    so.close()
    _Cache.drop("pf")
