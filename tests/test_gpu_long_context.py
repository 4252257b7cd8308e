"""Long context (cl_engine_config.context_length up to 131072) on the GPU.

1. The split-KV wgmma prefill attention (variant 2 of attn_prefill_tc.cu) against float64 at pos0 + T up to 131072, forced
   and planned split counts, GQA 4:1 and 8:1; NaN-filled outputs; two launches bit-identical (the op checks it: the
   counters re-arm); nsplit 1 equal to variant 1 bit for bit where variant 1 runs; variant -1 = the engine's rule.
2. The decode attention kernels (tensor-core shapes and the CUDA-core kernel) and the multi-row verify kernel behind
   contexts past 32768, with the bounds of test_gpu_step_kernels.
3. Whole model, 2-layer Llama-3.1-8B shape (llama3 RoPE scaling) with context_length 131072 behind cl_seq_fake_fill on
   both sides: a 300-row tile pass and a 40-row split-K pass past 100K run the split-KV kernel, a verify pass (k = 7)
   runs the multi-row verify kernel, and all match the oracle; teacher-forced steps on the persistent kernel, the per-op
   path and the batched step (B = 2); a context shift at the 131072 window, then steps; the head_dim-64 Llama-3.2-1B
   shape at 65536 (mma.sync prefill); the 32-layer model behind a fake fill past 32768 (FULL_FILL: its oracle's fp32
   cache takes 256 KiB per token, 8.5 GiB here next to 32 GB of fp32 weights in host memory).
4. Below 32768 tokens an engine with context_length 131072 computes the bits of an engine with the default window.
5. The scheduler: a 40K-token prompt through cl_generate_ids equals a token-level replay; a prompt larger than the pool
   fails with CL_ERR_OOM and leaks no page.

float64 references of the kernels are computed with torch on the device (numpy at 131072 keys x 4096 rows is too slow) on
the rows test_tile_pass_rows uses: the first and last row of every 128-row tile plus 64 seeded rows.
"""
import numpy as np
import pytest
import torch

from crowdllama_b200 import engine as eng
from oracle import oracle as oc
from test_gpu_longctx import _compare_steps, _oracle_steps
from test_gpu_step_kernels import DECODE_C, PREFILL_C, TC, attn64, attn_inputs, attn_ratio, bf16, check_decode, decode_inputs, f32

pytestmark = pytest.mark.gpu
LONG_FROM = 32768
N_TOKS = [10241, 32769, 65536, 131072]
TS = [1, 16, 17, 64, 300, 1024, 4096]
GQA = {"4:1": dict(n_heads=32, n_kv=8, hd=128), "8:1": dict(n_heads=32, n_kv=4, hd=128)}


def sample_rows(T, seed):
    rows = {r for t0 in range(0, T, 128) for r in (t0, min(t0 + 127, T - 1))}
    rows |= set(np.random.default_rng(seed).integers(0, T, 64).tolist())
    return np.array(sorted(rows))


def ref_rows(q, k, v, pos, n_heads, n_kv, hd):
    """float64 attention of query rows q [R][H*D] (bf16 bits) at positions pos over k, v [n][n_kv][D] (bf16 bits), on the
    device.  Returns (out, sum_t p_t |v_t|) as numpy [R][H*D]."""
    dev = torch.device("cuda")
    rep = n_heads // n_kv
    to64 = lambda a: torch.from_numpy(f32(a)).to(dev, torch.float64)
    qd = to64(q).reshape(len(pos), n_kv, rep, hd)
    pos_t = torch.as_tensor(pos, device=dev)
    n = int(pos.max()) + 1
    out = torch.empty((len(pos), n_kv, rep, hd), dtype=torch.float64, device=dev)
    pv = torch.empty_like(out)
    keys = torch.arange(n, device=dev)
    mask = keys[None, :] <= pos_t[:, None]
    for g in range(n_kv):
        kg = to64(k[:n, g])
        vg = to64(v[:n, g])
        s = torch.einsum("rhd,nd->rhn", qd[:, g], kg) / np.sqrt(hd)
        s = s.masked_fill(~mask[:, None, :], float("-inf"))
        p = torch.softmax(s, dim=-1)
        out[:, g] = torch.einsum("rhn,nd->rhd", p, vg)
        pv[:, g] = torch.einsum("rhn,nd->rhd", p, vg.abs())
        del kg, vg, s, p
    return out.reshape(len(pos), -1).cpu().numpy(), pv.reshape(len(pos), -1).cpu().numpy()


_inputs = {}


def long_inputs(n_tok, gqa):
    """q for the last 4096 positions of n_tok, k, v [n_tok][n_kv][128]; the key at each query's position boosted as in
    test_gpu_step_kernels.attn_inputs"""
    key = (n_tok, gqa)
    if key not in _inputs:
        sh = GQA[gqa]
        n_kv, hd, rep = sh["n_kv"], sh["hd"], sh["n_heads"] // sh["n_kv"]
        rng = np.random.default_rng(n_tok + rep)
        R = min(4096, n_tok)
        qpos = np.arange(n_tok - R, n_tok)
        q = f32(bf16(rng.standard_normal((R, n_kv, rep, hd)).astype(np.float32)))
        k = (rng.standard_normal((n_tok, n_kv, hd), dtype=np.float32) * 2.0)
        v = rng.standard_normal((n_tok, n_kv, hd), dtype=np.float32)
        q0 = q[:, :, 0].astype(np.float64)
        k[qpos] += (10.0 * np.sqrt(hd) * q0 / (q0 ** 2).sum(-1, keepdims=True)).astype(np.float32)
        _inputs[key] = (bf16(q.reshape(R, -1)), bf16(k), bf16(v))
    return _inputs[key]


def run_long(q, k, v, pos0, sh, variant=2, nsplit=0):
    out, ns, kind, _ = eng.op_attn_prefill_long(q, k, v, pos0, sh["n_heads"], sh["n_kv"], sh["hd"], variant=variant, nsplit=nsplit)
    assert not np.isnan(out).any(), f"variant {variant} nsplit {nsplit}: an output was not written"
    return out, ns, kind


def plan_max(pos0, T):
    return (pos0 + min(128, T) - 1) // 64 + 1                  # the first tile's KV blocks: the most splits the op takes


def most_splits(pos0, T, n_heads, budget=8 << 30):
    """the most splits the op takes, limited to a partial workspace of `budget` bytes (131072 x 4096 at 2048 splits would
    need 139 GB)"""
    items = (T + 127) // 128 * n_heads
    return min(plan_max(pos0, T), max(1, budget // (items * 128 * 130 * 4)))


@pytest.mark.parametrize("gqa", list(GQA))
@pytest.mark.parametrize("n_tok", N_TOKS)
@pytest.mark.parametrize("T", TS)
def test_split_kv_prefill_vs_float64(n_tok, T, gqa):
    sh = GQA[gqa]
    q_all, k, v = long_inputs(n_tok, gqa)
    q = q_all[-T:]
    pos0 = n_tok - T
    rows = sample_rows(T, n_tok + T) if T > 192 else np.arange(T)
    ref, pv = ref_rows(q[rows], k, v, pos0 + rows, **sh)
    worst, used = 0.0, set()
    outs = {}
    for force in (1, 2, 7, most_splits(pos0, T, sh["n_heads"]), 0):
        out, ns, kind = run_long(q, k, v, pos0, sh, nsplit=force)
        assert kind == "long"
        assert ns == (min(force, plan_max(pos0, T)) if force else eng_plan(pos0, T, sh["n_heads"]))
        used.add(ns)
        r = attn_ratio(out[rows], ref, pv, PREFILL_C)
        worst = max(worst, r)
        assert r <= 1.0, f"n_tok {n_tok} T {T} {gqa} nsplit {ns}: max err/tol {r:.3g}"
        outs[force] = out
    print(f"[long prefill] n_tok {n_tok} T {T} {gqa}: splits {sorted(used)} max err/tol {worst:.3g}")
    # the engine's rule: the split-KV kernel past 32768 tokens, the old choice at and below it
    auto, _, kind = run_long(q, k, v, pos0, sh, variant=-1)
    if n_tok > LONG_FROM and T <= 16 and gqa == "4:1":
        assert kind == "verify"                                 # the multi-row split-KV kernel of verify passes (4:1 only)
        r = attn_ratio(auto[rows], ref, pv, PREFILL_C)
        print(f"[long prefill] n_tok {n_tok} T {T} {gqa}: variant -1 (verify kernel) max err/tol {r:.3g}")
        assert r <= 1.0
    elif n_tok > LONG_FROM:
        assert kind == "long"
        np.testing.assert_array_equal(auto, outs[0])
    else:
        assert kind == "mma"                                    # 10241: past variant 1's block-table limit
        mma, _, _ = run_long(q, k, v, pos0, sh, variant=0)
        np.testing.assert_array_equal(auto, mma)


def eng_plan(pos0, T, n_heads):
    ns, part = C_int(), C_int64()
    assert eng.lib().cl_attn_prefill_long_plan(pos0, T, n_heads, torch.cuda.get_device_properties(0).multi_processor_count, 0,
                                               eng.C.byref(ns), eng.C.byref(part)) == eng.CL_OK
    return ns.value


C_int, C_int64 = eng.C.c_int32, eng.C.c_int64


@pytest.mark.parametrize("pos0,T", [(0, 1), (0, 300), (105, 150), (4096, 300), (6144, 4096), (10240 - 17, 17), (10240 - 1024, 1024)])
@pytest.mark.parametrize("gqa", list(GQA))
def test_one_split_is_variant_1_bit_for_bit(pos0, T, gqa):
    """nsplit = 1 at pos0 + T <= 10240 reproduces variant 1: the template left its arithmetic alone"""
    sh = GQA[gqa]
    q_all, k, v = long_inputs(10241, gqa)
    q, kk, vv = q_all[-T:], k[:pos0 + T], v[:pos0 + T]
    one, ns, _ = run_long(q, kk, vv, pos0, sh, nsplit=1)
    assert ns == 1
    v1, _, kind = run_long(q, kk, vv, pos0, sh, variant=1)
    assert kind == "wgmma"
    np.testing.assert_array_equal(one, v1)
    auto, _, kind = run_long(q, kk, vv, pos0, sh, variant=-1)
    assert kind == "wgmma"
    np.testing.assert_array_equal(auto, v1)


def test_engine_rule_at_the_boundary():
    """variant -1 at pos0 + T = 32768 keeps the mma.sync kernel; at 32769 up to 16 rows run the multi-row verify kernel and
    17 rows the split-KV kernel; head_dim 64 and page 64 keep mma.sync past it"""
    sh = GQA["4:1"]
    q_all, k, v = long_inputs(32769, "4:1")
    for n_tok, T, want in ((32768, 16, "mma"), (32768, 17, "mma"), (32769, 16, "verify"), (32769, 17, "long")):
        _, _, kind = run_long(q_all[-T:], k[:n_tok], v[:n_tok], n_tok - T, sh, variant=-1)
        assert kind == want, (n_tok, T)
    q64 = bf16(f32(q_all[-16:]).reshape(16, 32, 128)[:, :, :64].reshape(16, -1))
    k64, v64 = k[:, :, :64].copy(), v[:, :, :64].copy()
    out, _, _, _ = eng.op_attn_prefill_long(q64, k64, v64, 32769 - 16, 32, 8, 64, variant=-1)
    ref, pv = ref_rows(q64, k64, v64, 32769 - 16 + np.arange(16), 32, 8, 64)
    assert attn_ratio(out, ref, pv, PREFILL_C) <= 1.0
    _, _, kind, _ = eng.op_attn_prefill_long(q64, k64, v64, 32769 - 16, 32, 8, 64, variant=-1)
    assert kind == "mma"
    _, _, kind, _ = eng.op_attn_prefill_long(q_all[-16:], k, v, 32769 - 16, 32, 8, 128, page_size=64, variant=-1)
    assert kind == "mma"


# ---- decode and verify kernels behind long contexts ----------------------------------------------------------------------
@pytest.mark.parametrize("ctx", [32769, 65536, 131072])
@pytest.mark.parametrize("B", [1, 2, 4])
def test_decode_kernels_long_context(ctx, B):
    lens = [ctx - 977 * b for b in range(B)]
    q, kc, vc = decode_inputs(ctx + B, lens, **TC)
    refs = [attn64(q[b:b + 1], f32(kc[o:o + L]), f32(vc[o:o + L]), [L - 1], **TC)
            for b, (o, L) in enumerate(zip(np.cumsum([0] + lens[:-1]), lens))]
    for small in (0, 1):
        check_decode(f"tc ctx {ctx} B {B} small {small}", q, kc, vc, lens, **TC, refs=refs, variant=1, tc_small=small)
    sh = dict(n_heads=32, n_kv=8, hd=128)
    _, _, small = check_decode(f"cuda-core ctx {ctx} B {B}", q, kc, vc, lens, **sh, page=16, refs=refs, variant=-1)
    assert small == -1


@pytest.mark.parametrize("ctx", [131072 - 16])
def test_verify_kernel_behind_131072(ctx):
    rng = np.random.default_rng(5)
    rows = [16, 7, 1]
    lens = [ctx, ctx - 5000, 40000]
    qs, ks, vs = [], [], []
    for L, R in zip(lens, rows):
        q, k, v = attn_inputs(rng, L + R, L + np.arange(R), **TC)
        qs.append(q); ks.append(k); vs.append(v)
    q = np.concatenate(qs)
    out, ns = eng.op_attn_verify(q, np.concatenate(ks), np.concatenate(vs), lens, rows, 32, 8, 128)
    r0 = 0
    for b, (L, R) in enumerate(zip(lens, rows)):
        ref, pv = ref_rows(qs[b], ks[b], vs[b], L + np.arange(R), **TC)
        worst = attn_ratio(f32(out[r0:r0 + R]), ref, pv, DECODE_C)
        print(f"[verify] len {L} rows {R}: nsplit {ns} max err/tol {worst:.3g}")
        assert worst <= 1.0
        r0 += R


# ---- whole model behind a fake fill --------------------------------------------------------------------------------------
TOL2 = 0.05 + 0.03 * np.sqrt(2)                                 # 0.092: the 2-layer bar of tests/test_gpu_longctx.py


def _cfg(preset, n_layers=2):
    cfg = dict(oc.PRESETS[preset])
    cfg["n_layers"] = n_layers
    return cfg


_models = {}


def oracle_model(cfg, seed, max_seq_len):
    key = (cfg["n_layers"], cfg["head_dim"], seed, max_seq_len)
    if key not in _models:
        for m in _models.values():
            m.close()
        _models.clear()
        _models[key] = oc.Model(dict(cfg, max_seq_len=max_seq_len), seed=seed)
    return _models[key]


def test_llama31_8b_split_k_verify_and_steps_at_131072():
    """behind 100000 fake-filled tokens: a 40-row split-K pass (split-KV prefill kernel), 8 steps on the persistent kernel,
    then a verify pass of 1 + 7 rows (multi-row verify kernel), every logits row against the oracle"""
    cfg = _cfg("llama3.1-8b")
    m = oracle_model(cfg, 7, 131072)
    fill = 100000
    rng = np.random.default_rng(3)
    split = rng.integers(0, cfg["vocab_size"], 40).tolist()
    drafts = rng.integers(0, cfg["vocab_size"], 7).tolist()
    so = m.new_seq(131072)
    so.fake_fill(fill)
    ref_split = so.forward(split)
    with eng.Engine(model=cfg, seed=7, max_batch=2, context_length=131072) as e:
        assert e.cfg["max_seq_len"] == 131072
        s = e.seq_create()
        e.seq_fake_fill(s, fill)
        lg = e.prefill(s, np.array(split, np.int32))
        info = e.debug_pass_info()
        assert (info["path"], info["attn"]) == ("split-k", "long"), info
        err = float(np.abs(lg - ref_split).max())
        print(f"[llama3.1-8b x2 @131072] split-K pass 40 rows behind {fill}: max |dlogit| {err:.4f}")
        assert err < TOL2
        tok = int(ref_split.argmax())
        worst = 0.0
        for step in range(8):
            ref = so.forward([tok])
            lg, am = e.decode_step(s, tok)
            err = float(np.abs(lg - ref).max())
            worst = max(worst, err)
            assert err < TOL2, f"step {step}: {err:.4f}"
            tok = int(ref.argmax())
        print(f"[llama3.1-8b x2 @131072] 8 persistent-kernel steps: max |dlogit| {worst:.4f}")
        ref_v = so.forward([tok] + drafts, all_logits=True)
        _, lg_v = e.decode_verify(s, tok, drafts, want_logits=True)
        info = e.debug_pass_info()
        assert (info["path"], info["attn"]) == ("split-k", "verify"), info
        assert info["segs"][0][3] == fill + 40 + 8 and info["T"] == 8
        err = float(np.abs(lg_v - ref_v).max())
        print(f"[llama3.1-8b x2 @131072] verify pass k = 7 at {fill + 48}: max |dlogit| {err:.4f}")
        assert err < TOL2
    so.close()


@pytest.mark.parametrize("path", ["per-op", "batched"])
def test_llama31_8b_steps_at_131072(path, monkeypatch):
    """8 teacher-forced steps at the 131072 window on the per-op kernels (CL_MEGA=0) and on the batched step at B = 2"""
    cfg = _cfg("llama3.1-8b")
    m = oracle_model(cfg, 7, 131072)
    lens = [131072 - 16] if path == "per-op" else [131072 - 16, 100003]
    toks, logits = _oracle_steps(m, lens, [11, 12][:len(lens)], 8)
    if path == "per-op":
        monkeypatch.setenv("CL_MEGA", "0")
    with eng.Engine(model=cfg, seed=7, max_batch=2, context_length=131072) as e:
        seqs = [e.seq_create() for _ in lens]
        for s, n in zip(seqs, lens):
            e.seq_fake_fill(s, n)
        worst, mism = _compare_steps(f"{path} @131072", e, seqs, toks, logits, TOL2, batched=path == "batched")
        print(f"[llama3.1-8b x2 @131072] {path}: 8 steps, max |dlogit| {worst:.4f}, near-tie flips {mism}")


def test_llama31_8b_context_shift_at_131072():
    """a sequence at the 131072 window shifted as the scheduler would (num_keep 4, delta = 65504 tokens: 2047 pages
    re-rotated with rows of the 131072-row RoPE table), then 8 steps against the oracle shifted the same way"""
    from shift_util import oracle_shift
    cfg = _cfg("llama3.1-8b")
    m = oracle_model(cfg, 7, 131072)
    W, keep = 131072, 4
    n = W - 8
    delta = 32 * ((W - keep) // 64)
    so = m.new_seq(W)
    so.fake_fill(n)
    oracle_shift(so, keep, delta)
    with eng.Engine(model=cfg, seed=7, max_batch=2, context_length=W, context_shift=True, num_keep=keep) as e:
        s = e.seq_create()
        e.seq_fake_fill(s, n)
        e.seq_shift(s, keep, delta)
        tok, worst = 21, 0.0
        for step in range(8):
            ref = so.forward([tok])
            lg, _ = e.decode_step(s, tok)
            err = float(np.abs(lg - ref).max())
            worst = max(worst, err)
            assert err < TOL2, f"step {step}: {err:.4f}"
            tok = int(ref.argmax())
        print(f"[llama3.1-8b x2 @131072] shift of {delta} after {n} tokens, 8 steps: max |dlogit| {worst:.4f}")
    so.close()


FULL_FILL = 34000


def test_llama31_8b_full_depth_past_32768():
    """the 32-layer model behind FULL_FILL fake-filled tokens (past 32768; the oracle's fp32 cache costs 256 KiB per token
    at 32 layers, so this stays within the GPU machine's host memory next to the oracle's 32 GB of fp32 weights), 8 steps
    on the persistent kernel against the oracle within 0.05 + 0.03 sqrt(32) = 0.22"""
    cfg = _cfg("llama3.1-8b", n_layers=32)
    tol = 0.05 + 0.03 * np.sqrt(32)
    m = oracle_model(cfg, 5, FULL_FILL + 64)
    toks, logits = _oracle_steps(m, [FULL_FILL], [17], 8)
    with eng.Engine(model=cfg, seed=5, max_batch=1, context_length=65536) as e:
        s = e.seq_create()
        e.seq_fake_fill(s, FULL_FILL)
        worst, mism = _compare_steps("32 layers", e, [s], toks, logits, tol, batched=False)
        print(f"[llama3.1-8b x32 @{FULL_FILL}] 8 persistent-kernel steps: max |dlogit| {worst:.4f}, near-tie flips {mism}")
    for mm in _models.values():
        mm.close()
    _models.clear()


def test_llama32_1b_two_layers_at_65536():
    cfg = _cfg("llama3.2-1b")
    m = oc.Model(dict(cfg, max_seq_len=65536), seed=9)
    fill = 65000
    chunk = np.random.default_rng(4).integers(0, cfg["vocab_size"], 300).tolist()
    so = m.new_seq(65536)
    so.fake_fill(fill)
    ref = so.forward(chunk)
    with eng.Engine(model=cfg, seed=9, max_batch=2, context_length=65536) as e:
        s = e.seq_create()
        e.seq_fake_fill(s, fill)
        lg = e.prefill(s, np.array(chunk, np.int32))
        assert e.debug_pass_info()["attn"] == "mma"
        err = float(np.abs(lg - ref).max())
        print(f"[llama3.2-1b x2 @65536] tile pass 300 rows behind {fill}: max |dlogit| {err:.4f}")
        assert err < TOL2
    so.close()
    m.close()


def test_nothing_changes_below_the_boundary():
    """the same prompt ending at <= 32768 tokens: bit-identical logits and K/V with context_length 131072 and without"""
    cfg = _cfg("llama3.1-8b")
    ids = np.random.default_rng(8).integers(0, cfg["vocab_size"], 2000).astype(np.int32)
    got = []
    for ctx in (0, 131072):
        with eng.Engine(model=cfg, seed=11, max_batch=2, context_length=ctx) as e:
            s = e.seq_create()
            e.seq_fake_fill(s, 30000)
            lg = e.prefill(s, ids)
            kv = [e.debug_kv(s, 1, which, 30000, 2000) for which in (0, 1)]
            got.append((lg, kv))
    np.testing.assert_array_equal(got[0][0], got[1][0])
    for which in (0, 1):
        np.testing.assert_array_equal(got[0][1][which], got[1][1][which])


def test_scheduler_long_prompt_and_oversized_prompt():
    cfg = _cfg("llama3.1-8b")
    ids = np.random.default_rng(12).integers(0, cfg["vocab_size"], 40000).astype(np.int32)
    with eng.Engine(model=cfg, seed=13, max_batch=2, context_length=131072, start_scheduler=True) as e:
        r = e.generate_ids(ids, eng.greedy(16, ignore_eos=True))
        got = [int(t) for t in r.token_ids]
        s = e.seq_create()
        lg = e.prefill(s, ids)
        want = [int(lg.argmax())]
        for _ in range(15):
            lg, am = e.decode_step(s, want[-1])
            want.append(int(am))
        e.seq_free(s)
        assert got == want
    pool_tokens = 50000
    kv_per_token = 2 * cfg["n_layers"] * cfg["n_kv_heads"] * cfg["head_dim"] * 2
    with eng.Engine(model=cfg, seed=13, max_batch=2, context_length=131072, start_scheduler=True,
                    kv_pool_bytes=pool_tokens * kv_per_token) as e:
        assert e.stats()["kv_pages_used"] == 0
        big = np.random.default_rng(14).integers(0, cfg["vocab_size"], 60000).astype(np.int32)
        with pytest.raises(eng.EngineError) as ei:
            e.generate_ids(big, eng.greedy(4, ignore_eos=True))
        assert ei.value.status == eng.CL_ERR_OOM
        assert e.stats()["kv_pages_used"] == 0                  # no page leaked
        r = e.generate_ids(ids[:1000], eng.greedy(4, ignore_eos=True))    # the engine still serves
        assert r.n_generated == 4


def test_llama31_8b_tile_pass_at_131072():
    """a 300-row tile-path pass behind 100000 fake-filled tokens runs the split-KV prefill kernel; its last-row logits
    against the oracle's token step.  (The oracle needs minutes of CPU for these rows behind 100K; a 1024-row tile runs
    the same kernel with one split, checked against float64 at 131072 x 1024 in test_split_kv_prefill_vs_float64.)"""
    cfg = _cfg("llama3.1-8b")
    m = oracle_model(cfg, 7, 131072)
    fill = 100000
    chunk = np.random.default_rng(6).integers(0, cfg["vocab_size"], 300).astype(np.int32)
    so = m.new_seq(131072)
    so.fake_fill(fill)
    ref = so.forward(chunk)
    with eng.Engine(model=cfg, seed=7, max_batch=2, context_length=131072) as e:
        s = e.seq_create()
        e.seq_fake_fill(s, fill)
        lg = e.prefill(s, chunk)
        info = e.debug_pass_info()
        assert (info["path"], info["attn"], info["T"]) == ("tile", "long", 300), info
        err = float(np.abs(lg - ref).max())
        print(f"[llama3.1-8b x2 @131072] tile pass 300 rows behind {fill}: max |dlogit| {err:.4f}")
        assert err < TOL2
    so.close()
    for mm in _models.values():
        mm.close()
    _models.clear()
