"""Prefill path parity: tensor-core GEMM, causal paged attention, and the engine's chunked prefill vs the oracle."""
import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

pytestmark = pytest.mark.gpu


def _rand_bf16(rng, shape, scale=1.0):
    return oc.np_bf16_from_f32((rng.standard_normal(shape) * scale).astype(np.float32))


@pytest.mark.parametrize("t,n,k", [(16, 256, 128), (1, 128, 64), (33, 128, 64), (100, 384, 192), (300, 512, 256),
                                   (129, 320, 1024), (512, 6144, 4096), (64, 4096, 14336), (257, 1000, 4096)])
def test_gemm_tcgen05_matches_oracle(t, n, k):
    rng = np.random.default_rng(t + n + k)
    x = _rand_bf16(rng, (t, k))
    w = _rand_bf16(rng, (n, k), 0.05)
    got = eng.op_gemm_bf16(x, w)
    ref = oc.gemm(x, w)
    assert np.isfinite(got).all()          # the op pre-fills Y with NaNs: every element must be written
    tol = 2e-3 * float(np.sqrt((ref.astype(np.float64) ** 2).mean()))
    assert np.abs(got - ref).max() <= tol


@pytest.mark.parametrize("n_heads,n_kv,hd", [(4, 2, 64), (8, 2, 128), (2, 1, 64)])
@pytest.mark.parametrize("t", [1, 63, 64, 65, 200])
def test_attn_prefill_matches_oracle(n_heads, n_kv, hd, t):
    rng = np.random.default_rng(t * 3 + hd + n_heads)
    q = _rand_bf16(rng, (t, n_heads * hd))
    k = _rand_bf16(rng, (t, n_kv, hd))
    v = _rand_bf16(rng, (t, n_kv, hd))
    got = eng.op_attn_prefill(q, k, v, n_heads, n_kv, hd)
    qf, kf, vf = oc.np_f32_from_bf16(q), oc.np_f32_from_bf16(k), oc.np_f32_from_bf16(v)
    ref = np.stack([oc.attention(qf[i], kf[:i + 1], vf[:i + 1], n_heads, n_kv, hd) for i in range(t)])
    # P is rounded to bf16 before P.V on the tensor-core path: allow a bf16-sized band
    assert np.abs(got - ref).max() <= 2 ** -6 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("t,n_heads,n_kv", [(1, 4, 1), (127, 4, 1), (128, 8, 2), (129, 4, 4), (193, 4, 1), (255, 4, 1), (257, 8, 2), (640, 4, 1),
                                            (1000, 8, 2), (2049, 4, 1)])
def test_attn_prefill_kernels_head_dim_128(variant, t, n_heads, n_kv):
    """Both prefill attention kernels at head_dim 128 — variant 1 = wgmma (S and O in registers, K/V pages by 2-D TMA,
    V as an MN-major operand), variant 0 = the mma.sync kernel — against the oracle's per-position attention: ragged
    lengths around the 128-row item and 64-token KV block boundaries (127 / 128 / 129, 193 inside an item, 255 / 257, ...), reversed page order, GQA 1:1 ... 4:1.
    Score scale ~ N(0, 4): row maxima move between blocks and exercise the online-softmax rescale."""
    rng = np.random.default_rng(t * 5 + n_heads + n_kv)
    hd = 128
    q = _rand_bf16(rng, (t, n_heads * hd), 2.0)
    k = _rand_bf16(rng, (t, n_kv, hd), 2.0)
    v = _rand_bf16(rng, (t, n_kv, hd))
    got, _ = eng.op_attn_prefill_variant(q, k, v, n_heads, n_kv, hd, variant)
    assert np.isfinite(got).all()                  # the op pre-fills the output with NaNs: every row must be written
    qf, kf, vf = oc.np_f32_from_bf16(q), oc.np_f32_from_bf16(k), oc.np_f32_from_bf16(v)
    ref = np.stack([oc.attention(qf[i], kf[:i + 1], vf[:i + 1], n_heads, n_kv, hd) for i in range(t)])
    err = np.abs(got - ref)
    assert err.max() <= 2 ** -6 * max(1.0, np.abs(ref).max()), (int(err.argmax() // (n_heads * hd)), float(err.max()))


def _prompt(n, vocab, salt=0):
    return np.array([(i * 7919 + 13 + salt) % vocab for i in range(n)], np.int32)


@pytest.mark.parametrize("path", ["small", "tiles", "multi"])
@pytest.mark.parametrize("n_prompt", [16, 40, 97, 200])
def test_engine_chunked_prefill_matches_oracle(monkeypatch, n_prompt, path):
    """The tensor-core prefill paths against the oracle: "small" = short prompts (<= 256 tokens) on split-K projections
    (prefill_small, CL_PREFILL_SMALL_MAX=256); "tiles" = full tiles (the tiny model has head_dim 64: mma.sync attention);
    "multi" = the same tile pass entered through cl_prefill_batch with one prompt (batched LM head, and the device state
    it leaves behind must start decoding and a later prefill correctly)."""
    monkeypatch.setenv("CL_PREFILL_SMALL_MAX", "256" if path == "small" else "0")
    cfg = oc.PRESETS["tiny-test"]
    m = oc.Model(cfg, seed=1234)
    with eng.Engine(preset="tiny-test", seed=1234) as e:
        def fill(s, ids):
            return e.prefill_batch([s], [ids])[0] if path == "multi" else e.prefill(s, ids)
        p = _prompt(n_prompt, cfg["vocab_size"])
        so = m.new_seq()
        lo = so.forward(p)
        s = e.seq_create()
        lg = fill(s, p)                            # >= 16 tokens -> tensor-core path
        assert np.abs(lg - lo).max() < 0.125
        # decode continues from the prefix the prefill kernels wrote into the paged cache
        tok = int(lo.argmax())
        for _ in range(8):
            lo = so.forward([tok])
            lg, _ = e.decode_step(s, tok)
            assert np.abs(lg - lo).max() < 0.125
            tok = int(lo.argmax())
        # second prefill chunk appended to the same sequence (chunked prompt / multi-turn)
        p2 = _prompt(33, cfg["vocab_size"], salt=5)
        lo = so.forward(p2)
        lg = fill(s, p2)
        assert np.abs(lg - lo).max() < 0.125
        assert e.seq_len(s) == n_prompt + 8 + 33


@pytest.mark.parametrize("page", [32, 64])
def test_prefill_paths_agree_on_llama_shapes(monkeypatch, page):
    """Token-wise (decode kernels), full-tile (wgmma) and short-prompt (split-K) prefill of the same prompts give the same
    logits within tolerance at Llama-3-8B layer shapes (2 layers); the short-prompt path is also compared with the oracle
    directly.  Page 32 takes the wgmma prefill attention, page 64 the mma.sync kernel at head_dim 128."""
    monkeypatch.setenv("CL_PREFILL_SMALL_MAX", "256")
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["n_layers"] = 2
    cfg["max_seq_len"] = 512
    with eng.Engine(model=cfg, seed=1234, max_batch=2, page_size=page) as e:
        m = oc.Model(cfg, seed=1234)
        for n_small in (128, 250):
            ps = _prompt(n_small, cfg["vocab_size"], salt=3)
            so = m.new_seq()
            lo = so.prefill_block(ps)
            ss = e.seq_create()
            ls = e.prefill(ss, ps)                 # <= 256 tokens: split-K projections
            assert np.abs(ls - lo).max() < 0.125, float(np.abs(ls - lo).max())
            tok = int(lo.argmax())
            for _ in range(3):
                lo = so.forward([tok]); ls, _ = e.decode_step(ss, tok)
                assert np.abs(ls - lo).max() < 0.125
                tok = int(lo.argmax())
            e.seq_free(ss)
        p = _prompt(300, cfg["vocab_size"])
        s1 = e.seq_create()
        a = e.prefill(s1, p)                       # tensor-core tile path
        s2 = e.seq_create()
        b = None
        for i in range(0, 300, 10):                # 10-token pieces stay below the tile-path threshold
            b = e.prefill(s2, p[i:i + 10])
        assert np.abs(a - b).max() < 0.125
        assert int(a.argmax()) == int(b.argmax()) or np.sort(b)[-1] - np.sort(b)[-2] < 2e-2


@pytest.mark.parametrize("t2", [150, 300])
def test_prefill_continuation_at_an_unaligned_position_llama_shapes(monkeypatch, t2):
    """Multi-turn / chunked prompts: a second prefill appended at a position that is no multiple of the 64-token KV
    block (pos0 = 105) — the wgmma attention's diagonal then cuts through blocks, and keys come from pages written
    by an earlier prefill and by decode steps.  t2 = 150 takes the short-prompt path, 300 the full-tile path."""
    monkeypatch.setenv("CL_PREFILL_SMALL_MAX", "256")
    cfg = dict(oc.PRESETS["llama3-8b"])
    cfg["n_layers"] = 2
    cfg["max_seq_len"] = 512
    m = oc.Model(cfg, seed=4321)
    V = cfg["vocab_size"]
    with eng.Engine(model=cfg, seed=4321, max_batch=1) as e:
        so = m.new_seq()
        s = e.seq_create()
        p1 = _prompt(100, V, salt=1)
        lo = so.prefill_block(p1)
        lg = e.prefill(s, p1)
        assert np.abs(lg - lo).max() < 0.125
        tok = int(lo.argmax())
        for _ in range(5):
            lo = so.forward([tok]); lg, _ = e.decode_step(s, tok)
            tok = int(lo.argmax())
        p2 = _prompt(t2, V, salt=9)
        lo = so.prefill_block(p2)
        lg = e.prefill(s, p2)
        err = float(np.abs(lg - lo).max())
        assert err < 0.125, err
        tok = int(lo.argmax())
        for _ in range(4):
            lo = so.forward([tok]); lg, _ = e.decode_step(s, tok)
            assert np.abs(lg - lo).max() < 0.125
            tok = int(lo.argmax())
        assert e.seq_len(s) == 100 + 5 + t2 + 4


def test_multi_prompt_prefill_is_bit_identical_to_one_prompt_at_a_time(monkeypatch):
    """Engine::prefill_multi (cl_prefill_batch): several prompts as the rows of ONE tile-path pass.  A row's results do
    not depend on its neighbours, so the cached K / V of every position and the greedy continuation must equal, bit for
    bit, the same prompts prefilled alone through the tile path (CL_PREFILL_SMALL_MAX=0) — at Llama-3-8B layer shapes
    (wgmma attention) and on the tiny preset (head_dim 64).  The last-position logits come from the batched LM head
    (wgmma GEMM) instead of the single-sequence GEMV: same bf16 inputs, another summation order (<= 2e-4)."""
    monkeypatch.setenv("CL_PREFILL_SMALL_MAX", "0")
    for preset, layers, lens in (("llama3-8b", 2, [130, 17, 256, 33, 64, 300, 129]), ("tiny-test", 2, [40, 16, 97, 31])):
        cfg = dict(oc.PRESETS[preset])
        cfg["n_layers"] = layers
        cfg["max_seq_len"] = 1024
        V = cfg["vocab_size"]
        prompts = [np.array([(i * 7919 + 13 * b + 5) % V for i in range(n)], np.int32) for b, n in enumerate(lens)]
        with eng.Engine(model=cfg, seed=31, max_batch=8, max_seqs=16) as e:
            alone, alone_kv, alone_next = [], [], []
            for p in prompts:
                s = e.seq_create()
                alone.append(e.prefill(s, p))
                alone_kv.append([e.debug_kv(s, layers - 1, w, 0, len(p)) for w in (0, 1)])
                alone_next.append(e.decode_greedy(s, int(alone[-1].argmax()), 6)[0])
                e.seq_free(s)
            seqs = [e.seq_create() for _ in prompts]
            lg = e.prefill_batch(seqs, prompts)
            for b, s in enumerate(seqs):
                assert np.abs(lg[b] - alone[b]).max() < 2e-4 and int(lg[b].argmax()) == int(alone[b].argmax())
                assert e.seq_len(s) == lens[b]
                for w in (0, 1):
                    np.testing.assert_array_equal(e.debug_kv(s, layers - 1, w, 0, lens[b]), alone_kv[b][w])
            for b, s in enumerate(seqs):                       # the device state left behind (tok / pos) starts decoding correctly
                np.testing.assert_array_equal(e.decode_greedy(s, int(lg[b].argmax()), 6)[0], alone_next[b])
            # oracle check of one prompt of the batch (the tile path itself is pinned in the tests above)
            if preset == "tiny-test":
                m = oc.Model(cfg, seed=31)
                ref = m.new_seq().forward(prompts[2])
                assert np.abs(lg[2] - ref).max() < 0.05 + 0.03 * np.sqrt(layers)
            with pytest.raises(eng.EngineError):
                e.prefill_batch([seqs[0], seqs[0]], prompts[:2])   # duplicate sequence
