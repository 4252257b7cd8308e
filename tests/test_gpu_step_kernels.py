"""Kernel-level float64 parity of the batched decode step and of prefill behind a cached prefix.

Covers what the whole-model tests only see through logits: the tensor-core decode attention (both kernel shapes, the split
combine, the persistent item loop, slots, the bf16 copy), the CUDA-core decode attention at batch > 1, the wgmma GEMM's
split-K partials, PDL launch, in-place residual and SiLU epilogues, and both prefill attention kernels at pos0 > 0.

Every reference is plain float64 numpy on the exact bf16 values the kernels see.  Each bound follows from the kernel's
rounding points (see the constants below), is checked per element, and the observed max(err / tol) is printed (-s).  The
CPU tests at the end show that each bound is tight enough to catch a dropped page, a dropped current token, the wrong kv
head and a dropped k-block.
"""
import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc

gpu = pytest.mark.gpu

# Attention: out = bf16(sum_t p_t v_t / sum_t p_t).  Bound per element = one bf16 ulp of the reference (the output rounding,
# including a carry into the next binade) + C * sum_t p_t |v_t| (normalised p).
#   decode (both kernels): P is fp32-accurate (the tensor-core kernel feeds P.V a hi + lo bf16 pair, |p - hi - lo| <= 2^-17 p);
#     what is left are fp32 scores (a few 2^-23 of sum |q k| / sqrt(d) ~ 2^-16) and exp2f: C = 2^-14.
#   prefill (both kernels): P is rounded to bf16 before P.V, |bf16(p) - p| <= 2^-9 p, while the normaliser sums fp32 p:
#     C = 2^-7.
DECODE_C = 2.0 ** -14
PREFILL_C = 2.0 ** -7
# GEMM partial: fp32 accumulation over the split's k range, K/16 wgmma k-steps, each rounding a partial sum bounded by
# sum |x w| at most twice (the in-MMA product sum and the accumulate), each <= 2^-23 relative: 2 * (16384 / 16) * 2^-23 = 2^-12
# for K <= 16384.  Products of two bf16 are exact in fp32.  This worst case lies far above the observed errors (~2^-20 of
# sum |x w|) and, for a partial over thousands of k, above a bf16 rounding of the fp32 result (2^-9 |y|, with |y| ~ sum|x w| /
# 40 at K = 4096).  low_bits_zero_share() therefore checks separately that such partials keep every fp32 mantissa bit.
GEMM_C = 2.0 ** -12
BK = 64                                                   # k-block of the GEMM (split-K splits whole k-blocks)


def bf16(x):
    return oc.np_bf16_from_f32(np.asarray(x, dtype=np.float32))


def f32(h):
    return oc.np_f32_from_bf16(np.asarray(h, dtype=np.uint16))


def ulp_bf16(y):
    e = np.floor(np.log2(np.maximum(np.abs(np.asarray(y, np.float64)), 2.0 ** -126)))
    return 2.0 ** (e - 7)


# ---- attention: inputs and float64 reference ----------------------------------------------------------------------------
def attn_inputs(rng, n_keys, q_pos, n_heads, n_kv, hd, boost=10.0):
    """q [R][H*D], k, v [n_keys][n_kv][D] as bf16 bits.  q.k / sqrt(D) ~ N(0, 4): peaked scores, so the row maximum moves
    between pages and splits.  The key at each query's own position gets +boost on the score of the first q head of its kv
    group, as real attention often weights the current token: without it a dropped current token would hide in 8K others."""
    q_pos = np.asarray(q_pos)
    R, rep = len(q_pos), n_heads // n_kv
    q = f32(bf16(rng.standard_normal((R, n_kv, rep, hd))))
    k = rng.standard_normal((n_keys, n_kv, hd)) * 2.0
    v = rng.standard_normal((n_keys, n_kv, hd))
    if boost:
        q0 = q[:, :, 0].astype(np.float64)
        k[q_pos] += boost * np.sqrt(hd) * q0 / (q0 ** 2).sum(-1, keepdims=True)
    return bf16(q.reshape(R, -1)), bf16(k), bf16(v)


def attn64(q, k, v, q_pos, n_heads, n_kv, hd, page=32, mutate=None):
    """Float64 causal attention with an explicit softmax: query r (q [R][H*D]) sees keys 0 .. q_pos[r] of k, v [n][n_kv][D].
    Returns (out [R][H*D], sum_t p_t |v_t| [R][H*D]).  mutate: "page" drops the page (of `page` keys) with the largest weight,
    "current" drops key q_pos[r], "kv_head" reads kv head g + 1 instead of g."""
    q_pos = np.asarray(q_pos)
    R, n, rep = q.shape[0], k.shape[0], n_heads // n_kv
    q = np.asarray(q, np.float64).reshape(R, n_kv, rep, hd)
    k = np.asarray(k, np.float64)
    v = np.asarray(v, np.float64)
    keys = np.arange(n)
    vis = keys[None, :] <= q_pos[:, None]
    if mutate == "current":
        vis = vis & (keys[None, :] != q_pos[:, None])
    out = np.empty((R, n_kv, rep, hd))
    pv = np.empty_like(out)

    def softmax(s, m):
        s = np.where(m, s, -np.inf)
        e = np.exp(s - s.max(-1, keepdims=True))
        return e / e.sum(-1, keepdims=True)

    for g in range(n_kv):
        src = (g + 1) % n_kv if mutate == "kv_head" else g
        s = (q[:, g].reshape(R * rep, hd) @ k[:, src].T).reshape(R, rep, n) / np.sqrt(hd)
        m = np.broadcast_to(vis[:, None, :], s.shape)
        p = softmax(s, m)
        if mutate == "page":
            n_pg = (n + page - 1) // page
            w = np.pad(p, ((0, 0), (0, 0), (0, n_pg * page - n))).reshape(R, rep, n_pg, page).sum(-1)
            m = m & ((keys // page)[None, None, :] != w.argmax(-1)[..., None])
            p = softmax(s, m)
        out[:, g] = p @ v[:, src]
        pv[:, g] = p @ np.abs(v[:, src])
    return out.reshape(R, -1), pv.reshape(R, -1)


def attn_ratio(got, ref, pv, c):
    return float((np.abs(np.asarray(got, np.float64) - ref) / (ulp_bf16(ref) + c * pv)).max())


# ---- decode attention (cl_op_attn_decode_batch) ------------------------------------------------------------------------
def decode_inputs(seed, lens, n_heads, n_kv, hd, boost=10.0):
    """One batch: q [B][H*D] fp32, k, v [sum(lens)][n_kv][D] bf16, each sequence's current token last."""
    rng = np.random.default_rng(seed)
    qs, ks, vs = [], [], []
    for L in lens:
        q, k, v = attn_inputs(rng, L, [L - 1], n_heads, n_kv, hd, boost)
        qs.append(f32(q))
        ks.append(k)
        vs.append(v)
    return np.concatenate(qs), np.concatenate(ks), np.concatenate(vs)


def decode_refs(q, kc, vc, lens, n_heads, n_kv, hd):
    refs, off = [], 0
    for b, L in enumerate(lens):
        refs.append(attn64(q[b:b + 1], f32(kc[off:off + L]), f32(vc[off:off + L]), [L - 1], n_heads, n_kv, hd))
        off += L
    return refs


def check_decode(name, q, kc, vc, lens, n_heads, n_kv, hd, page=32, slots=None, n_slots=None, refs=None, **kw):
    """Runs the op, asserts the exact properties and the per-element bound; returns (out rows of the batch, nsplit, tc_small)."""
    B = len(lens)
    n_slots = n_slots or B
    slots = list(range(B)) if slots is None else list(slots)
    init = np.random.default_rng(99).standard_normal((n_slots, n_heads * hd)).astype(np.float32)
    out, ob, ns, small = eng.op_attn_decode_batch(q, kc, vc, lens, n_heads, n_kv, hd, page, slots=slots, n_slots=n_slots,
                                                  out_init=init, **kw)
    rows = out[slots]
    assert not np.isnan(rows).any(), name
    others = sorted(set(range(n_slots)) - set(slots))
    assert np.array_equal(out[others].view(np.uint32), init[others].view(np.uint32)), f"{name}: a slot outside the batch was written"
    np.testing.assert_array_equal(ob, bf16(rows), err_msg=f"{name}: out_bf16 differs from the fp32 out")
    refs = refs or decode_refs(q, kc, vc, lens, n_heads, n_kv, hd)
    worst = max(attn_ratio(rows[b:b + 1], ref, pv, DECODE_C) for b, (ref, pv) in enumerate(refs))
    print(f"[decode] {name}: nsplit {ns} tc_small {small} max err/tol {worst:.3g}")
    assert worst <= 1.0, f"{name}: max err/tol {worst:.3g}"
    return rows, ns, small


TC = dict(n_heads=32, n_kv=8, hd=128)                     # Llama-3-8B / Mistral-7B attention
LONGCTX_B16 = [L + 1 for L in [8188, 4096, 4095, 31, 32, 33, 0, 1000, 2047, 2048, 6000, 100, 64, 500, 3000, 7]]


def _wide_lens(B):                                         # test_gpu_longctx's B = 40 / 100 lengths, + the current token
    return [((i * 97 + 13) % 600 if i % 7 else (31, 32, 33, 0, 64, 95, 96)[(i // 7) % 7]) + 1 for i in range(B)]


@gpu
@pytest.mark.parametrize("ctx", [1, 2, 31, 32, 33, 63, 64, 65, 4095, 4096, 4097, 8192])
def test_decode_tc_context_lengths(ctx):
    q, kc, vc = decode_inputs(ctx, [ctx], **TC)
    _, ns, small = check_decode(f"tc ctx {ctx}", q, kc, vc, [ctx], **TC, variant=1)
    assert small == 0 and ns > 1                           # one sequence: 8-warp shape, many splits (empty ones at short ctx)


@gpu
@pytest.mark.parametrize("lens,slots,n_slots", [
    ([8190, 4097, 100], [5, 0, 2], 7),
    (LONGCTX_B16, [3, 17, 0, 9, 4, 12, 19, 1, 8, 15, 6, 2, 11, 18, 5, 13], 20),
])
def test_decode_tc_mixed_batch(lens, slots, n_slots):
    q, kc, vc = decode_inputs(len(lens), lens, **TC)
    check_decode(f"tc B {len(lens)}", q, kc, vc, lens, **TC, slots=slots, n_slots=n_slots, variant=-1)


@gpu
@pytest.mark.parametrize("B", [40, 100])
def test_decode_tc_wide_batch_persistent(B):
    """Under the step's plan: the 4-warp shape, one split, more items than resident CTAs (persistent item loop); then the
    8-warp shape forced on the same inputs."""
    lens = _wide_lens(B)
    q, kc, vc = decode_inputs(B, lens, **TC)
    slots = list(np.random.default_rng(B).permutation(B + 5)[:B])
    refs = decode_refs(q, kc, vc, lens, **TC)
    _, ns, small = check_decode(f"tc B {B} plan", q, kc, vc, lens, **TC, slots=slots, n_slots=B + 5, refs=refs, variant=-1)
    assert (ns, small) == (1, 1)
    check_decode(f"tc B {B} 8-warp", q, kc, vc, lens, **TC, slots=slots, n_slots=B + 5, refs=refs, variant=1, tc_small=0)


@gpu
def test_decode_tc_explicit_splits_and_shapes():
    """nsplit 1, 2, 7, 16 and more splits than pages (empty splits), each with both kernel shapes."""
    lens = [3000, 100, 33, 1]
    q, kc, vc = decode_inputs(7, lens, **TC)
    refs = decode_refs(q, kc, vc, lens, **TC)
    for ns in (1, 2, 7, 16, 40):
        for small in (0, 1):
            _, used, su = check_decode(f"tc nsplit {ns} small {small}", q, kc, vc, lens, **TC, refs=refs, variant=1, nsplit=ns,
                                       tc_small=small)
            assert (used, su) == (ns, small)


@gpu
def test_decode_tc_one_kv_head_max_splits():
    """H = 4 / n_kv = 1 with nsplit 64 (the kernel's MAXS): 94 pages, and 32 pages (half the splits empty)."""
    shape = dict(n_heads=4, n_kv=1, hd=128)
    lens = [3000, 1000]
    q, kc, vc = decode_inputs(11, lens, **shape)
    for small in (0, 1):
        check_decode(f"tc H4/kv1 nsplit 64 small {small}", q, kc, vc, lens, **shape, variant=1, nsplit=64, tc_small=small)
    with pytest.raises(eng.EngineError) as ei:
        eng.op_attn_decode_batch(q, kc, vc, lens, 4, 1, 128, variant=1, nsplit=65)
    assert ei.value.status == eng.CL_ERR_INVALID_ARG


@gpu
def test_decode_tc_dominant_and_flat_scores():
    """One key that takes nearly all the weight in a middle split; and all scores equal (k = 0)."""
    L, j = 4097, 2050
    q, kc, vc = decode_inputs(13, [L], **TC)
    q0 = q.reshape(8, 4, 128)[:, 0].astype(np.float64)
    kc[j] = bf16(30.0 * np.sqrt(128) * q0 / (q0 ** 2).sum(-1, keepdims=True))
    check_decode("tc dominant key", q, kc, vc, [L], **TC, variant=1, nsplit=16)
    check_decode("tc k = 0", q, np.zeros_like(kc), vc, [L], **TC, variant=1, nsplit=16)


@gpu
@pytest.mark.parametrize("n_heads,n_kv,hd", [(32, 4, 64), (32, 8, 128)])
@pytest.mark.parametrize("page", [16, 64])
def test_decode_cuda_core_batch(n_heads, n_kv, hd, page):
    """CUDA-core kernel at batch > 1 with slots and the step's split plan (TinyLlama's head_dim 64 with 8 q heads per kv head,
    and head_dim 128 at the page sizes the tensor-core kernel does not take)."""
    shape = dict(n_heads=n_heads, n_kv=n_kv, hd=hd)
    lens = [1, 64, 65, 700, 2049]
    q, kc, vc = decode_inputs(page + hd, lens, **shape)
    _, _, small = check_decode(f"cuda-core H{n_heads}/kv{n_kv} d{hd} page {page}", q, kc, vc, lens, **shape, page=page,
                               slots=[6, 2, 0, 4, 1], n_slots=8, variant=-1)
    assert small == -1                                     # the step's choice at these shapes is the CUDA-core kernel


# ---- prefill attention behind a cached prefix (cl_op_attn_prefill_cached) ---------------------------------------------
def prefill_inputs(seed, pos0, T, n_heads, n_kv, hd, boost=10.0):
    rng = np.random.default_rng(seed)
    return attn_inputs(rng, pos0 + T, pos0 + np.arange(T), n_heads, n_kv, hd, boost)


def check_prefill(name, q, k, v, pos0, n_heads, n_kv, hd, page, variant, ref=None):
    T = q.shape[0]
    out = eng.op_attn_prefill_cached(q, k, v, pos0, n_heads, n_kv, hd, page_size=page, variant=variant)
    assert not np.isnan(out).any(), name
    ref, pv = ref or attn64(f32(q), f32(k), f32(v), pos0 + np.arange(T), n_heads, n_kv, hd)
    worst = attn_ratio(out, ref, pv, PREFILL_C)
    print(f"[prefill] {name}: max err/tol {worst:.3g}")
    assert worst <= 1.0, f"{name}: max err/tol {worst:.3g}"
    return out


PREFILL_CASES = [(1, 1), (31, 1), (32, 1), (1024, 1), (1024, 40), (63, 65), (105, 150), (105, 300), (127, 129), (4096, 300)]


@gpu
@pytest.mark.parametrize("pos0,T", PREFILL_CASES)
def test_prefill_cached_both_kernels(pos0, T):
    q, k, v = prefill_inputs(pos0 * 7 + T, pos0, T, **TC)
    ref = attn64(f32(q), f32(k), f32(v), pos0 + np.arange(T), **TC)
    for variant in (0, 1):
        check_prefill(f"variant {variant} pos0 {pos0} T {T}", q, k, v, pos0, **TC, page=32, variant=variant, ref=ref)


@gpu
def test_prefill_cached_wgmma_block_table_limit():
    """pos0 + T = 10240 fills the wgmma kernel's 320 staged block-table entries; at 10241 variant 1 is refused and the
    engine's rule (-1) takes the mma.sync kernel."""
    T = 64
    for n_tok, wgmma in ((10240, True), (10241, False)):
        pos0 = n_tok - T
        q, k, v = prefill_inputs(n_tok, pos0, T, **TC)
        ref = attn64(f32(q), f32(k), f32(v), pos0 + np.arange(T), **TC)
        auto = check_prefill(f"variant -1 pos0+T {n_tok}", q, k, v, pos0, **TC, page=32, variant=-1, ref=ref)
        mma = check_prefill(f"variant 0 pos0+T {n_tok}", q, k, v, pos0, **TC, page=32, variant=0, ref=ref)
        if wgmma:
            tc = check_prefill(f"variant 1 pos0+T {n_tok}", q, k, v, pos0, **TC, page=32, variant=1, ref=ref)
            np.testing.assert_array_equal(auto, tc)
        else:
            with pytest.raises(eng.EngineError) as ei:
                eng.op_attn_prefill_cached(q, k, v, pos0, 32, 8, 128, variant=1)
            assert ei.value.status == eng.CL_ERR_INVALID_ARG
            np.testing.assert_array_equal(auto, mma)


@gpu
@pytest.mark.parametrize("n_heads,n_kv,hd", [(8, 8, 128), (32, 8, 128), (32, 4, 128), (8, 8, 64), (32, 8, 64), (32, 4, 64)])
@pytest.mark.parametrize("page", [16, 32, 64])
def test_prefill_cached_shapes(n_heads, n_kv, hd, page):
    """GQA 1:1, 4:1 and 8:1 at head_dim 64 and 128: the mma.sync kernel at every page size, the wgmma kernel where it
    applies (head_dim 128, page 32)."""
    shape = dict(n_heads=n_heads, n_kv=n_kv, hd=hd)
    pos0, T = 105, 150
    q, k, v = prefill_inputs(n_heads * hd + page, pos0, T, **shape)
    ref = attn64(f32(q), f32(k), f32(v), pos0 + np.arange(T), **shape)
    check_prefill(f"variant 0 H{n_heads}/kv{n_kv} d{hd} page {page}", q, k, v, pos0, **shape, page=page, variant=0, ref=ref)
    if hd == 128 and page == 32:
        check_prefill(f"variant 1 H{n_heads}/kv{n_kv} d{hd}", q, k, v, pos0, **shape, page=page, variant=1, ref=ref)


# ---- GEMM: split-K partials, PDL, residual and SiLU epilogues (cl_op_gemm_bf16_epi) ----------------------------------
def split_ranges(K, ks):
    """k ranges (in elements) of the ks split-K partials: whole k-blocks of 64, ceil(nkb / ks) per split, the last one short."""
    nkb = -(-K // BK)
    per = -(-nkb // ks)
    return [(s * per * BK, min(K, (s + 1) * per * BK)) for s in range(ks)]


def splits_valid(K, ks):
    """The counts launch_gemm_bf16 takes: every split owns at least one k-block."""
    nkb = -(-K // BK)
    return ks == 1 or (1 <= ks <= nkb and -(-nkb // ks) * (ks - 1) < nkb)


def gemm_inputs(seed, T, N, K):
    rng = np.random.default_rng(seed)
    x = bf16(rng.standard_normal((T, K)))
    w = bf16(rng.standard_normal((N, K)) * 2.0 / np.sqrt(K))   # outputs ~ N(0, 4): SiLU sees both of its regimes
    return x, w


def gemm_refs(x, w, ks):
    """Float64 partials [ks][T][N] and the matching sum_k |x_k w_k|."""
    xf, wf = f32(x).astype(np.float64), f32(w).astype(np.float64)
    ref = np.stack([xf[:, a:b] @ wf[:, a:b].T for a, b in split_ranges(x.shape[1], ks)])
    mag = np.stack([np.abs(xf[:, a:b]) @ np.abs(wf[:, a:b]).T for a, b in split_ranges(x.shape[1], ks)])
    return ref, mag


def low_bits_zero_share(y):
    """Share of the nonzero values whose 8 lowest fp32 mantissa bits are all 0: about 1/256 for an fp32 sum of many bf16
    products, 1 for a value rounded to 16 or fewer significant bits on the way (bf16, fp16, tf32)."""
    y = np.asarray(y, np.float32)
    u = y[y != 0].view(np.uint32)
    return float(((u & 0xFF) == 0).mean())


def check_partials(name, y, x, w, ks):
    assert y.shape[0] == ks and not np.isnan(y).any(), name
    ref, mag = gemm_refs(x, w, ks)
    worst = float((np.abs(y - ref) / (GEMM_C * mag)).max())
    print(f"[gemm] {name}: k_splits {ks} max err/tol {worst:.3g}")
    assert worst <= 1.0, f"{name}: max err/tol {worst:.3g}"
    if split_ranges(x.shape[1], ks)[0][1] >= 16 * BK:     # partials over >= 16 k-blocks: no rounding below fp32 on the way
        assert low_bits_zero_share(y) <= 1 / 16, f"{name}: k_splits {ks} lost fp32 mantissa bits"


GEMM_SHAPES = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336), (136, 72), (1000, 200), (320, 1000)]


@gpu
@pytest.mark.parametrize("N,K", [(6144, 4096), (136, 72)])
def test_gemm_token_counts(N, K):
    """Every token tile (32 / 64 / 128) and its ragged edges, split as the batched step splits."""
    for T in (1, 2, 31, 32, 33, 64, 65, 100, 128, 129, 256):
        x, w = gemm_inputs(T * 3 + N, T, N, K)
        y, ks = eng.op_gemm_bf16_epi(x, w, epi=0, k_splits=0, pdl=True)
        check_partials(f"T {T} N {N} K {K}", y, x, w, ks)


@gpu
@pytest.mark.parametrize("N,K", GEMM_SHAPES)
def test_gemm_splits_pdl_and_epilogues(N, K):
    """Split counts 0 (the step's choice), 1, 2 and the largest the GEMM takes, with and without PDL (identical bits); the
    residual epilogue = float32(resid + the unsplit partial) bit for bit; SiLU within one bf16 ulp of silu(g) * u."""
    nkb = -(-K // BK)
    largest = max(s for s in range(1, nkb + 1) if splits_valid(K, s))
    x129, w = gemm_inputs(N + K, 129, N, K)
    for T in (33, 129):
        x = x129[:T]
        base = {}
        for ks in sorted({0, 1, 2, largest}):
            y0, used = eng.op_gemm_bf16_epi(x, w, epi=0, k_splits=ks, pdl=False)
            y1, used1 = eng.op_gemm_bf16_epi(x, w, epi=0, k_splits=ks, pdl=True)
            assert used == used1 and (ks == 0 or used == ks)
            np.testing.assert_array_equal(y0.view(np.uint32), y1.view(np.uint32), err_msg=f"PDL changed k_splits {ks}")
            check_partials(f"T {T} N {N} K {K}", y0, x, w, used)
            base[used] = y0
        y = base[1][0]
        resid = np.random.default_rng(T).standard_normal((T, N)).astype(np.float32)
        for pdl in (False, True):
            r, _ = eng.op_gemm_bf16_epi(x, w, epi=1, k_splits=0, pdl=pdl, resid=resid)
            np.testing.assert_array_equal(r.view(np.uint32), (resid + y).view(np.uint32), err_msg=f"residual, pdl {pdl}")
        act, _ = eng.op_gemm_bf16_epi(x, w, epi=2)
        g, u = y[:, 0::2].astype(np.float64), y[:, 1::2].astype(np.float64)
        ref = g / (1.0 + np.exp(-g)) * u
        worst = float((np.abs(f32(act) - ref) / ulp_bf16(ref)).max())
        print(f"[gemm] SiLU T {T} N {N} K {K}: max err/ulp {worst:.3g}")
        assert worst <= 1.0


@gpu
def test_gemm_refused_split_counts():
    x, w = gemm_inputs(1, 8, 1000, 200)
    for ks in range(1, 7):
        if splits_valid(200, ks):
            y, used = eng.op_gemm_bf16_epi(x, w, epi=0, k_splits=ks)
            assert used == ks and not np.isnan(y).any()
        else:
            with pytest.raises(eng.EngineError) as ei:
                eng.op_gemm_bf16_epi(x, w, epi=0, k_splits=ks)
            assert ei.value.status == eng.CL_ERR_INVALID_ARG, ks
    assert [s for s in range(1, 7) if not splits_valid(200, s)] == [3, 5, 6]
    with pytest.raises(eng.EngineError) as ei:
        eng.op_gemm_bf16_epi(x, w, epi=1, k_splits=2, resid=np.zeros((8, 1000), np.float32))
    assert ei.value.status == eng.CL_ERR_INVALID_ARG


# ---- CPU: entry points without a device, the references, and the power of every bound ---------------------------------
def test_new_ops_report_no_device():
    if eng.device_count() > 0:
        pytest.skip("GPU present")
    q, kc, vc = decode_inputs(0, [3], 4, 2, 64)
    for call in (lambda: eng.op_attn_decode_batch(q, kc, vc, [3], 4, 2, 64),
                 lambda: eng.op_attn_prefill_cached(bf16(np.zeros((1, 256))), kc, vc, 2, 4, 2, 64),
                 lambda: eng.op_gemm_bf16_epi(np.zeros((1, 64), np.uint16), np.zeros((2, 64), np.uint16))):
        with pytest.raises(eng.EngineError) as ei:
            call()
        assert ei.value.status == eng.CL_ERR_NO_DEVICE


@pytest.mark.parametrize("ctx,n_heads,n_kv,hd", [(1, 4, 2, 64), (7, 8, 8, 64), (40, 8, 2, 128), (300, 32, 8, 128)])
def test_attention_reference_matches_oracle(ctx, n_heads, n_kv, hd):
    q, kc, vc = decode_inputs(ctx, [ctx], n_heads, n_kv, hd)
    ref, _ = attn64(q, f32(kc), f32(vc), [ctx - 1], n_heads, n_kv, hd)
    got = oc.attention(q[0], f32(kc), f32(vc), n_heads, n_kv, hd)
    np.testing.assert_allclose(got, ref[0], rtol=1e-5, atol=1e-5 * np.abs(ref).max())


@pytest.mark.parametrize("K", [72, 200, 1000, 4096])
def test_split_references_sum_to_unsplit(K):
    x, w = gemm_inputs(K, 5, 24, K)
    full, _ = gemm_refs(x, w, 1)
    for ks in range(1, -(-K // BK) + 1):
        if splits_valid(K, ks):
            parts, _ = gemm_refs(x, w, ks)
            assert split_ranges(K, ks)[-1][1] == K and split_ranges(K, ks)[-1][0] < K
            np.testing.assert_allclose(parts.sum(0), full[0], rtol=0, atol=1e-9)


# Representative inputs of every attention family, built by the generators the GPU tests use.
POWER_DECODE = [(8192, 32, 8, 128, 32), (4097, 32, 8, 128, 32), (65, 32, 8, 128, 32), (2049, 32, 4, 64, 16),
                (700, 32, 8, 128, 64)]
POWER_PREFILL = [(4096, 300, 32, 8, 128, 32), (10176, 64, 32, 8, 128, 32), (105, 150, 32, 4, 64, 16), (63, 65, 8, 8, 128, 64),
                 (1024, 1, 32, 8, 128, 32)]


def _power(q, k, v, q_pos, shape, page, c):
    ref, pv = attn64(q, k, v, q_pos, **shape, page=page)
    tol = ulp_bf16(ref) + c * pv
    with np.errstate(invalid="ignore"):                    # a query whose only page is dropped has nothing left: NaN, skipped
        return {m: float(np.nanmax(np.abs(attn64(q, k, v, q_pos, **shape, page=page, mutate=m)[0] - ref) / tol))
                for m in ("page", "current", "kv_head")}


@pytest.mark.parametrize("ctx,n_heads,n_kv,hd,page", POWER_DECODE)
def test_decode_bound_catches_dropped_page_token_and_head(ctx, n_heads, n_kv, hd, page):
    shape = dict(n_heads=n_heads, n_kv=n_kv, hd=hd)
    q, kc, vc = decode_inputs(ctx, [ctx], **shape)
    r = _power(q, f32(kc), f32(vc), [ctx - 1], shape, page, DECODE_C)
    print(f"[power] decode ctx {ctx} H{n_heads}/kv{n_kv} d{hd} page {page}: {r}")
    assert min(r.values()) >= 4.0, r


@pytest.mark.parametrize("pos0,T,n_heads,n_kv,hd,page", POWER_PREFILL)
def test_prefill_bound_catches_dropped_page_token_and_head(pos0, T, n_heads, n_kv, hd, page):
    shape = dict(n_heads=n_heads, n_kv=n_kv, hd=hd)
    q, k, v = prefill_inputs(pos0 * 7 + T, pos0, T, **shape)
    r = _power(f32(q), f32(k), f32(v), pos0 + np.arange(T), shape, page, PREFILL_C)
    print(f"[power] prefill pos0 {pos0} T {T} H{n_heads}/kv{n_kv} d{hd} page {page}: {r}")
    assert min(r.values()) >= 4.0, r


@pytest.mark.parametrize("T,N,K", [(1, 4096, 14336), (33, 1000, 1000), (1, 6144, 4096), (129, 4096, 4096)])
def test_gemm_precision_check_catches_a_rounded_partial(T, N, K):
    """The fp32 rounding of the exact unsplit partial passes the mantissa check; the same rounded to bf16, fp16 or tf32 (which
    the 2^-12 bound lets through at large K) fails it."""
    x, w = gemm_inputs(K + T, T, N, K)
    ref, _ = gemm_refs(x, w, 1)
    assert low_bits_zero_share(ref.astype(np.float32)) <= 1 / 64
    assert low_bits_zero_share(f32(bf16(ref))) == 1.0
    assert low_bits_zero_share(ref.astype(np.float16).astype(np.float32)) == 1.0
    tf32 = (ref.astype(np.float32).view(np.uint32) + 0x1000) & np.uint32(0xFFFFE000)
    assert low_bits_zero_share(tf32.view(np.float32)) == 1.0


@pytest.mark.parametrize("T,N,K", [(1, 4096, 14336), (33, 1000, 200), (33, 136, 72), (2, 512, 4096)])
def test_gemm_bound_catches_dropped_k_block(T, N, K):
    """Dropping any one k-block of any partial moves some element of that partial by >= 4x its bound."""
    x, w = gemm_inputs(K + T, T, N, K)
    xf, wf = f32(x).astype(np.float64), f32(w).astype(np.float64)
    for ks in sorted({1, 2, max(s for s in range(1, -(-K // BK) + 1) if splits_valid(K, s))}):
        for a, b in split_ranges(K, ks):
            tol = GEMM_C * (np.abs(xf[:, a:b]) @ np.abs(wf[:, a:b]).T)
            weakest = min(float((np.abs(xf[:, k0:k0 + BK] @ wf[:, k0:k0 + BK].T) / tol).max()) for k0 in range(a, b, BK))
            assert weakest >= 4.0, (ks, a, b, weakest)
