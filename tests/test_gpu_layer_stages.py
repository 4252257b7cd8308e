"""Stage-by-stage float64 parity of one transformer layer as the decode step, the prefill passes and the verify passes run it.

What the whole-model tests only see through logits is checked here stage by stage on engines whose every weight the test
owns (cl_engine_set_tensor), with the buffers cl_debug_seq_hidden, cl_debug_pass_rows and cl_debug_kv expose:

  1. RMSNorm -> q|k|v projection -> RoPE -> bf16 -> cache append      q, and the K / V rows written at `pos`
  2. split-KV attention + combine                                       attention output
  3. o-projection + residual, RMSNorm -> gate|up -> SiLU * up           activation
  4. down projection + residual (and the o-projection's rows again)     residual stream after the layer
  5. final RMSNorm + LM head                                            logits

Every stage is teacher-forced: its float64 reference starts from the kernel's own output of the stage before, so the
bound of a stage holds its own rounding points only and is checked per element.  The constants are derived from the
kernels' summation structure below; none is fitted to an observation.  The observed max(err / bound) is printed (-s).

Covered: decode_mega_kernel, the per-op path with both GEMV kernels, the batched step (wgmma projections, batch_* glue,
tensor-core attention, graph and PDL as shipped) — parts (a), (b) — and, part (d), the rows of every multi-row pass: the
split-K pass (prompts of 16 .. 256 tokens, the verify passes) and the tile pass (longer prompts, chunk by chunk, and
cl_prefill_batch), with the mma.sync, wgmma and multi-row verify attention kernels.  cl_debug_pass_info asserts which path
and kernel a case ran; the rejected rows of a verify pass are read through cl_debug_kv's which 2 / 3.  Long passes are
checked stage by stage on sampled rows, and stage 1 of K / V on every row of every pass.  The intermediates
h_mid (after the o-projection) and xn are not kept by any path: stage 3 and 4 start from the attention output and compose
the o-projection's bound.

The CPU tests at the end feed the same checks with mutated "kernel outputs" (each must exceed its bound by the stated
margin) and with a float32 numpy layer that sums in another order (must stay inside every bound).
"""
import functools

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from test_gpu_speculative_batch import ATTN_C
from test_gpu_step_kernels import DECODE_C, LONGCTX_B16, PREFILL_C, _wide_lens, attn64, bf16, f32, ulp_bf16

gpu = pytest.mark.gpu
U = 2.0 ** -24                                             # unit roundoff of fp32 (round to nearest)

# ---- constants, each from the code it bounds -----------------------------------------------------------------------------
# GEMV (decode_mega.cu consume_dynamic, decode_kernels.cu gemv_ring_kernel / gemv_ldg_kernel): every term w*x (exact in fp32:
# bf16 x bf16) passes through a chain of fp32 roundings, each <= U relative to a partial sum <= sum |w x|:
#   ring / persistent kernel: 8 * CPL fmaf per lane, 5 warp-shuffle adds, then the S slice partials (S - 1 adds in sequence,
#     or two levels of pairs in the persistent kernel: never more than S);  K = S * CPL * 256
#   LDG kernel: K / 32 fmaf per lane (16 per 32-byte chunk, K / 512 chunks), 5 warp-shuffle adds.
# These are worst cases over sum |w x|.  Rounding errors follow the partial sums, about sqrt(K) smaller than sum |w x| for
# signed terms, and add like sqrt(depth), so stages 4 and 5 (no bf16 term) sit near 0.003 of their bound at K = 4096 and
# 0.04 at K = 256; the CPU tests show that a dropped row or k-slice still lands tens of bounds outside.
RING_CFG = {1024: (4, 1), 2048: (4, 2), 4096: (4, 4), 8192: (8, 4), 14336: (8, 7)}   # K -> (S, CPL)


def gemv_c(K, ring):
    if ring and K in RING_CFG:
        S, CPL = RING_CFG[K]
        return (8 * CPL + 5 + S) * U
    return (K // 32 + 5) * U


# wgmma GEMM (batched step, prefill, verify): the bound of tests/test_gpu_step_kernels.py, 2 roundings per 16-wide k-step,
# K / 16 steps: K * 2^-26 of sum |w x| for an unsplit row; split-K partials are shorter, so this also covers them.  Their
# fixed-order fp32 sum (batch_rope_append_kernel, batch_silu_kernel, batch_resid_norm_kernel, rope_scatter_kernel) adds
# n_split roundings of partial sums <= sum_s |y_s| <= sum |w x|; n_split <= 16 (pick_splits).
def gemm_c(K):
    return K * 2.0 ** -26 + 16 * U


# RMSNorm, xn = bf16(h * inv * gain), inv = 1 / sqrtf(tot / K + eps): relative fp32 error of h * inv * gain before the bf16
# rounding.  tot is a sum of squares (all terms positive, so the chain bound is relative): the deepest chain of any variant
# is batch_resid_norm_kernel's 8 fmaf + 5 shuffles + 32 warp partials = 45 roundings (persistent / ring kernels 40, LDG 29,
# rmsnorm_bf16_kernel 29); the square root halves it: 22.5.  tot / K and + eps: 2 roundings, halved: 1.  sqrtf, the
# reciprocal and the two multiplies: 4.  Total 27.5 -> 28 U ~ 2^-19.2.
REL_XN = 28 * U
# RoPE r0 = y0 c - y1 s in fp32 (one product may be fused): 2 roundings of terms <= |y0| + |y1|, and c, s are the double
# table rounded to fp32 (U relative each): 4 U (|y0| + |y1|).
ROPE_C = 4 * U
# SiLU: __expf(-g) = ex2.approx(-g * log2e): the product's rounding moves the exponent by <= |g| log2e U, i.e. |g| U
# relative on e^-g; ex2.approx <= 2^-22 = 4 U; 1 + e, the division and the multiply by up: 3 U.  (|g| + 7) U, rounded up.
SILU_DERIV = 1.1                                           # max |d silu / dg|


def silu_rel(g):
    return (np.abs(g) + 8) * U


# ---- shapes and weights ---------------------------------------------------------------------------------------------------
VOCAB = 512
LLAMA = dict(d_model=4096, n_heads=32, n_kv_heads=8, head_dim=128, d_ff=14336, max_seq_len=8192, rope_theta=5e5)
MISTRAL = dict(LLAMA, max_seq_len=8704, rope_theta=1e6)
LLAMA31 = dict(LLAMA, max_seq_len=32768, rope_factor=8.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0,
               rope_original_max_pos=8192)
TINYLLAMA = dict(d_model=2048, n_heads=32, n_kv_heads=4, head_dim=64, d_ff=5632, max_seq_len=2048, rope_theta=1e4)
LLAMA32_1B = dict(d_model=2048, n_heads=32, n_kv_heads=8, head_dim=64, d_ff=8192, max_seq_len=8192, rope_theta=5e5,
                  rope_factor=32.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0, rope_original_max_pos=8192)
TINY = dict(d_model=256, n_heads=4, n_kv_heads=2, head_dim=64, d_ff=512, max_seq_len=1024, rope_theta=1e4)
EPS = 1e-5


def rope_table(shape, positions):
    """cos, sin [len(positions)][head_dim / 2] as the engine tabulates them (DESIGN.md section 3): the angle in double,
    pos * theta^(-2i / head_dim), with the "llama3" frequency scaling where configured, rounded to fp32."""
    hd = shape["head_dim"]
    inv = np.float64(np.float32(shape["rope_theta"])) ** (-2.0 * np.arange(hd // 2) / hd)
    factor = shape.get("rope_factor", 0.0)
    if factor > 1.0:
        lo, hi, old = shape["rope_low_freq_factor"], shape["rope_high_freq_factor"], float(shape["rope_original_max_pos"])
        wavelen = 2.0 * np.pi / inv
        smooth = (old / wavelen - lo) / (hi - lo)
        inv = np.where(wavelen > old / lo, inv / factor, np.where(wavelen < old / hi, inv, (1 - smooth) * inv / factor + smooth * inv))
    ang = np.asarray(positions, np.float64)[:, None] * inv[None, :]
    return np.cos(ang).astype(np.float32).astype(np.float64), np.sin(ang).astype(np.float32).astype(np.float64)


def exact_bf16(x):
    return f32(bf16(x)).astype(np.float64)


class Net:
    """Seeded weights of one layer shape, float64 copies of the exact bf16 values, layers generated on demand (every
    engine of a module shares them, so layer l of any depth is the same layer).  Gains are 1 + 0.3 N(0, 1); wq has 1.5 x the
    scale of the others and each kv head's K rows are 0.4 x the Q rows of the first query head of its group, so a token's
    own key (and earlier occurrences of its id in layer 0) carries real attention weight."""

    def __init__(self, shape, seed):
        self.shape, self.seed = dict(shape), seed
        d = shape["d_model"]
        rng = np.random.default_rng(seed)
        self.embed = exact_bf16(rng.standard_normal((VOCAB, d)))
        self.lm_head = exact_bf16(rng.standard_normal((VOCAB, d)) / np.sqrt(d))
        self.final_norm = exact_bf16(1 + 0.3 * rng.standard_normal(d))
        self._layers = {}

    def layer(self, l):
        if l not in self._layers:
            s = self.shape
            d, F, hd, H, G = s["d_model"], s["d_ff"], s["head_dim"], s["n_heads"], s["n_kv_heads"]
            rng = np.random.default_rng((self.seed, l))
            w = lambda n, k, sc=1.0: exact_bf16(rng.standard_normal((n, k)) * (sc / np.sqrt(k)))
            L = dict(ATTN_NORM=exact_bf16(1 + 0.3 * rng.standard_normal(d)), FFN_NORM=exact_bf16(1 + 0.3 * rng.standard_normal(d)),
                     WQ=w(H * hd, d, 1.5), WV=w(G * hd, d), WO=w(d, H * hd), WGATE=w(F, d), WUP=w(F, d), WDOWN=w(d, F))
            L["WK"] = exact_bf16(0.4 * L["WQ"].reshape(G, H // G, hd, d)[:, 0].reshape(G * hd, d))
            L["WQKV"] = np.concatenate([L["WQ"], L["WK"], L["WV"]])
            self._layers[l] = L
        return self._layers[l]

    def model(self, n_layers, **over):
        return dict(dict(self.shape, n_layers=n_layers, vocab_size=VOCAB, rms_eps=EPS), **over)

    def engine(self, n_layers=1, zero_branch0=False, **kw):
        """zero_branch0: layer 0's WO and WDOWN are zero, so layer 0 leaves every row's embedding unchanged (x + 0 is
        exact in fp32) and layer 1 sees the embedding as its input."""
        e = eng.Engine(model=self.model(n_layers), **kw)
        e.set_tensor(0, "EMBED", bf16(self.embed))
        e.set_tensor(0, "LM_HEAD", bf16(self.lm_head))
        e.set_tensor(0, "FINAL_NORM", bf16(self.final_norm))
        for l in range(n_layers):
            for kind in ("ATTN_NORM", "FFN_NORM", "WQ", "WK", "WV", "WO", "WGATE", "WUP", "WDOWN"):
                w = self.layer(l)[kind]
                e.set_tensor(l, kind, bf16(np.zeros_like(w) if zero_branch0 and l == 0 and kind in ("WO", "WDOWN") else w))
        return e


@functools.lru_cache(maxsize=None)
def net(name):
    return Net(dict(llama=LLAMA, mistral=MISTRAL, llama31=LLAMA31, tinyllama=TINYLLAMA, llama32=LLAMA32_1B, tiny=TINY)[name],
               seed=20240 + len(name))


def prompt_ids(seed, n):
    """Ids with many repeats (32 distinct values): earlier occurrences of the current id carry weight in layer 0, in pages
    and splits that move with the seed."""
    return np.random.default_rng(seed).integers(0, 32, size=n).astype(np.int32) * 16 + 3


# ---- float64 references and bounds (rows of a batch of observations at once) ------------------------------------------
def norm_round(h, gain, extra=0.0):
    """xn = bf16(rmsnorm(h) * gain) in float64 and, per element, the slack a kernel may differ by: one bf16 ulp where the
    float64 value lies within the kernel's fp32 error (REL_XN, plus `extra`, an absolute error already on h, carried
    through the norm) of a rounding boundary, 0 elsewhere."""
    inv = 1.0 / np.sqrt((h * h).mean(-1, keepdims=True) + EPS)
    x = h * inv * gain
    r = exact_bf16(x)
    u = ulp_bf16(x)
    band = REL_XN * np.abs(x) + np.abs(extra * inv * gain)
    if np.ndim(extra):                                     # an error on h also moves inv: relative |h . e| / |h|^2 <= |e| / |h|
        band = band + np.abs(x) * np.linalg.norm(extra, axis=-1, keepdims=True) / np.linalg.norm(h, axis=-1, keepdims=True)
    return r, np.where(u / 2 - np.abs(x - r) <= band, u, 0.0)


def proj(W, x, slack, c):
    """y = W x and its bound c * sum |w x| + sum_k |w_k| slack_k."""
    aW = np.abs(W)
    b = c * (np.abs(x) @ aW.T)
    if slack is not None and slack.any():
        b = b + slack @ aW.T
    return x @ W.T, b


def rope_ref(y, b, cos, sin, n_rot, hd):
    """Rotate-half RoPE of the first n_rot heads of y [R][heads * hd] (dims j, j + hd / 2 form a pair); later heads pass.
    Returns the unrounded reference and the bound before the bf16 rounding."""
    R, half = y.shape[0], hd // 2
    y, b = y.reshape(R, -1, hd), b.reshape(R, -1, hd)
    ref, tol = y.copy(), b.copy()
    y0, y1, b0, b1 = y[:, :n_rot, :half], y[:, :n_rot, half:], b[:, :n_rot, :half], b[:, :n_rot, half:]
    c, s = cos[:, None, :], sin[:, None, :]
    ref[:, :n_rot, :half], ref[:, :n_rot, half:] = y0 * c - y1 * s, y1 * c + y0 * s
    sl = ROPE_C * (np.abs(y0) + np.abs(y1))
    tol[:, :n_rot, :half], tol[:, :n_rot, half:] = b0 * np.abs(c) + b1 * np.abs(s) + sl, b1 * np.abs(c) + b0 * np.abs(s) + sl
    return ref.reshape(R, -1), tol.reshape(R, -1)


def ratio(got, ref, tol):
    return np.abs(np.asarray(got, np.float64) - ref) / tol


def stage1(nt, l, h_in, pos, c):
    """(reference, bound) of q | k | v [R][qkv_dim] as written: roped q and k, plain v, all rounded to bf16."""
    s, L = nt.shape, nt.layer(l)
    xn, slack = norm_round(h_in, L["ATTN_NORM"])
    y, b = proj(L["WQKV"], xn, slack, c)
    cos, sin = rope_table(s, pos)
    ref, tol = rope_ref(y, b, cos, sin, s["n_heads"] + s["n_kv_heads"], s["head_dim"])
    return ref, tol + ulp_bf16(ref)


def check_layer(nt, l, obs, C, page=32):
    """obs: arrays with one row per observed row — h_in, pos, q, k_new, v_new, attn, act, h_out; K, V: lists of caches,
    rows 0 .. (at least) pos of every row that reads them, and kv_seg, each row's index into K / V (default: one cache per
    row); optionally logits, of the rows logit_rows (default: all).  C: c_qkv, c_o, c_gu, c_dn, c_lm, and c_attn (default
    DECODE_C), h_adds (default 1).  Returns {stage: max err / bound per row} (stage 5: 0 on rows without logits)."""
    s, L = nt.shape, nt.layer(l)
    H, G, hd = s["n_heads"], s["n_kv_heads"], s["head_dim"]
    qd, kvd = H * hd, G * hd
    h_in = np.asarray(obs["h_in"], np.float64)
    pos = np.asarray(obs["pos"]).reshape(-1)
    out = {}
    ref, tol = stage1(nt, l, h_in, pos, C["c_qkv"])
    got = np.concatenate([obs["q"], obs["k_new"], obs["v_new"]], axis=1)
    r1 = ratio(got, ref, tol)
    out["1 q"], out["1 k"], out["1 v"] = r1[:, :qd].max(1), r1[:, qd:qd + kvd].max(1), r1[:, qd + kvd:].max(1)
    kv_seg = np.asarray(obs.get("kv_seg", np.arange(len(pos))))
    r2 = np.empty(len(pos))
    for g in np.unique(kv_seg):                            # one float64 attention per cache, with all of its rows
        i = np.flatnonzero(kv_seg == g)
        a_ref, pv = attn64(obs["q"][i], obs["K"][g].reshape(-1, G, hd), obs["V"][g].reshape(-1, G, hd), pos[i], H, G, hd, page=page)
        r2[i] = ratio(obs["attn"][i], a_ref, ulp_bf16(a_ref) + C.get("c_attn", DECODE_C) * pv).max(1)
    out["2 attn"] = r2
    attn, act = np.asarray(obs["attn"], np.float64), np.asarray(obs["act"], np.float64)
    o, b_o = proj(L["WO"], attn, None, C["c_o"])
    h_mid = h_in + o
    e_mid = b_o + U * np.abs(h_mid) * C.get("h_adds", 1)    # the kernel's fp32 h_mid: the projection's error + the add(s)
    xn, slack = norm_round(h_mid, L["FFN_NORM"], extra=e_mid)
    g, b_g = proj(L["WGATE"], xn, slack, C["c_gu"])
    u, b_u = proj(L["WUP"], xn, slack, C["c_gu"])
    sg = g / (1.0 + np.exp(-g))
    a_ref = sg * u
    tol = SILU_DERIV * b_g * np.abs(u) + np.abs(sg) * b_u + SILU_DERIV * b_g * b_u + silu_rel(g) * np.abs(a_ref) + ulp_bf16(a_ref)
    out["3 act"] = ratio(act, a_ref, tol).max(1)
    dn, b_d = proj(L["WDOWN"], act, None, C["c_dn"])
    h_ref = h_mid + dn
    hmax = np.maximum(np.maximum(np.abs(h_in), np.abs(h_mid)), np.abs(h_ref))
    out["4 h"] = ratio(obs["h_out"], h_ref, b_o + b_d + 2 * U * hmax * C.get("h_adds", 1)).max(1)
    if "logits" in obs:
        lr = np.asarray(obs.get("logit_rows", np.arange(len(pos))))
        xn, slack = norm_round(np.asarray(obs["h_out"], np.float64)[lr], nt.final_norm)
        lg, b_l = proj(nt.lm_head, xn, slack, C["c_lm"])
        out["5 logits"] = np.zeros(len(pos))
        out["5 logits"][lr] = ratio(obs["logits"], lg, b_l).max(1)
    return out


def report(name, labels, res):
    worst = {k: float(v.max()) for k, v in res.items()}
    for i, lab in enumerate(labels):
        print(f"[stages] {name} {lab}: " + "  ".join(f"{k} {v[i]:.3g}" for k, v in res.items()))
    print(f"[stages] {name} worst err/bound: " + "  ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, f"{name}: err / bound above 1: {bad}"
    return worst


def consts(shape, path):
    """path: "mega" | "ring" | "ldg" | "gemm" (batched step)."""
    d, F, qd = shape["d_model"], shape["d_ff"], shape["n_heads"] * shape["head_dim"]
    if path == "gemm":
        # h takes one add per split-K partial of the o and down projections (batch_resid_norm_kernel): up to 16 each
        return dict(c_qkv=gemm_c(d), c_o=gemm_c(qd), c_gu=gemm_c(d), c_dn=gemm_c(F), c_lm=gemm_c(d), h_adds=16)
    ring = path != "ldg"                                   # the persistent kernel's GEMV has the ring kernel's structure
    return dict(c_qkv=gemv_c(d, ring), c_o=gemv_c(qd, ring), c_gu=gemv_c(d, ring), c_dn=gemv_c(F, ring), c_lm=gemv_c(d, ring))


# ---- GPU: observations --------------------------------------------------------------------------------------------------
def observe_step(e, s, layer, tok, h_in, logits):
    """The buffers of sequence s after a single-sequence step that appended `tok`."""
    pos = e.seq_len(s) - 1
    K, V = e.debug_kv(s, layer, 0, 0, pos + 1), e.debug_kv(s, layer, 1, 0, pos + 1)
    return dict(h_in=h_in, pos=pos, q=e.debug_seq_hidden(s, "q"), k_new=K[pos], v_new=V[pos], K=K, V=V,
                attn=e.debug_seq_hidden(s, "attn"), act=e.debug_seq_hidden(s, "act"), h_out=e.debug_seq_hidden(s, "h"), logits=logits)


def stack(rows):
    return {k: ([r[k] for r in rows] if k in ("K", "V") else np.stack([r[k] for r in rows])) for k in rows[0]}


def scattered_seq(e, seed):
    """A live neighbour in slot 0 and a sequence in a later slot whose pages interleave with freed ones."""
    live, tmp, tmp2 = e.seq_create(), e.seq_create(), e.seq_create()
    e.prefill(live, prompt_ids(seed + 1, 70), want_logits=False)
    e.prefill(tmp, prompt_ids(seed + 2, 40), want_logits=False)
    e.prefill(tmp2, prompt_ids(seed + 3, 40), want_logits=False)
    e.seq_free(tmp)
    s = e.seq_create()
    assert s != 0 and s != live
    return live, tmp2, s


STEP_RUNS = [[0], [1], [31, 32, 33], [255, 256, 257], [4095, 4096, 4097], [8191]]   # first position -> consecutive steps


def run_single(nt, path, graph, runs, n_layers=1, h_in_of=None, monkeypatch=None):
    monkeypatch.setenv("CL_MEGA", "1" if path == "mega" else "0")
    monkeypatch.setenv("CL_GRAPH", "1" if graph else "0")
    rows, labels = [], []
    with nt.engine(n_layers, max_batch=4, decode_path=1 if path == "ldg" else 2, use_cuda_graph=graph) as e:
        assert e.runs_mega_kernel() == (path == "mega"), "the single-sequence step does not run the kernel this case is about"
        for run in runs:
            live, tmp2, s = scattered_seq(e, run[0])
            before = [e.debug_kv(live, n_layers - 1, w, 0, 70) for w in (0, 1)]
            ids = prompt_ids(run[0], run[0] + len(run))
            if run[0]:
                e.prefill(s, ids[:run[0]], want_logits=False)
            for p in run:
                logits, _ = e.decode_step(s, int(ids[p]))
                h_in = nt.embed[ids[p]] if h_in_of is None else h_in_of[p]
                rows.append(observe_step(e, s, n_layers - 1, int(ids[p]), h_in, logits))
                assert rows[-1]["pos"] == p
                labels.append(f"pos {p}")
            for w in (0, 1):
                np.testing.assert_array_equal(before[w], e.debug_kv(live, n_layers - 1, w, 0, 70), err_msg="a neighbour's K / V changed")
            for q in (live, tmp2, s):
                e.seq_free(q)
    return stack(rows), labels


@gpu
@pytest.mark.parametrize("path,graph", [("mega", True), ("mega", False), ("ring", True), ("ldg", True), ("ldg", False)])
def test_single_step_llama_layer(path, graph, monkeypatch):
    """Llama-3-8B layer shape: empty cache, page edges, split edges (16 splits of the 8-page split plan), the last RoPE row
    and block-table entry; three consecutive steps across 32 and 4096 (a counter left stale by one step shows on the next)."""
    nt = net("llama")
    runs = STEP_RUNS if graph else [[31, 32, 33], [4095, 4096, 4097]]
    obs, labels = run_single(nt, path, graph, runs, monkeypatch=monkeypatch)
    report(f"{path} graph {int(graph)}", labels, check_layer(nt, 0, obs, consts(nt.shape, path)))


@gpu
@pytest.mark.parametrize("name,pos", [("mistral", 8703), ("llama31", 20000)])
def test_single_step_rope_tables(name, pos, monkeypatch):
    """theta 1e6 at the last position of Mistral-7B's table, and the frequency-scaled table of Llama-3.1 at 20000."""
    nt = net(name)
    obs, labels = run_single(nt, "mega", True, [[pos]], monkeypatch=monkeypatch)
    report(f"mega {name}", labels, check_layer(nt, 0, obs, consts(nt.shape, "mega")))


@gpu
def test_single_step_layer_chain(monkeypatch):
    """Layers 0, 1, 2 of the persistent kernel: layer l of an (l + 1)-layer engine, its input the residual stream an l-layer
    engine left for the same token and cache (per-layer weight pointers, KV layer stride, barrier and tile counters)."""
    nt = net("llama")
    h_in_of = None
    for l in range(3):
        obs, labels = run_single(nt, "mega", True, [[33], [4096]], n_layers=l + 1, h_in_of=h_in_of, monkeypatch=monkeypatch)
        report(f"mega layer {l}", labels, check_layer(nt, l, obs, consts(nt.shape, "mega")))
        h_in_of = {int(p): obs["h_out"][i].astype(np.float64) for i, p in enumerate(obs["pos"])}


@gpu
@pytest.mark.parametrize("name", ["tinyllama", "llama32", "tiny"])
@pytest.mark.parametrize("path", ["ring", "ldg"])
def test_single_step_small_shapes(name, path, monkeypatch):
    """Per-op path only: head_dim 64 with 8 and 4 query heads per kv head, d_ff 5632 (LDG fallback of the ring path), 8192."""
    nt = net(name)
    obs, labels = run_single(nt, path, True, [[0], [31, 32], [600]], monkeypatch=monkeypatch)
    C = consts(nt.shape, path)
    report(f"{path} {name}", labels, check_layer(nt, 0, obs, C))


# ---- GPU: batched step --------------------------------------------------------------------------------------------------
def run_batched(nt, lens, monkeypatch, batch_gemm=True):
    B = len(lens)
    s = nt.shape
    monkeypatch.setenv("CL_BATCH_GEMM", "1" if batch_gemm else "0")
    pages = sum(-(-L // 32) for L in lens) + 2 * B + 8
    pool = pages * 32 * 2 * s["n_kv_heads"] * s["head_dim"] * 2
    with nt.engine(1, max_batch=max(B + 3, 4), kv_pool_bytes=pool) as e:
        seqs = [e.seq_create() for _ in range(B + 3)]
        for q in (seqs[0], seqs[2]):
            e.seq_free(q)
        outsider, seqs = seqs[1], seqs[3:]
        order = list(np.random.default_rng(B).permutation(B))
        seqs = [seqs[i] for i in order]                    # batch index != slot
        ids = [prompt_ids(100 + b, L) for b, L in enumerate(lens)]
        for q, t in zip(seqs + [outsider], ids + [prompt_ids(7, 40)]):
            if len(t) > 1:
                e.prefill(q, t[:-1], want_logits=False)
        e.decode_step(outsider, 5)
        out_before = [e.debug_seq_hidden(outsider, w) for w in ("h", "q")]
        kv_before = [[e.debug_kv(q, 0, w, 0, L - 1) if L > 1 else None for w in (0, 1)] for q, L in zip(seqs, lens)]
        logits, _ = e.decode_step_batch(seqs, [int(t[-1]) for t in ids])
        rows = []
        for b, (q, L) in enumerate(zip(seqs, lens)):
            K, V = e.debug_kv(q, 0, 0, 0, L), e.debug_kv(q, 0, 1, 0, L)
            for w, full in ((0, K), (1, V)):
                if L > 1:
                    np.testing.assert_array_equal(kv_before[b][w], full[:L - 1], err_msg="cached K / V below the length changed")
            attn = e.debug_seq_hidden(q, "attn")
            if batch_gemm:
                np.testing.assert_array_equal(bf16(e.debug_seq_hidden(q, "attn_bf16")), bf16(attn), err_msg="bf16 attention operand")
            act = e.debug_seq_hidden(q, "act_bf16" if batch_gemm else "act")
            rows.append(dict(h_in=nt.embed[ids[b][-1]], pos=L - 1, q=e.debug_seq_hidden(q, "q"), k_new=K[L - 1], v_new=V[L - 1], K=K, V=V,
                             attn=attn, act=act, h_out=e.debug_seq_hidden(q, "h"), logits=logits[b]))
        for w, before in zip(("h", "q"), out_before):
            np.testing.assert_array_equal(before.view(np.uint32), e.debug_seq_hidden(outsider, w).view(np.uint32),
                                          err_msg=f"{w} of a slot outside the batch changed")
    return stack(rows), [f"b {b} len {L}" for b, L in enumerate(lens)]


@gpu
@pytest.mark.parametrize("B", [2, 3, 8, 33, 100])
def test_batched_step_llama_layer(B, monkeypatch):
    nt = net("llama")
    lens = LONGCTX_B16[:B] if B <= 16 else _wide_lens(B)
    obs, labels = run_batched(nt, lens, monkeypatch)
    report(f"batched B {B}", labels, check_layer(nt, 0, obs, consts(nt.shape, "gemm")))


@gpu
def test_batched_step_gemv_fallback(monkeypatch):
    """CL_BATCH_GEMM=0: two sequences through the per-sequence GEMV kernels (grid y = batch)."""
    nt = net("llama")
    obs, labels = run_batched(nt, [4097, 33], monkeypatch, batch_gemm=False)
    report("batched B 2 GEMV", labels, check_layer(nt, 0, obs, consts(nt.shape, "ring")))


@gpu
def test_batched_step_head_dim_64(monkeypatch):
    """d 2048, head_dim 64: the CUDA-core attention at B = 3 and batch_resid_norm_kernel with one float4 per thread."""
    nt = net("llama32")
    obs, labels = run_batched(nt, [601, 33, 1], monkeypatch)
    report("batched B 3 d 2048", labels, check_layer(nt, 0, obs, consts(nt.shape, "gemm")))


# ---- GPU: every row of the multi-row passes (part d) ---------------------------------------------------------------------
# The split-K pass (small_pass: prompts of 16 .. 256 tokens, every verify pass) and the tile pass (prefill_pass: longer prompts,
# one per chunk, and cl_prefill_batch), read back through cl_debug_pass_info / cl_debug_pass_rows after the pass.
def pass_consts(shape, info, c_lm):
    """The wgmma constants; the tile path adds each residual projection to h once, in the GEMM epilogue (the split-K pass
    folds up to 16 partials); the prefill kernels round P to bf16, the multi-row verify kernel does not."""
    C = dict(consts(shape, "gemm"), c_lm=c_lm, c_attn=ATTN_C if info["attn"] == "verify" else PREFILL_C)
    if info["path"] == "tile":
        C["h_adds"] = 1
    return C


def sample_rows(info, seed):
    """The rows checked stage by stage: every row of a pass of up to 300 rows; of a longer one the first and last row of
    every 128-row tile and of every segment, and 64 seeded random rows.  (Stage 1 of K / V covers every row of every pass:
    check_pass.)"""
    T = info["T"]
    if T <= 300:
        return np.arange(T)
    edges = [r for t0 in range(0, T, 128) for r in (t0, min(t0 + 127, T - 1))]
    edges += [r for _, r0, n, _ in info["segs"] for r in (r0, r0 + n - 1)]
    return np.unique(np.concatenate([edges, np.random.default_rng(seed).choice(T, 64, replace=False)]))


def pass_rows(e, what, rows):
    """Rows `rows` (sorted) of the latest pass, one cl_debug_pass_rows call per run of consecutive rows."""
    cuts = np.flatnonzero(np.diff(rows) != 1) + 1
    return np.concatenate([e.debug_pass_rows(what, int(run[0]), len(run)) for run in np.split(rows, cuts)])


def kv_upto(e, s, layer, end):
    """K, V rows 0 .. end - 1 of sequence s: below its length through debug_kv which 0 / 1, past it (the rejected rows of a
    verify pass) through which 2 / 3."""
    n = min(e.seq_len(s), end)
    return [np.concatenate(([e.debug_kv(s, layer, w, 0, n)] if n else []) + ([e.debug_kv(s, layer, w + 2, n, end - n)] if end > n else []))
            for w in (0, 1)]


def observe_pass(e, nt, ids, layer=0, seed=0, logits=None, logit_rows=(), kept=None):
    """The latest pass's rows (sample_rows) with the K / V of their sequences.  ids: the pass's token ids in row order;
    logits: rows of the pass logit_rows; kept: rows of each segment its sequence kept (a verify pass), the others are
    reported apart as rejected.  Returns obs, the label of every row group and the pass info."""
    info = e.debug_pass_info()
    ids = np.asarray(ids)
    assert len(ids) == info["T"] and sum(g[2] for g in info["segs"]) == info["T"]
    rows = sample_rows(info, seed)
    lr = np.asarray(logit_rows, int)
    rows = np.union1d(rows, lr).astype(int)
    seg_of = np.concatenate([np.full(n, i) for i, (_, _, n, _) in enumerate(info["segs"])])[rows]
    pos = np.array([info["segs"][g][3] + r - info["segs"][g][1] for g, r in zip(seg_of, rows)])
    K, V = zip(*[kv_upto(e, q, layer, p0 + n) for q, _, n, p0 in info["segs"]])
    group_all, labels = np.zeros(info["T"], int), []      # the group of every row of the pass
    for i, (q, r0, n, p0) in enumerate(info["segs"]):
        a = n if kept is None else kept[i]
        group_all[r0:r0 + n] = len(labels)
        labels.append(f"seq {q} rows {r0}..{r0 + min(a, n) - 1} at {p0}" + (f" ({a} kept)" if kept is not None else ""))
        if a < n:
            group_all[r0 + a:r0 + n] = len(labels)
            labels.append(f"seq {q} rejected rows {r0 + a}..{r0 + n - 1} at {p0 + a}")
    obs = dict(h_in=nt.embed[ids[rows]], pos=pos, q=pass_rows(e, "q", rows), attn=pass_rows(e, "attn", rows),
               act=pass_rows(e, "act", rows), h_out=pass_rows(e, "h", rows), K=list(K), V=list(V), kv_seg=seg_of,
               k_new=np.stack([K[g][p] for g, p in zip(seg_of, pos)]), v_new=np.stack([V[g][p] for g, p in zip(seg_of, pos)]),
               group=group_all[rows], group_all=group_all)
    if logits is not None:
        obs["logits"], obs["logit_rows"] = np.asarray(logits).reshape(len(lr), -1), np.searchsorted(rows, lr)
    return obs, labels, info


def kv_rows_ratio(nt, l, ids, pos, K, V, c):
    """Stage 1 of the K and V rows [R][kv_dim] written for tokens ids at positions pos, whose layer input is their embedding
    row: max err / bound per row of K and of V.  Before RoPE a row depends on its id only, so the projection runs once per
    distinct id (prompt_ids has 32), and a pass of thousands of rows is checked whole."""
    s, L = nt.shape, nt.layer(l)
    qd = s["n_heads"] * s["head_dim"]
    uniq, inv = np.unique(ids, return_inverse=True)
    xn, slack = norm_round(nt.embed[uniq], L["ATTN_NORM"])
    y, b = proj(L["WQKV"][qd:], xn, slack, c)
    cos, sin = rope_table(s, pos)
    ref, tol = rope_ref(y[inv], b[inv], cos, sin, s["n_kv_heads"], s["head_dim"])
    r = ratio(np.concatenate([K, V], axis=1), ref, tol + ulp_bf16(ref))
    kvd = K.shape[1]
    return r[:, :kvd].max(1), r[:, kvd:].max(1)


def check_pass(name, nt, e, ids, expect, c_lm, layer=0, seed=0, **kw):
    """Asserts that the latest pass ran the path and attention kernel `expect`, checks every sampled row stage by stage,
    and stage 1 of the K / V of every row of the pass ("1 K all", "1 V all")."""
    obs, labels, info = observe_pass(e, nt, ids, layer, seed, **kw)
    assert (info["path"], info["attn"]) == expect, f"{name}: the pass ran {info['path']} / {info['attn']}, not {expect}"
    C = pass_consts(nt.shape, info, c_lm)
    res = check_layer(nt, layer, obs, C)
    grouped = {k: np.array([v[obs["group"] == g].max() for g in range(len(labels))]) for k, v in res.items()}
    segs = info["segs"]
    rk, rv = kv_rows_ratio(nt, layer, np.asarray(ids), np.concatenate([np.arange(p0, p0 + n) for _, _, n, p0 in segs]),
                           np.concatenate([obs["K"][i][p0:p0 + n] for i, (_, _, n, p0) in enumerate(segs)]),
                           np.concatenate([obs["V"][i][p0:p0 + n] for i, (_, _, n, p0) in enumerate(segs)]), C["c_qkv"])
    grouped["1 K all"] = np.array([rk[obs["group_all"] == g].max() for g in range(len(labels))])
    grouped["1 V all"] = np.array([rv[obs["group_all"] == g].max() for g in range(len(labels))])
    return report(f"{name} ({info['path']}, {info['attn']}, T {info['T']}, {len(obs['pos'])} rows)", labels, grouped)


def prefill_case(name, nt, e, ids, expect, prefix=None, layer=0):
    """A fresh sequence (after `prefix`, prefilled first), prefilled with ids; checks the pass and the last row's logits
    (cl_prefill's GEMV head).  A prompt longer than one chunk leaves its last chunk's pass."""
    s = e.seq_create()
    if prefix is not None:
        e.prefill(s, prefix, want_logits=False)
    lg = e.prefill(s, ids)
    info = e.debug_pass_info()
    T = info["T"]
    assert info["segs"] == [(s, 0, T, e.seq_len(s) - T)]
    check_pass(name, nt, e, np.asarray(ids)[len(ids) - T:], expect, gemv_c(nt.shape["d_model"], True), layer,
               seed=len(ids), logits=lg, logit_rows=[T - 1])
    e.seq_free(s)


@gpu
def test_split_k_pass_rows():
    """Llama-3-8B layer: prompts of 16, 40, 128, 129 and 256 tokens, a continuation 33 + 40 and 40 rows behind 4096 cached
    tokens, each through the split-K pass with the wgmma prefill attention."""
    nt = net("llama")
    with nt.engine(1, max_batch=4) as e:
        for n in (16, 40, 128, 129, 256):
            prefill_case(f"split-k {n}", nt, e, prompt_ids(n, n), ("split-k", "wgmma"))
        ids = prompt_ids(9, 33 + 40)
        prefill_case("split-k 33 + 40", nt, e, ids[33:], ("split-k", "wgmma"), prefix=ids[:33])
        ids = prompt_ids(11, 4096 + 40)
        prefill_case("split-k 4096 + 40", nt, e, ids[4096:], ("split-k", "wgmma"), prefix=ids[:4096])


@gpu
def test_tile_pass_rows():
    """Llama-3-8B layer: prompts of 257, 300, 1024 and 4096 tokens, a continuation 33 + 300, 300 rows behind 4096 cached
    tokens, the last chunk (700 rows at 4096) of a 4796-token prompt; Mistral-7B (theta 1e6) at 8192 with T = 300."""
    nt = net("llama")
    with nt.engine(1, max_batch=4) as e:
        for n in (257, 300, 1024, 4096):
            prefill_case(f"tile {n}", nt, e, prompt_ids(n, n), ("tile", "wgmma"))
        ids = prompt_ids(9, 33 + 300)
        prefill_case("tile 33 + 300", nt, e, ids[33:], ("tile", "wgmma"), prefix=ids[:33])
        ids = prompt_ids(12, 4096 + 300)
        prefill_case("tile 4096 + 300", nt, e, ids[4096:], ("tile", "wgmma"), prefix=ids[:4096])
        prefill_case("tile last chunk of 4796", nt, e, prompt_ids(13, 4096 + 700), ("tile", "wgmma"))
    nt = net("mistral")
    with nt.engine(1, max_batch=2) as e:
        ids = prompt_ids(14, 8192 + 300)
        prefill_case("mistral tile 8192 + 300", nt, e, ids[8192:], ("tile", "wgmma"), prefix=ids[:8192])


@gpu
@pytest.mark.parametrize("name,page", [("llama", 16), ("llama", 64), ("llama32", 32)])
def test_pass_rows_mma_prefill_attention(name, page):
    """The mma.sync prefill kernel, which the wgmma kernel leaves to pages 16 and 64 and to head_dim 64 (Llama-3.2-1B
    shape): a split-K and a tile pass, each behind a cached prefix."""
    nt = net(name)
    with nt.engine(1, max_batch=4, page_size=page) as e:
        ids = prompt_ids(page, 33 + 300)
        prefill_case(f"{name} page {page} split-k 40", nt, e, ids[:40], ("split-k", "mma"))
        prefill_case(f"{name} page {page} split-k 33 + 40", nt, e, ids[33:73], ("split-k", "mma"), prefix=ids[:33])
        prefill_case(f"{name} page {page} tile 300", nt, e, ids[:300], ("tile", "mma"))
        prefill_case(f"{name} page {page} tile 33 + 300", nt, e, ids[33:], ("tile", "mma"), prefix=ids[:33])


@gpu
def test_prefill_batch_pass_rows():
    """cl_prefill_batch of prompts of 1, 40, 300 and 1000 tokens in one tile pass (segments at rows 0, 1, 41, 341): rows of
    every segment and the last row of each, whose logits come from the batched wgmma head."""
    nt = net("llama")
    with nt.engine(1, max_batch=4) as e:
        seqs = [e.seq_create() for _ in range(4)]
        prompts = [prompt_ids(20 + i, n) for i, n in enumerate((1, 40, 300, 1000))]
        lg = e.prefill_batch(seqs, prompts)
        last = np.cumsum([len(p) for p in prompts]) - 1
        assert e.debug_pass_info()["segs"] == [(q, int(r - len(p) + 1), len(p), 0) for q, p, r in zip(seqs, prompts, last)]
        check_pass("prefill_batch 1 / 40 / 300 / 1000", nt, e, np.concatenate(prompts), ("tile", "wgmma"),
                   gemm_c(nt.shape["d_model"]), logits=lg, logit_rows=last)


def greedy_drafts(e, ids, x0, k, wrong, salt):
    """k drafts after x0 for a sequence holding ids: what greedy decoding of a twin emits, with draft `wrong` (if < k)
    replaced, so that the verify pass keeps the rows before it and rejects the rest."""
    if k == 0:
        return []
    twin = e.seq_create()
    e.prefill(twin, ids, want_logits=False)
    d = [int(t) for t in e.decode_greedy(twin, x0, k)[0]]
    e.seq_free(twin)
    if wrong < k:
        d[wrong] = (d[wrong] + 16 * (1 + salt % 7)) % VOCAB
    return d


def verify_case(name, nt, e, lens, ks, wrong, attn, batch=True, layer=0):
    """Sequences holding prompts of `lens` tokens, verified with ks drafts (partly wrong) in one decode_verify_batch pass, or
    (batch False) one decode_verify pass each.  Every row is checked, rejected ones through debug_kv which 2 / 3, and every
    row's logits (the verify pass's wgmma head).  Returns the number of rejected rows."""
    seqs = [e.seq_create() for _ in lens]
    prompts = [prompt_ids(100 * len(lens) + i, n) for i, n in enumerate(lens)]
    for q, p in zip(seqs, prompts):
        e.prefill(q, p, want_logits=False)
    x0 = [int(p[-1]) ^ 16 for p in prompts]
    drafts = [greedy_drafts(e, p, x, k, w, i) for i, (p, x, k, w) in enumerate(zip(prompts, x0, ks, wrong))]
    rejected = 0
    for grp in [list(range(len(lens)))] if batch else [[i] for i in range(len(lens))]:
        if batch:
            outs, lg = e.decode_verify_batch([seqs[i] for i in grp], [x0[i] for i in grp], [drafts[i] for i in grp], want_logits=True)
        else:
            out, lg = e.decode_verify(seqs[grp[0]], x0[grp[0]], drafts[grp[0]], want_logits=True)
            outs = [out]
        kept = [len(o) for o in outs]
        rejected += sum(ks[i] + 1 - a for i, a in zip(grp, kept))
        ids = np.concatenate([[x0[i]] + drafts[i] for i in grp])
        check_pass(f"{name} k {[ks[i] for i in grp]}", nt, e, ids, ("split-k", attn), gemm_c(nt.shape["d_model"]), layer,
                   logits=lg, logit_rows=np.arange(len(ids)), kept=kept)
    for q in seqs:
        e.seq_free(q)
    return rejected


@gpu
def test_verify_pass_rows():
    """cl_decode_verify with k = 1 and 15 (the per-segment prefill attention; rows 20 .. 35 cross a page boundary) and
    cl_decode_verify_batch over 2 and 8 sequences (the multi-row kernel; sequences behind 4096 cached tokens take 17
    splits), drafts right up to a wrong one: the rejected rows are checked too."""
    nt = net("llama")
    with nt.engine(1, max_batch=8, max_seqs=10) as e:
        rej = verify_case("verify", nt, e, [20, 60], [15, 1], [9, 0], "wgmma", batch=False)
        rej += verify_case("verify_batch B 2", nt, e, [40, 4096], [15, 6], [3, 4], "verify")
        rej += verify_case("verify_batch B 8", nt, e, [4096, 40, 17, 4100, 1, 300, 33, 64], [15, 3, 0, 7, 15, 1, 4, 9],
                           [5, 1, 0, 7, 12, 0, 2, 9], "verify")
    assert rej > 0, "no rejected row was checked"


@gpu
@pytest.mark.parametrize("page", [32, 64])
def test_pass_rows_layer_1(page):
    """A 2-layer engine whose layer 0 has WO = WDOWN = 0: layer 1's input is the embedding and the pass buffers hold layer
    1, so its rows check the per-layer pool offsets and tensor-map rows (l * n_pages * n_kv * page) of rope_scatter, of the
    prefill kernel (wgmma at page 32, mma.sync at 64) and of the multi-row verify kernel."""
    nt = net("llama")
    kern = "wgmma" if page == 32 else "mma"
    with nt.engine(2, zero_branch0=True, max_batch=4, page_size=page) as e:
        ids = prompt_ids(5, 33 + 300)
        prefill_case(f"layer 1 page {page} split-k 33 + 40", nt, e, ids[33:73], ("split-k", kern), prefix=ids[:33], layer=1)
        prefill_case(f"layer 1 page {page} tile 33 + 300", nt, e, ids[33:], ("tile", kern), prefix=ids[:33], layer=1)
        # the multi-row kernel takes page 32 only; at page 64 a verify pass runs the prefill kernel per segment
        verify_case(f"layer 1 page {page} verify_batch", nt, e, [300, 40], [15, 5], [6, 2], "verify" if page == 32 else "mma", layer=1)


@gpu
def test_pass_rows_on_prefix_cache_pages(monkeypatch):
    """CL_PREFIX_CACHE=1: 40- and 300-token suffixes prefilled on 256 attached tokens (split-K and tile pass)."""
    monkeypatch.setenv("CL_PREFIX_CACHE", "1")
    nt = net("llama")
    with nt.engine(1, max_batch=4) as e:
        A = prompt_ids(30, 256)
        x = e.seq_create()
        e.prefill(x, A, want_logits=False)
        e.seq_free(x)
        for n, path in ((40, "split-k"), (300, "tile")):
            Q = prompt_ids(31 + n, n)
            s = e.seq_create()
            assert e.attach_prefix(s, np.concatenate([A, Q])) == 256
            lg = e.prefill(s, Q)
            assert e.debug_pass_info()["segs"] == [(s, 0, n, 256)]
            check_pass(f"prefix cache 256 + {n}", nt, e, Q, (path, "wgmma"), gemv_c(nt.shape["d_model"], True),
                       logits=lg, logit_rows=[n - 1])
            e.seq_free(s)


@gpu
def test_pass_accessor_refuses():
    """No pass yet, a token-wise prefill since the last pass, a wrong selector or row range: CL_ERR_INVALID_ARG, never
    another pass's rows.  debug_kv which 2 / 3 stop at the end of the pages the sequence holds."""
    nt = net("tiny")
    with nt.engine(1, max_batch=2, page_size=16) as e:
        s = e.seq_create()
        for call in (e.debug_pass_info, lambda: e.debug_pass_rows("h", 0, 1)):
            with pytest.raises(eng.EngineError) as ei:
                call()
            assert ei.value.status == eng.CL_ERR_INVALID_ARG
        e.prefill(s, prompt_ids(1, 40), want_logits=False)
        assert e.debug_pass_info()["T"] == 40
        for what, r0, n in (("h", -1, 1), ("h", 0, 41), ("act", 40, 1), ("q", 0, 0)):
            with pytest.raises(eng.EngineError) as ei:
                e.debug_pass_rows(what, r0, n)
            assert ei.value.status == eng.CL_ERR_INVALID_ARG, (what, r0, n)
        out = np.empty(nt.shape["d_model"], np.float32)
        assert eng.lib().cl_debug_pass_rows(e._h, 4, 0, 1, eng._ptr(out)) == eng.CL_ERR_INVALID_ARG
        assert e.debug_kv(s, 0, 2, 40, 8).shape == (8, nt.shape["n_kv_heads"] * nt.shape["head_dim"])   # 48 = 3 pages
        for which, t0, n in ((2, 40, 9), (3, 0, 49), (1, 40, 1), (4, 0, 1)):
            with pytest.raises(eng.EngineError) as ei:
                e.debug_kv(s, 0, which, t0, n)
            assert ei.value.status == eng.CL_ERR_INVALID_ARG, (which, t0, n)
        e.prefill(s, prompt_ids(2, 3), want_logits=False)     # token-wise: decode steps, no multi-row pass
        for call in (e.debug_pass_info, lambda: e.debug_pass_rows("h", 0, 1)):
            with pytest.raises(eng.EngineError) as ei:
                call()
            assert ei.value.status == eng.CL_ERR_INVALID_ARG


# ---- CPU: the bounds hold for an honest float32 layer and catch every mutation -------------------------------------------
def pairwise32(W, x):
    """float32 GEMV with pairwise summation (another order than any kernel's)."""
    p = (W.astype(np.float32) * x.astype(np.float32)[None, :])
    while p.shape[1] > 1:
        if p.shape[1] & 1:
            p = np.concatenate([p[:, :-2], p[:, -2:-1] + p[:, -1:]], axis=1)
        p = p[:, 0::2] + p[:, 1::2]
    return p[:, 0]


def bf16r(x):
    return f32(bf16(np.asarray(x, np.float32)))


def layer32(nt, l, h_in, pos, K_prev, V_prev, mutate=None):
    """One decode step of layer l in float32 numpy with pairwise sums: the observation a correct kernel could produce.
    mutate names one defect (see MUTATIONS)."""
    s, L = nt.shape, nt.layer(l)
    H, G, hd, d, F = s["n_heads"], s["n_kv_heads"], s["head_dim"], s["d_model"], s["d_ff"]
    half, qd, kvd = hd // 2, H * hd, G * hd
    f = np.float32

    def norm(h, gain, eps=EPS, use_gain=True):
        h = h.astype(f)
        inv = f(1) / np.sqrt(np.sort(h * h).sum(dtype=f) / f(len(h)) + f(eps))
        return bf16r(h * inv * (gain.astype(f) if use_gain else f(1)))

    h_in = np.asarray(h_in, f)
    xn = norm(h_in, L["ATTN_NORM"], eps=0.0 if mutate == "no_eps" else EPS, use_gain=mutate != "no_gain")
    y = pairwise32(L["WQKV"], xn)
    if mutate == "splitk":                                  # one of four split-K partials (k 1024 .. 2047) left out of the sum
        y = y - pairwise32(L["WQKV"][:, 1024:2048], xn[1024:2048])
    yh = y.reshape(-1, hd)

    def rope(p):
        cos, sin = rope_table(s, [p])
        c, sn = cos[0].astype(f), sin[0].astype(f)
        return np.concatenate([yh[:H + G, :half] * c - yh[:H + G, half:] * sn, yh[:H + G, half:] * c + yh[:H + G, :half] * sn], axis=1)

    rot = rope({"rope_pos": pos + 1, "rope_rel": pos - ROPE_REL_POS0}.get(mutate, pos))
    q, k_new, v_new = bf16r(rot[:H].reshape(-1)), bf16r(rot[H:].reshape(-1)), bf16r(y[qd + kvd:])
    if mutate == "q_perm":                                  # the heads of the first group in another order
        q = q.reshape(H, hd)[[1, 0] + list(range(2, H))].reshape(-1)
    if mutate == "v_interleave":                            # V stored in the projection's rope-pair-interleaved column order
        v_new = v_new.reshape(G, 2, half).transpose(0, 2, 1).reshape(-1)
    K, V = np.concatenate([K_prev, k_new[None]]).astype(f), np.concatenate([V_prev, v_new[None]]).astype(f)
    am = {"drop_current": "current", "drop_page": "page"}.get(mutate)
    Ka, Va, qp = K, V, pos
    if mutate == "future_key":                              # the causal mask one key late: the next row (the same id) visible
        K, V = np.concatenate([K, bf16r(rope(pos + 1)[H:].reshape(1, -1))]), np.concatenate([V, v_new[None]])
        Ka, Va, qp = K, V, pos + 1
    if mutate == "other_seg":                               # another segment's sequence: its K / V rows 0 .. pos
        Ka, Va, _ = fake_cache(nt, 77, pos + 1)
    if mutate == "drop_split":                              # the split of pages 0 .. pps - 1 never reaches the combine
        pps = -(-(-(-(pos + 1) // 32)) // 16)
        Ka, Va, qp = K[pps * 32:], V[pps * 32:], pos - pps * 32
    a64, _ = attn64(q[None], Ka.reshape(-1, G, hd), Va.reshape(-1, G, hd), [qp], H, G, hd, mutate=am)
    attn = bf16r(a64[0])
    # neighbour_row: the o-projection adds another row's residual.  In a pass, a row offset off by one reads the neighbouring
    # token's row, which in layer 0 is the same embedding whenever the two ids agree (1 in 32 for prompt_ids), and then that
    # row cannot show the defect; the pass's other rows do.  The mutation takes id 7, which no prompt_ids id is (3 mod 16),
    # to stand for the rows that can show it.
    h_mid = (np.asarray(nt.embed[7], f) if mutate == "neighbour_row" else h_in) + pairwise32(L["WO"], attn)
    if mutate == "resid_twice":                             # Y aliases resid: the residual added twice
        h_mid = h_mid + h_in
    xn2 = norm(h_in if mutate == "stale_xn" else h_mid, L["FFN_NORM"])
    g, u = pairwise32(L["WGATE"], xn2), pairwise32(L["WUP"], xn2)
    act = bf16r(g / (f(1) + np.exp(-g)) * u)
    dn = pairwise32(L["WDOWN"], act)
    if mutate == "row_dropped":
        dn[5] = 0
    if mutate == "row_twice":
        dn[5] *= 2
    if mutate == "k_slice":
        dn[5] -= pairwise32(L["WDOWN"][5:6, 4096:8192], act[4096:8192])[0]
    h_out = h_mid + dn
    lg = pairwise32(nt.lm_head, norm(h_out, nt.final_norm))
    return dict(h_in=h_in.astype(np.float64), pos=pos, q=q, k_new=k_new, v_new=v_new, K=K, V=V, attn=attn, act=act, h_out=h_out, logits=lg)


def fake_cache(nt, seed, n):
    """A plausible layer-0 cache: K / V rows of a repeated-id prompt, computed in float64 from stage 1."""
    if n == 0:
        kvd = nt.shape["n_kv_heads"] * nt.shape["head_dim"]
        return np.zeros((0, kvd), np.float32), np.zeros((0, kvd), np.float32), prompt_ids(seed, 1)
    ids = prompt_ids(seed, n + 1)
    uniq, inv = np.unique(ids[:n], return_inverse=True)
    ref, _ = stage1(nt, 0, nt.embed[uniq], np.zeros(len(uniq)), 0.0)
    s = nt.shape
    qd, kvd, hd = s["n_heads"] * s["head_dim"], s["n_kv_heads"] * s["head_dim"], s["head_dim"]
    k0, v = ref[inv, qd:qd + kvd], ref[inv, qd + kvd:]
    cos, sin = rope_table(s, np.arange(n))
    k, _ = rope_ref(k0, np.zeros_like(k0), cos, sin, s["n_kv_heads"], hd)
    return bf16r(k), bf16r(v), ids


@pytest.mark.parametrize("name,pos", [("llama", 0), ("llama", 33), ("llama", 4096), ("tinyllama", 600), ("llama32", 32), ("tiny", 31),
                                      ("llama", 4395)])
def test_float32_layer_stays_inside_every_bound(name, pos):
    """Rehearsal that no bound is too tight: a float32 layer with pairwise sums against the tightest constants of any path,
    and against the tile pass's (one residual add, the prefill attention constant: the last row of 4096 + 300)."""
    nt = net(name)
    K, V, ids = fake_cache(nt, pos, pos)
    obs = stack([layer32(nt, 0, nt.embed[ids[pos]], pos, K, V)])
    tile = dict(consts(nt.shape, "gemm"), h_adds=1, c_attn=PREFILL_C)
    for path, C in (("ring", consts(nt.shape, "ring")), ("ldg", consts(nt.shape, "ldg")), ("tile", tile)):
        worst = report(f"float32 {name} {path}", [f"pos {pos}"], check_layer(nt, 0, obs, C))
        assert max(worst.values()) > 0.01                   # and none is idle: the bf16 stages sit near half an ulp


# mutation -> (stage that must see it, least err / bound); the second line: the defects of the multi-row passes
MUTATIONS = {
    "row_dropped": ("4 h", 10), "row_twice": ("4 h", 10), "k_slice": ("4 h", 10), "stale_xn": ("3 act", 10),
    "no_gain": ("1 q", 10), "rope_pos": ("1 k", 10), "q_perm": ("1 q", 10), "v_interleave": ("1 v", 10),
    "drop_current": ("2 attn", 4), "drop_page": ("2 attn", 4), "drop_split": ("2 attn", 4), "splitk": ("1 v", 10),
    "future_key": ("2 attn", 4), "rope_rel": ("1 k", 10), "other_seg": ("2 attn", 4), "resid_twice": ("4 h", 10),
    "neighbour_row": ("4 h", 10),
}
ROPE_REL_POS0 = 4096                                       # rope_rel: RoPE at pos - pos0, as if positions restarted per chunk


@pytest.mark.parametrize("mutate", sorted(MUTATIONS))
def test_bounds_catch_mutation(mutate):
    """The widest constants of the decode paths (the GEMM's, 16 residual adds, DECODE_C) and of the multi-row passes (the
    same with the prefill kernels' attention constant PREFILL_C, 128 x DECODE_C) still put each defect outside its stage's
    bound by the stated factor."""
    nt = net("llama")
    pos = 4096
    K, V, ids = fake_cache(nt, 1, pos)
    obs = stack([layer32(nt, 0, nt.embed[ids[pos]], pos, K, V, mutate=mutate)])
    stage, least = MUTATIONS[mutate]
    for name, C in (("decode", consts(nt.shape, "gemm")), ("pass", dict(consts(nt.shape, "gemm"), c_attn=PREFILL_C))):
        res = check_layer(nt, 0, obs, C)
        print(f"[power] {mutate} {name}: " + "  ".join(f"{k} {v[0]:.3g}" for k, v in res.items()))
        assert res[stage][0] >= least, (mutate, name, res[stage][0])


def test_bounds_catch_missing_eps_at_small_norm():
    """An input of rms 1e-3 (mean square 1e-6 against eps 1e-5): without eps the norm is 3.3 x too large."""
    nt = net("llama")
    h = nt.embed[3] * 1e-3
    obs = stack([layer32(nt, 0, h, 0, *fake_cache(nt, 0, 0)[:2], mutate="no_eps")])
    res = check_layer(nt, 0, obs, consts(nt.shape, "gemm"))
    assert res["1 v"][0] >= 100, res


def test_rope_shift_is_caught_on_the_pairs_that_can_show_it():
    """K roped at pos + 1: pair i turns by theta^(-2i / head_dim) rad more, which moves a value by at most that times
    |y0| + |y1|.  Below about half a bf16 ulp (2^-9) the rounding hides it: at theta 5e5 that is every pair from i = 31
    on, at any position — a wrong row index of the table cannot show there, only a wrong table can (which pos 8191, 8703
    and 20000 check).  The pairs below 24 must each exceed the bound."""
    nt = net("llama")
    pos = 4096
    K, V, ids = fake_cache(nt, 1, pos)
    obs = stack([layer32(nt, 0, nt.embed[ids[pos]], pos, K, V, mutate="rope_pos")])
    ref, tol = stage1(nt, 0, obs["h_in"], obs["pos"], gemm_c(4096))
    r = ratio(obs["k_new"], ref[:, 4096:5120], tol[:, 4096:5120]).reshape(8, 2, 64).max(axis=(0, 1))
    assert (r[:24] > 1.0).all(), r[:24]
    assert 4096 * 5e5 ** (-2 * 31 / 128) < 2.0 ** -9 * 4096


def test_rope_at_segment_relative_position_is_caught():
    """K roped at pos - pos0 (positions restarting at a chunk or segment): at pos 4096, pos0 4096 pair i is off by a turn of
    4096 theta^(-2i / head_dim) rad, which moves a value by 2 |sin(turn / 2)| (|y0| + |y1|) at most.  Every pair whose turn
    moves it by more than 2^-5 of that must exceed the bound; that is pairs 0 .. 50 at theta 5e5 save those whose turn
    lands near a multiple of 2 pi."""
    nt = net("llama")
    pos = 4096
    K, V, ids = fake_cache(nt, 1, pos)
    obs = stack([layer32(nt, 0, nt.embed[ids[pos]], pos, K, V, mutate="rope_rel")])
    ref, tol = stage1(nt, 0, obs["h_in"], obs["pos"], gemm_c(4096))
    r = ratio(obs["k_new"], ref[:, 4096:5120], tol[:, 4096:5120]).reshape(8, 2, 64).max(axis=(0, 1))
    turn = ROPE_REL_POS0 * np.float64(np.float32(5e5)) ** (-2.0 * np.arange(64) / 128)
    shows = 2 * np.abs(np.sin(turn / 2)) > 2.0 ** -5
    assert shows.sum() >= 40, shows.sum()
    assert (r[shows] > 1.0).all(), np.flatnonzero(shows & (r <= 1.0))
