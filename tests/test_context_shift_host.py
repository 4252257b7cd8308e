"""CPU-only tests of the context shift: the paged-KV allocator's part (cl_kvpool_shift) against a Python model of its rules,
with the prefix index and its host tier, and the oracle's restatement of the K rotation against float64 (with two wrong
rotations that the bound must catch)."""
import random

import numpy as np
import pytest

from crowdllama_b200 import engine as eng
from oracle import oracle as oc
import shift_util as su


def _model_shift(pages, length, keep, discard, P):
    """The rules of cl_kvpool_shift on a page list: (kept entries, dropped entries, the written old entries with their rows,
    the partial item (source entry, rows) or None)."""
    k0, r, d = keep // P, keep % P, discard // P
    used = -(-length // P)
    head = k0 + (1 if r else 0)
    tail = head + d
    part_end = min(P, length - (k0 + d) * P) if r else 0
    part = (k0 + d, r, part_end) if part_end > r else None
    rotated = [(j, min(P, length - j * P)) for j in range(tail, used)]
    return list(range(head)) + list(range(tail, len(pages))), list(range(head, tail)), rotated, part


def _ids(n, salt):
    return [(i * 7919 + 13 + salt * 104729) % 500 + 3 for i in range(n)]


@pytest.mark.parametrize("P", [16, 32, 64])
def test_private_pages_shift_in_place(P):
    rng = random.Random(P)
    for _ in range(60):
        pool = eng.KvPool(256, P)
        pool.reserve(7, rng.randrange(0, 5) * P)               # another owner, so the sequence's pages are not 0..n
        length = rng.randrange(2 * P, 40 * P)
        extra = rng.choice([0, 1])
        assert pool.reserve(0, length + extra) == 0
        before = pool.pages_of(0)
        keep = rng.choice([0, 4, P - 1, P, P + 3, rng.randrange(0, length - P)])
        keep = min(keep, length - P)
        discard = P * rng.randrange(1, (length - keep) // P + 1)
        free0 = pool.free_pages
        rc, items = pool.shift(0, length, keep, discard)
        assert rc == 0
        kept, dropped, rotated, part = _model_shift(before, length, keep, discard, P)
        after = pool.pages_of(0)
        assert after == [before[j] for j in kept]
        assert pool.free_pages == free0 + len(dropped)
        want = []
        if part:
            want.append((before[part[0]], before[keep // P], part[1], part[2], 1))
        want += [(before[j], before[j], 0, rows, 1) for j, rows in rotated]
        assert items == want
        assert pool.release(0) == 0 and pool.release(7) == 0
        assert pool.used_pages == 0 and pool.free_pages == 256


@pytest.mark.parametrize("P", [16, 32])
def test_bad_arguments_change_nothing(P):
    pool = eng.KvPool(64, P)
    pool.reserve(0, 10 * P)
    before, free0 = pool.pages_of(0), pool.free_pages
    for keep, discard, length in [(4, P + 1, 10 * P), (4, 0, 10 * P), (-1, P, 10 * P), (9 * P + 1, P, 10 * P), (0, P, 11 * P)]:
        rc, items = pool.shift(0, length, keep, discard)
        assert rc == -1 and items == []
        assert pool.pages_of(0) == before and pool.free_pages == free0
    assert pool.shift(3, P, 0, P)[0] == -1                       # no such owner


def _check_index_invariant(pool, prompts, P, owner_pages):
    """Every prompt's attach finds exactly the pages that were published for it (owner_pages[i]: the original pages)."""
    for i, ids in enumerate(prompts):
        o = 100 + i
        n = pool.attach(o, ids + [1])
        got = pool.pages_of(o)
        assert n == len(ids) // P * P
        assert got == owner_pages[i][:len(got)], (i, got, owner_pages[i])
        pool.release(o)


@pytest.mark.parametrize("host_pages", [0, 64])
@pytest.mark.parametrize("P", [16, 32])
@pytest.mark.parametrize("keep", [0, 4, 16, 19])
def test_shared_and_indexed_pages_are_copied(P, keep, host_pages):
    """Owner A publishes a prompt; B attaches its prefix (shared pages), extends it and publishes a cached descendant;
    C holds its own published pages.  B and C shift: every page they write is a fresh page, A's and the index's pages keep
    their bytes' owners, and attach of the original ids still finds the original pages."""
    keep = min(keep, P + 3)
    pool = eng.KvPool(200, P)
    pool.set_host_pages(host_pages)
    A = _ids(8 * P, 1)
    pool.reserve(0, len(A))
    pool.publish(0, A)
    a_pages = pool.pages_of(0)
    B = A[:6 * P] + _ids(4 * P, 2)                              # shares 6 pages with A, then its own
    assert pool.attach(1, B) == 6 * P
    pool.reserve(1, len(B) + 1)
    pool.publish(1, B)
    b_pages = pool.pages_of(1)
    assert b_pages[:6] == a_pages[:6]
    C = _ids(10 * P, 3)
    pool.reserve(2, len(C))
    pool.publish(2, C)
    c_pages = pool.pages_of(2)
    moves0 = pool.take_moves()
    assert moves0 == []
    for owner, ids, pages in ((1, B, b_pages), (2, C, c_pages)):
        length = len(ids)
        discard = 4 * P
        rc, items = pool.shift(owner, length, keep, discard)
        assert rc == 0
        kept, dropped, rotated, part = _model_shift(pages, length, keep, discard, P)
        after = pool.pages_of(owner)
        assert len(after) == len(kept)
        written = {it[1] for it in items}
        # every written page is new: no other owner's page, no indexed original
        assert not written & set(a_pages) and not written & set(pages)
        # the unwritten head is the original
        assert after[:keep // P] == pages[:keep // P]
        # copy-on-write items read the originals, at the right rows
        srcs = [it for it in items if it[4] == 1]
        want_src = ([pages[part[0]]] if part else []) + [pages[j] for j, _ in rotated]
        assert [it[0] for it in srcs] == want_src
        copies = [it for it in items if it[4] == 0]
        if part:
            assert copies == [(pages[keep // P], after[keep // P], 0, keep % P, 0)]
        else:
            assert copies == []
        # publishing after a shift indexes nothing
        cached0 = pool.cached_pages
        pool.publish(owner, ids[:keep] + ids[keep + discard:])
        pool.release(owner)
        assert pool.cached_pages >= cached0
        for p in written:
            assert p not in pool.pages_of(0)
    # the original pages still answer the original ids (B's descendant chain too), never the shifted copies
    pool.release(0)
    _check_index_invariant(pool, [A, B, C], P, [a_pages, b_pages, c_pages])
    assert pool.used_pages == 0
    assert pool.free_pages == 200


@pytest.mark.parametrize("P", [16, 32])
def test_copy_on_write_needs_free_pages(P):
    pool = eng.KvPool(12, P)
    A = _ids(10 * P, 4)
    pool.reserve(0, len(A))
    pool.publish(0, A)
    pool.reserve(1, 2 * P)                                      # the pool is full
    before = pool.pages_of(0)
    rc, _ = pool.shift(0, len(A), 4, 2 * P)
    assert rc == -4                                             # CL_ERR_OOM: needs 8 copies, none free
    assert pool.pages_of(0) == before
    pool.release(1)                                             # 2 free: still too few
    assert pool.shift(0, len(A), 4, 2 * P)[0] == -4
    pool.release(0)
    assert pool.used_pages == 0


@pytest.mark.parametrize("P", [16, 32])
def test_host_tier_evictions_for_copies(P):
    """Copies that evict cached pages spill them to the host tier first; the spilled entries still answer their ids."""
    pool = eng.KvPool(16, P)
    pool.set_host_pages(8)
    old = _ids(6 * P, 5)
    pool.reserve(5, len(old))
    pool.publish(5, old)
    old_pages = pool.pages_of(5)
    pool.release(5)                                             # 6 cached pages
    A = _ids(8 * P, 6)
    pool.reserve(0, len(A))
    pool.publish(0, A)
    assert pool.take_moves() == []
    rc, items = pool.shift(0, len(A), 0, 2 * P)                 # 6 copies: 2 free pages, then 4 evictions
    assert rc == 0
    moves = pool.take_moves()
    assert len(moves) == 4 and all(m[0] == 0 for m in moves)
    assert {m[1] for m in moves} <= set(old_pages)
    assert {it[1] for it in items} & set(pool.pages_of(0))
    pool.release(0)
    assert pool.attach(9, old + [1]) == 6 * P                  # 4 fills from the host, 2 still on the device
    pool.release(9)
    assert pool.used_pages == 0


def _rand_k(rng, shape):
    return oc.np_bf16_round(rng.standard_normal(shape).astype(np.float32) * 3)


@pytest.mark.parametrize("preset", ["tiny-test", "llama3.1-8b"])
def test_rotation_matches_float64(preset):
    cfg = dict(oc.PRESETS[preset])
    tab = su.rope_table(cfg, 8192)
    rng = np.random.default_rng(5)
    k = _rand_k(rng, (3, 64, 2, cfg["head_dim"]))
    for delta in (16, 32, 992, 4064, 4096):
        cs = tab[delta]
        assert su.shift_err(su.rotate_back(k, cs), k, cs) <= 1.0


def test_bounds_catch_wrong_rotations():
    cfg = dict(oc.PRESETS["llama3-8b"])
    tab = su.rope_table(cfg, 8192)
    rng = np.random.default_rng(6)
    k = _rand_k(rng, (2, 64, 2, 128))
    for delta in (32, 4064):
        cs = tab[delta]
        plus = tab[delta] * np.array([1.0, -1.0], np.float32)     # R(+delta)
        assert su.shift_err(su.rotate_back(k, plus), k, cs) > 4.0
        for off in (-1, 1):
            assert su.shift_err(su.rotate_back(k, tab[delta + off]), k, cs) > 4.0


def test_numpy_table_is_the_oracles():
    for preset in ("tiny-test",):
        cfg = dict(oc.PRESETS[preset])
        m = oc.Model(cfg, seed=1)
        assert np.array_equal(su.oracle_rope_table(m), su.rope_table(cfg, cfg["max_seq_len"]))
    cfg = dict(oc.PRESETS["tiny-test"], rope_factor=8.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0,
               rope_original_max_pos=64, rope_theta=5e5)
    m = oc.Model(cfg, seed=1)
    assert np.abs(su.oracle_rope_table(m) - su.rope_table(cfg, cfg["max_seq_len"])).max() < 1e-6


@pytest.mark.parametrize("keep", [0, 4, 17])
def test_oracle_shift_against_float64(keep):
    """oracle_shift on a prefilled oracle sequence: positions < keep exact, V moved exactly, K within the bound."""
    cfg = dict(oc.PRESETS["tiny-test"])
    m = oc.Model(cfg, seed=11)
    s = m.new_seq()
    ids = np.array(_ids(200, 7), np.int32)
    s.forward(ids)
    L = cfg["n_layers"]
    K0 = [s.kv(l, 0, 0, 200) for l in range(L)]
    V0 = [s.kv(l, 1, 0, 200) for l in range(L)]
    tab = su.oracle_rope_table(m)
    delta = 64
    su.oracle_shift(s, keep, delta)
    assert len(s) == 200 - delta
    hd = cfg["head_dim"]
    for l in range(L):
        K1, V1 = s.kv(l, 0, 0, 200 - delta), s.kv(l, 1, 0, 200 - delta)
        assert np.array_equal(K1[:keep], K0[l][:keep]) and np.array_equal(V1[:keep], V0[l][:keep])
        assert np.array_equal(V1[keep:], V0[l][keep + delta:])
        old = K0[l][keep + delta:].reshape(-1, cfg["n_kv_heads"], hd)
        assert su.shift_err(K1[keep:].reshape(old.shape), old, tab[delta]) <= 1.0
        assert np.array_equal(K1[keep:].reshape(old.shape), su.rotate_back(old, tab[delta]))   # the engine's roundings
