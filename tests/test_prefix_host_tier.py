"""CPU-only tests of the prefix cache's host tier in the paged-KV allocator (cl_kvpool_set_host_pages / take_moves /
host_cached_pages): randomised runs against a Python model of the tier's rules, with the page contents simulated by
executing the recorded moves in order, plus directed cases for the two order hazards."""
import random

import pytest

from crowdllama_b200 import engine as eng
from test_prefix_pool import PoolModel, check_state

SPILL, FILL = 0, 1


class TierModel:
    """The allocator's rules with a host tier of H pages.  An index entry (key -> [location, uid]) lives on a device page
    (location >= 0) or a host page h (location ~h).  Evicting a cached device page moves its entry to a free host page, or
    to the host LRU front's page after dropping that entry, or erases it when the tier has no page to give.  attach takes
    the longest prefix of the chain whose host entries can all get a device page now, protects the chain, then fills
    its host entries in chain order."""

    def __init__(self, n_pages, page, H):
        self.n, self.P, self.H = n_pages, page, H
        self.free = list(range(n_pages - 1, -1, -1))
        self.ref = [0] * n_pages
        self.key = [None] * n_pages       # index key of the entry on a device page
        self.hkey = [None] * H            # index key of the entry on a host page
        self.hfree = list(range(H - 1, -1, -1))
        self.index = {}                   # key -> [loc, uid]
        self.lru, self.hlru = [], []
        self.owned, self.chain = {}, {}
        self.next_uid = 1
        self.moves = []
        self.to_host = self.from_host = 0

    def take_host(self):
        if self.hfree:
            return self.hfree.pop()
        if self.hlru:
            h = self.hlru.pop(0)
            del self.index[self.hkey[h]]
            self.hkey[h] = None
            return h
        return None

    def take_page(self):
        if self.free:
            return self.free.pop()
        p = self.lru.pop(0)
        key, self.key[p] = self.key[p], None
        h = self.take_host()
        if h is None:
            del self.index[key]
        else:
            self.index[key][0] = ~h
            self.hkey[h] = key
            self.hlru.append(h)
            self.moves.append((SPILL, p, h))
            self.to_host += 1
        return p

    def reserve(self, o, n):
        v = self.owned.setdefault(o, [])
        extra = -(-n // self.P) - len(v)
        if extra <= 0:
            return 0
        if extra > len(self.free) + len(self.lru):
            return eng.CL_ERR_OOM
        for _ in range(extra):
            p = self.take_page()
            self.ref[p] = 1
            v.append(p)
        return 0

    def release(self, o):
        self.chain.pop(o, None)
        for p in reversed(self.owned.pop(o, [])):
            self.ref[p] -= 1
            if self.ref[p] == 0:
                (self.lru if self.key[p] is not None else self.free).append(p)

    def walk(self, ids):
        locs, parent = [], 0
        for k in range((len(ids) - 1) // self.P if len(ids) > 1 else 0):
            e = self.index.get((parent, tuple(ids[k * self.P:(k + 1) * self.P])))
            if e is None:
                break
            locs.append(e[0])
            parent = e[1]
        return locs

    def lookup(self, ids):
        locs = self.walk(ids)
        return len(locs) * self.P, sum(1 for l in locs if l < 0 or self.ref[l] == 0)

    def attach(self, o, ids):
        if self.owned.get(o):
            return None
        locs, avail, k = self.walk(ids), len(self.free) + len(self.lru), 0
        while k < len(locs):
            if locs[k] < 0 or self.ref[locs[k]] == 0:
                if avail == 0:
                    break
                avail -= 1
            k += 1
        locs = locs[:k]
        for l in locs:
            if l >= 0:
                if self.ref[l] == 0:
                    self.lru.remove(l)
                self.ref[l] += 1
            else:
                self.hlru.remove(~l)
        v = []
        for l in locs:
            if l >= 0:
                v.append(l)
                continue
            h, p = ~l, self.take_page()
            key, self.hkey[h] = self.hkey[h], None
            self.index[key][0] = p
            self.key[p] = key
            self.ref[p] = 1
            self.moves.append((FILL, p, h))
            self.from_host += 1
            self.hfree.append(h)
            v.append(p)
        self.owned[o] = v
        self.chain[o] = [len(v), self.index[self.key[v[-1]]][1] if v else 0]
        return len(v) * self.P

    def publish(self, o, ids, n_known):
        if o not in self.owned:
            return
        v, c = self.owned[o], self.chain.setdefault(o, [0, 0])
        k = c[0]
        while k < len(v) and (k + 1) * self.P <= n_known:
            key = (c[1], tuple(ids[k * self.P:(k + 1) * self.P]))
            if key in self.index:
                c[1] = self.index[key][1]
            else:
                self.index[key] = [v[k], self.next_uid]
                self.key[v[k]] = key
                self.next_uid += 1
                c[1] = self.index[key][1]
            k += 1
            c[0] = k


class Contents:
    """What the device and host pages hold, driven the way the engine drives them: the moves run in the order recorded,
    then the owner writes the pages it reserved; publishing names a page by the uid of its entry."""

    def __init__(self, n_pages, H):
        self.dev, self.host = [None] * n_pages, [None] * H

    def run(self, moves):
        for kind, p, h in moves:
            if kind == SPILL:
                self.host[h] = self.dev[p]
            else:
                self.dev[p] = self.host[h]

    def check(self, m):
        for key, (loc, uid) in m.index.items():
            got = self.dev[loc] if loc >= 0 else self.host[~loc]
            assert got == ("entry", key), (key, loc, got)


def check_tier(pool, m):
    held = {p for v in m.owned.values() for p in v}
    for o, v in m.owned.items():
        assert pool.pages_of(o) == v, (o, pool.pages_of(o), v)
    cached, free = set(m.lru), set(m.free)
    assert not (held & cached) and not (held & free) and not (cached & free)
    assert len(held) + len(cached) + len(free) == m.n                      # no device page leaks
    hcached, hfree = set(m.hlru), set(m.hfree)
    assert not (hcached & hfree) and len(hcached) + len(hfree) == m.H        # no host page leaks
    assert all(m.hkey[h] is not None for h in hcached) and all(m.hkey[h] is None for h in hfree)
    # the index: every entry sits where its page says it does, and nowhere else
    assert len(m.index) == sum(k is not None for k in m.key) + len(hcached)
    for key, (loc, _) in m.index.items():
        assert (m.key[loc] if loc >= 0 else m.hkey[~loc]) == key
    assert pool.used_pages == len(held) and pool.cached_pages == len(cached) and pool.host_cached_pages == len(hcached)
    assert pool.free_pages + pool.used_pages == m.n


def publish_both(pool, m, c, o, ids, n_known):
    before = set(m.index)
    pool.publish(o, ids, n_known)
    m.publish(o, ids, n_known)
    for key in set(m.index) - before:
        c.dev[m.index[key][0]] = ("entry", key)      # the owner computed this page's K/V before publishing it


def reserve_both(pool, m, c, o, n):
    before = len(m.owned.get(o, []))
    rc = pool.reserve(o, n)
    assert rc == m.reserve(o, n)
    moves = pool.take_moves()
    assert moves == m.moves, (moves, m.moves)
    c.run(moves)
    m.moves = []
    for p in m.owned.get(o, [])[before:]:
        c.dev[p] = ("written", o)                      # kernels then write the new pages
    return rc, moves


def attach_both(pool, m, c, o, ids):
    want_tokens, want_cached = m.lookup(ids)
    got = pool.attach(o, ids)
    assert got == m.attach(o, ids)
    moves = pool.take_moves()
    assert moves == m.moves, (moves, m.moves)
    c.run(moves)
    m.moves = []
    assert got <= want_tokens
    return got, moves


@pytest.mark.parametrize("page,n_pages,H,seed", [(4, 24, 8, 0), (4, 40, 3, 1), (8, 16, 16, 2), (2, 64, 40, 3), (4, 20, 1, 4)])
def test_host_tier_matches_model(page, n_pages, H, seed):
    rng = random.Random(seed)
    pool, m, c = eng.KvPool(n_pages, page), TierModel(n_pages, page, H), Contents(n_pages, H)
    pool.set_host_pages(H)
    families = [[rng.randrange(6) for _ in range(page * 8)] for _ in range(3)]
    toks = {}
    n_fill = n_spill = n_both = 0
    for step in range(4000):
        o = rng.randrange(6)
        if o not in toks:
            f = families[rng.randrange(3)]
            ids = f[:rng.randrange(1, len(f))] + [rng.randrange(6) for _ in range(rng.randrange(0, 2 * page))]
            if rng.random() < 0.8:
                got, moves = attach_both(pool, m, c, o, ids)
                assert got % page == 0 and got <= page * ((len(ids) - 1) // page)
                n_fill += any(k == FILL for k, _, _ in moves)
                n_both += any(k == SPILL for k, _, _ in moves) and any(k == FILL for k, _, _ in moves)
            rc, moves = reserve_both(pool, m, c, o, len(ids))
            n_spill += bool(moves)
            if rc:
                pool.release(o)
                m.release(o)
            else:
                toks[o] = ids
                publish_both(pool, m, c, o, ids, len(ids) if rng.random() < 0.7 else rng.randrange(len(ids) + 1))
        else:
            r = rng.random()
            if r < 0.35:
                pool.release(o)
                m.release(o)
                del toks[o]
            elif r < 0.7:
                ids = toks[o] + [rng.randrange(6) for _ in range(rng.randrange(1, 2 * page))]
                rc, moves = reserve_both(pool, m, c, o, len(ids))
                n_spill += bool(moves)
                if rc == 0:
                    toks[o] = ids
                    publish_both(pool, m, c, o, ids, len(ids))
            else:
                with pytest.raises(eng.EngineError):
                    pool.attach(o, toks[o])
        check_tier(pool, m)
        c.check(m)
        assert pool.take_moves() == []
    assert pool.host_cached_pages == len(m.hlru)
    assert n_fill > 20 and n_spill > 20, (n_fill, n_spill, n_both)


def test_host_tier_off_hands_out_what_the_allocator_always_did():
    """H = 0 (set explicitly, and after a tier was freed): the same pages and states as the allocator without a host
    tier, and no moves."""
    for resize in (False, True):
        rng = random.Random(11)
        pool, m = eng.KvPool(24, 4), PoolModel(24, 4)
        if resize:
            pool.set_host_pages(8)
        pool.set_host_pages(0)
        fam = [rng.randrange(5) for _ in range(40)]
        toks = {}
        for _ in range(2000):
            o = rng.randrange(6)
            if o not in toks:
                ids = fam[:rng.randrange(1, 40)] + [rng.randrange(5) for _ in range(rng.randrange(8))]
                assert pool.attach(o, ids) == m.attach(o, ids)
                rc = pool.reserve(o, len(ids))
                assert rc == m.reserve(o, len(ids))
                if rc:
                    pool.release(o)
                    m.release(o)
                    continue
                toks[o] = ids
                pool.publish(o, ids)
                m.publish(o, ids, len(ids))
            else:
                pool.release(o)
                m.release(o)
                del toks[o]
            check_state(pool, m)
            assert pool.take_moves() == [] and pool.host_cached_pages == 0


def _publish_chain(pool, o, ids):
    assert pool.reserve(o, len(ids)) == 0
    pool.publish(o, ids)
    pages = pool.pages_of(o)
    pool.release(o)
    return pages


def test_spill_then_fill_of_one_device_page_in_one_attach():
    """The pool is full of cached pages of B; attaching A, which sits on the host, evicts a page of B to the host and
    fills A into that same page: the spill must run before the fill."""
    P = 4
    pool = eng.KvPool(4, P)
    pool.set_host_pages(8)
    a, b = list(range(10, 10 + 4 * P)), list(range(50, 50 + 4 * P))
    _publish_chain(pool, 0, a)
    pb = _publish_chain(pool, 1, b)                        # evicts all four pages of A to the host
    spills = pool.take_moves()
    assert [k for k, _, _ in spills] == [SPILL] * 4 and pool.host_cached_pages == 4
    assert pool.attach(2, a + [0]) == 4 * P                # every page of A comes back, every page of B leaves
    moves = pool.take_moves()
    assert [k for k, _, _ in moves] == [SPILL, FILL] * 4
    for i in range(0, 8, 2):
        (k0, p0, h0), (k1, p1, h1) = moves[i], moves[i + 1]
        assert p0 == p1 and p0 in pb and h0 != h1           # one device page: out to the host, then A's bytes in
    assert pool.pages_of(2) == [p for _, p, _ in moves[1::2]]
    pool.release(2)
    assert pool.attach(3, b + [0]) == 4 * P                 # and B comes back from the host in turn
    pool.release(3)


def test_host_page_freed_by_a_fill_is_reused_by_a_later_spill():
    """The host tier is full of A's pages and the pool full of cached pages of B.  The first fill finds no host page for
    the page of B it evicts (the host pages all hold the chain being attached), so that entry is dropped; the host page
    the fill frees then takes the next page of B: fill before spill."""
    P = 4
    pool = eng.KvPool(3, P)
    pool.set_host_pages(3)
    a, b = list(range(10, 10 + 3 * P)), list(range(50, 50 + 3 * P))
    _publish_chain(pool, 0, a)
    _publish_chain(pool, 1, b)
    pool.take_moves()
    assert pool.host_cached_pages == 3 and pool.cached_pages == 3
    assert pool.attach(2, a + [0]) == 3 * P
    moves = pool.take_moves()
    assert [k for k, _, _ in moves] == [FILL, SPILL, FILL, SPILL, FILL]
    for i in (0, 2):
        assert moves[i][2] == moves[i + 1][2]                 # the host page a fill read is the next spill's target
    pool.release(2)
    # B's deepest page was dropped; its other two pages went to the host in chain order
    assert pool.host_cached_pages == 2
    assert pool.attach(3, b + [0]) == 2 * P
    pool.release(3)


def test_host_lru_drops_deepest_page_first():
    P = 4
    pool = eng.KvPool(4, P)
    pool.set_host_pages(3)
    a = list(range(10, 10 + 4 * P))
    chain = _publish_chain(pool, 0, a)
    assert pool.reserve(1, 4 * P) == 0                      # four evictions, deepest page first, into three host pages
    moves = pool.take_moves()
    assert moves[:3] == [(SPILL, chain[3], 0), (SPILL, chain[2], 1), (SPILL, chain[1], 2)]
    assert moves[3] == (SPILL, chain[0], 0)                 # the root took the host page of the deepest one, dropped
    assert pool.host_cached_pages == 3
    pool.release(1)
    assert pool.attach(2, a + [0]) == 3 * P                 # the first three pages come back
    assert [k for k, _, _ in pool.take_moves()] == [FILL] * 3
    pool.release(2)


def test_chain_whose_root_was_dropped_is_not_attached():
    """The root of A is indexed on W's page and A's second page on X's (X's own root page stayed private).  W goes first,
    so the host LRU holds the root before the child and drops it first: the child stays on the host, unreachable."""
    P = 4
    pool = eng.KvPool(4, P)
    pool.set_host_pages(2)
    a, b = list(range(10, 10 + 2 * P)), list(range(50, 50 + 4 * P))
    assert pool.reserve(0, P) == 0
    pool.publish(0, a[:P])
    assert pool.reserve(1, 2 * P) == 0
    pool.publish(1, a)
    pool.release(0)
    pool.release(1)
    assert pool.cached_pages == 2
    _publish_chain(pool, 2, b)                              # two free pages, then root and child of A go to the host
    assert [k for k, _, _ in pool.take_moves()] == [SPILL, SPILL] and pool.host_cached_pages == 2
    assert pool.reserve(4, 2 * P) == 0                      # B's two deepest pages: the first spill drops A's root ...
    moves = pool.take_moves()
    assert [k for k, _, _ in moves] == [SPILL, SPILL]
    pool.release(4)
    assert pool.attach(5, a + [0]) == 0                     # ... and A's child, still on the host, is never attached
    pool.release(5)
    assert pool.attach(6, b + [0]) == 4 * P


def test_attach_takes_only_the_prefix_that_fits():
    """Two host pages of A, one free device page and nothing cached on the device: attach takes the first page of A
    and leaves the second on the host."""
    P = 4
    pool = eng.KvPool(3, P)
    pool.set_host_pages(4)
    a = list(range(10, 10 + 2 * P))
    _publish_chain(pool, 0, a)
    assert pool.reserve(1, 3 * P) == 0                      # the two pages of A go to the host
    pool.take_moves()
    pool.release(1)                                         # three free pages (private)
    assert pool.reserve(4, 2 * P) == 0                      # one free page left
    assert pool.attach(2, a + [0]) == P
    assert [k for k, _, _ in pool.take_moves()] == [FILL]
    assert pool.host_cached_pages == 1 and pool.free_pages == 0
    pool.release(2)
    pool.release(4)
    assert pool.attach(3, a + [0]) == 2 * P


def test_set_host_pages_validates():
    pool = eng.KvPool(4, 4)
    with pytest.raises(eng.EngineError):
        pool.set_host_pages(-1)
    pool.set_host_pages(2)
    a = list(range(10, 18))
    _publish_chain(pool, 0, a)
    assert pool.reserve(1, 16) == 0
    with pytest.raises(eng.EngineError):                    # moves pending
        pool.set_host_pages(4)
    assert len(pool.take_moves()) == 2
    pool.set_host_pages(0)                                  # drops what the tier held
    assert pool.host_cached_pages == 0
    pool.release(1)
    assert pool.attach(2, a + [0]) == 0
