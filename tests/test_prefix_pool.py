"""CPU-only tests of the paged-KV allocator's prefix sharing (cl_kvpool_attach / publish / cached_pages): a randomised
run against a small Python model of the sharing rules, plus directed cases."""
import random

import pytest

from crowdllama_b200 import engine as eng


class PoolModel:
    """The allocator's rules restated: pages are free (a stack, low ids first), referenced (refcount > 0) or cached
    (refcount 0, still indexed, on an LRU list).  The index maps (parent entry uid, the page's token ids) to a page."""

    def __init__(self, n_pages, page):
        self.n, self.P = n_pages, page
        self.free = list(range(n_pages - 1, -1, -1))
        self.ref = [0] * n_pages
        self.key = [None] * n_pages       # index key of a published page
        self.uid = [0] * n_pages
        self.index = {}
        self.lru = []
        self.owned = {}
        self.chain = {}                   # owner -> [pages published or matched, uid of the last]
        self.next_uid = 1
        self.evicted = []

    def reserve(self, o, n):
        v = self.owned.setdefault(o, [])
        extra = -(-n // self.P) - len(v)
        if extra <= 0:
            return 0
        if extra > len(self.free) + len(self.lru):
            return eng.CL_ERR_OOM
        for _ in range(extra):
            if self.free:
                p = self.free.pop()
            else:
                p = self.lru.pop(0)
                del self.index[self.key[p]]
                self.key[p] = None
                self.evicted.append(p)
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
        pages, parent = [], 0
        for k in range((len(ids) - 1) // self.P if len(ids) > 1 else 0):
            p = self.index.get((parent, tuple(ids[k * self.P:(k + 1) * self.P])))
            if p is None:
                break
            pages.append(p)
            parent = self.uid[p]
        return pages

    def attach(self, o, ids):
        if self.owned.get(o):
            return None
        pages = self.walk(ids)
        for p in pages:
            if self.ref[p] == 0:
                self.lru.remove(p)
            self.ref[p] += 1
        self.owned[o] = list(pages)
        self.chain[o] = [len(pages), self.uid[pages[-1]] if pages else 0]
        return len(pages) * self.P

    def publish(self, o, ids, n_known):
        if o not in self.owned:
            return
        v, c = self.owned[o], self.chain.setdefault(o, [0, 0])
        k = c[0]
        while k < len(v) and (k + 1) * self.P <= n_known:
            key = (c[1], tuple(ids[k * self.P:(k + 1) * self.P]))
            if key in self.index:
                c[1] = self.uid[self.index[key]]
            else:
                self.index[key] = v[k]
                self.key[v[k]] = key
                self.uid[v[k]] = self.next_uid
                self.next_uid += 1
                c[1] = self.uid[v[k]]
            k += 1
            c[0] = k


def check_state(pool, m):
    held = set()
    for o, v in m.owned.items():
        assert pool.pages_of(o) == v, (o, pool.pages_of(o), v)
        held |= set(v)
    cached, free = set(m.lru), set(m.free)
    # every page is in exactly one state
    assert not (held & cached) and not (held & free) and not (cached & free)
    assert len(held) + len(cached) + len(free) == m.n
    assert all(m.ref[p] > 0 for p in held) and all(m.ref[p] == 0 for p in cached | free)
    assert all(m.key[p] is not None for p in cached) and all(m.key[p] is None for p in free)
    assert pool.used_pages == len(held)
    assert pool.cached_pages == len(cached)
    assert pool.free_pages + pool.used_pages == m.n


@pytest.mark.parametrize("page,n_pages,seed", [(4, 24, 0), (4, 40, 1), (8, 16, 2), (2, 64, 3)])
def test_prefix_pool_matches_model(page, n_pages, seed):
    rng = random.Random(seed)
    pool, m = eng.KvPool(n_pages, page), PoolModel(n_pages, page)
    # a few prompt families with long common prefixes, tokens from a tiny vocabulary so that chains collide often
    families = [[rng.randrange(6) for _ in range(page * 8)] for _ in range(3)]
    toks = {}
    n_hit = n_evict = 0
    for step in range(4000):
        o = rng.randrange(6)
        if o not in toks:
            f = families[rng.randrange(3)]
            ids = f[:rng.randrange(1, len(f))] + [rng.randrange(6) for _ in range(rng.randrange(0, 2 * page))]
            if rng.random() < 0.8:
                got, want = pool.attach(o, ids), m.attach(o, ids)
                assert got == want, (step, got, want)
                assert got % page == 0 and got <= page * ((len(ids) - 1) // page)
                n_hit += got > 0
            others = {p for o2, v in m.owned.items() if o2 != o for p in v}
            before = list(m.owned.get(o, []))
            rc = pool.reserve(o, len(ids))
            assert rc == m.reserve(o, len(ids))
            if rc:
                assert pool.pages_of(o) == before            # atomic on OOM
                pool.release(o)
                m.release(o)
            else:
                assert not (set(m.owned[o][len(before):]) & others)   # never a page somebody holds
                toks[o] = ids
                n_known = len(ids) if rng.random() < 0.7 else rng.randrange(len(ids) + 1)
                pool.publish(o, ids, n_known)
                m.publish(o, ids, n_known)
        else:
            r = rng.random()
            if r < 0.35:
                pool.release(o)
                m.release(o)
                del toks[o]
            elif r < 0.7:
                ids = toks[o] + [rng.randrange(6) for _ in range(rng.randrange(1, 2 * page))]
                ev0 = len(m.evicted)
                rc = pool.reserve(o, len(ids))
                assert rc == m.reserve(o, len(ids))
                n_evict += len(m.evicted) > ev0
                if rc == 0:
                    toks[o] = ids
                    pool.publish(o, ids, len(ids))
                    m.publish(o, ids, len(ids))
            else:
                assert m.owned[o]
                with pytest.raises(eng.EngineError):          # attach needs an owner without pages
                    pool.attach(o, toks[o])
        check_state(pool, m)
    assert n_hit > 50 and n_evict > 20, (n_hit, n_evict)


def test_prefix_pool_one_token_difference_stops_the_match():
    P = 16
    pool = eng.KvPool(32, P)
    a = list(range(100, 100 + 6 * P))
    assert pool.attach(0, a) == 0
    assert pool.reserve(0, len(a)) == 0
    pool.publish(0, a)
    pool.release(0)
    assert pool.cached_pages == 6 and pool.used_pages == 0 and pool.free_pages == 32
    for k in range(6):
        b = list(a)
        b[k * P + 5] += 1                                   # one token of page k differs
        assert pool.attach(1, b + [7]) == k * P
        pool.release(1)
    assert pool.attach(1, a + [7]) == 6 * P                 # all six pages
    pool.release(1)
    assert pool.attach(1, a) == 5 * P                       # capped: the last token is always computed
    pool.release(1)
    assert pool.attach(1, a[:1]) == 0


def test_prefix_pool_duplicate_publish_keeps_the_first_page():
    P = 16
    pool = eng.KvPool(16, P)
    a = list(range(3, 3 + 3 * P))
    for o in (0, 1):                                        # the same text prefilled twice, independently
        assert pool.reserve(o, len(a)) == 0
        pool.publish(o, a)
    first, second = pool.pages_of(0), pool.pages_of(1)
    pool.release(1)                                         # its pages stayed private: straight back to the free list
    assert pool.cached_pages == 0 and pool.free_pages == 16 - 3
    pool.release(0)
    assert pool.cached_pages == 3
    assert pool.attach(2, a + [1]) == 3 * P and pool.pages_of(2) == first
    assert not set(first) & set(second)


def test_prefix_pool_evicts_deepest_pages_first_and_forgets_their_chains():
    P = 4
    pool = eng.KvPool(8, P)
    a = list(range(10, 10 + 4 * P))
    assert pool.reserve(0, len(a)) == 0
    pool.publish(0, a)
    chain = pool.pages_of(0)
    pool.release(0)
    assert pool.reserve(1, 4 * P) == 0                      # the four free pages
    assert pool.reserve(2, P) == 0 and pool.pages_of(2) == [chain[3]]     # then the deepest cached page
    assert pool.attach(3, a + [0]) == 3 * P                 # the rest of the chain still hits
    pool.release(3)
    assert pool.reserve(2, 4 * P) == 0 and pool.pages_of(2) == [chain[3], chain[2], chain[1], chain[0]]
    assert pool.cached_pages == 0 and pool.free_pages == 0
    assert pool.reserve(4, 1) == eng.CL_ERR_OOM
    pool.release(2)
    assert pool.attach(3, a + [0]) == 0                     # evicted pages never hit, the chain is gone
    pool.release(3)
    pool.release(1)
    assert pool.free_pages == 8 and pool.used_pages == 0


def test_prefix_pool_without_sharing_hands_out_the_same_pages():
    """publish / attach never called: page order and counts are the allocator's as before."""
    rng = random.Random(7)
    pool, m = eng.KvPool(40, 16), PoolModel(40, 16)
    for _ in range(1000):
        o = rng.randrange(8)
        if rng.random() < 0.3:
            pool.release(o)
            m.release(o)
        else:
            n = rng.randrange(1, 200)
            assert pool.reserve(o, n) == m.reserve(o, n)
        check_state(pool, m)
        assert pool.cached_pages == 0
