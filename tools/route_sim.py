"""Closed-loop routing simulation behind the two-level Load rule (router.advertised_load).

N identical workers, each decoding up to `max_batch` requests at once (step time grows with the batch, fitted to one
H100 SXM: 5.5 ms at B = 1, 7.5 ms at B = 63, 9.8 ms at B = 126), requests of 256 tokens, a gateway that applies FindBestWorker
(manager.go:338-387: strict max of T / (1 + Load), random order) to metadata that is refreshed every `refresh` seconds.
Prints requests/s for a set of Load thresholds: Load = 1 iff (active + queued) / max_batch >= threshold.

    python tools/route_sim.py [--workers 8] [--concurrency 256] [--refresh 2] [--seconds 60]
"""
import argparse
import random


def simulate(n_workers, conc, refresh, thr, seconds, max_batch=32, gen=256, seed=0, dt=0.005):
    rng = random.Random(seed)
    work = [[] for _ in range(n_workers)]          # remaining tokens per request; the first max_batch are active
    adv = [0.0] * n_workers
    acc = [0.0] * n_workers                        # fractional decode steps
    done, t, next_refresh = 0, 0.0, 0.0

    def route():
        order = list(range(n_workers)); rng.shuffle(order)
        best, sel = 0.0, None
        for w in order:
            sc = 1.0 / (1.0 + adv[w])
            if sc > best:
                best, sel = sc, w
        work[sel].append(gen)

    for _ in range(conc):
        route()
    while t < seconds:
        if t >= next_refresh:
            adv = [1.0 if len(q) / max_batch >= thr else 0.0 for q in work]
            next_refresh += refresh
        finished = 0
        for w in range(n_workers):
            q = work[w]
            b = min(len(q), max_batch)
            if not b:
                continue
            acc[w] += dt / ((5.5 + 0.034 * b) * 1e-3)
            k = int(acc[w]); acc[w] -= k
            if k:
                for i in range(b):
                    q[i] -= k
                n0 = len(q)
                q[:] = [r for r in q if r > 0]
                finished += n0 - len(q)
        for _ in range(finished):
            route()
        done += finished
        t += dt
    return done / seconds


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--concurrency", type=int, default=256)
    ap.add_argument("--refresh", type=float, default=2.0)
    ap.add_argument("--seconds", type=float, default=60.0)
    a = ap.parse_args()
    ideal = a.workers * min(32, a.concurrency / a.workers) / (256 * (5.5 + 0.034 * min(32, a.concurrency / a.workers)) * 1e-3)
    print(f"{a.workers} workers, {a.concurrency} closed-loop clients, metadata refresh {a.refresh}s; perfectly balanced: {ideal:.1f} req/s")
    for thr in (1.0, 1.25, 1.5, 2.0, 1e9):
        r = [simulate(a.workers, a.concurrency, a.refresh, thr, a.seconds, seed=s) for s in range(3)]
        print(f"  Load=1 iff load >= {thr:<6g}: {sum(r) / len(r):7.1f} req/s  ({sum(r) / len(r) / ideal:.2f} of balanced)")
