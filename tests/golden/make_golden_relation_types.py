"""Generate tests/golden/relation_types.npz from the UNMODIFIED reference's splitRelationType.

    KGREC_REFERENCE=<reference checkout> python tests/golden/make_golden_relation_types.py

Synthetic train / valid / test triples cover all four categories, relations whose mean head or tail count per key
lands exactly on 1.5 or 2.5 (Python 3 round: half to even), duplicated triples, relations present only in valid or
test, and a relation absent from every split.  The reference classifies train + valid + test as
preprocessTriples.py:253 does; its four sets are recorded as one int8 category per relation
(0 = 1-1, 1 = 1-N, 2 = N-1, 3 = N-N, -1 = absent).
"""
import os
import sys

import numpy as np

REF = os.environ["KGREC_REFERENCE"]
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)

from jTransUP.data.preprocessTriples import Triple, splitRelationType  # noqa: E402


def triples():
    rng = np.random.RandomState(7)
    rows = []
    e = iter(range(10_000))                          # fresh entity ids
    for _ in range(20):                              # r0: 1-1
        rows.append((next(e), next(e), 0))
    for _ in range(10):                              # r1: 1-N, 3 tails per head
        h = next(e)
        rows += [(h, next(e), 1) for _ in range(3)]
    for _ in range(10):                              # r2: N-1, 4 heads per tail
        t = next(e)
        rows += [(next(e), t, 2) for _ in range(4)]
    hs, ts = [next(e) for _ in range(6)], [next(e) for _ in range(6)]
    rows += [(h, t, 3) for h in hs for t in ts]      # r3: N-N, complete bipartite
    # r4: mean heads per (t, r) = 1.5 (keys with 1 and 2 heads) -> round 2; one tail per head -> N-1
    t1, t2 = next(e), next(e)
    rows += [(next(e), t1, 4), (next(e), t2, 4), (next(e), t2, 4)]
    # r5: mean tails per (h, r) = 2.5 (keys with 2 and 3 tails) -> round 2; one head per tail -> 1-N
    h1, h2 = next(e), next(e)
    rows += [(h1, next(e), 5), (h1, next(e), 5), (h2, next(e), 5), (h2, next(e), 5), (h2, next(e), 5)]
    # r6: one key with 2 heads and one with 2 tails, both means 4/3 -> round 1 -> 1-1
    a, b, c, d = next(e), next(e), next(e), next(e)
    rows += [(a, b, 6), (c, b, 6), (d, next(e), 6), (a, next(e), 6)]
    # r7: a duplicated triple counts once (the reference's sets): heads per key 1 and 2 -> 1.5 -> N-1
    t3, t4 = next(e), next(e)
    x = next(e)
    rows += [(x, t3, 7), (x, t3, 7), (next(e), t4, 7), (next(e), t4, 7)]
    # r8..r11: random relations over a small entity range (many keys share entities)
    for r, (nh, nt) in zip(range(8, 12), ((3, 12), (12, 3), (6, 6), (40, 40))):
        rows += [(int(rng.randint(0, nh)) + 20_000, int(rng.randint(0, nt)) + 20_100, r) for _ in range(30)]
    rows = np.asarray(rows, dtype=np.int64)
    rng.shuffle(rows)
    n = len(rows)
    train, valid, test = rows[: int(0.7 * n)], rows[int(0.7 * n): int(0.85 * n)], rows[int(0.85 * n):]
    only_valid = np.asarray([(30_000, 30_001, 12), (30_002, 30_001, 12)], dtype=np.int64)           # r12: valid only
    only_test = np.asarray([(30_003, 30_004, 13), (30_003, 30_005, 13), (30_006, 30_007, 13)], dtype=np.int64)  # r13
    valid = np.concatenate([valid, only_valid, train[:3]])                   # triples repeated across splits
    test = np.concatenate([test, only_test])
    return train, valid, test                                               # r14: absent everywhere


def main():
    train, valid, test = triples()
    n_rel = 15
    allt = [Triple(int(h), int(t), int(r)) for h, t, r in np.concatenate([train, valid, test])]
    sets = splitRelationType(allt)
    cat = np.full(n_rel, -1, dtype=np.int8)
    for c, s in enumerate(sets):
        for r in s:
            cat[r] = c
    np.savez_compressed(os.path.join(OUT, "relation_types.npz"), train=train, valid=valid, test=test,
                        n_rel=np.int64(n_rel), category=cat)
    print("categories:", cat.tolist())


if __name__ == "__main__":
    main()
