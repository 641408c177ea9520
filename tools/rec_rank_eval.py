"""Cost of the recommendation-side rank counts (RecModelBase.rank_counts_items / RecEvaluator(ranks=True)) next to the
top-10 pass of the same path.

    python tools/rec_rank_eval.py [--quick]

Shape (synthetic, seeded; the one tools/device_eval.py uses for RecEvaluator): U = I = 50k, d = 100, P = 20, 10k
validation users with 5 golds and 100 filtered training items each; TUP soft and ST-Gumbel (L2), random tables (the
worst case for the count pass: about half of all pairs sort before a gold and reach the filter lookup).
Per model, device time by CUDA events, median of 5 after a warm-up, the passes alternated:
  topk_ms         filtered top-10 of every user (RecEvaluator.topk, which also builds the augmented catalog)
  gold_scores_ms  the sweep that captures the gold scores (kgrec_rec_gold_scores), augmented rows given
  rank_count_ms   gold sort + count sweep + prefix sums (kgrec_rec_rank_count), augmented rows and gold scores given
  run_ms / run_ranks_ms   RecEvaluator.run without and with ranks (catalog build included)
One JSON line per model, plus the GPU's name, power limit and SM clock limit.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "joint-kg-recommender_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.device_eval import emit, gpu_info      # noqa: E402


def timed(fns, reps=5):
    """Median device ms of every callable in `fns` (a dict), alternating them."""
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    for _ in range(reps):
        for name, fn in fns.items():
            start.record()
            fn()
            stop.record()
            stop.synchronize()
            res[name].append(start.elapsed_time(stop))
    return {k + "_ms": float(np.median(v)) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="smaller shapes (a rehearsal, not the measurement)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rec_rank_eval.py measures the GPU path and needs a CUDA device")
    import kgrec_b200 as K
    from kgrec_b200 import metrics as KM
    emit(gpu=gpu_info(), torch=torch.__version__)
    U = I = 10_000 if a.quick else 50_000
    n_users, d, P = (2_000 if a.quick else 10_000), 100, 20
    rng = np.random.RandomState(1)
    users = rng.choice(U, n_users, replace=False)
    eval_dict = {int(u): set(int(x) for x in rng.choice(I, 5, replace=False)) for u in users}
    train = {u: set(int(x) for x in rng.choice(I, 100, replace=False)) - eval_dict[u] for u in eval_dict}
    for gumbel in (False, True):
        torch.manual_seed(2)
        m = K.TransUPModel(False, d, U, I, P, gumbel)
        rv = KM.RecEvaluator(m, eval_dict, [train], topn=10, ranks=True)
        plain = KM.RecEvaluator(m, eval_dict, [train], topn=10)
        gold = (rv.gold_ptr, rv.gold_ids)
        cat = m.gumbel_catalog() if gumbel else m.soft_catalog()
        kw = dict(soft_catalog=cat, seed=7, topn=10, n_gold=rv.n_gold)
        gs = m.gold_scores_items(rv.users, gold, **kw)
        t = timed({
            "topk": lambda: rv.topk(seed=7),
            "gold_scores": lambda: m.gold_scores_items(rv.users, gold, **kw),
            "rank_count": lambda: m.rank_counts_items(rv.users, gold, rv.filter_csr, gold_scores=gs, **kw),
            "run": lambda: plain.run(seed=7),
            "run_ranks": lambda: rv.run(seed=7),
        })
        c = rv.rank_counts(seed=7).double()
        emit(case="rec_rank", model="tup_gumbel" if gumbel else "tup_soft", U=U, I=I, d=d, P=P, users=n_users, golds=rv.n_gold,
             items_before_gold_fraction=float(c.mean()) / I, rank_pass_over_topk=(t["gold_scores_ms"] + t["rank_count_ms"]) / t["topk_ms"],
             run_ranks_over_run=t["run_ranks_ms"] / t["run_ms"], result=rv.result(rv.run(seed=7)), **t)
        del m, rv, plain, cat
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
