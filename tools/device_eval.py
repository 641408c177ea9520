"""Wall time of the driver-level validation (metrics.evaluate_kg / evaluate_rec) against the device-resident
evaluators (metrics.KGEvaluator / RecEvaluator: run() + result()), the evaluators' kernel time (torch.profiler), and
the cost of the in-kernel filter in the rank-count pass.

    python tools/device_eval.py [--quick] [--only kg,rec,filter]

Shapes are synthetic (seeded):
  kg      E = 100k, R = 500, d = 100; ~20k validation triples split over head and tail queries with 1-20 golds each,
          500k training triples as the filter (half of them on the validation queries); TransE, TransH, TransR
  rec     U = I = 50k, d = 100, P = 20; 10k validation users with 5 golds and 100 filtered training items each;
          TUP soft and ST-Gumbel (L2)
  filter  configs[4]: E = 5M, d = 128, random tables, 4096 queries with random golds (about half the catalog sorts
          before the gold, so half the rows reach the id lookup) and 100 excluded ids each: the filtered rank pass
          (kgrec_eval_rank_count_ex) against the unfiltered one (kgrec_eval_rank_count)
Wall times are medians of 5 after one warm-up; every timed call ends in a device synchronisation.  One JSON line per
result, plus the GPU's name, power limit and SM clock limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "joint-kg-recommender_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def wall(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def kernel_ms(fn):
    """Device time of one call (sum over the GPU activities torch.profiler records)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        tot += getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0.0)
    return tot / 1e3


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        out = "nvidia-smi unavailable: %s" % e
    return out


def kg_case(quick):
    import kgrec_b200 as K
    from kgrec_b200 import metrics as KM
    E, R, d = (20_000, 100, 100) if quick else (100_000, 500, 100)
    n_val, n_train = (4_000, 100_000) if quick else (20_000, 500_000)
    rng = np.random.RandomState(0)
    evals = {}
    for side in ("head", "tail"):
        ev, n = {}, 0
        while n < n_val // 2:
            key = (int(rng.randint(0, E)), int(rng.randint(0, R)))
            if key in ev:
                continue
            g = set(int(x) for x in rng.randint(0, E, rng.randint(1, 21)))
            ev[key] = g
            n += len(g)
        evals[side] = ev
    # training triples: half on the validation queries (so the filter reaches them), half uniform
    filt = {"head": {}, "tail": {}}
    keys = {s: list(evals[s]) for s in evals}
    for i in range(n_train):
        if i % 2 == 0:
            side = "head" if i % 4 == 0 else "tail"
            key = keys[side][rng.randint(0, len(keys[side]))]
            filt[side].setdefault(key, set()).add(int(rng.randint(0, E)))
        else:
            h, t, r = (int(x) for x in (rng.randint(0, E), rng.randint(0, E), rng.randint(0, R)))
            filt["head"].setdefault((t, r), set()).add(h)
            filt["tail"].setdefault((h, r), set()).add(t)
    n_pairs = sum(len(g) for s in evals for g in evals[s].values())
    n_q = sum(len(evals[s]) for s in evals)
    for name, cls in (("transe", K.TransEModel), ("transh", K.TransHModel), ("transr", K.TransRModel)):
        torch.manual_seed(1)
        m = cls(False, d, E, R)
        args = (m, evals["head"], evals["tail"], [filt["head"]], [filt["tail"]])
        t_drv = wall(lambda: KM.evaluate_kg(*args, topn=10))
        t0 = time.perf_counter()
        ev = KM.KGEvaluator(*args, topn=10)
        t_init = (time.perf_counter() - t0) * 1e3
        t_dev = wall(lambda: ev.result(ev.run()))
        k_dev = kernel_ms(lambda: ev.result(ev.run()))
        same = ev.result(ev.run()) == KM.evaluate_kg(*args, topn=10)
        emit(case="kg", model=name, E=E, R=R, d=d, queries=n_q, pairs=n_pairs, golds_per_query=n_pairs / n_q,
             evaluate_kg_ms=t_drv, evaluator_ms=t_dev, evaluator_kernel_ms=k_dev, evaluator_init_ms=t_init,
             speedup=t_drv / t_dev, wall_over_kernel=t_dev / k_dev, results_equal=same)
        del m, ev
        torch.cuda.empty_cache()


def rec_case(quick):
    import kgrec_b200 as K
    from kgrec_b200 import metrics as KM
    U = I = 10_000 if quick else 50_000
    n_users, d, P = (2_000 if quick else 10_000), 100, 20
    rng = np.random.RandomState(1)
    users = rng.choice(U, n_users, replace=False)
    eval_dict = {int(u): set(int(x) for x in rng.choice(I, 5, replace=False)) for u in users}
    train = {u: set(int(x) for x in rng.choice(I, 100, replace=False)) - eval_dict[u] for u in eval_dict}
    for gumbel in (False, True):
        torch.manual_seed(2)
        m = K.TransUPModel(False, d, U, I, P, gumbel)
        t_drv = wall(lambda: KM.evaluate_rec(m, eval_dict, [train], topn=10))
        t0 = time.perf_counter()
        rv = KM.RecEvaluator(m, eval_dict, [train], topn=10)
        t_init = (time.perf_counter() - t0) * 1e3
        t_dev = wall(lambda: rv.result(rv.run(seed=7)))
        k_dev = kernel_ms(lambda: rv.result(rv.run(seed=7)))
        got = rv.result(rv.run(seed=7))
        want = KM.evaluate_rec(m, eval_dict, [train], topn=10) if not gumbel else None
        emit(case="rec", model="tup_gumbel" if gumbel else "tup_soft", U=U, I=I, d=d, P=P, users=n_users,
             evaluate_rec_ms=t_drv, evaluator_ms=t_dev, evaluator_kernel_ms=k_dev, evaluator_init_ms=t_init,
             speedup=t_drv / t_dev, wall_over_kernel=t_dev / k_dev,
             max_rel_diff=None if want is None else float(np.max(np.abs(np.subtract(got, want)) / np.maximum(np.abs(want), 1e-300))))
        del m, rv
        torch.cuda.empty_cache()


def filter_case(quick):
    import kgrec_b200 as K
    from kgrec_b200 import _lib, functional as KF
    lib = _lib.load()
    E, d, nq, n_excl = (500_000 if quick else 5_000_000), 128, 4096, 100
    torch.manual_seed(3)
    m = K.TransEModel(False, d, E, 50)
    g = torch.Generator(device="cuda").manual_seed(4)
    q = torch.randint(0, E, (nq,), device="cuda", generator=g)
    r = torch.randint(0, 50, (nq,), device="cuda", generator=g)
    gold = torch.randint(0, E, (nq,), device="cuda", generator=g)
    gs = m.gold_scores("tail", q, r, gold)
    gold32 = gold.to(torch.int32)
    excl_ids = torch.sort(torch.randint(0, E, (nq, n_excl), device="cuda", generator=g), dim=1).values.to(torch.int32).contiguous()
    excl_ptr = torch.arange(nq + 1, device="cuda", dtype=torch.int64) * n_excl
    excl_row = torch.arange(nq, device="cuda", dtype=torch.int32)
    cat = m.ent_embeddings.weight.detach()
    T = KF.make_tables(m._weights(), d, False)
    counts = torch.zeros(nq, dtype=torch.int32, device="cuda")

    def plain():
        counts.zero_()
        _lib.check(lib.kgrec_eval_rank_count(C.byref(T), _lib.TRANSE, _lib.SIDE_TAIL, KF._ptr(q), KF._ptr(r), 8, None, nq,
                                             KF._ptr(cat), d, E, 0, KF._ptr(gs), KF._ptr(gold32), KF._ptr(counts), KF._stream()))

    def filtered():
        counts.zero_()
        _lib.check(lib.kgrec_eval_rank_count_ex(C.byref(T), _lib.TRANSE, _lib.SIDE_TAIL, KF._ptr(q), KF._ptr(r), 8, None, nq,
                                                KF._ptr(cat), d, E, 0, KF._ptr(gs), KF._ptr(gold32), KF._ptr(counts),
                                                KF._ptr(excl_row), KF._ptr(excl_ptr), KF._ptr(excl_ids), KF._stream()))
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {"plain": [], "filtered": []}
    for fn in (plain, filtered):
        fn()
    torch.cuda.synchronize()
    for _ in range(5):                       # alternate the two passes
        for name, fn in (("plain", plain), ("filtered", filtered)):
            start.record()
            fn()
            stop.record()
            stop.synchronize()
            res[name].append(start.elapsed_time(stop))
    plain()
    frac_before = float(counts.double().mean()) / E
    t_p, t_f = float(np.median(res["plain"])), float(np.median(res["filtered"]))
    emit(case="filter", E=E, d=d, queries=nq, excluded_per_query=n_excl, rows_before_gold_fraction=frac_before,
         unfiltered_ms=t_p, filtered_ms=t_f, ratio=t_f / t_p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="smaller shapes (a rehearsal, not the measurement)")
    ap.add_argument("--only", default="kg,rec,filter")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("device_eval.py measures the GPU path and needs a CUDA device")
    emit(gpu=gpu_info(), torch=torch.__version__)
    todo = a.only.split(",")
    if "filter" in todo:
        filter_case(a.quick)
    if "rec" in todo:
        rec_case(a.quick)
    if "kg" in todo:
        kg_case(a.quick)


if __name__ == "__main__":
    main()
