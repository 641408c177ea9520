"""Cost of the link-prediction metrics (KGEvaluator(link=True)): the dual rank count against the filtered pass alone
and against two separate passes, and run() with link=False / link=True.

    python tools/kg_link_eval.py [--quick] [--only kg,worst]

Shapes are synthetic (seeded):
  kg     the DESIGN section 6 validation shape of tools/device_eval.py: E = 100k, R = 500, d = 100, ~20k validation
         pairs over ~1.9k head and tail queries (1-20 golds each), 500k training triples as the filter (half of them on
         the validation queries); TransE, TransH, TransR with fresh (untrained) tables.  Kernel time of both sides'
         rank passes over every (query, gold) pair: the filtered pass (kgrec_*eval_rank_count_ex, exclusion CSR), the
         dual pass (kgrec_*eval_rank_count_dual) and the two passes it replaces (_ex with the exclusion CSR, then _ex
         with the gold CSR); then run() of KGEvaluator(link=False) and of KGEvaluator(link=True, rel_category).
  worst  configs[4]: E = 5M, d = 128, TransE L2, random tables, 4096 queries with random golds (about half the catalog
         sorts before the gold, so half the rows reach the exclusion lookup), 100 excluded ids each of which 10 are
         the query's golds: the same three pass variants.
Times are CUDA-event medians of 5 after one warm-up, the variants alternating.  One JSON line per result, plus the
GPU's name, power limit and SM clock limit read in the same run.
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "joint-kg-recommender_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from device_eval import emit, gpu_info  # noqa: E402


def timed(variants, reps=5):
    """{name: median ms} of callables, one warm-up each, then `reps` rounds alternating the variants."""
    for fn in variants.values():
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {k: [] for k in variants}
    for _ in range(reps):
        for name, fn in variants.items():
            start.record()
            fn()
            stop.record()
            stop.synchronize()
            res[name].append(start.elapsed_time(stop))
    return {k: float(np.median(v)) for k, v in res.items()}


class Passes:
    """The three pass variants over one set of (query, gold) pairs per side.  side: (sd, q, r, gold32, gold_scores,
    excl_row, (excl_ptr, excl_ids), (gold_ptr, gold_ids), TransR runs or None)."""

    def __init__(self, lib, T, kg, catalog, sides, ws=None, status=None):
        self.lib, self.T, self.kg, self.cat, self.sides, self.ws, self.status = lib, T, kg, catalog, sides, ws, status
        self.bufs = [[torch.zeros(s[1].numel(), dtype=torch.int32, device="cuda") for _ in range(2)] for s in sides]

    def _common(self, s):
        from kgrec_b200 import functional as KF
        sd, q, r, g32, gs, row, excl, gcsr, runs = s
        cat = self.cat
        if runs is not None:
            begin, rel = runs
            return [C.byref(self.T), sd, KF._ptr(q), KF._ptr(r), 8, q.numel(), C.c_void_p(begin.data_ptr()),
                    C.c_void_p(rel.data_ptr()), rel.numel(), KF._ptr(cat), cat.stride(0), cat.shape[0], 0, KF._ptr(self.ws),
                    KF._ptr(gs), KF._ptr(g32)]
        return [C.byref(self.T), self.kg, sd, KF._ptr(q), KF._ptr(r), 8, None, q.numel(), KF._ptr(cat), cat.stride(0),
                cat.shape[0], 0, KF._ptr(gs), KF._ptr(g32)]

    def ex(self, csr_of):
        from kgrec_b200 import _lib, functional as KF
        for s, (a, _) in zip(self.sides, self.bufs):
            a.zero_()
            ptr, ids = csr_of(s)
            tail = [KF._ptr(a), KF._ptr(s[5]), KF._ptr(ptr), KF._ptr(ids)]
            if s[8] is not None:
                _lib.check(self.lib.kgrec_transr_eval_rank_count_ex(*self._common(s), *tail, KF._ptr(self.status), KF._stream()))
            else:
                _lib.check(self.lib.kgrec_eval_rank_count_ex(*self._common(s), *tail, KF._stream()))

    def filtered(self):
        self.ex(lambda s: s[6])

    def two_passes(self):
        self.ex(lambda s: s[6])
        self.ex(lambda s: s[7])

    def dual(self):
        from kgrec_b200 import _lib, functional as KF
        for s, (a, b) in zip(self.sides, self.bufs):
            a.zero_()
            b.zero_()
            tail = [KF._ptr(a), KF._ptr(s[5]), KF._ptr(s[6][0]), KF._ptr(s[6][1]), KF._ptr(s[7][0]), KF._ptr(s[7][1]), KF._ptr(b)]
            if s[8] is not None:
                _lib.check(self.lib.kgrec_transr_eval_rank_count_dual(*self._common(s), *tail, KF._ptr(self.status), KF._stream()))
            else:
                _lib.check(self.lib.kgrec_eval_rank_count_dual(*self._common(s), *tail, KF._stream()))

    def run(self):
        t = timed({"filtered": self.filtered, "dual": self.dual, "two_passes": self.two_passes})
        return dict(filtered_ms=t["filtered"], dual_ms=t["dual"], two_passes_ms=t["two_passes"],
                    dual_over_filtered=t["dual"] / t["filtered"], two_passes_over_filtered=t["two_passes"] / t["filtered"])


def kg_dicts(quick):
    E, R = (20_000, 100) if quick else (100_000, 500)
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
    filt = {"head": {}, "tail": {}}
    keys = {s: list(evals[s]) for s in evals}
    triples = []
    for i in range(n_train):
        if i % 2 == 0:
            side = "head" if i % 4 == 0 else "tail"
            key = keys[side][rng.randint(0, len(keys[side]))]
            filt[side].setdefault(key, set()).add(int(rng.randint(0, E)))
        else:
            h, t, r = (int(x) for x in (rng.randint(0, E), rng.randint(0, E), rng.randint(0, R)))
            filt["head"].setdefault((t, r), set()).add(h)
            filt["tail"].setdefault((h, r), set()).add(t)
            triples.append((h, t, r))
    return E, R, evals, filt, np.asarray(triples, dtype=np.int64)


def kg_case(quick):
    import kgrec_b200 as K
    from kgrec_b200 import _lib, dataio as KD, metrics as KM
    lib = _lib.load()
    d = 100
    E, R, evals, filt, triples = kg_dicts(quick)
    rel_category = KD.relation_categories(triples, R)
    for name, cls in (("transe", K.TransEModel), ("transh", K.TransHModel), ("transr", K.TransRModel)):
        torch.manual_seed(1)
        m = cls(False, d, E, R)
        args = (m, evals["head"], evals["tail"], [filt["head"]], [filt["tail"]])
        plain = KM.KGEvaluator(*args, topn=10)
        link = KM.KGEvaluator(*args, topn=10, link=True, rel_category=rel_category)
        T = link._tables()
        catalog = m.ent_embeddings.weight.detach()
        sides = []
        for s in link.sides:
            runs = (s.run_begin, s.run_rel) if link._transr else None
            sides.append((s.sd, s.q, s.r, s.gold32, link._gold_scores(T, s, catalog), s.excl_row, (s.excl_ptr, s.excl_ids),
                          (s.gold_ptr, s.gold_ids), runs))
        passes = Passes(lib, T, link._kg, catalog, sides, link._ws, m._status_buf(catalog.device) if link._transr else None)
        k = passes.run()
        t = timed({"link_false": plain.run, "link_true": link.run})
        same = link.result(link.run()) == plain.result(plain.run())
        emit(case="kg", model=name, E=E, R=R, d=d, queries=sum(len(e) for e in evals.values()),
             pairs=sum(s.n for s in link.sides), filtered_pairs=sum(s.n_filt for s in link.sides), **k,
             run_link_false_ms=t["link_false"], run_link_true_ms=t["link_true"],
             run_ratio=t["link_true"] / t["link_false"], filtered_results_equal=same)
        del m, plain, link, passes, sides
        torch.cuda.empty_cache()


def worst_case(quick):
    import kgrec_b200 as K
    from kgrec_b200 import _lib, functional as KF
    lib = _lib.load()
    E, d, nq, n_excl, n_gold = (500_000 if quick else 5_000_000), 128, 4096, 100, 10
    torch.manual_seed(3)
    m = K.TransEModel(False, d, E, 50)
    g = torch.Generator(device="cuda").manual_seed(4)
    q = torch.randint(0, E, (nq,), device="cuda", generator=g)
    r = torch.randint(0, 50, (nq,), device="cuda", generator=g)
    excl = torch.sort(torch.randint(0, E, (nq, n_excl), device="cuda", generator=g), dim=1).values
    gold_set = excl[:, ::n_excl // n_gold].contiguous()                    # 10 of the excluded ids are the golds
    gold = gold_set[torch.arange(nq, device="cuda"), torch.randint(0, n_gold, (nq,), device="cuda", generator=g)]
    gs = m.gold_scores("tail", q, r, gold)
    row = torch.arange(nq, device="cuda", dtype=torch.int32)
    excl_csr = (torch.arange(nq + 1, device="cuda", dtype=torch.int64) * n_excl, excl.to(torch.int32).contiguous())
    gold_csr = (torch.arange(nq + 1, device="cuda", dtype=torch.int64) * n_gold, gold_set.to(torch.int32).contiguous())
    T = KF.make_tables(m._weights(), d, False)
    passes = Passes(lib, T, _lib.TRANSE, m.ent_embeddings.weight.detach(),
                    [(_lib.SIDE_TAIL, q, r, gold.to(torch.int32), gs, row, excl_csr, gold_csr, None)])
    k = passes.run()
    passes.dual()
    raw, filt = passes.bufs[0][1], passes.bufs[0][0]
    emit(case="worst", E=E, d=d, queries=nq, excluded_per_query=n_excl, golds_per_query=n_gold,
         rows_before_gold_fraction=float(raw.double().mean()) / E, filtered_below_gold_per_query=float((raw - filt).double().mean()),
         **k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="smaller shapes (a rehearsal, not the measurement)")
    ap.add_argument("--only", default="kg,worst")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kg_link_eval.py measures the GPU path and needs a CUDA device")
    emit(gpu=gpu_info(), torch=torch.__version__)
    todo = a.only.split(",")
    if "worst" in todo:
        worst_case(a.quick)
    if "kg" in todo:
        kg_case(a.quick)


if __name__ == "__main__":
    main()
