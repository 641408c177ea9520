"""Driver-level evaluation on the reduced kernel outputs (SURVEY 8f, next row 3).

The reference's evaluate() functions copy a [B, N] score matrix to the host for every batch,
fork `num_processes` workers per batch and argsort each row (item_recommendation.py:27-75,
knowledge_representation.py:28-105, utils/misc.py:61-248).  These two functions produce the
same numbers -- mean F1 / precision / recall / hit / NDCG@n for recommendation, hit@n and mean
filtered rank for KG completion -- from the on-chip top-K lists and rank counts, so that only
K ids (or one count) per query ever leave the GPU.

Semantics restated from the reference (ties broken by (score, id), see oracle/kg_oracle.py):
  rec : top-n ids of the user after dropping the filter set (train + other eval files),
        misc.py:213-248; users with an empty gold set are skipped (misc.py:169).
  KG  : for every gold id g of a query, rank(g) = #{ e not in filter, not gold : e sorts before g };
        hit = rank < topn (misc.py:125-146).  A gold id that is itself in the filter set is never
        reached by the reference's walk and is skipped here too.

evaluate_rec / evaluate_kg rebuild the per-query filter sets on the host at every call.  KGEvaluator and
RecEvaluator do that host work once, for a fixed set of eval / filter dicts, and then evaluate the current
tables with device work only (the loop-with-validation form, INTEGRATION section 4).
"""
import ctypes as C
import itertools

import numpy as np
import torch

from . import _lib
from . import dataio as KD
from . import evaluation as KE
from . import functional as KF


def evaluate_rec(model, eval_dict, all_dicts=None, topn=10, batch=4096):
    """Mean (f1, precision, recall, hit, ndcg) over the users of eval_dict.

    eval_dict: {user: set(gold items)}; all_dicts: dicts whose items are filtered per user
    (the drivers pass [train_dict] + the other eval files' dicts, item_recommendation.py:108-111).
    """
    dev = model._require_cuda()
    users = [u for u, gold in eval_dict.items() if len(gold) > 0]
    rows = []
    for lo in range(0, len(users), batch):
        chunk = users[lo:lo + batch]
        csr = KE.build_filter_csr(chunk, all_dicts, dev) if all_dicts else None
        keys = model.topk_items(torch.tensor(chunk, dtype=torch.int64, device=dev), k=topn, filter_csr=csr)
        ids, _ = KE.keys_to_ids_scores(keys)
        rows.extend(KE.rec_metrics_from_topk(ids.cpu().tolist(), [eval_dict[u] for u in chunk]))
    if not rows:
        return (0.0,) * 5
    return tuple(float(x) for x in np.asarray(rows, dtype=np.float64).mean(axis=0))


def _kg_side(model, side, eval_dict, all_dicts, topn, batch):
    """[(hit, rank)] for every (query, gold id) of one side.  eval_dict: {(q, r): set(gold)}."""
    dev = model._require_cuda()
    from . import _lib
    kg = _lib.TRANSH if model.MODEL == _lib.KTUP else model.MODEL
    sd = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
    transr = model.MODEL == _lib.TRANSR

    def sub_scores(qq, rr, rows, ids):
        """[len(qq), len(ids)] scores against gathered catalog rows, by the catalog pass's own arithmetic (bit-identical
        to the scores the rank-count kernel compares).  TransR projects the gathered rows per distinct relation
        (TransRModel._scores -> csrc/eval_transr.cu)."""
        if transr:
            return model._scores(sd, qq, rr, catalog=rows, cat_ids=ids)
        return model._eval(kg, sd, qq, rr, "scores", catalog=rows, cat_ids=ids)
    queries = [k for k, gold in eval_dict.items() if len(gold) > 0]
    results = []
    catalog = model.ent_embeddings.weight.detach()
    for lo in range(0, len(queries), batch):
        chunk = queries[lo:lo + batch]
        # one row per (query, gold id): the rank-count kernel takes one gold per query row
        qid, gold, excl = [], [], []
        for qi, key in enumerate(chunk):
            g_all = eval_dict[key]
            filt = set()
            for d in all_dicts or ():
                if key in d:
                    filt.update(d[key])
            for g in g_all:
                if g in filt:
                    continue                      # the reference's walk skips filtered ids before testing gold
                qid.append(qi)
                gold.append(g)
                excl.append(sorted((filt | g_all) - {g}))
        if not gold:
            continue
        q = torch.tensor([chunk[i][0] for i in qid], dtype=torch.int64, device=dev)
        r = torch.tensor([chunk[i][1] for i in qid], dtype=torch.int64, device=dev)
        gt = torch.tensor(gold, dtype=torch.int64, device=dev)
        # gold scores from the evaluation kernel itself (bit-identical to the catalog pass)
        gs = torch.empty(gt.numel(), dtype=torch.float32, device=dev)
        for glo in range(0, gt.numel(), 512):
            ghi = min(gt.numel(), glo + 512)
            gs[glo:ghi] = sub_scores(q[glo:ghi], r[glo:ghi], catalog[gt[glo:ghi]].contiguous(), gt[glo:ghi]).diagonal()
        if transr:
            counts = model.rank_counts(side, q, r, gt, gold_scores=gs).to(torch.int64)
        else:
            counts = model._eval(kg, sd, q, r, "rank", catalog=catalog, gold_scores=gs, gold_ids=gt).to(torch.int64)
        # correction: filtered ids and the other gold ids that sort before the gold do not count.
        # Their scores come from the same evaluation kernel on the gathered rows (bit-identical).
        flat_row = torch.tensor([i for i, e in enumerate(excl) for _ in e], dtype=torch.int64, device=dev)
        flat_ids = torch.tensor([x for e in excl for x in e], dtype=torch.int64, device=dev)
        if flat_ids.numel():
            uniq, inv = torch.unique(flat_ids, return_inverse=True)
            sub = catalog[uniq].contiguous()
            before = torch.zeros_like(counts)
            for qlo in range(0, q.numel(), 2048):          # [rows, n_unique] score blocks
                qhi = min(q.numel(), qlo + 2048)
                sel = (flat_row >= qlo) & (flat_row < qhi)
                if not bool(sel.any()):
                    continue
                m = sub_scores(q[qlo:qhi], r[qlo:qhi], sub, uniq)
                rr, cc = flat_row[sel] - qlo, inv[sel]
                s_e = m[rr, cc]
                s_g, i_g = gs[flat_row[sel]], gt[flat_row[sel]]
                lt = (s_e < s_g) | ((s_e == s_g) & (flat_ids[sel] < i_g))
                before.index_add_(0, flat_row[sel], lt.to(torch.int64))
            counts = counts - before
        ranks = counts.cpu().tolist()
        results.extend((1 if rk < topn else 0, rk) for rk in ranks)
    return results


def evaluate_kg(model, eval_head_dict, eval_tail_dict, all_head_dicts=None, all_tail_dicts=None, topn=10, batch=2048):
    """(avg_hit, avg_mean_rank, head (hit, rank), tail (hit, rank)) as knowledge_representation.py:66-87
    logs them.  eval_head_dict: {(t, r): set(gold heads)}, eval_tail_dict: {(h, r): set(gold tails)}."""
    head = _kg_side(model, "head", eval_head_dict, all_head_dicts, topn, batch)
    tail = _kg_side(model, "tail", eval_tail_dict, all_tail_dicts, topn, batch)
    h = np.asarray(head, dtype=np.float64).mean(axis=0) if head else np.zeros(2)
    t = np.asarray(tail, dtype=np.float64).mean(axis=0) if tail else np.zeros(2)
    n_h, n_t = len(head), len(tail)
    tot = max(1, n_h + n_t)
    return (float(h[0] * n_h + t[0] * n_t) / tot, float(h[1] * n_h + t[1] * n_t) / tot,
            (float(h[0]), float(h[1])), (float(t[0]), float(t[1])))


# ---- evaluators: host work once per (eval dicts, filter dicts), device work per evaluation ---------------
def _flatten_sets(keys, dct):
    """(lengths [len(keys)], ids) of dct[key] for every key, each set in its own iteration order."""
    sets = [dct[k] for k in keys]
    lens = np.fromiter((len(s) for s in sets), dtype=np.int64, count=len(sets))
    ids = np.fromiter(itertools.chain.from_iterable(sets), dtype=np.int64, count=int(lens.sum()))
    return lens, ids


def _csr(codes, n_rows, width):
    """Sorted (row * width + id) codes -> (ptr int64 [n_rows + 1], ids int64)."""
    ptr = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(np.bincount(codes // width, minlength=n_rows), out=ptr[1:])
    return ptr, codes % width


def side_arrays(keys, eval_dict, all_dicts, drop_filtered_gold):
    """Host arrays of one evaluation side (query keys = the eval dict's keys with a non-empty gold set).

    Returns a dict of int64 numpy arrays:
      pair_q, pair_gold  one entry per (query index, gold id), queries in `keys` order and each gold set in
                         its iteration order -- the order evaluate_kg / evaluate_rec visit them; with
                         drop_filtered_gold, golds inside the query's filter set are left out (the reference's
                         walk never reaches them, misc.py:125-146)
      filt_ptr, filt_ids the filter CSR: per query the ascending union over all_dicts of dict[key]
      excl_ptr, excl_ids the exclusion CSR: per query the ascending union of its filter and gold sets
      gold_ptr, gold_ids the gold CSR: per query its ascending gold set
    """
    nq = len(keys)
    g_len, g_ids = _flatten_sets(keys, eval_dict)
    g_q = np.repeat(np.arange(nq, dtype=np.int64), g_len)
    f_q, f_ids = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for d in all_dicts or ():
        present = [i for i, k in enumerate(keys) if k in d]
        lens, ids = _flatten_sets([keys[i] for i in present], d)
        f_q.append(np.repeat(np.asarray(present, dtype=np.int64), lens))
        f_ids.append(ids)
    f_q, f_ids = np.concatenate(f_q), np.concatenate(f_ids)
    if (g_ids.size and g_ids.min() < 0) or (f_ids.size and f_ids.min() < 0):
        raise ValueError("kgrec_b200: negative ids in the eval / filter dicts")
    width = 1 + int(max(g_ids.max(initial=0), f_ids.max(initial=0)))
    f_code = np.unique(f_q * width + f_ids)
    g_code = g_q * width + g_ids
    keep = ~np.isin(g_code, f_code) if drop_filtered_gold else np.ones(g_code.size, dtype=bool)
    out = {"pair_q": g_q[keep], "pair_gold": g_ids[keep]}
    out["filt_ptr"], out["filt_ids"] = _csr(f_code, nq, width)
    out["excl_ptr"], out["excl_ids"] = _csr(np.union1d(f_code, g_code), nq, width)
    out["gold_ptr"], out["gold_ids"] = _csr(np.sort(g_code), nq, width)
    return out


def _dev_ids(a, dev, dtype):
    """Host id array -> device tensor; an empty CSR id array still gets one (never read) element."""
    a = np.asarray(a)
    if a.size and (a.min() < np.iinfo(np.int32).min or a.max() > np.iinfo(np.int32).max) and dtype == torch.int32:
        raise ValueError("kgrec_b200: ids must fit 32 bits")
    return torch.as_tensor(a if a.size else np.zeros(1, a.dtype), device=dev).to(dtype).contiguous()


def link_side_arrays(keys, eval_dict, all_dicts, rel_category=None):
    """side_arrays(..., drop_filtered_gold=False) -- every (query, gold) pair, the filter, exclusion and gold CSRs --
    plus, per pair:
      has_filt  bool: the gold is not in its query's filter set, so it has a filtered rank (these are the pairs
                side_arrays keeps with drop_filtered_gold=True, in the same order)
      pair_cat  int8 category of the query's relation (rel_category given); a key of eval_dict whose relation has
                no category (-1, or beyond rel_category) raises ValueError
    Keys are (entity, relation) tuples."""
    a = side_arrays(keys, eval_dict, all_dicts, drop_filtered_gold=False)
    width = 1 + int(max(a["pair_gold"].max(initial=0), a["filt_ids"].max(initial=0)))
    f_q = np.repeat(np.arange(len(keys), dtype=np.int64), np.diff(a["filt_ptr"]))
    a["has_filt"] = ~np.isin(a["pair_q"] * width + a["pair_gold"], f_q * width + a["filt_ids"])
    if rel_category is not None:
        cat = np.asarray(rel_category)
        rels = np.fromiter((k[1] for k in eval_dict), dtype=np.int64, count=len(eval_dict))
        if rels.size and (rels.min() < 0 or rels.max() >= cat.size or (cat[rels] < 0).any()):
            raise ValueError("kgrec_b200: a relation of the eval dict has no category in rel_category")
        kr = np.fromiter((k[1] for k in keys), dtype=np.int64, count=len(keys))
        a["pair_cat"] = cat[kr[a["pair_q"]]].astype(np.int8)
    return a


class _KGSide:
    """Device arrays of one KG side.  TransR keeps its pairs sorted by relation (kgrec_transr_eval_* take the queries
    of one relation as one run) and maps the ranks back to the driver's order with `inv`.

    link=True keeps every (query, gold) pair, `has_filt` (link_side_arrays), the gold CSR and, with rel_category,
    the per-pair group masks `grp` [1 + 4, n] (row 0: all pairs; row 1 + c: pairs of category c)."""

    def __init__(self, model, side, eval_dict, all_dicts, chunk, transr, link=False, rel_category=None):
        dev = model.device
        self.sd = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
        keys = [k for k, gold in eval_dict.items() if len(gold) > 0]
        a = link_side_arrays(keys, eval_dict, all_dicts, rel_category) if link else \
            side_arrays(keys, eval_dict, all_dicts, drop_filtered_gold=True)
        kq = np.fromiter((k[0] for k in keys), dtype=np.int64, count=len(keys))
        kr = np.fromiter((k[1] for k in keys), dtype=np.int64, count=len(keys))
        q, r, gold, row = kq[a["pair_q"]], kr[a["pair_q"]], a["pair_gold"], a["pair_q"]
        n_ent, n_rel = model.ent_embeddings.weight.shape[0], model.rel_embeddings.weight.shape[0]
        for name, ids, bound in (("query", q, n_ent), ("relation", r, n_rel), ("gold", gold, n_ent)):
            if ids.size and (ids.min() < 0 or ids.max() >= bound):
                raise IndexError("kgrec_b200: a %s id of the %s eval dict is out of range for its table" % (name, side))
        self.n = int(q.size)
        if link:
            self.n_filt = int(a["has_filt"].sum())
            self.has_filt = torch.as_tensor(a["has_filt"], device=dev)
            self.kept = torch.as_tensor(np.flatnonzero(a["has_filt"]), device=dev)
            self.gold_ptr = torch.as_tensor(a["gold_ptr"], device=dev)
            self.gold_ids = _dev_ids(a["gold_ids"], dev, torch.int32)
            grp = [np.ones(self.n, dtype=bool)]
            if rel_category is not None:
                grp += [a["pair_cat"] == c for c in range(4)]
            self.grp = torch.as_tensor(np.stack(grp), device=dev)                        # [groups, n] (driver order)
            self.grp_filt = self.grp & self.has_filt[None, :]
        self.inv = None
        if transr and self.n:
            order = np.argsort(r, kind="stable")
            q, r, gold, row = q[order], r[order], gold[order], row[order]
            inv = np.empty_like(order)
            inv[order] = np.arange(order.size)
            self.inv = torch.as_tensor(inv, device=dev)
            cut = np.flatnonzero(np.diff(r)) + 1
            self.run_begin = torch.as_tensor(np.concatenate([[0], cut, [self.n]]).astype(np.int64))   # host arrays
            self.run_rel = torch.as_tensor(r[np.concatenate([[0], cut])].astype(np.int64))
            # gold-score chunks of the sorted pairs, each with the run boundaries inside it
            self.chunks = []
            for lo in range(0, self.n, chunk):
                hi = min(self.n, lo + chunk)
                b = np.concatenate([[lo], cut[(cut > lo) & (cut < hi)], [hi]]).astype(np.int64)
                self.chunks.append((lo, hi, torch.as_tensor(b - lo), torch.as_tensor(r[b[:-1]].astype(np.int64))))
        self.q = torch.as_tensor(q, device=dev)
        self.r = torch.as_tensor(r, device=dev)
        self.gold = torch.as_tensor(gold, device=dev)
        self.gold32 = _dev_ids(gold, dev, torch.int32)
        self.excl_row = _dev_ids(row, dev, torch.int32)
        self.excl_ptr = torch.as_tensor(a["excl_ptr"], device=dev)
        self.excl_ids = _dev_ids(a["excl_ids"], dev, torch.int32)
        self.pairs = (kq[a["pair_q"]], kr[a["pair_q"]], a["pair_gold"])    # host copy, driver order


LINK_FIELDS = ("n", "rank_sum", "rr_sum", "hits@1", "hits@3", "hits@10", "hits@topn")


class KGEvaluator:
    """Filtered KG validation (hit@topn and mean rank of both sides, as evaluate_kg) with the host work done once.

    The constructor turns the eval and filter dicts into device arrays: one row per (query, gold) pair, the query's
    exclusion CSR (filter set + gold set, ascending) and, for TransR, the relation-sorted order with its runs.
    run() then scores the current tables with device work only:
      1. gold scores by the catalog pass's own arithmetic (the gathered gold rows as an id-tagged sub-catalog, in
         chunks of `chunk` pairs; the diagonal of each [chunk, chunk] block), bit-identical to what the count compares;
      2. one filtered rank-count pass per side (kgrec_eval_rank_count_ex / kgrec_transr_eval_rank_count_ex);
      3. hit and rank sums as a [4] float64 device tensor.
    result(m) reads it back (the one synchronisation) and returns evaluate_kg's tuple.
    Models: TransE, TransH, TransR, and jTransUP's KG branch (TransH kernels on the KTUP tables, padding row included).

    link=True adds the link-prediction metrics of both settings from the same single sweep per side
    (kgrec_eval_rank_count_dual / kgrec_transr_eval_rank_count_dual).  For a query q (a key of the eval dict) with
    gold set G_q and filter set F_q (the union of all_dicts[k][q]), and a gold g of G_q, in (score, id) order:
      raw(q, g)  = #{ e in catalog : e not in G_q, (s(q, e), e) < (s(q, g), g) }   (the reference's walk without the
                   filter, -nofilter_wrong_corrupted); every gold has one
      filt(q, g) = #{ e in catalog : e not in F_q U G_q, (s(q, e), e) < (s(q, g), g) }   (the rank above); a gold
                   inside F_q has none (-1 in dual_ranks) and is left out of the filtered numbers
    Ranks are 0-based: MR = mean rank, MRR = mean 1 / (rank + 1), Hits@k = share of pairs with rank < k, for
    k in (1, 3, 10, topn).  Head and tail are reported apart and combined weighted by their pair counts.  With
    rel_category (int8 [n_rel], dataio.relation_categories / load_relation_types) every pair is also counted in the
    category of its relation (1-1 / 1-N / N-1 / N-N), so the categories partition the pairs; a relation of the eval
    dicts without a category raises.  run() then returns the float64 sums [setting (raw, filtered), side (head, tail),
    group (all, then the four categories when given), field (LINK_FIELDS)]; link_result(m) turns them into metrics
    and result(m) still returns evaluate_kg's tuple (the filtered numbers), bit for bit.
    """

    def __init__(self, model, eval_head_dict, eval_tail_dict, all_head_dicts=None, all_tail_dicts=None, topn=10, chunk=512,
                 link=False, rel_category=None):
        self.model = model
        self.topn = int(topn)
        self.chunk = int(chunk)
        self.link = bool(link)
        if rel_category is not None and not self.link:
            raise ValueError("kgrec_b200: rel_category needs link=True")
        self.groups = ("all",) + (tuple(KD.REL_CATEGORIES) if rel_category is not None else ())
        dev = model._require_cuda()
        self._transr = model.MODEL == _lib.TRANSR
        self._kg = _lib.TRANSH if model.MODEL == _lib.KTUP else model.MODEL
        self.sides = (_KGSide(model, "head", eval_head_dict, all_head_dicts, self.chunk, self._transr, self.link, rel_category),
                      _KGSide(model, "tail", eval_tail_dict, all_tail_dicts, self.chunk, self._transr, self.link, rel_category))
        n_cat, d = model.ent_embeddings.weight.shape
        n_max = max(s.n for s in self.sides)
        c = min(self.chunk, max(1, n_max))
        self._blk = torch.empty((c, c), dtype=torch.float32, device=dev)         # gold-score blocks
        self._ws = self._ws_gold = None
        if self._transr:
            lib = _lib.load()
            self._ws = torch.empty(int(lib.kgrec_transr_workspace_floats(max(1, n_max), n_cat, d)), dtype=torch.float32, device=dev)
            self._ws_gold = torch.empty(int(lib.kgrec_transr_workspace_floats(c, c, d)), dtype=torch.float32, device=dev)

    def _tables(self):
        m = self.model
        if self._transr:
            return KF.make_tables(m._weights(), m.embedding_size, m.L1_flag)
        return KF.make_tables(m._weights(), m.embedding_size, m.L1_flag, m.use_st_gumbel, m._item2ent)

    def _gold_scores(self, T, s, catalog):
        lib = _lib.load()
        rows = catalog.index_select(0, s.gold)
        gs = torch.empty(s.n, dtype=torch.float32, device=catalog.device)
        stream = KF._stream()
        if self._transr:
            status = self.model._status_buf(catalog.device)
            for lo, hi, begin, rel in s.chunks:
                n = hi - lo
                _lib.check(lib.kgrec_transr_eval_scores(
                    C.byref(T), s.sd, KF._ptr(s.q[lo:hi]), KF._ptr(s.r[lo:hi]), 8, n, C.c_void_p(begin.data_ptr()),
                    C.c_void_p(rel.data_ptr()), rel.numel(), KF._ptr(rows[lo:hi]), rows.stride(0), n, 0,
                    KF._ptr(s.gold32[lo:hi]), KF._ptr(self._ws_gold), KF._ptr(self._blk), self._blk.stride(0),
                    KF._ptr(status), stream))
                gs[lo:hi].copy_(self._blk[:n, :n].diagonal())
        else:
            for lo in range(0, s.n, self.chunk):
                hi = min(s.n, lo + self.chunk)
                KE.run(T, self._kg, s.sd, s.q[lo:hi], s.r[lo:hi], "scores", rows[lo:hi], cat_ids=s.gold32[lo:hi],
                       out=self._blk[:hi - lo, :hi - lo])
                gs[lo:hi].copy_(self._blk[:hi - lo, :hi - lo].diagonal())
        return gs

    def ranks(self):
        """Filtered rank of every (query, gold) pair of the head and the tail side under the current tables: two
        int32 device tensors in the order evaluate_kg visits the pairs (`sides[i].pairs` holds them on the host;
        with link=True, the pairs of `has_filt`)."""
        if self.link:
            return tuple(filt.index_select(0, s.kept) for s, (_, filt) in zip(self.sides, self._dual_counts()))
        m = self.model
        dev = m._require_cuda()
        lib = _lib.load()
        T = self._tables()
        catalog = m.ent_embeddings.weight.detach()
        n_cat = catalog.shape[0]
        out = []
        for s in self.sides:
            counts = torch.zeros(s.n, dtype=torch.int32, device=dev)
            if s.n:
                gs = self._gold_scores(T, s, catalog)
                if self._transr:
                    _lib.check(lib.kgrec_transr_eval_rank_count_ex(
                        C.byref(T), s.sd, KF._ptr(s.q), KF._ptr(s.r), 8, s.n, C.c_void_p(s.run_begin.data_ptr()),
                        C.c_void_p(s.run_rel.data_ptr()), s.run_rel.numel(), KF._ptr(catalog), catalog.stride(0), n_cat, 0,
                        KF._ptr(self._ws), KF._ptr(gs), KF._ptr(s.gold32), KF._ptr(counts), KF._ptr(s.excl_row),
                        KF._ptr(s.excl_ptr), KF._ptr(s.excl_ids), KF._ptr(m._status_buf(dev)), KF._stream()))
                    counts = counts.index_select(0, s.inv)
                else:
                    _lib.check(lib.kgrec_eval_rank_count_ex(
                        C.byref(T), self._kg, s.sd, KF._ptr(s.q), KF._ptr(s.r), 8, None, s.n, KF._ptr(catalog),
                        catalog.stride(0), n_cat, 0, KF._ptr(gs), KF._ptr(s.gold32), KF._ptr(counts), KF._ptr(s.excl_row),
                        KF._ptr(s.excl_ptr), KF._ptr(s.excl_ids), KF._stream()))
                    KF.count_launches(1)
            out.append(counts)
        return tuple(out)

    def _dual_counts(self):
        """link=True: (raw, filtered) int32 counts of every pair per side, driver order, from one dual sweep per side
        (a filtered count of a gold inside its filter set is computed but means nothing)."""
        m = self.model
        dev = m._require_cuda()
        lib = _lib.load()
        T = self._tables()
        catalog = m.ent_embeddings.weight.detach()
        n_cat = catalog.shape[0]
        out = []
        for s in self.sides:
            raw = torch.zeros(s.n, dtype=torch.int32, device=dev)
            filt = torch.zeros(s.n, dtype=torch.int32, device=dev)
            if s.n:
                gs = self._gold_scores(T, s, catalog)
                if self._transr:
                    _lib.check(lib.kgrec_transr_eval_rank_count_dual(
                        C.byref(T), s.sd, KF._ptr(s.q), KF._ptr(s.r), 8, s.n, C.c_void_p(s.run_begin.data_ptr()),
                        C.c_void_p(s.run_rel.data_ptr()), s.run_rel.numel(), KF._ptr(catalog), catalog.stride(0), n_cat, 0,
                        KF._ptr(self._ws), KF._ptr(gs), KF._ptr(s.gold32), KF._ptr(filt), KF._ptr(s.excl_row),
                        KF._ptr(s.excl_ptr), KF._ptr(s.excl_ids), KF._ptr(s.gold_ptr), KF._ptr(s.gold_ids), KF._ptr(raw),
                        KF._ptr(m._status_buf(dev)), KF._stream()))
                    raw, filt = raw.index_select(0, s.inv), filt.index_select(0, s.inv)
                else:
                    _lib.check(lib.kgrec_eval_rank_count_dual(
                        C.byref(T), self._kg, s.sd, KF._ptr(s.q), KF._ptr(s.r), 8, None, s.n, KF._ptr(catalog),
                        catalog.stride(0), n_cat, 0, KF._ptr(gs), KF._ptr(s.gold32), KF._ptr(filt), KF._ptr(s.excl_row),
                        KF._ptr(s.excl_ptr), KF._ptr(s.excl_ids), KF._ptr(s.gold_ptr), KF._ptr(s.gold_ids), KF._ptr(raw),
                        KF._stream()))
                    KF.count_launches(1)
            out.append((raw, filt))
        return out

    def dual_ranks(self):
        """link=True: ((head raw, head filtered), (tail raw, tail filtered)) int32 device tensors, one entry per
        (query, gold) pair in the order evaluate_kg visits them (`sides[i].pairs`); a gold inside its query's filter
        set has filtered rank -1."""
        if not self.link:
            raise ValueError("kgrec_b200: dual_ranks needs KGEvaluator(..., link=True)")
        return tuple((raw, torch.where(s.has_filt, filt, torch.full_like(filt, -1)))
                     for s, (raw, filt) in zip(self.sides, self._dual_counts()))

    def _link_sums(self, c, w):
        """[groups, fields] float64 sums of LINK_FIELDS over the pairs of each group (w: bool [groups, n]).  A plain
        reduction over a fixed shape, no atomics: the reciprocal-rank sums repeat bit for bit."""
        c = c.to(torch.float64)
        vals = torch.stack([torch.ones_like(c), c, 1.0 / (c + 1.0), (c < 1).to(c.dtype), (c < 3).to(c.dtype),
                            (c < 10).to(c.dtype), (c < self.topn).to(c.dtype)])                  # [fields, n]
        return torch.where(w[:, None, :], vals[None], torch.zeros((), dtype=c.dtype, device=c.device)).sum(-1)

    def run(self):
        """[4] float64 device tensor: (head hits, head rank sum, tail hits, tail rank sum), queued on the current
        stream with no host synchronisation.  link=True: the [2, 2, groups, 7] sums of the class docstring."""
        if self.link:
            per_side = [torch.stack([self._link_sums(raw, s.grp), self._link_sums(filt, s.grp_filt)])
                        for s, (raw, filt) in zip(self.sides, self._dual_counts())]
            return torch.stack(per_side, 1)
        parts = []
        for c in self.ranks():
            c = c.to(torch.int64)
            parts += [(c < self.topn).sum(), c.sum()]
        return torch.stack(parts).to(torch.float64)

    def link_result(self, m):
        """{"raw" | "filtered": {"head" | "tail" | "both": {group: {mr, mrr, hits@1, hits@3, hits@10, hits@topn, n}}}}
        from the sums run() returned with link=True; "both" pools head and tail pairs; a group without pairs reads 0."""
        v = m.tolist()
        out = {}
        for si, setting in enumerate(("raw", "filtered")):
            out[setting] = {}
            for side in ("head", "tail", "both"):
                out[setting][side] = {}
                for gi, g in enumerate(self.groups):
                    if side == "both":
                        f = [a + b for a, b in zip(v[si][0][gi], v[si][1][gi])]
                    else:
                        f = v[si][0 if side == "head" else 1][gi]
                    n = f[0]
                    mean = (lambda x: x / n) if n else (lambda x: 0.0)
                    out[setting][side][g] = {"mr": mean(f[1]), "mrr": mean(f[2]), "hits@1": mean(f[3]), "hits@3": mean(f[4]),
                                             "hits@10": mean(f[5]), "hits@topn": mean(f[6]), "n": int(n)}
        return out

    def result(self, m):
        """(avg_hit, avg_mean_rank, (head hit, head rank), (tail hit, tail rank)) -- evaluate_kg's tuple, bit for bit."""
        if self.link:
            v = m.tolist()
            hh, hr, th, tr = v[1][0][0][6], v[1][0][0][1], v[1][1][0][6], v[1][1][0][1]
            n_h, n_t = self.sides[0].n_filt, self.sides[1].n_filt
        else:
            hh, hr, th, tr = m.tolist()
            n_h, n_t = self.sides[0].n, self.sides[1].n
        h = (hh / n_h, hr / n_h) if n_h else (0.0, 0.0)
        t = (th / n_t, tr / n_t) if n_t else (0.0, 0.0)
        tot = max(1, n_h + n_t)
        return (float(h[0] * n_h + t[0] * n_t) / tot, float(h[1] * n_h + t[1] * n_t) / tot, (h[0], h[1]), (t[0], t[1]))


class RecEvaluator:
    """Rec-side validation (mean f1 / precision / recall / hit / NDCG@topn, as evaluate_rec) with the host work done
    once: the users with a non-empty gold set, their filter CSR and their gold CSR live on the device.  run() builds the
    catalog of the current tables (TUP soft / ST-Gumbel augmented rows, KTUP's item + entity table), takes the
    filtered top-n of every user in one call and reduces them on the device (kgrec_rec_topk_metrics); result(m) reads
    back five numbers.  ST-Gumbel draws come from `seed` (passed by value; one draw per (user position, item,
    preference)) or from explicit uniforms `gumbel_u` [n_users, n_items, P].

    ranks=True adds the whole-catalog numbers of the gold items (RecModelBase.rank_counts_items on the path of the
    top-n pass, same users, same noise): run() returns ten sums, result(m) (f1, p, r, hit, ndcg, mean_rank, mrr, auc).
      mean_rank  mean over the kept golds of the filtered 0-based rank (a gold inside its user's filter set is left out)
      mrr        mean over the kept golds of 1 / (rank + 1)
      auc        mean over the users with a kept gold and N_u > 0 of 1 - sum(ranks) / (kept golds * N_u), where
                 N_u = item_total - |filter set U gold set| is the number of unfiltered non-gold items: the share of
                 (gold, other item) pairs the model orders correctly, which is what the BPR loss optimises
    """

    def __init__(self, model, eval_dict, all_dicts=None, topn=10, ranks=False):
        self.model = model
        self.topn = int(topn)
        self.ranks = bool(ranks)
        dev = model._require_cuda()
        users = [u for u, gold in eval_dict.items() if len(gold) > 0]
        a = side_arrays(users, eval_dict, all_dicts, drop_filtered_gold=False)
        u = np.asarray(users, dtype=np.int64)
        if u.size and (u.min() < 0 or u.max() >= model.user_embeddings.weight.shape[0]):
            raise IndexError("kgrec_b200: a user id of the eval dict is out of range for its table")
        self.n = int(u.size)
        self.users = torch.as_tensor(u, device=dev)
        self.filter_csr = (torch.as_tensor(a["filt_ptr"], device=dev), _dev_ids(a["filt_ids"], dev, torch.int32))
        self.gold_ptr = torch.as_tensor(a["gold_ptr"], device=dev)
        self.gold_ids = _dev_ids(a["gold_ids"], dev, torch.int32)
        if self.ranks:
            n_items = model.item_embeddings.weight.shape[0]
            if a["gold_ids"].size and a["gold_ids"].max() >= n_items:
                raise IndexError("kgrec_b200: a gold id of the eval dict is out of range for the item table")
            self.n_gold = int(a["gold_ids"].size)
            self.gold_user = torch.as_tensor(np.repeat(np.arange(self.n, dtype=np.int64), np.diff(a["gold_ptr"])), device=dev)
            self.n_other = torch.as_tensor((n_items - np.diff(a["excl_ptr"])).astype(np.float64), device=dev)     # N_u

    def topk(self, seed=0, gumbel_u=None):
        """[n_users, topn] filtered top-n keys of the current tables (the dispatch of RecModelBase._rec_call)."""
        m, k = self.model, self.topn
        user_rows = m.user_embeddings.weight.detach()
        kw = dict(k=k, filter_csr=self.filter_csr)
        if m._gumbel_aug_ok(k):
            cat = m.gumbel_catalog()
            qrows = m._gumbel_rows(user_rows, ids=self.users, with_consts=True)
            return m._eval(m.MODEL, _lib.SIDE_REC, None, None, "topk", catalog=cat, qvec=qrows, gumbel_u=gumbel_u, seed=seed, **kw)
        if m._pref_aug_ok(k):
            cat = m.soft_catalog()
            qrows = m._aug_rows(user_rows, True, ids=self.users)
            return m._eval(m.MODEL, _lib.SIDE_REC, None, None, "topk", catalog=cat, qvec=qrows, **kw)
        return m._eval(m.MODEL, _lib.SIDE_REC, self.users, None, "topk", catalog=m._rec_catalog(), gumbel_u=gumbel_u,
                       seed=seed if m.use_st_gumbel else 0, **kw)

    def per_user(self, seed=0, gumbel_u=None):
        """[n_users, 5] float64 device tensor: (f1, p, r, hit, ndcg) per user, users in eval_dict order."""
        dev = self.model._require_cuda()
        out = torch.empty((self.n, 5), dtype=torch.float64, device=dev)
        if self.n:
            keys = self.topk(seed, gumbel_u)
            _lib.check(_lib.load().kgrec_rec_topk_metrics(KF._ptr(keys), self.n, self.topn, KF._ptr(self.gold_ptr),
                                                          KF._ptr(self.gold_ids), KF._ptr(out), KF._stream()))
            KF.count_launches(1)
        return out

    def run(self, seed=0, gumbel_u=None):
        """[5] float64 device tensor of the per-user sums, queued on the current stream with no host synchronisation
        (the hit sum is an exact count; result() divides on the host, as evaluate_rec's mean does)."""
        if not self.n:
            return torch.zeros(10 if self.ranks else 5, dtype=torch.float64, device=self.model._require_cuda())
        five = self.per_user(seed, gumbel_u).sum(0)
        return torch.cat([five, self.rank_sums(seed, gumbel_u)]) if self.ranks else five

    def rank_counts(self, seed=0, gumbel_u=None):
        """int32 [n_gold] filtered rank of every gold (gold CSR order; -1: the gold is in its user's filter set)."""
        m = self.model
        return m.rank_counts_items(self.users, (self.gold_ptr, self.gold_ids), self.filter_csr, gumbel_u=gumbel_u,
                                   seed=seed if m.use_st_gumbel else 0, topn=self.topn, n_gold=self.n_gold)

    def rank_sums(self, seed=0, gumbel_u=None):
        """[5] float64: (rank sum, reciprocal-rank sum, per-user AUC sum, kept golds, users in the AUC mean).  The
        per-user sums are integer scatter-adds, so the result repeats bit for bit."""
        c = self.rank_counts(seed, gumbel_u).to(torch.int64)
        kept = c >= 0
        c = torch.where(kept, c, torch.zeros_like(c))
        rr = torch.where(kept, 1.0 / (c.to(torch.float64) + 1.0), torch.zeros((), dtype=torch.float64, device=c.device))
        s_u = torch.zeros(self.n, dtype=torch.int64, device=c.device).index_add_(0, self.gold_user, c)
        n_u = torch.zeros(self.n, dtype=torch.int64, device=c.device).index_add_(0, self.gold_user, kept.to(torch.int64))
        use = (n_u > 0) & (self.n_other > 0)
        auc = torch.where(use, 1.0 - s_u.to(torch.float64) / (n_u.to(torch.float64) * self.n_other).clamp_min(1.0),
                          torch.zeros((), dtype=torch.float64, device=c.device))
        return torch.stack([c.sum().to(torch.float64), rr.sum(), auc.sum(), kept.sum().to(torch.float64),
                            use.sum().to(torch.float64)])

    def result(self, m):
        """(f1, precision, recall, hit, ndcg) -- evaluate_rec's tuple; with ranks, followed by (mean_rank, mrr, auc)."""
        v = m.tolist()
        five = tuple(x / self.n for x in v[:5]) if self.n else (0.0,) * 5
        if not self.ranks:
            return five
        rank_sum, rr_sum, auc_sum, n_kept, n_auc = v[5:]
        return five + (rank_sum / n_kept if n_kept else 0.0, rr_sum / n_kept if n_kept else 0.0, auc_sum / n_auc if n_auc else 0.0)
