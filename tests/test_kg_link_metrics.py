"""KG link-prediction metrics: the dual rank count (kgrec_eval_rank_count_dual / kgrec_transr_eval_rank_count_dual),
KGEvaluator(link=True) with MRR / Hits@k of the raw and filtered settings and the 1-1 / 1-N / N-1 / N-N breakdown,
and the relation categories of dataio.  On the CPU: the categories against the reference's splitRelationType, the
relation_type.dat reader, the host-side rejections of the two entry points and the constructor's host arrays."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import kg_oracle as O

FAKE = 0x7000_0000_1000
INVALID, UNSUPPORTED = 1, 2            # KGREC_ERR_INVALID / KGREC_ERR_UNSUPPORTED


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_relation_categories_match_the_reference_split(golden):
    from kgrec_b200 import dataio as KD
    g = golden("relation_types")
    allt = np.concatenate([g["train"], g["valid"], g["test"]])
    got = KD.relation_categories(allt, int(g["n_rel"]))
    assert got.dtype == np.int8
    assert got.tolist() == g["category"].tolist()
    assert set(got.tolist()) == {-1, 0, 1, 2, 3}                       # every category and an absent relation
    only_eval = np.setdiff1d(np.concatenate([g["valid"][:, 2], g["test"][:, 2]]), g["train"][:, 2])
    assert only_eval.size and (got[only_eval] >= 0).all()              # relations seen only in valid / test
    # the x.5 means: r4 (heads 1.5) and r5 (tails 2.5) are "many" on that side, r7 (1.5 after a duplicate) too
    assert got[4] == 2 and got[5] == 1 and got[7] == 2
    assert KD.relation_categories(np.zeros((0, 3), np.int64), 3).tolist() == [-1, -1, -1]
    with pytest.raises(IndexError):
        KD.relation_categories(allt, 5)


def test_relation_categories_round_half_to_even():
    from kgrec_b200 import dataio as KD
    # heads per (t, r): 2 and 3 -> mean 2.5 -> 2 (N); 1, 1, 1, 2 -> 1.25 -> 1; 1 and 2 -> 1.5 -> 2 (N)
    rows = [(0, 10, 0), (1, 10, 0), (2, 11, 0), (3, 11, 0), (4, 11, 0),
            (0, 10, 1), (1, 11, 1), (2, 12, 1), (3, 13, 1), (4, 13, 1),
            (0, 10, 2), (1, 11, 2), (2, 11, 2)]
    got = KD.relation_categories(np.asarray(rows), 3)
    assert got.tolist() == [2, 0, 2]                                   # r1's heads 1.25 and tails 1 -> 1-1


def test_load_relation_types_reads_labels_not_positions(tmp_path):
    from kgrec_b200 import dataio as KD
    p = tmp_path / "relation_type.dat"
    # as preprocessTriples.py:280-284 writes it when there is no 1-N relation: an empty category line
    p.write_text("one2one\t0\t4\none2many\t\nmany2one\t2\t5\nmany2many\t1\t3\n", encoding="utf-8")
    assert KD.load_relation_types(str(p)).tolist() == [0, 3, 2, 3, 0, 2]
    assert KD.load_relation_types(str(p), n_rel=8).tolist() == [0, 3, 2, 3, 0, 2, -1, -1]
    (tmp_path / "bad.dat").write_text("one2few\t1\n", encoding="utf-8")
    with pytest.raises(ValueError):
        KD.load_relation_types(str(tmp_path / "bad.dat"))


def test_rank_count_dual_host_rejections_without_a_gpu():
    from kgrec_b200 import _lib
    lib = _lib.load()

    def err():
        return lib.kgrec_last_error().decode()

    t = _lib.Tables(dim=100, ld=100, n_ent=5000, n_rel=7, ent=FAKE, rel=FAKE, norm=FAKE)

    def dual(excl_row=FAKE, excl_ptr=FAKE, excl_ids=FAKE, gold_ptr=FAKE, gold_set=FAKE, raw=FAKE, filt=FAKE, gold_scores=FAKE,
             side=_lib.SIDE_TAIL, model=_lib.TRANSH, id_base=0, tt=t):
        return lib.kgrec_eval_rank_count_dual(C.byref(tt), model, side, FAKE, FAKE, 8, None, 16, FAKE, 100, 5000, id_base,
                                              gold_scores, FAKE, filt, excl_row, excl_ptr, excl_ids, gold_ptr, gold_set, raw, None)
    assert dual(raw=None) == INVALID and "raw_counts" in err()
    assert dual(filt=None) == INVALID and "NULL argument" in err()
    assert dual(gold_scores=None) == INVALID and "NULL argument" in err()
    assert dual(excl_row=None) == INVALID and "exclusion CSR" in err()
    assert dual(excl_ptr=None) == INVALID and dual(excl_ids=None) == INVALID
    assert dual(gold_ptr=None) == INVALID and "gold CSR" in err()
    assert dual(gold_set=None) == INVALID and "gold CSR" in err()
    assert dual(excl_ptr=FAKE + 4) == INVALID and "aligned" in err()
    for kw in ({"gold_ptr": FAKE + 4}, {"gold_set": FAKE + 2}, {"raw": FAKE + 1}, {"filt": FAKE + 2}):
        assert dual(**kw) == INVALID and "aligned" in err(), kw
    assert dual(id_base=1 << 32) != 0 and "fit 32 bits" in err()
    assert dual(id_base=(1 << 32) - 4999) != 0 and "fit 32 bits" in err()
    assert dual(model=42) != 0 and "unknown model" in err()
    rt = _lib.Tables(dim=100, ld=100, n_user=50, n_item=60, n_pref=4, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE)
    assert dual(side=_lib.SIDE_REC, model=_lib.TUP, tt=rt) == UNSUPPORTED and "KG sides" in err()

    rr = _lib.Tables(dim=64, ld=64, n_ent=5000, n_rel=7, ent=FAKE, rel=FAKE, proj=FAKE)
    begin = (C.c_int64 * 2)(0, 16)
    rel = (C.c_int64 * 1)(3)

    def tr(excl_row=FAKE, excl_ptr=FAKE, excl_ids=FAKE, gold_ptr=FAKE, gold_set=FAKE, raw=FAKE, filt=FAKE, id_base=0,
           rels=rel, b=begin, tt=rr):
        return lib.kgrec_transr_eval_rank_count_dual(C.byref(tt), _lib.SIDE_HEAD, FAKE, FAKE, 8, 16, b, rels, 1, FAKE, 64, 5000,
                                                     id_base, FAKE, FAKE, FAKE, filt, excl_row, excl_ptr, excl_ids, gold_ptr,
                                                     gold_set, raw, None, None)
    assert tr(raw=None) == INVALID and "NULL argument" in err()
    assert tr(filt=None) == INVALID and "NULL argument" in err()
    assert tr(excl_ids=None) == INVALID and "exclusion CSR" in err()
    assert tr(excl_row=None) == INVALID and tr(excl_ptr=None) == INVALID
    assert tr(gold_ptr=None) == INVALID and "gold CSR" in err()
    assert tr(gold_set=None) == INVALID and "gold CSR" in err()
    for kw in ({"excl_ptr": FAKE + 4}, {"gold_ptr": FAKE + 4}, {"gold_set": FAKE + 2}, {"raw": FAKE + 1}, {"filt": FAKE + 2}):
        assert tr(**kw) == INVALID and "aligned" in err(), kw
    assert tr(id_base=-1) != 0 and "fit 32 bits" in err()
    assert tr(rels=(C.c_int64 * 1)(9)) != 0 and "bad run" in err()                      # the TransR run checks
    assert tr(b=(C.c_int64 * 2)(0, 15)) != 0 and "run boundaries" in err()
    assert tr(tt=_lib.Tables(dim=132, ld=132, n_ent=5000, n_rel=7, ent=FAKE, rel=FAKE, proj=FAKE)) == UNSUPPORTED


def _restated_link_side(keys, eval_dict, all_dicts, rel_category):
    """Plain-Python statement of metrics.link_side_arrays."""
    pq, pg, has, cat, eptr, eids, gptr, gids = [], [], [], [], [0], [], [0], []
    for qi, key in enumerate(keys):
        gold = eval_dict[key]
        filt = set()
        for d in all_dicts or ():
            filt |= d.get(key, set())
        for g in gold:
            pq.append(qi)
            pg.append(g)
            has.append(g not in filt)
            cat.append(int(rel_category[key[1]]))
        eids += sorted(filt | gold)
        eptr.append(len(eids))
        gids += sorted(gold)
        gptr.append(len(gids))
    return dict(pair_q=pq, pair_gold=pg, has_filt=has, pair_cat=cat, excl_ptr=eptr, excl_ids=eids, gold_ptr=gptr, gold_ids=gids)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_link_side_arrays_match_a_plain_python_restatement(seed):
    from kgrec_b200 import metrics as KM
    rng = np.random.RandomState(seed)
    E, R = 300, 6
    ev = {}
    while len(ev) < 60:
        ev[(int(rng.randint(0, E)), int(rng.randint(0, R)))] = set(int(x) for x in rng.choice(E, rng.randint(0, 21), replace=False))
    keys_all = list(ev)
    train = {k: set(int(x) for x in rng.choice(E, rng.randint(0, 40), replace=False)) for k in keys_all[::2]}
    other = {}
    for k in keys_all[::3]:
        if ev[k]:
            other[k] = set(list(ev[k])[: rng.randint(1, len(ev[k]) + 1)])  # golds inside the filter, up to all of them
    rel_category = rng.randint(0, 4, R).astype(np.int8)
    keys = [k for k, g in ev.items() if len(g) > 0]
    for all_dicts in ([train, other], None):
        got = KM.link_side_arrays(keys, ev, all_dicts, rel_category)
        want = _restated_link_side(keys, ev, all_dicts, rel_category)
        for name, v in want.items():
            assert got[name].tolist() == v, name
        # the dual count's precondition: every gold-row id is in its exclusion row
        for q in range(len(keys)):
            g_row = got["gold_ids"][got["gold_ptr"][q]:got["gold_ptr"][q + 1]]
            x_row = got["excl_ids"][got["excl_ptr"][q]:got["excl_ptr"][q + 1]]
            assert np.isin(g_row, x_row).all()
        # the pairs with a filtered rank are the pairs the filtered evaluator keeps, in its order
        kept = KM.side_arrays(keys, ev, all_dicts, drop_filtered_gold=True)
        assert got["pair_q"][got["has_filt"]].tolist() == kept["pair_q"].tolist()
        assert got["pair_gold"][got["has_filt"]].tolist() == kept["pair_gold"].tolist()
        assert got["has_filt"].all() == (all_dicts is None)
    bad = rel_category.copy()
    bad[keys_all[-1][1]] = -1
    with pytest.raises(ValueError, match="no category"):
        KM.link_side_arrays(keys, ev, [train], bad)
    with pytest.raises(ValueError, match="no category"):
        KM.link_side_arrays(keys, ev, [train], rel_category[:max(k[1] for k in ev)])     # a relation beyond the array


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _lt(x):
    return torch.as_tensor(np.asarray(x), dtype=torch.long, device="cuda")


def _kg_model(name, l1, d, E, R, rng):
    import kgrec_b200 as K
    if name == "jtransup":
        I = 200
        new_map = {i: ((int(rng.randint(0, E)) if rng.rand() < 0.7 else -1), i) for i in range(I)}
        m = K.jTransUPModel(l1, d, 150, I, E, R, {i: i for i in range(I)}, new_map, False, False)
    else:
        m = {"transe": K.TransEModel, "transh": K.TransHModel, "transr": K.TransRModel}[name](l1, d, E, R)
    with torch.no_grad():                                               # duplicated catalog rows: equal scores, ties by id
        w = m.ent_embeddings.weight
        n = w.shape[0]
        src = torch.as_tensor(rng.choice(n, min(40, n // 3), replace=False), device=w.device)
        w[(src + 7) % n] = w[src]
    return m


def _csr(rows):
    ptr = np.concatenate([[0], np.cumsum([len(s) for s in rows])]).astype(np.int64)
    ids = np.concatenate([np.asarray(sorted(s), dtype=np.int32) for s in rows] + [np.zeros(0, np.int32)])
    return torch.as_tensor(ptr, device="cuda"), torch.as_tensor(ids if ids.size else np.zeros(1, np.int32), device="cuda")


def _dual_case(name, l1, d, E, rng, n_rows=60):
    """A model, pairs (one gold each) over n_rows CSR rows and the two CSRs: row j's gold set has 0, 1 or many ids
    (0: the pair's gold is outside its gold row), its filter holds some of its golds, and pairs share rows."""
    R = 5
    m = _kg_model(name, l1, d, E, R, rng)
    n_ent = m.ent_embeddings.weight.shape[0]
    gold_rows, excl_rows = [], []
    for j in range(n_rows):
        k = (0, 1, int(rng.randint(2, 30)))[j % 3]
        g = set(int(x) for x in rng.choice(n_ent, k, replace=False))
        f = set(int(x) for x in rng.choice(n_ent, int(rng.randint(0, min(60, n_ent))), replace=False))
        if g and j % 2:
            f |= set(list(g)[: 1 + j % len(g)])                        # golds inside the filter
        gold_rows.append(g)
        excl_rows.append(f | g)
    row, gold = [], []
    for j, g in enumerate(gold_rows):
        for x in (sorted(g) if g else [int(rng.randint(0, n_ent))]):
            row.append(j)
            gold.append(x)
    row += list(rng.randint(0, n_rows, 40))                          # more pairs on shared rows
    gold += [int(rng.choice(sorted(gold_rows[j]))) if gold_rows[j] else int(rng.randint(0, n_ent)) for j in row[len(gold):]]
    n = len(row)
    q, r = rng.randint(0, n_ent if name != "jtransup" else E, n), rng.randint(0, R, n)
    return m, np.asarray(q), np.asarray(r), np.asarray(gold), np.asarray(row, dtype=np.int32), _csr(excl_rows), _csr(gold_rows)


def _counts_dual_and_ex(m, name, side, q, r, gold, row, excl, gcsr, shards):
    """(raw, filt) of the dual entry and (raw, filt) of two kgrec_*_rank_count_ex passes (the gold CSR as the
    exclusion for raw), summed over catalog shards [lo, hi) with id_base = lo."""
    from kgrec_b200 import _lib, functional as KF
    lib = _lib.load()
    d = m.embedding_size
    kg = _lib.TRANSH if name == "jtransup" else m.MODEL
    sd = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
    transr = name == "transr"
    n = q.size
    order = np.argsort(r, kind="stable") if transr else np.arange(n)
    q, r, gold, row = q[order], r[order], gold[order], row[order]
    qt, rt, gt = _lt(q), _lt(r), _lt(gold)
    full = m.evaluateHead(qt, rt) if side == "head" else m.evaluateTail(qt, rt)
    gs = full[torch.arange(n, device="cuda"), gt].contiguous()          # any gold scores do: both sides of the test share them
    g32 = gt.to(torch.int32)
    row_t = torch.as_tensor(row, device="cuda")
    cat = m.ent_embeddings.weight.detach()
    T = KF.make_tables(m._weights(), d, m.L1_flag) if transr else KF.make_tables(m._weights(), d, m.L1_flag, m.use_st_gumbel, m._item2ent)
    st = KF._stream()
    out = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(4)]   # dual raw, dual filt, ex raw, ex filt
    if transr:
        cut = np.flatnonzero(np.diff(r)) + 1
        begin = torch.as_tensor(np.concatenate([[0], cut, [n]]).astype(np.int64))
        rels = torch.as_tensor(r[np.concatenate([[0], cut])].astype(np.int64))
        status = m._status_buf(torch.device("cuda"))
    for lo, hi in shards:
        c = cat[lo:hi]
        if transr:
            ws = torch.empty(int(lib.kgrec_transr_workspace_floats(n, hi - lo, d)), dtype=torch.float32, device="cuda")
            common = [C.byref(T), sd, KF._ptr(qt), KF._ptr(rt), 8, n, C.c_void_p(begin.data_ptr()), C.c_void_p(rels.data_ptr()),
                      rels.numel(), KF._ptr(c), c.stride(0), hi - lo, lo, KF._ptr(ws), KF._ptr(gs), KF._ptr(g32)]
            _lib.check(lib.kgrec_transr_eval_rank_count_dual(*common, KF._ptr(out[1]), KF._ptr(row_t), KF._ptr(excl[0]), KF._ptr(excl[1]),
                                                             KF._ptr(gcsr[0]), KF._ptr(gcsr[1]), KF._ptr(out[0]), KF._ptr(status), st))
            for o, (p, i) in ((out[2], gcsr), (out[3], excl)):
                _lib.check(lib.kgrec_transr_eval_rank_count_ex(*common, KF._ptr(o), KF._ptr(row_t), KF._ptr(p), KF._ptr(i),
                                                               KF._ptr(status), st))
        else:
            common = [C.byref(T), kg, sd, KF._ptr(qt), KF._ptr(rt), 8, None, n, KF._ptr(c), c.stride(0), hi - lo, lo,
                      KF._ptr(gs), KF._ptr(g32)]
            _lib.check(lib.kgrec_eval_rank_count_dual(*common, KF._ptr(out[1]), KF._ptr(row_t), KF._ptr(excl[0]), KF._ptr(excl[1]),
                                                      KF._ptr(gcsr[0]), KF._ptr(gcsr[1]), KF._ptr(out[0]), st))
            for o, (p, i) in ((out[2], gcsr), (out[3], excl)):
                _lib.check(lib.kgrec_eval_rank_count_ex(*common, KF._ptr(o), KF._ptr(row_t), KF._ptr(p), KF._ptr(i), st))
    return [x.cpu().numpy() for x in out]


@pytest.mark.gpu
@pytest.mark.parametrize("d", [32, 100, 128])
@pytest.mark.parametrize("name,l1", [("transe", True), ("transe", False), ("transh", True), ("transh", False),
                                     ("jtransup", False), ("transr", False), ("transr", True)])
def test_dual_count_equals_two_filtered_passes(name, l1, d):
    rng = np.random.RandomState(sum(map(ord, name)) * 5 + 3 * int(l1) + d)
    torch.manual_seed(3)
    E = 700
    m, q, r, gold, row, excl, gcsr = _dual_case(name, l1, d, E, rng)
    n_cat = m.ent_embeddings.weight.shape[0]
    for side in ("head", "tail"):
        whole = _counts_dual_and_ex(m, name, side, q, r, gold, row, excl, gcsr, [(0, n_cat)])
        assert np.array_equal(whole[0], whole[2]) and np.array_equal(whole[1], whole[3]), side
        assert (whole[0] >= whole[1]).all() and (whole[0] > whole[1]).any()
        cuts = [0, 211, 452, n_cat]                                    # three shards with id_base: the counts add
        shards = _counts_dual_and_ex(m, name, side, q, r, gold, row, excl, gcsr, list(zip(cuts[:-1], cuts[1:])))
        for a, b in zip(shards, whole):
            assert np.array_equal(a, b), side


@pytest.mark.gpu
@pytest.mark.parametrize("E", [31, 32, 33, 63, 64, 65, 127, 128, 129, 257])
@pytest.mark.parametrize("name", ["transe", "transh"])
def test_dual_count_at_catalog_tile_edges(name, E):
    rng = np.random.RandomState(E * 3 + len(name))
    torch.manual_seed(4)
    m, q, r, gold, row, excl, gcsr = _dual_case(name, False, 100, E, rng, n_rows=9)
    for side in ("head", "tail"):
        got = _counts_dual_and_ex(m, name, side, q, r, gold, row, excl, gcsr, [(0, E)])
        assert np.array_equal(got[0], got[2]) and np.array_equal(got[1], got[3])


def _kg_dicts(rng, E, R, n_head=45, n_tail=55):
    def rand_dict(n):
        out = {}
        while len(out) < n:
            out[(int(rng.randint(0, E)), int(rng.randint(0, R)))] = set(int(x) for x in rng.choice(E, rng.randint(1, 21), replace=False))
        return out
    head_eval, tail_eval = rand_dict(n_head), rand_dict(n_tail)
    head_all = [{k: set(int(x) for x in rng.choice(E, 30, replace=False)) for k in list(head_eval)[::2]}]
    tail_all = [{k: set(int(x) for x in rng.choice(E, 25, replace=False)) for k in list(tail_eval)[::3]}, {}]
    for k in list(tail_eval)[::4]:
        tail_all[1][k] = {next(iter(tail_eval[k]))}                     # gold ids inside the filter
    k0 = list(head_eval)[1]
    head_all[0][k0] = set(head_eval[k0])                               # every gold of a query filtered
    head_eval[(int(rng.randint(0, E)), 0)] = set()                      # empty gold set: skipped
    return head_eval, tail_eval, head_all, tail_all


def _walk(m, side, e, a):
    """(raw, filtered) ranks of every pair from the reference's walk on the model's own score matrix (driver order;
    filtered -1 for a gold inside the filter)."""
    keys = [k for k, g in e.items() if g]
    q, r = _lt([k[0] for k in keys]), _lt([k[1] for k in keys])
    full = (m.evaluateHead(q, r) if side == "head" else m.evaluateTail(q, r)).cpu().numpy()
    raw, filt = [], []
    for b, key in enumerate(keys):
        f = set()
        for dct in a or ():
            f |= dct.get(key, set())
        w_raw = O.kg_ranks(full[b], e[key], None, 10)
        w_f = O.kg_ranks(full[b], e[key], f, 10)
        raw += [w_raw[g][1] for g in e[key]]
        filt += [w_f[g][1] if g in w_f else -1 for g in e[key]]
    return raw, filt


def _np_link(raw_or_filt, topn):
    c = np.asarray([x for x in raw_or_filt if x >= 0], dtype=np.float64)
    return dict(n=c.size, mr=c.mean() if c.size else 0.0, mrr=(1.0 / (c + 1.0)).sum() / c.size if c.size else 0.0,
                **{"hits@%d" % k: float((c < k).mean()) if c.size else 0.0 for k in (1, 3, 10)},
                **{"hits@topn": float((c < topn).mean()) if c.size else 0.0})


@pytest.mark.gpu
@pytest.mark.parametrize("d", [32, 100, 128])
@pytest.mark.parametrize("l1", [True, False])
@pytest.mark.parametrize("name", ["transe", "transh", "transr", "jtransup"])
def test_link_evaluator_matches_separate_evaluators_and_the_walk(name, l1, d):
    from kgrec_b200 import metrics as KM
    rng = np.random.RandomState(sum(map(ord, name)) * 11 + 3 * int(l1) + d)
    torch.manual_seed(5)
    E, R, topn = 700, 5, 7
    m = _kg_model(name, l1, d, E, R, rng)
    h, t, ha, ta = _kg_dicts(rng, E, R)
    ev = KM.KGEvaluator(m, h, t, ha, ta, topn=topn, link=True)
    sums = ev.run()
    assert sums.shape == (2, 2, 1, 7) and sums.dtype == torch.float64
    # filtered totals == today's evaluator; raw totals == the evaluator without the filter
    filtered = KM.KGEvaluator(m, h, t, ha, ta, topn=topn)
    assert ev.result(sums) == filtered.result(filtered.run())
    plain = KM.KGEvaluator(m, h, t, None, None, topn=topn)
    raw_want = plain.result(plain.run())
    lr = ev.link_result(sums)
    n_h, n_t = lr["raw"]["head"]["all"]["n"], lr["raw"]["tail"]["all"]["n"]
    tot = n_h + n_t
    hr, th = lr["raw"]["head"]["all"], lr["raw"]["tail"]["all"]
    assert (hr["hits@topn"], hr["mr"]) == raw_want[2] and (th["hits@topn"], th["mr"]) == raw_want[3]
    assert (float(hr["hits@topn"] * n_h + th["hits@topn"] * n_t) / tot, float(hr["mr"] * n_h + th["mr"] * n_t) / tot) == raw_want[:2]
    # every rank against the walk on the model's own score matrices; metrics against a float64 numpy reduction
    dual = ev.dual_ranks()
    for i, (side, e, a) in enumerate((("head", h, ha), ("tail", t, ta))):
        raw_w, filt_w = _walk(m, side, e, a)
        raw_g, filt_g = dual[i][0].cpu().tolist(), dual[i][1].cpu().tolist()
        assert raw_g == raw_w and filt_g == filt_w, side
        assert ev.ranks()[i].cpu().tolist() == [x for x in filt_w if x >= 0]
        for setting, ranks in (("raw", raw_g), ("filtered", filt_g)):
            want, got = _np_link(ranks, topn), lr[setting][side]["all"]
            assert got["n"] == want["n"] and got["mr"] == want["mr"]
            for k in ("hits@1", "hits@3", "hits@10", "hits@topn"):
                assert got[k] == want[k], (setting, side, k)
            assert got["mrr"] == pytest.approx(want["mrr"], rel=1e-12, abs=0)
    both = _np_link(dual[0][0].cpu().tolist() + dual[1][0].cpu().tolist(), topn)
    assert lr["raw"]["both"]["all"]["n"] == both["n"] and lr["raw"]["both"]["all"]["hits@3"] == both["hits@3"]
    assert lr["raw"]["both"]["all"]["mrr"] == pytest.approx(both["mrr"], rel=1e-12, abs=0)
    assert lr["filtered"]["head"]["all"]["n"] < lr["raw"]["head"]["all"]["n"]       # golds inside the filter drop out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["transe", "transh", "transr", "jtransup"])
def test_category_breakdown_equals_evaluators_on_restricted_dicts(name):
    from kgrec_b200 import dataio as KD, metrics as KM
    rng = np.random.RandomState(17 + len(name))
    torch.manual_seed(6)
    E, R, topn = 600, 8, 10
    m = _kg_model(name, False, 100, E, R, rng)
    h, t, ha, ta = _kg_dicts(rng, E, R, 70, 70)
    cat = np.asarray([0, 1, 2, 3, 0, 1, 2, 3], dtype=np.int8)
    ev = KM.KGEvaluator(m, h, t, ha, ta, topn=topn, link=True, rel_category=cat)
    sums = ev.run()
    assert sums.shape == (2, 2, 5, 7)
    exact = [0, 1, 3, 4, 5, 6]                                          # every field but the reciprocal-rank sum
    assert torch.equal(sums[:, :, 1:, exact].sum(2), sums[:, :, 0, exact])          # the categories partition the pairs
    lr = ev.link_result(sums)
    assert ev.groups == ("all",) + KD.REL_CATEGORIES
    for c, g in enumerate(KD.REL_CATEGORIES):
        sub = lambda dct: {k: v for k, v in dct.items() if cat[k[1]] == c}          # noqa: E731
        one = KM.KGEvaluator(m, sub(h), sub(t), ha, ta, topn=topn, link=True)
        want = one.link_result(one.run())
        for setting in ("raw", "filtered"):
            for side in ("head", "tail", "both"):
                got, w = lr[setting][side][g], want[setting][side]["all"]
                assert got["n"] == w["n"] and got["n"] > 0
                for k in ("mr", "hits@1", "hits@3", "hits@10", "hits@topn"):
                    assert got[k] == w[k], (g, setting, side, k)
                assert got["mrr"] == pytest.approx(w["mrr"], rel=1e-12, abs=0)
    bad = cat.copy()
    bad[3] = -1
    with pytest.raises(ValueError, match="no category"):
        KM.KGEvaluator(m, h, t, ha, ta, topn=topn, link=True, rel_category=bad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["transe", "transh", "transr", "jtransup"])
def test_link_run_has_no_host_sync_and_repeats_bit_for_bit(name):
    from kgrec_b200 import metrics as KM
    rng = np.random.RandomState(23)
    m = _kg_model(name, False, 100, 700, 4, rng)
    h, t, ha, ta = _kg_dicts(rng, 700, 4)
    ev = KM.KGEvaluator(m, h, t, ha, ta, topn=10, link=True, rel_category=np.asarray([0, 1, 2, 3], dtype=np.int8))
    ev.run()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = ev.run()
        b = ev.run()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a, b)
    assert a.view(torch.int64).equal(b.view(torch.int64))             # bit for bit, reciprocal-rank sums included


@pytest.mark.gpu
def test_link_evaluator_sees_tables_after_graphed_training():
    import kgrec_b200 as K
    from kgrec_b200 import metrics as KM
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import TripleNegativeSampler
    from kgrec_b200.train import GraphedTrainLoop
    rng = np.random.RandomState(9)
    torch.manual_seed(9)
    E, R = 600, 7
    m = K.TransEModel(False, 64, E, R)
    data = np.stack([rng.randint(0, E, 2000), rng.randint(0, E, 2000), rng.randint(0, R, 2000)], 1)
    it, sampler = DeviceTrainIterator(data, 200, device="cuda", seed=1), TripleNegativeSampler(E, R, known_triples=data)
    opt = SparseRowOptimizer(m, optimizer_type="Adagrad", lr=0.05, l2_lambda=0.0, clip=1.0)
    loop = GraphedTrainLoop(m, opt, it, sampler, 1, steps_per_graph=5, sample_seed=3)
    h, t, ha, ta = _kg_dicts(np.random.RandomState(4), E, R, 30, 30)
    ev = KM.KGEvaluator(m, h, t, ha, ta, topn=10, link=True)

    def fresh():
        e2 = KM.KGEvaluator(m, h, t, ha, ta, topn=10, link=True)
        return e2.link_result(e2.run())
    before = ev.link_result(ev.run())
    assert before == fresh()
    loop.run(20)
    after = ev.link_result(ev.run())
    assert after != before
    assert after == fresh()
    assert ev.result(ev.run()) == KM.evaluate_kg(m, h, t, ha, ta, topn=10)
