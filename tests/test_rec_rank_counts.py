"""Rank counts of the recommendation side: kgrec_rec_gold_scores / kgrec_rec_rank_count, RecModelBase.rank_counts_items
and RecEvaluator(ranks=True) against a restatement of the definition applied to the model's own score matrix; on the
CPU, the restatement on a hand-computed example and the host-side rejections of the new entry points."""
import ctypes as C

import numpy as np
import pytest
import torch

FAKE = 0x7000_0000_1000
INVALID, UNSUPPORTED = 1, 2


# ---- the definition, restated from a full fp32 score matrix -----------------------------------------------------------
def oracle_counts(scores, golds, filts, id_base=0):
    """counts per (user, gold) in CSR order (users in row order, golds ascending): the number of catalog columns e
    (global id id_base + column) with (score bits, id) < (gold's score bits, gold id), e not in the user's filter set and
    not one of the user's golds; -1 for a gold inside the filter set.  `scores` holds every gold's column."""
    scores = np.ascontiguousarray(scores, dtype=np.float32)
    ids = np.arange(scores.shape[1], dtype=np.uint64) + np.uint64(id_base)
    out = []
    for q, (gold, filt) in enumerate(zip(golds, filts)):
        key = (scores[q].view(np.uint32).astype(np.uint64) << np.uint64(32)) | ids
        skip = np.isin(ids, np.fromiter(set(gold) | set(filt), dtype=np.uint64, count=len(set(gold) | set(filt))))
        for g in sorted(gold):
            out.append(-1 if g in filt else int(np.count_nonzero((key < key[g - id_base]) & ~skip)))
    return np.asarray(out, dtype=np.int64)


def oracle_metrics(counts, golds, filts, item_total):
    """(mean_rank, mrr, auc) in float64 from oracle_counts' output."""
    kept = counts >= 0
    mean_rank = float(counts[kept].mean()) if kept.any() else 0.0
    mrr = float((1.0 / (counts[kept] + 1.0)).mean()) if kept.any() else 0.0
    aucs, j = [], 0
    for gold, filt in zip(golds, filts):
        c = counts[j:j + len(gold)]
        j += len(gold)
        c = c[c >= 0]
        n_other = item_total - len(set(gold) | set(filt))
        if c.size and n_other > 0:
            aucs.append(1.0 - float(c.sum()) / (c.size * n_other))
    return mean_rank, mrr, float(np.mean(aucs)) if aucs else 0.0


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_oracle_on_a_hand_computed_example_with_a_tie():
    s = np.asarray([[0.5, 0.25, 0.25, 1.0, 0.75, 0.25],      # items 1, 2, 5 tie
                    [3.0, 2.0, 1.0, 0.5, 4.0, 5.0],
                    [1.0, 1.0, 1.0, 1.0, 1.0, 1.0]], dtype=np.float32)
    golds = [{2, 4}, {0, 3}, {5}]
    filts = [{0}, {3, 2}, {5, 0}]            # user 1: gold 3 is filtered; user 2: its only gold is filtered
    c = oracle_counts(s, golds, filts)
    # user 0: order by (score, id) = 1, 2, 5, 0, 4, 3; item 0 filtered, golds 2 and 4 never count each other:
    #   gold 2: {1} -> 1 (5 ties on score and has the larger id); gold 4: {1, 5} -> 2
    # user 1: order 3, 2, 1, 0, 4, 5; filter {3, 2}: gold 0: {1} -> 1; gold 3 is filtered -> -1
    assert c.tolist() == [1, 2, 1, -1, -1]
    mean_rank, mrr, auc = oracle_metrics(c, golds, filts, 6)
    assert mean_rank == pytest.approx(4 / 3) and mrr == pytest.approx((1 / 2 + 1 / 3 + 1 / 2) / 3)
    # N_0 = 6 - |{0, 2, 4}| = 3, N_1 = 6 - |{0, 2, 3}| = 3; user 2 has no kept gold
    assert auc == pytest.approx(((1 - 3 / (2 * 3)) + (1 - 1 / (1 * 3))) / 2)


def test_rec_rank_host_rejections_without_a_gpu():
    from kgrec_b200 import _lib
    lib = _lib.load()

    def err():
        return lib.kgrec_last_error().decode()

    rt = _lib.Tables(dim=100, ld=100, n_user=50, n_item=60, n_pref=4, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE)
    kt = _lib.Tables(dim=100, ld=100, n_ent=500, n_rel=7, ent=FAKE, rel=FAKE, norm=FAKE)
    base = dict(tt=rt, model=_lib.TUP, q=FAKE, idx=8, qvec=None, nq=16, cat=FAKE, ld=100, n_cat=60, id_base=0, gptr=FAKE, gids=FAKE)

    def head(a):
        return (C.byref(a["tt"]), a["model"], a["q"], a["idx"], a["qvec"], a["nq"], a["cat"], a["ld"], a["n_cat"], a["id_base"],
                a["gptr"], a["gids"])

    def gs(out=FAKE, **kw):
        return lib.kgrec_rec_gold_scores(*head({**base, **kw}), None, 0, out, None)

    def rc(n_gold=40, scores=FAKE, fptr=FAKE, fids=FAKE, counts=FAKE, ws=FAKE, ws_bytes=1 << 20, **kw):
        return lib.kgrec_rec_rank_count(*head({**base, **kw}), n_gold, scores, fptr, fids, None, 0, counts, ws, ws_bytes, None)

    for call in (gs, rc):
        assert call(model=_lib.TRANSH, tt=kt) == INVALID and "not a recommendation model" in err()
        assert call(model=42) == INVALID
        assert call(gptr=None) == INVALID and "NULL argument" in err()
        assert call(gids=None) == INVALID
        assert call(gptr=FAKE + 4) == INVALID and "aligned" in err()
        assert call(q=None) == INVALID and "query ids" in err()
        assert call(idx=3) == INVALID and "idx_bytes" in err()
        assert call(id_base=1 << 32) == INVALID and "fit 32 bits" in err()
        assert call(n_cat=1 << 32) == INVALID
        assert call(cat=None) == INVALID
        assert call(nq=-1) == INVALID
        assert call(nq=0, gptr=None) == 0                                     # no users: nothing to do
        assert call(ld=102) != 0                                              # not a multiple of 4
        # augmented rows: the catalog's leading dimension must be the path's
        assert call(qvec=FAKE, ld=100) == INVALID and "leading dimension" in err()
        wide = _lib.Tables(dim=260, ld=260, n_user=50, n_item=60, n_pref=4, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE)
        assert call(tt=wide, ld=260) == UNSUPPORTED and "[1, 256]" in err()
        big = _lib.Tables(dim=256, ld=256, n_user=50, n_item=60, n_pref=128, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE)
        assert not lib.kgrec_pref_eval_supported(256, 128, 0, 0)
        assert call(tt=big, ld=256) == UNSUPPORTED and "limit" in err()          # outside the plain path's envelope
    assert gs(out=None) == INVALID and "gold_scores" in err()
    assert rc(scores=None) == INVALID and rc(counts=None) == INVALID and "NULL argument" in err()
    assert rc(fptr=None) == INVALID and "filter CSR" in err()
    assert rc(fids=FAKE + 2) == INVALID and "aligned" in err()
    assert rc(n_gold=-1) == INVALID
    assert rc(n_gold=0, scores=None, counts=None, ws=None) == 0               # no golds: nothing to do
    need = lib.kgrec_rec_rank_workspace_bytes(16, 40)
    assert need >= 16 * 8 + 40 * 24
    assert rc(ws=None) == INVALID and "workspace" in err()
    assert rc(ws_bytes=need - 1) == INVALID and str(need) in err()
    assert rc(ws=FAKE + 4) == INVALID

    # the KG entry points keep turning the rec side away
    assert lib.kgrec_eval_rank_count_ex(C.byref(rt), _lib.TUP, _lib.SIDE_REC, FAKE, FAKE, 8, None, 16, FAKE, 100, 60, 0,
                                        FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None) == UNSUPPORTED and "KG sides" in err()
    lda = lib.kgrec_pref_aug_ld(100)
    assert lib.kgrec_eval_rank_count(C.byref(rt), _lib.TUP, _lib.SIDE_REC, None, None, 8, FAKE, 16, FAKE, lda, 60, 0,
                                     FAKE, FAKE, FAKE, None) == UNSUPPORTED and "KG sides" in err()


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _model(name, l1, d, P, U, I, rng, dup=True):
    import kgrec_b200 as K
    if name.startswith("ktup"):
        E = I + 40
        new_map = {i: ((int(rng.randint(0, E)) if rng.rand() < 0.7 else -1), i) for i in range(I)}
        m = K.jTransUPModel(l1, d, U, I, E, P, {i: i for i in range(I)}, new_map, False, name.endswith("gumbel"))
    else:
        m = K.TransUPModel(l1, d, U, I, P, name.endswith("gumbel"))
    if dup and I > 40:
        with torch.no_grad():                                  # duplicated item rows: equal scores, ties broken by id
            w = m.item_embeddings.weight
            src = torch.as_tensor(rng.choice(I, I // 8, replace=False), device=w.device)
            w[(src + 3) % I] = w[src]
            if name.startswith("ktup"):
                m._item2ent[(src + 3) % I] = m._item2ent[src]
    return m


def _sets(rng, n_users, I, big=70):
    """Gold and filter sets per user: 0, 1, several and `big` golds; empty filter rows, a row filtering the whole
    catalog, filtered golds, filter ids beyond the catalog."""
    golds, filts = [], []
    for q in range(n_users):
        n_g = [0, 1, 3, 5, min(big, I), 2][q % 6] if I > 8 else min(I, q % 3)
        g = set(int(x) for x in rng.choice(I, n_g, replace=False))
        f = set(int(x) for x in rng.choice(I, min(I, rng.randint(0, 40)), replace=False)) if q % 4 else set()
        if q % 5 == 2 and g:
            f.add(sorted(g)[0])                                # a gold that is filtered
        if q % 7 == 3:
            f |= {I + 5, I + 90}                               # ids outside every shard
        if q == 9:
            f = set(range(I))                                  # the whole catalog
        golds.append(g)
        filts.append(f)
    return golds, filts


def _csr(sets, dev="cuda"):
    ptr = np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.int64)
    ids = np.concatenate([np.asarray(sorted(s), dtype=np.int32) for s in sets] + [np.zeros(0, np.int32)])
    return torch.as_tensor(ptr, device=dev), torch.as_tensor(ids if ids.size else np.zeros(1, np.int32), device=dev), int(ids.size)


def _matrix(m, u, gumbel_u=None, seed=None):
    if seed is not None:
        m._next_seed = lambda: seed                            # the hashed noise of this seed
    return (m.evaluateRec(u, None, gumbel_u) if hasattr(m, "evaluateRec") else m.evaluate(u, gumbel_u)).cpu().numpy()


SHAPES = [(n, l1, 100, 20) for n in ("tup_soft", "tup_gumbel", "ktup_soft", "ktup_gumbel") for l1 in (True, False)]
SHAPES += [("tup_soft", False, 128, 20), ("tup_gumbel", False, 128, 20), ("ktup_gumbel", True, 128, 20)]      # one per path
SHAPES += [("tup_soft", False, 200, 8), ("tup_gumbel", False, 200, 8), ("tup_gumbel", True, 200, 8)]         # wide rows


@pytest.mark.gpu
@pytest.mark.parametrize("name,l1,d,P", SHAPES)
def test_rank_counts_equal_the_definition_on_the_models_own_matrix(name, l1, d, P):
    from kgrec_b200 import evaluation as KE
    rng = np.random.RandomState(sum(map(ord, name)) + 2 * int(l1) + d)
    torch.manual_seed(5)
    U, I, B = 200, 300, 150                                    # 150 users: more than one query tile, the last one partial
    m = _model(name, l1, d, P, U, I, rng)
    u = torch.as_tensor(rng.choice(U, B, replace=False), device="cuda")
    golds, filts = _sets(rng, B, I)
    gptr, gids, n_gold = _csr(golds)
    fcsr = _csr(filts)[:2]
    gumbel = name.endswith("gumbel")
    gu = torch.rand(B, I, P, device="cuda") if gumbel else None
    full = _matrix(m, u, gu)
    want = oracle_counts(full, golds, filts)
    assert (want == -1).any() and (want > 0).any()
    got = m.rank_counts_items(u, (gptr, gids), fcsr, gumbel_u=gu, n_gold=n_gold)
    assert got.dtype == torch.int32 and got.cpu().tolist() == want.tolist()
    # the gold scores are the matrix's own entries, bit for bit
    gs = m.gold_scores_items(u, (gptr, gids), gumbel_u=gu, n_gold=n_gold).cpu().numpy()
    rows = np.repeat(np.arange(B), [len(g) for g in golds])
    assert np.array_equal(gs.view(np.uint32), full[rows, gids.cpu().numpy()[:n_gold]].view(np.uint32))
    # ties exist among the golds' neighbours: some item shares a gold's score
    assert any((full[q] == full[q, g]).sum() > 1 for q, gold in enumerate(golds) for g in gold)
    # no filter at all = the unfiltered count
    assert m.rank_counts_items(u, (gptr, gids), None, gumbel_u=gu, n_gold=n_gold).cpu().tolist() == \
        oracle_counts(full, golds, [set()] * B).tolist()
    # three catalog shards with id_base: gold scores and counts add
    seed = 0x5eed_1234 if gumbel else 0
    if gumbel:                                                 # hashed noise: the matrix the same seed and user list produce
        full = _matrix(m, u, seed=seed)
        want = oracle_counts(full, golds, filts)
        assert m.rank_counts_items(u, (gptr, gids), fcsr, seed=seed, n_gold=n_gold).cpu().tolist() == want.tolist()
    cat = m._rec_catalog()
    bounds = [KE.shard_bounds(I, 3, r) for r in range(3)]
    gs = sum(m.gold_scores_items(u, (gptr, gids), catalog=cat[lo:hi], id_base=lo, seed=seed, n_gold=n_gold) for lo, hi in bounds)
    total = sum(m.rank_counts_items(u, (gptr, gids), fcsr, catalog=cat[lo:hi], id_base=lo, seed=seed, gold_scores=gs, n_gold=n_gold)
                for lo, hi in bounds)
    assert torch.where(total < 0, torch.full_like(total, -1), total).cpu().tolist() == want.tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("name,l1", [("tup_soft", False), ("tup_gumbel", False), ("tup_gumbel", True), ("ktup_soft", True)])
def test_rank_counts_at_tile_and_piece_edges(name, l1):
    d, P = 100, 20
    for I in (1, 31, 32, 33, 39, 41, 63, 65, 257):             # tiles of 32 / 64 (augmented rows) and 40 (plain) catalog rows
        rng = np.random.RandomState(I)
        m = _model(name, l1, d, P, 40, I, rng)
        u = torch.arange(37, device="cuda")
        golds, filts = _sets(rng, 37, I, big=20)
        gptr, gids, n_gold = _csr(golds)
        seed = 77 + I
        want = oracle_counts(_matrix(m, u, seed=seed), golds, filts)
        got = m.rank_counts_items(u, (gptr, gids), _csr(filts)[:2], seed=seed, n_gold=n_gold)
        assert got.cpu().tolist()[:n_gold] == want.tolist(), I
    empty = m.rank_counts_items(torch.zeros(0, dtype=torch.long, device="cuda"),
                                (torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")), n_gold=0)
    assert empty.numel() == 0


def _rec_dicts(rng, U, I):
    eval_dict = {int(u): set(int(x) for x in rng.choice(I, rng.randint(0, 6), replace=False)) for u in rng.choice(U, 90, replace=False)}
    train = {u: set(int(x) for x in rng.choice(I, 60, replace=False)) for u in eval_dict}
    other = {u: set(int(x) for x in rng.choice(I, 5, replace=False)) for u in list(eval_dict)[::3]}
    for u in list(eval_dict)[::4]:
        if eval_dict[u]:
            other.setdefault(u, set()).add(next(iter(eval_dict[u])))            # a gold that is filtered
    return eval_dict, [train, other]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_soft", "tup_gumbel", "ktup_soft", "ktup_gumbel"])
def test_rec_evaluator_ranks_agree_with_its_top_n_and_the_definition(name):
    from kgrec_b200 import metrics as KM
    rng = np.random.RandomState(len(name))
    torch.manual_seed(3)
    U, I, topn, seed = 160, 300, 10, 0xabc_def0
    m = _model(name, False, 100, 20, U, I, rng)
    eval_dict, all_dicts = _rec_dicts(rng, U, I)
    ev = KM.RecEvaluator(m, eval_dict, all_dicts, topn=topn, ranks=True)
    plain = KM.RecEvaluator(m, eval_dict, all_dicts, topn=topn)
    users = [u for u, g in eval_dict.items() if g]
    golds = [eval_dict[u] for u in users]
    filts = [set().union(*[dd.get(u, set()) for dd in all_dicts]) for u in users]
    assert ev.n_other.cpu().tolist() == [float(I - len(g | f)) for g, f in zip(golds, filts)]
    counts = ev.rank_counts(seed=seed).cpu().numpy()
    want = oracle_counts(_matrix(m, ev.users, seed=seed), golds, filts)
    assert counts.tolist() == want.tolist() and (want < 0).any()
    # a kept gold is in the filtered top-n list exactly when fewer than topn items rank before it
    top = (ev.topk(seed=seed) & 0xFFFFFFFF).cpu().tolist()
    j = 0
    for q, g in enumerate(golds):
        for item in sorted(g):
            if counts[j] >= 0:
                assert (counts[j] < topn) == (item in top[q]), (q, item)
            else:
                assert item not in top[q]
            j += 1
    ev.run(seed=seed)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = ev.run(seed=seed)
        b = ev.run(seed=seed)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert a.dtype == torch.float64 and a.shape == (10,) and torch.equal(a, b)
    five = plain.run(seed=seed)
    assert five.shape == (5,) and torch.equal(a[:5], five)
    res = ev.result(a)
    assert len(res) == 8 and res[:5] == plain.result(five)
    assert res[5:] == pytest.approx(oracle_metrics(want, golds, filts, I), rel=1e-12, abs=0)


@pytest.mark.gpu
def test_rec_evaluator_ranks_see_the_tables_after_graphed_training():
    import kgrec_b200 as K
    from kgrec_b200 import metrics as KM
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import RatingNegativeSampler
    from kgrec_b200.train import GraphedTrainLoop
    rng = np.random.RandomState(9)
    torch.manual_seed(9)
    U, I = 200, 300
    m = K.TransUPModel(False, 64, U, I, 5, False)
    data = np.stack([rng.randint(0, U, 2000), rng.randint(0, I, 2000)], 1)
    it, sampler = DeviceTrainIterator(data, 200, device="cuda", seed=1), RatingNegativeSampler(I, known_ratings=data)
    opt = SparseRowOptimizer(m, optimizer_type="Adagrad", lr=0.05, l2_lambda=0.0, clip=1.0)
    loop = GraphedTrainLoop(m, opt, it, sampler, 1, steps_per_graph=5, sample_seed=3)
    eval_dict, all_dicts = _rec_dicts(rng, U, I)
    ev = KM.RecEvaluator(m, eval_dict, all_dicts, topn=10, ranks=True)
    users = [u for u, g in eval_dict.items() if g]
    golds = [eval_dict[u] for u in users]
    filts = [set().union(*[dd.get(u, set()) for dd in all_dicts]) for u in users]

    def want():
        return oracle_metrics(oracle_counts(_matrix(m, ev.users), golds, filts), golds, filts, I)
    before = ev.result(ev.run())
    assert before[5:] == pytest.approx(want(), rel=1e-12, abs=0)
    loop.run(20)
    after = ev.result(ev.run())
    assert after[5:] != before[5:]
    assert after[5:] == pytest.approx(want(), rel=1e-12, abs=0)
