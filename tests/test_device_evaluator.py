"""Device-resident validation: kgrec_b200.metrics.KGEvaluator / RecEvaluator against the driver-level metrics
(evaluate_kg / evaluate_rec) and the reference's ranking walk, the filtered rank count kgrec_eval_rank_count_ex and
the rec metrics kernel kgrec_rec_topk_metrics; on the CPU, their host-side rejections and the constructor's CSRs."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import kg_oracle as O

FAKE = 0x7000_0000_1000


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_rank_count_ex_and_rec_metrics_host_rejections_without_a_gpu():
    from kgrec_b200 import _lib
    lib = _lib.load()

    def err():
        return lib.kgrec_last_error().decode()

    t = _lib.Tables(dim=100, ld=100, n_ent=5000, n_rel=7, ent=FAKE, rel=FAKE, norm=FAKE)

    def ex(excl_row=FAKE, excl_ptr=FAKE, excl_ids=FAKE, gold_scores=FAKE, side=_lib.SIDE_TAIL, model=_lib.TRANSH, id_base=0, tt=t):
        return lib.kgrec_eval_rank_count_ex(C.byref(tt), model, side, FAKE, FAKE, 8, None, 16, FAKE, 100, 5000, id_base,
                                            gold_scores, FAKE, FAKE, excl_row, excl_ptr, excl_ids, None)
    assert ex(excl_row=None) == _lib_err_invalid() and "exclusion CSR" in err()
    assert ex(excl_ptr=None) == _lib_err_invalid() and "NULL array" in err()
    assert ex(excl_ids=None) == _lib_err_invalid()
    assert ex(excl_ptr=FAKE + 4) == _lib_err_invalid() and "aligned" in err()
    assert ex(excl_row=FAKE + 2) == _lib_err_invalid() and ex(excl_ids=FAKE + 1) == _lib_err_invalid()
    assert ex(gold_scores=None) != 0 and "NULL argument" in err()          # the checks of kgrec_eval_rank_count still apply
    assert ex(id_base=1 << 32) != 0 and "fit 32 bits" in err()
    assert ex(model=42) != 0 and "unknown model" in err()
    rt = _lib.Tables(dim=100, ld=100, n_user=50, n_item=60, n_pref=4, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE)
    assert ex(side=_lib.SIDE_REC, model=_lib.TUP, tt=rt) == 2 and "KG sides" in err()          # KGREC_ERR_UNSUPPORTED

    rr = _lib.Tables(dim=64, ld=64, n_ent=5000, n_rel=7, ent=FAKE, rel=FAKE, proj=FAKE)
    begin = (C.c_int64 * 2)(0, 16)
    rel = (C.c_int64 * 1)(3)

    def tr(excl_row=FAKE, excl_ptr=FAKE, excl_ids=FAKE, counts=FAKE, id_base=0, rels=rel):
        return lib.kgrec_transr_eval_rank_count_ex(C.byref(rr), _lib.SIDE_HEAD, FAKE, FAKE, 8, 16, begin, rels, 1, FAKE, 64, 5000,
                                                   id_base, FAKE, FAKE, FAKE, counts, excl_row, excl_ptr, excl_ids, None, None)
    assert tr(excl_ids=None) == _lib_err_invalid() and "exclusion CSR" in err()
    assert tr(excl_row=None) == _lib_err_invalid() and tr(excl_ptr=None) == _lib_err_invalid()
    assert tr(excl_ptr=FAKE + 4) == _lib_err_invalid() and "aligned" in err()
    assert tr(counts=None) != 0 and "NULL argument" in err()
    assert tr(id_base=-1) != 0 and "fit 32 bits" in err()
    assert tr(rels=(C.c_int64 * 1)(9)) != 0 and "bad run" in err()                                 # transr_check runs first

    assert lib.kgrec_rec_topk_metrics(FAKE, 10, 0, FAKE, FAKE, FAKE, None) == _lib_err_invalid() and "k >= 1" in err()
    assert lib.kgrec_rec_topk_metrics(FAKE, -1, 10, FAKE, FAKE, FAKE, None) == _lib_err_invalid()
    for i in range(4):
        args = [FAKE, 10, 10, FAKE, FAKE, FAKE]
        args[[0, 3, 4, 5][i]] = None
        assert lib.kgrec_rec_topk_metrics(*args, None) == _lib_err_invalid() and "NULL argument" in err()
    assert lib.kgrec_rec_topk_metrics(None, 0, 10, None, None, None, None) == 0                     # no users: nothing to do


def _lib_err_invalid():
    return 1      # KGREC_ERR_INVALID


def _restated_side(keys, eval_dict, all_dicts, drop_filtered_gold):
    """Plain-Python statement of metrics.side_arrays (the per-pair loop of metrics._kg_side)."""
    pq, pg, fptr, fids, eptr, eids, gptr, gids = [], [], [0], [], [0], [], [0], []
    for qi, key in enumerate(keys):
        gold = eval_dict[key]
        filt = set()
        for d in all_dicts or ():
            if key in d:
                filt.update(d[key])
        for g in gold:
            if drop_filtered_gold and g in filt:
                continue
            pq.append(qi)
            pg.append(g)
        fids += sorted(filt)
        fptr.append(len(fids))
        eids += sorted(filt | gold)
        eptr.append(len(eids))
        gids += sorted(gold)
        gptr.append(len(gids))
    return dict(pair_q=pq, pair_gold=pg, filt_ptr=fptr, filt_ids=fids, excl_ptr=eptr, excl_ids=eids, gold_ptr=gptr, gold_ids=gids)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_evaluator_csr_building_matches_a_plain_python_restatement(seed):
    from kgrec_b200 import metrics as KM
    rng = np.random.RandomState(seed)
    E = 300
    ev = {}
    while len(ev) < 60:
        ev[(int(rng.randint(0, E)), int(rng.randint(0, 4)))] = set(int(x) for x in rng.choice(E, rng.randint(0, 21), replace=False))
    keys_all = list(ev)
    train = {k: set(int(x) for x in rng.choice(E, rng.randint(0, 40), replace=False)) for k in keys_all[::2]}
    other = {k: set(int(x) for x in rng.choice(E, 5, replace=False)) for k in keys_all[1::3]}
    shared = set(int(x) for x in rng.choice(E, 8, replace=False))
    for k in keys_all[::5]:
        train.setdefault(k, set()).update(shared)                       # filter ids shared between queries
    for k in keys_all[::4]:
        if ev[k]:
            other.setdefault(k, set()).add(next(iter(ev[k])))           # a gold id that is itself filtered
    other[("unused", 0)] = {1, 2, 3}                                    # filter keys without an eval query are ignored
    keys = [k for k, g in ev.items() if len(g) > 0]
    assert len(keys) < len(ev)                                          # some empty gold sets
    for all_dicts in ([train, other], None, [{}]):
        for drop in (True, False):
            got = KM.side_arrays(keys, ev, all_dicts, drop)
            want = _restated_side(keys, ev, all_dicts, drop)
            for name, v in want.items():
                assert got[name].dtype == np.int64
                assert got[name].tolist() == v, (name, all_dicts is None, drop)
    got = KM.side_arrays([], {}, [train], True)
    assert got["pair_q"].size == 0 and got["excl_ptr"].tolist() == [0] and got["gold_ptr"].tolist() == [0]


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
        src = torch.as_tensor(rng.choice(E, 40, replace=False), device=w.device)
        w[(src + 7) % E] = w[src]
    return m


def _kg_dicts(rng, E, R, n_head=45, n_tail=55):
    def rand_dict(n):
        out = {}
        while len(out) < n:
            out[(int(rng.randint(0, E)), int(rng.randint(0, R)))] = set(int(x) for x in rng.choice(E, rng.randint(1, 21), replace=False))
        return out
    head_eval, tail_eval = rand_dict(n_head), rand_dict(n_tail)
    shared = set(int(x) for x in rng.choice(E, 12, replace=False))
    head_all = [{k: set(int(x) for x in rng.choice(E, 30, replace=False)) | shared for k in list(head_eval)[::2]}]
    tail_all = [{k: set(int(x) for x in rng.choice(E, 25, replace=False)) for k in list(tail_eval)[::3]}, {}]
    for k in list(tail_eval)[::4]:
        tail_all[1][k] = {next(iter(tail_eval[k]))}                     # gold ids inside the filter
    k0 = list(tail_eval)[1]
    tail_all[0][k0] = set(range(E)) - set(list(tail_eval[k0])[:1]) - set(rng.choice(E, 4).tolist())   # < topn unfiltered rows
    head_eval[(int(rng.randint(0, E)), 0)] = set()                      # empty gold set: skipped
    return head_eval, tail_eval, head_all, tail_all


@pytest.mark.gpu
@pytest.mark.parametrize("d", [32, 100, 128])
@pytest.mark.parametrize("l1", [True, False])
@pytest.mark.parametrize("name", ["transe", "transh", "transr", "jtransup"])
def test_kg_evaluator_matches_driver_metrics_and_ranking_walk(name, l1, d):
    from kgrec_b200 import metrics as KM
    rng = np.random.RandomState(sum(map(ord, name)) * 7 + 3 * int(l1) + d)
    torch.manual_seed(1)
    E, R, topn = 700, 5, 10
    m = _kg_model(name, l1, d, E, R, rng)
    head_eval, tail_eval, head_all, tail_all = _kg_dicts(rng, E, R)
    ev = KM.KGEvaluator(m, head_eval, tail_eval, head_all, tail_all, topn=topn)
    ranks = ev.ranks()
    for i, (s, side, e, a) in enumerate(zip(ev.sides, ("head", "tail"), (head_eval, tail_eval), (head_all, tail_all))):
        want = KM._kg_side(m, side, e, a, topn, 2048)
        assert len(want) == s.n
        assert ranks[i].cpu().tolist() == [rk for _, rk in want], side
    got = ev.result(ev.run())
    assert got == KM.evaluate_kg(m, head_eval, tail_eval, head_all, tail_all, topn=topn)
    # the reference's walk over the full score matrices
    for i, (side, e, a) in enumerate(zip(("head", "tail"), (head_eval, tail_eval), (head_all, tail_all))):
        keys = [k for k, g in e.items() if g]
        q, r = _lt([k[0] for k in keys]), _lt([k[1] for k in keys])
        full = (m.evaluateHead(q, r) if side == "head" else m.evaluateTail(q, r)).cpu().numpy()
        want = []
        for b, key in enumerate(keys):
            filt = set()
            for dct in a:
                filt |= dct.get(key, set())
            walk = O.kg_ranks(full[b], e[key], filt, topn)
            want += [walk[g][1] for g in e[key] if g in walk]
        assert ranks[i].cpu().tolist() == want


def _rec_model(name, l1, d, rng):
    import kgrec_b200 as K
    U, I, P = 160, 300, 4
    if name.startswith("ktup"):
        E = 260
        new_map = {i: ((int(rng.randint(0, E)) if rng.rand() < 0.7 else -1), i) for i in range(I)}
        m = K.jTransUPModel(l1, d, U, I, E, P, {i: i for i in range(I)}, new_map, False, name.endswith("gumbel"))
    else:
        m = K.TransUPModel(l1, d, U, I, P, name.endswith("gumbel"))
    with torch.no_grad():
        w = m.item_embeddings.weight
        src = torch.as_tensor(rng.choice(I, 30, replace=False), device=w.device)
        w[(src + 3) % I] = w[src]
    return m, U, I


def _rec_dicts(rng, U, I):
    eval_dict = {int(u): set(int(x) for x in rng.choice(I, rng.randint(0, 6), replace=False)) for u in rng.choice(U, 90, replace=False)}
    train = {u: set(int(x) for x in rng.choice(I, 60, replace=False)) for u in eval_dict}
    other = {u: set(int(x) for x in rng.choice(I, 5, replace=False)) for u in list(eval_dict)[::3]}
    u0 = [u for u in eval_dict if eval_dict[u]][0]
    train[u0] = set(range(I)) - set(list(eval_dict[u0])[:1]) - {7, 8}   # fewer than topn unfiltered items
    return eval_dict, [train, other]


@pytest.mark.gpu
@pytest.mark.parametrize("d", [32, 100, 128])
@pytest.mark.parametrize("l1", [True, False])
@pytest.mark.parametrize("name", ["tup_soft", "tup_gumbel", "ktup_soft", "ktup_gumbel"])
def test_rec_evaluator_matches_driver_metrics(name, l1, d):
    from kgrec_b200 import evaluation as KE, metrics as KM
    rng = np.random.RandomState(sum(map(ord, name)) * 7 + 3 * int(l1) + d)
    torch.manual_seed(2)
    m, U, I = _rec_model(name, l1, d, rng)
    eval_dict, all_dicts = _rec_dicts(rng, U, I)
    topn, seed = 10, 0x1234_5678_9abc
    rv = KM.RecEvaluator(m, eval_dict, all_dicts, topn=topn)
    per_user = rv.per_user(seed=seed).cpu().numpy()
    m._next_seed = lambda: seed                                        # evaluate_rec draws the same ST-Gumbel noise
    want = KM.evaluate_rec(m, eval_dict, all_dicts, topn=topn)
    got = rv.result(rv.run(seed=seed))
    assert got[3] == want[3]                                           # hit: exact
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    users = [u for u in eval_dict if eval_dict[u]]
    keys = rv.topk(seed=seed)
    ids, _ = KE.keys_to_ids_scores(keys)
    rows = np.asarray(KE.rec_metrics_from_topk(ids.cpu().tolist(), [eval_dict[u] for u in users]), dtype=np.float64)
    np.testing.assert_allclose(per_user, rows, rtol=1e-12, atol=0)
    n_free = len(set(range(I)) - all_dicts[0][users[0]] - all_dicts[1].get(users[0], set()))
    assert 0 < n_free < topn and int((ids[0] >= 0).sum()) == n_free    # a list shorter than topn: p = hits / n_free
    if name.endswith("soft"):                                          # the reference's walk over the full score matrix
        full = (m.evaluateRec(_lt(users)) if name.startswith("ktup") else m.evaluate(_lt(users))).cpu().numpy()
        walk = [O.rec_metrics(O.rec_topk(full[b], all_dicts[0][u] | all_dicts[1].get(u, set()), topn), eval_dict[u])
                for b, u in enumerate(users)]
        np.testing.assert_allclose(per_user, np.asarray(walk, dtype=np.float64), rtol=1e-12, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["transe", "transh"])
def test_rank_count_ex_kernel(name):
    """Empty exclusion == kgrec_eval_rank_count; with exclusions == unfiltered count minus the excluded rows that sort
    before the gold (from the full score matrix); counts over two catalog shards add up to the whole."""
    from kgrec_b200 import _lib, functional as KF
    lib = _lib.load()
    rng = np.random.RandomState(5)
    E, R, d, n = 900, 4, 100, 300
    m = _kg_model(name, False, d, E, R, rng)
    q, r, gold = _lt(rng.randint(0, E, n)), _lt(rng.randint(0, R, n)), _lt(rng.randint(0, E, n))
    gs = m.gold_scores("tail", q, r, gold)
    gold32 = gold.to(torch.int32)
    cat = m.ent_embeddings.weight.detach()
    T = KF.make_tables(m._weights(), d, False)
    st = KF._stream()

    def count(excl_row, ptr, ids, lo=0, hi=E):
        c = torch.zeros(n, dtype=torch.int32, device="cuda")
        if excl_row is None:
            _lib.check(lib.kgrec_eval_rank_count(C.byref(T), m.MODEL, _lib.SIDE_TAIL, KF._ptr(q), KF._ptr(r), 8, None, n,
                                                 KF._ptr(cat[lo:hi]), d, hi - lo, lo, KF._ptr(gs), KF._ptr(gold32), KF._ptr(c), st))
        else:
            _lib.check(lib.kgrec_eval_rank_count_ex(C.byref(T), m.MODEL, _lib.SIDE_TAIL, KF._ptr(q), KF._ptr(r), 8, None, n,
                                                    KF._ptr(cat[lo:hi]), d, hi - lo, lo, KF._ptr(gs), KF._ptr(gold32), KF._ptr(c),
                                                    KF._ptr(excl_row), KF._ptr(ptr), KF._ptr(ids), st))
        return c
    plain = count(None, None, None)
    rows = torch.arange(n, dtype=torch.int32, device="cuda")
    empty_ptr = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    assert torch.equal(count(rows, empty_ptr, torch.zeros(1, dtype=torch.int32, device="cuda")), plain)
    # exclusion rows shared by pairs (row i uses CSR row i % 50), each 0..80 ascending ids, some containing the gold
    sets = [np.unique(rng.choice(E, rng.randint(0, 81))) for _ in range(50)]
    ptr = torch.as_tensor(np.concatenate([[0], np.cumsum([len(s) for s in sets])]), device="cuda")
    ids = torch.as_tensor(np.concatenate(sets).astype(np.int32), device="cuda")
    excl_row = (rows % 50).to(torch.int32)
    got = count(excl_row, ptr, ids)
    full = m.evaluateTail(q, r)
    ent = torch.arange(E, device="cuda")
    before = (full < gs[:, None]) | ((full == gs[:, None]) & (ent[None, :] < gold[:, None]))
    mask = torch.zeros(50, E, dtype=torch.bool, device="cuda")
    for i, s in enumerate(sets):
        mask[i, torch.as_tensor(s, device="cuda")] = True
    excluded_before = (before & mask[excl_row.long()]).sum(1).to(torch.int32)
    assert torch.equal(plain, before.sum(1).to(torch.int32))
    assert torch.equal(got, plain - excluded_before)
    assert int(excluded_before.sum()) > 0
    # two catalog shards: global ids in the exclusion rows, id_base per shard
    half = 437
    assert torch.equal(count(excl_row, ptr, ids, 0, half) + count(excl_row, ptr, ids, half, E), got)


@pytest.mark.gpu
def test_rec_topk_metrics_kernel_on_hand_built_lists():
    from kgrec_b200 import _lib, evaluation as KE, functional as KF
    lib = _lib.load()
    k = 40
    inf = -1                                                           # UINT64_MAX in int64 storage
    lists = [
        list(range(100, 140)),                                         # full list, hits at 0, 1, 17, 39
        [5, 6, 7],                                                     # short list, no hit
        [],                                                            # all places empty
        [3, 9, 1, 4],                                                  # hits at 2, 3
        list(range(200, 240)),                                         # every place a hit
        [77],                                                          # one place, a hit, gold of 3
    ]
    golds = [{100, 101, 117, 139, 999}, {1, 2}, {4}, {1, 4, 8}, set(range(200, 240)), {77, 78, 79}]
    keys = np.full((len(lists), k), inf, dtype=np.int64)
    for i, ids in enumerate(lists):
        for j, x in enumerate(ids):
            keys[i, j] = (((j + 1) * 1000) << 32) | x                 # any ascending score bits
    gptr = np.concatenate([[0], np.cumsum([len(g) for g in golds])]).astype(np.int64)
    gids = np.concatenate([sorted(g) for g in golds]).astype(np.int32)
    keys_t = torch.as_tensor(keys, device="cuda")
    gptr_t, gids_t = torch.as_tensor(gptr, device="cuda"), torch.as_tensor(gids, device="cuda")
    out = torch.full((len(lists), 5), float("nan"), dtype=torch.float64, device="cuda")
    _lib.check(lib.kgrec_rec_topk_metrics(KF._ptr(keys_t), len(lists), k, KF._ptr(gptr_t), KF._ptr(gids_t), KF._ptr(out), KF._stream()))
    ids, _ = KE.keys_to_ids_scores(keys_t)
    want = np.asarray(KE.rec_metrics_from_topk(ids.cpu().tolist(), golds), dtype=np.float64)
    got = out.cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    assert got[1].tolist() == [0.0] * 5 and got[2].tolist() == [0.0] * 5
    assert got[4, 4] == 1.0 and got[5, 1] == 1.0


def _loop_env(kind):
    import kgrec_b200 as K
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import RatingNegativeSampler, TripleNegativeSampler
    from kgrec_b200.train import GraphedTrainLoop
    rng = np.random.RandomState(9)
    torch.manual_seed(9)
    if kind == "kg":
        E, R = 600, 7
        m = K.TransEModel(False, 64, E, R)
        data = np.stack([rng.randint(0, E, 2000), rng.randint(0, E, 2000), rng.randint(0, R, 2000)], 1)
        it, sampler = DeviceTrainIterator(data, 200, device="cuda", seed=1), TripleNegativeSampler(E, R, known_triples=data)
    else:
        U, I = 200, 300
        m = K.TransUPModel(False, 64, U, I, 5, False)
        data = np.stack([rng.randint(0, U, 2000), rng.randint(0, I, 2000)], 1)
        it, sampler = DeviceTrainIterator(data, 200, device="cuda", seed=1), RatingNegativeSampler(I, known_ratings=data)
    opt = SparseRowOptimizer(m, optimizer_type="Adagrad", lr=0.05, l2_lambda=0.0, clip=1.0)
    return m, GraphedTrainLoop(m, opt, it, sampler, 1, steps_per_graph=5, sample_seed=3)


def _evaluators(name, rng):
    from kgrec_b200 import metrics as KM
    if name in ("transe", "transh", "transr", "jtransup"):
        m = _kg_model(name, False, 100, 700, 5, rng)
        h, t, ha, ta = _kg_dicts(rng, 700, 5)
        return m, KM.KGEvaluator(m, h, t, ha, ta, topn=10), {}
    m, U, I = _rec_model(name, False, 100, rng)
    ev, ad = _rec_dicts(rng, U, I)
    return m, KM.RecEvaluator(m, ev, ad, topn=10), {"seed": 99}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["transe", "transh", "transr", "jtransup", "tup_soft", "tup_gumbel", "ktup_soft", "ktup_gumbel"])
def test_evaluator_run_has_no_host_sync_and_repeats_bit_for_bit(name):
    m, ev, kw = _evaluators(name, np.random.RandomState(3))
    ev.run(**kw)                                                       # warm-up: first-call allocations and attributes
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = ev.run(**kw)
        b = ev.run(**kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert a.dtype == torch.float64 and torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["kg", "rec"])
def test_evaluator_sees_tables_after_graphed_training(kind):
    from kgrec_b200 import metrics as KM
    m, loop = _loop_env(kind)
    rng = np.random.RandomState(4)
    if kind == "kg":
        h, t, ha, ta = _kg_dicts(rng, 600, 7, 30, 30)
        ev = KM.KGEvaluator(m, h, t, ha, ta, topn=10)
        want = lambda: KM.evaluate_kg(m, h, t, ha, ta, topn=10)      # noqa: E731
    else:
        e, ad = _rec_dicts(rng, 200, 300)
        ev = KM.RecEvaluator(m, e, ad, topn=10)
        want = lambda: KM.evaluate_rec(m, e, ad, topn=10)            # noqa: E731
    def same(got, ref):                                               # KG: evaluate_kg's tuple exactly; rec: to 1e-12
        return got == ref if kind == "kg" else got == pytest.approx(ref, rel=1e-12, abs=0)
    before = ev.result(ev.run())
    assert same(before, want())
    loop.run(20)
    after = ev.result(ev.run())
    assert after != before
    assert same(after, want())
