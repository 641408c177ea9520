"""The whole envelope the evaluation entry points accept (csrc/eval.cu, csrc/eval_transr.cu), against float64.

Every GPU case runs the three modes on one call shape and checks
  * scores (kgrec_eval_scores): |kernel - ref| <= 8 (d [+ P]) 2^-24 sum|terms| at every (query, row), where ref is the
    oracle's score on float64 copies of the tables and sum|terms| is the same sum taken over the magnitudes of every
    operand (so the bound follows each pair's own cancellation, and a dropped or doubled 4-float chunk fails at any d);
  * top-K (kgrec_eval_topk via topk / topk_items): ids and score bits equal a stable (score, id) sort of the kernel's
    own score matrix after filtering; empty places hold id -1 / +inf; and wherever the float64 gap at the K-th place
    exceeds the bound, the id set equals the float64 top-K;
  * rank counts (kgrec_eval_rank_count and _ex): exact against the (score, id) walk over the kernel's own scores, with
    the exclusion of KGEvaluator (filter + other golds).

Which case covers which part of the envelope:
  models, every d % 4 == 0 up to 256 (TransR 128), k in K_SWEEP ... test_kg_d_sweep, test_rec_d_sweep
  n_pref in {1, 4, 20, 64, 128} ....................................... test_rec_preference_counts
  nq / n_cat at the tile edges (RQ = 8, TQT = 64 / 128, TN) ........... test_tile_edges
  n_splits > 1 with a CTA range across a query tile, ties across pieces,
    shard merge, all-zero table, gold among tied rows ................ test_multi_piece_ties_and_shards
  strided catalog, padded / unpadded tile_pitch, id_base > 0, cat_ids,
    int32 / int64 ids, short filters, filters outside the shard ...... test_catalog_layouts_ids_and_filters
  KGEvaluator / RecEvaluator at topn 1 / 50 / 128, d 136 / 200 / 256 . test_evaluators_at_large_topn_and_wide_rows
  KGREC_EVAL_SHARE=0 / KGREC_EVAL_ROTATE=0 ............................. test_scheduling_switches_change_nothing
  the soft-preference limits that remain (host-side rejection) ........ test_plain_rec_path_limit_is_stated
On the CPU: the support queries' form, monotonicity and pinned limits, and the construction-time warning.
"""
import ctypes as C
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from oracle import kg_oracle as O

U24 = 2.0 ** -24
K_SWEEP = (1, 10, 28, 29, 31, 32, 33, 61, 62, 64, 74, 75, 127, 128)
NAMED_D = (4, 32, 64, 100, 128, 132, 136, 148, 200, 252, 256)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_support_queries_form_monotonicity_and_pinned_limits():
    from kgrec_b200 import _lib
    lib = _lib.load()
    assert {"kgrec_pref_aug_supported", "kgrec_pref_eval_supported", "kgrec_gumbel_aug_supported"} <= set(_lib.EXPORTS)
    aug, plain, gum = lib.kgrec_pref_aug_supported, lib.kgrec_pref_eval_supported, lib.kgrec_gumbel_aug_supported
    # the form of kgrec_gumbel_aug_supported: 0 / 1, k = 0 is the score matrix, 0 outside the accepted arguments
    for bad in ((0, 10), (6, 10), (260, 10), (64, -1), (64, 129)):
        assert aug(*bad) == 0 and plain(bad[0], 4, 0, bad[1]) == 0 and gum(bad[0], 4, bad[1]) == 0
    assert plain(64, 0, 0, 10) == 0 and plain(64, 129, 0, 10) == 0
    for d in range(4, 257, 4):
        for k in range(0, 129):
            v = aug(d, k)
            assert v in (0, 1)
            if v and k:
                assert aug(d, k - 1)
            if v and d > 4:
                assert aug(d - 4, k)
    for g in (0, 1):
        for d in (4, 64, 128, 148, 200, 256):
            for P in (1, 4, 20, 64, 128):
                for k in (0, 1, 10, 64, 128):
                    if plain(d, P, g, k):      # (not in d: the plain path's catalog tile holds ~16 KB whatever d is)
                        assert plain(d, P, g, max(0, k - 1)) and (P == 1 or plain(d, P - 1, g, k))
    # the augmented soft path: every mode fails for 148 <= d <= 256, top-K from 62 at d = 128
    assert [d for d in range(4, 257, 4) if not aug(d, 0)] == list(range(148, 257, 4))
    assert min(k for k in range(1, 129) if not aug(128, k)) == 62
    # the plain path's limit in preference_total x embedding_size: largest n_pref at k = 0 / 10 / 128
    pinned = {(0, 148): (90, 87, 48), (0, 200): (66, 64, 32), (0, 256): (53, 51, 25),
              (1, 148): (108, 105, 66), (1, 200): (83, 80, 48), (1, 256): (67, 64, 39)}
    for (g, d), want in pinned.items():
        got = tuple(max([P for P in range(1, 129) if plain(d, P, g, k)] or [0]) for k in (0, 10, 128))
        assert got == want, (g, d)
    # below those corners every rec-side call has a path: (d, k) for the models the sweeps build (n_pref = 4)
    for d in range(4, 257, 4):
        for k in (0,) + K_SWEEP:
            assert aug(d, k) or plain(d, 4, 0, k)
            assert gum(d, 4, k) or plain(d, 4, 1, k)


def test_construction_warns_about_the_rec_evaluation_limit():
    import kgrec_b200 as K

    def built(*a):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            m = K.TransUPModel(*a)
        return m, [str(x.message) for x in w if "kgrec_b200" in str(x.message)]
    m, w = built(False, 256, 5, 6, 4, False)
    assert w == [] and m.rec_eval_max_topn() == 128
    m, w = built(False, 256, 5, 6, 26, False)
    assert m.rec_eval_max_topn() == 126 and len(w) == 1 and "topn <= 126" in w[0]
    m, w = built(False, 256, 5, 6, 60, False)
    assert m.rec_eval_max_topn() == -1 and len(w) == 1 and "evaluateRec" in w[0] and "raise" in w[0]
    m, w = built(True, 200, 5, 6, 60, True)                  # ST-Gumbel L1: the plain path only
    assert m.rec_eval_max_topn() == 87 and "topn <= 87" in w[0]
    _, w = built(False, 130, 5, 6, 4, False)
    assert len(w) == 1 and "multiple of 4" in w[0]           # the existing warning, unchanged


# ---- GPU helpers ------------------------------------------------------------------------------------------------------
def _lt(x, dtype=torch.int64):
    return torch.as_tensor(np.asarray(x), dtype=dtype, device="cuda")


def _f64(m):
    return {k: v.detach().double().cpu().numpy() for k, v in m._weights().items()}


def _kg_model(name, l1, d, E, R=3, seed=0):
    import kgrec_b200 as K
    torch.manual_seed(seed)
    if name == "jtransup":
        I = 20
        new_map = {i: (i * 7 % (E - 1), i) for i in range(I)}
        return K.jTransUPModel(l1, d, 10, I, E - 1, R, {i: i for i in range(I)}, new_map, False, False)  # E rows with padding
    return {"transe": K.TransEModel, "transh": K.TransHModel, "transr": K.TransRModel}[name](l1, d, E, R)


def _kg_ref(name, W, q, r, side, cat, l1):
    """float64 scores [nq, N] and the bound 8 d 2^-24 sum|terms| of every pair."""
    ent, rel = W["ent"], W["rel"]
    if name == "transe":
        S = O.transe_eval(ent, rel, q, r, l1, side, catalog=cat)
    elif name == "transr":
        S = O.transr_eval(ent, rel, W["proj"], q, r, l1, side, catalog=cat)
    else:
        S = O.transh_eval(ent, rel, W["norm"], q, r, l1, side, catalog=cat)
    d = ent.shape[1]
    B = np.empty_like(S)
    ac = np.abs(cat)
    for b in range(len(q)):
        e, rr = np.abs(ent[q[b]]), np.abs(rel[r[b]])
        if name == "transe":
            m = e + rr + ac
        elif name == "transr":
            M = np.abs(W["proj"][r[b]]).reshape(d, d)
            m = M @ e + rr + ac @ M.T
        else:
            w = np.abs(W["norm"][r[b]])
            m = e + (e @ w) * w + rr + ac + (ac @ w)[:, None] * w
        B[b] = 8 * d * U24 * (m if l1 else m * m).sum(-1) + 1e-30
    return S, B


def _gumbel(u):
    return -np.log(-np.log(u + O.EPS_GUMBEL) + O.EPS_GUMBEL)


def _rec_ref(m, W, u, gu):
    """float64 scores, bounds 8 (d + P) 2^-24 sum|terms|, and a mask of the ST-Gumbel pairs whose arg-max is a near tie."""
    ktup = m.MODEL == 4
    l1 = m.L1_flag
    item = W["item"] + (W["ent"][m.item2ent.cpu().numpy().astype(np.int64)] if ktup else 0)
    Pm = W["pref"] + (W["rel"] if ktup else 0)
    Nm = W["pref_norm"] + (W["norm"] if ktup else 0)
    hf = 0.5 if ktup else 1.0
    if ktup:
        S = O.ktup_rec_eval(W["user"], W["item"], W["ent"], W["rel"], W["norm"], W["pref"], W["pref_norm"],
                            m.item2ent.cpu().numpy().astype(np.int64), u, l1, gu)
    else:
        S = O.tup_eval(W["user"], W["item"], W["pref"], W["pref_norm"], u, l1, gu)
    d, P = item.shape[1], Pm.shape[0]
    B = np.empty_like(S)
    near = np.zeros(S.shape, dtype=bool)
    aP, aN, ai = np.abs(Pm), np.abs(Nm), np.abs(item)
    for b in range(len(u)):
        a = np.abs(W["user"][u[b]]) + ai
        za = a @ aP.T / 2
        if gu is None:
            ra, wa = hf * za @ aP, hf * za @ aN
        else:
            z = (W["user"][u[b]] + item) @ Pm.T / 2 + _gumbel(gu[b])
            ks = z.argmax(-1)
            top2 = np.sort(z, axis=-1)[:, -2:] if P > 1 else np.zeros((len(z), 2))
            near[b] = (top2[:, 1] - top2[:, 0] < 1e-3) if P > 1 else False
            ra, wa = hf * aP[ks], hf * aN[ks]
        sa = (a * wa).sum(-1)
        mm = a + ra + sa[:, None] * wa
        B[b] = 8 * (d + P) * U24 * (mm if l1 else mm * mm).sum(-1) + 1e-30
    return S, B, near


def _csr(rows):
    ptr = np.concatenate([[0], np.cumsum([len(x) for x in rows])]).astype(np.int64)
    ids = np.concatenate([np.sort(np.asarray(list(x), dtype=np.int64)) for x in rows] + [np.zeros(0, np.int64)])
    return _lt(ptr), _lt(ids if ids.size else [0], torch.int32)


def _check_scores(S, ref, B, tag, skip=None):
    err = np.abs(S.astype(np.float64) - ref)
    bad = err > B
    if skip is not None:
        bad &= ~skip
    assert not bad.any(), "%s: %d pairs over the bound, first %s: kernel %r ref %r bound %r" % (
        tag, bad.sum(), np.argwhere(bad)[0], S[bad][0], ref[bad][0], B[bad][0])


def _check_topk(keys, S, ids, k, filt, ref, B, tag, skip=None):
    """keys [nq, k] against the stable (score, id) sort of the kernel's own scores S [nq, N] (global ids `ids`)."""
    from kgrec_b200 import evaluation as KE
    gi, gs = KE.keys_to_ids_scores(keys)
    gi, gs = gi.cpu().numpy(), gs.cpu().numpy()
    for b in range(S.shape[0]):
        keep = ~np.isin(ids, list(filt[b])) if filt is not None else np.ones(len(ids), bool)
        s, i = S[b, keep], ids[keep]
        o = np.lexsort((i, s))[:k]
        n = len(o)
        assert gi[b, :n].tolist() == i[o].tolist(), "%s q%d ids" % (tag, b)
        assert np.array_equal(gs[b, :n].view(np.uint32), s[o].view(np.uint32)), "%s q%d scores" % (tag, b)
        assert (gi[b, n:] == -1).all() and np.isinf(gs[b, n:]).all(), "%s q%d empty places" % (tag, b)
        if n == k and len(s) > k and (skip is None or not skip[b].any()):
            r64 = ref[b, keep]
            o64 = np.argsort(r64, kind="stable")
            if r64[o64[k]] - r64[o64[k - 1]] > 2 * B[b, keep].max():
                assert set(i[o64[:k]].tolist()) == set(gi[b, :k].tolist()), "%s q%d float64 set" % (tag, b)


def _want_counts(S, ids, gold, excl=None):
    out = []
    for b, g in enumerate(gold):
        j = int(np.flatnonzero(ids == g)[0])
        before = (S[b] < S[b, j]) | ((S[b] == S[b, j]) & (ids < g))
        if excl is not None:
            before &= ~np.isin(ids, list(excl[b]))
        out.append(int(before.sum()))
    return out


class KGCall:
    """One KG model's evaluation calls on a catalog (ids id_base + row, or cat_ids)."""

    def __init__(self, m, name, side, q, r):
        from kgrec_b200 import _lib
        self.m, self.name, self.side, self.q, self.r = m, name, side, q, r
        self.sd = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
        self.kg = _lib.TRANSH if name == "jtransup" else m.MODEL

    def scores(self, cat, id_base=0, cat_ids=None):
        if self.name == "transr":
            return self.m._scores(self.sd, self.q, self.r, catalog=cat, id_base=id_base, cat_ids=cat_ids)
        return self.m._eval(self.kg, self.sd, self.q, self.r, "scores", catalog=cat, id_base=id_base, cat_ids=cat_ids)

    def topk(self, cat, k, filt=None, id_base=0):
        csr = _csr(filt) if filt is not None else None
        if self.name == "transr":
            return self.m.topk(self.side, self.q, self.r, k=k, filter_csr=csr, catalog=cat, id_base=id_base)
        return self.m._eval(self.kg, self.sd, self.q, self.r, "topk", catalog=cat, id_base=id_base, k=k, filter_csr=csr)

    def counts(self, cat, gold, gs, id_base=0):
        g = _lt(gold)
        if self.name == "transr":
            return self.m.rank_counts(self.side, self.q, self.r, g, gold_scores=gs, catalog=cat, id_base=id_base)
        return self.m._eval(self.kg, self.sd, self.q, self.r, "rank", catalog=cat, id_base=id_base, gold_scores=gs, gold_ids=g)

    def counts_ex(self, cat, gold, gs, excl, id_base=0):
        from kgrec_b200 import _lib, functional as KF
        lib = _lib.load()
        T = KF.make_tables(self.m._weights(), self.m.embedding_size, self.m.L1_flag)
        nq = len(gold)
        c = torch.zeros(nq, dtype=torch.int32, device="cuda")
        g32, row = _lt(gold, torch.int32), torch.arange(nq, dtype=torch.int32, device="cuda")
        ptr, ids = _csr(excl)
        _lib.check(lib.kgrec_eval_rank_count_ex(C.byref(T), self.kg, self.sd, KF._ptr(self.q), KF._ptr(self.r),
                                                self.q.element_size(), None, nq, KF._ptr(cat), cat.stride(0), cat.shape[0],
                                                id_base, KF._ptr(gs), KF._ptr(g32), KF._ptr(c), KF._ptr(row), KF._ptr(ptr),
                                                KF._ptr(ids), KF._stream()))
        return c


def _kg_case(m, name, side, q, r, ks, cat=None, id_base=0, filt=None, gold=None, excl=None, tag=""):
    """The three modes of one KG call shape against float64; returns the kernel's score matrix."""
    call = KGCall(m, name, side, q if isinstance(q, torch.Tensor) else _lt(q), r if isinstance(r, torch.Tensor) else _lt(r))
    cat = m.ent_embeddings.weight.detach() if cat is None else cat
    N = cat.shape[0]
    ids = id_base + np.arange(N)
    S = call.scores(cat, id_base).cpu().numpy()
    W = _f64(m)
    qn, rn = call.q.cpu().numpy().astype(np.int64), call.r.cpu().numpy().astype(np.int64)
    ref, B = _kg_ref("transh" if name == "jtransup" else name, W, qn, rn, side, cat.double().cpu().numpy(), m.L1_flag)
    _check_scores(S, ref, B, tag)
    for k in ks:
        _check_topk(call.topk(cat, k, filt, id_base), S, ids, k, filt, ref, B, "%s k%d" % (tag, k))
    if gold is not None:
        gs = torch.as_tensor(S[np.arange(len(gold)), np.asarray(gold) - id_base], device="cuda")
        assert call.counts(cat, gold, gs, id_base).cpu().tolist() == _want_counts(S, ids, gold), tag + " rank"
        if excl is not None and name != "transr":
            assert call.counts_ex(cat, gold, gs, excl, id_base).cpu().tolist() == _want_counts(S, ids, gold, excl), tag + " rank_ex"
    return S


def _rec_model(name, d, U, I, P, seed=0):
    import kgrec_b200 as K
    torch.manual_seed(seed)
    l1 = "l1" in name
    gumbel = "gumbel" in name
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if name.startswith("ktup"):
            E = 30
            new_map = {i: ((i * 5) % E if i % 4 else -1, i) for i in range(I)}
            return K.jTransUPModel(l1, d, U, I, E, P, {i: i for i in range(I)}, new_map, False, gumbel)
        return K.TransUPModel(l1, d, U, I, P, gumbel)


def _rec_path(m, k):
    """The path RecModelBase._rec_call takes for top-k k (0: the score matrix)."""
    return "gumbel_aug" if m._gumbel_aug_ok(k) else "soft_aug" if m._pref_aug_ok(k) else "plain"


def _rec_case(m, u, ks, filt=None, rng=None, tag=""):
    """Every path's score matrix against float64, then top-K of each k against the score matrix of the path the call
    takes (bit-exact), or, past the stated limit (rec_eval_max_topn), the host-side rejection."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    W = _f64(m)
    I, P, d = m.item_embeddings.weight.shape[0], m.pref_embeddings.weight.shape[0], m.embedding_size
    gu = rng.uniform(0.0, 1.0, (len(u), I, P)) if m.use_st_gumbel else None
    gut = torch.as_tensor(gu, dtype=torch.float32, device="cuda") if gu is not None else None
    ut = _lt(u)
    ref, B, near = _rec_ref(m, W, np.asarray(u), gu.astype(np.float32).astype(np.float64) if gu is not None else None)
    S = {}
    path0 = _rec_path(m, 0)
    if path0 != "plain":
        S[path0] = (m.evaluateRec(ut, gumbel_u=gut) if m.MODEL == 4 else m.evaluate(ut, gumbel_u=gut)).cpu().numpy()
    if lib.kgrec_pref_eval_supported(d, P, int(m.use_st_gumbel), 0):
        S["plain"] = m._eval(m.MODEL, _lib.SIDE_REC, ut, None, "scores", catalog=m._rec_catalog(), gumbel_u=gut).cpu().numpy()
    for path, Sp in S.items():
        _check_scores(Sp, ref, B, "%s %s" % (tag, path), near)
    kmax = m.rec_eval_max_topn()
    for k in ks:
        csr = _csr(filt) if filt is not None else None
        if k > kmax:
            with pytest.raises(RuntimeError, match="kgrec_pref_eval_supported"):
                m.topk_items(ut, k=k, filter_csr=csr, gumbel_u=gut)
            continue
        keys = m.topk_items(ut, k=k, filter_csr=csr, gumbel_u=gut)
        _check_topk(keys, S[_rec_path(m, k)], np.arange(I), k, filt, ref, B, "%s k%d" % (tag, k), near)
    return S


# ---- GPU: sweeps ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,l1", [("transe", False), ("transe", True), ("transh", True), ("transr", True), ("jtransup", False)])
def test_kg_d_sweep(name, l1):
    """Every d % 4 == 0 up to 256 (TransR 128) at every k of K_SWEEP: the 16 -> 8 -> 4 warp fallbacks of eval_plan."""
    rng = np.random.RandomState(1)
    E = 140
    for d in range(4, (128 if name == "transr" else 256) + 1, 4):
        m = _kg_model(name, l1, d, E, seed=d)
        q, r = rng.randint(0, E - 1, 9), rng.randint(0, 3, 9)
        side = "head" if d % 8 else "tail"
        gold = rng.randint(0, E - 1, 9)
        _kg_case(m, name, side, q, r, K_SWEEP, gold=gold, excl=[{int(x)} for x in rng.randint(0, E, 9)],
                 tag="%s l1=%d d=%d" % (name, l1, d))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_soft_l1", "tup_soft_l2", "tup_gumbel_l2", "tup_gumbel_l1", "ktup_soft_l2", "ktup_gumbel_l2"])
def test_rec_d_sweep(name):
    """Soft preferences at every d (augmented rows up to d = 144 / k = 61 at d = 128, the plain path beyond); the
    ST-Gumbel and KTUP paths at a stride of 12 plus the named widths."""
    rng = np.random.RandomState(2)
    U, I = 12, 140
    ds = range(4, 257, 4) if name.startswith("tup_soft") else sorted(set(range(4, 257, 12)) | set(NAMED_D))
    for d in ds:
        m = _rec_model(name, d, U, I, 4, seed=d)
        _rec_case(m, rng.choice(U, 9, replace=False), K_SWEEP, rng=rng, tag="%s d=%d" % (name, d))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_soft_l2", "tup_gumbel_l2", "tup_gumbel_l1", "ktup_soft_l1", "ktup_gumbel_l2"])
@pytest.mark.parametrize("P", [1, 4, 20, 64, 128])
def test_rec_preference_counts(name, P):
    rng = np.random.RandomState(P)
    m = _rec_model(name, 64, 20, 150, P, seed=P)
    filt = [set(rng.choice(150, rng.randint(0, 30), replace=False).tolist()) for _ in range(11)]
    _rec_case(m, rng.choice(20, 11, replace=False), (1, 10, 128), filt=filt, rng=rng, tag="%s P=%d" % (name, P))


# ---- GPU: tiles, pieces, ties -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,d,tn", [("transe", 100, 128), ("transh", 200, 32), ("tup_soft_l2", 64, 32)])
def test_tile_edges(name, d, tn):
    """nq around RQ = 8 and the query tiles (64 / 128), n_cat around k and the catalog tile TN of the plan."""
    rng = np.random.RandomState(d)
    k = 10
    for n_cat in (1, k - 1, k, k + 1, tn - 1, tn, tn + 1):
        for nq in (1, 7, 8, 9, 63, 64, 65, 127, 128, 129):
            tag = "%s n_cat=%d nq=%d" % (name, n_cat, nq)
            if name.startswith("tup"):
                m = _rec_model(name, d, 130, max(n_cat, 1), 4, seed=n_cat)
                _rec_case(m, rng.randint(0, 130, nq), (k,), rng=rng, tag=tag)
            else:
                m = _kg_model(name, False, d, max(n_cat, 2), seed=n_cat)
                cat = m.ent_embeddings.weight.detach()[:n_cat]
                q, r = rng.randint(0, max(n_cat, 2), nq), rng.randint(0, 3, nq)
                gold = rng.randint(0, n_cat, nq)
                _kg_case(m, name, "tail", q, r, (k,), cat=cat, gold=gold, tag=tag)


def _pieces(nq, n_cat, tn, tqt, sm):
    """eval_plan's tiling of a tiled top-K call: (n_splits, units_per_cta, does some CTA range cross a query tile)."""
    n_tiles, n_qt = -(-n_cat // tn), -(-nq // tqt)
    total = n_tiles * n_qt
    ctas = min(sm, total)
    upc = -(-total // ctas)
    grid = -(-total // upc)
    crosses = any((b * upc) // n_tiles != (min(total, (b + 1) * upc) - 1) // n_tiles for b in range(grid))
    return -(-n_tiles // upc) + 1, upc, crosses


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["transe", "transh"])
def test_multi_piece_ties_and_shards(name):
    """Many pieces per query (n_splits > 1, CTA ranges across query tiles); rows i and i + n_cat / 2 identical, so tied
    keys sit in different pieces and shards; a gold among tied rows; an all-zero table (every key tied)."""
    from kgrec_b200 import evaluation as KE
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    d, n_cat = 32, 600
    tn, tqt = (128, 128) if name == "transe" else (64, 128)          # 16-warp plans at d = 32 (k <= 28)
    nq = 0
    for nqt in range(1, 200):
        n_splits, upc, crosses = _pieces(nqt * tqt, n_cat, tn, tqt, sm)
        if n_splits > 1 and crosses and nqt * -(-n_cat // tn) > sm:
            nq = nqt * tqt - 3
            break
    n_splits, upc, crosses = _pieces(nq, n_cat, tn, tqt, sm)
    assert nq > 0 and n_splits > 1 and crosses
    rng = np.random.RandomState(7)
    m = _kg_model(name, False, d, n_cat)
    w = m.ent_embeddings.weight
    with torch.no_grad():
        w[n_cat // 2:] = w[:n_cat // 2]
    q, r = rng.randint(0, n_cat, nq), rng.randint(0, 3, nq)
    S = _kg_case(m, name, "tail", q, r, (1, 5, 11, 28), tag=name + " pieces")
    # a gold id among tied rows: the query's own best row and its twin
    best = S.argmin(1)
    gold = np.where(np.arange(nq) % 2, best, (best + n_cat // 2) % n_cat)
    call = KGCall(m, name, "tail", _lt(q), _lt(r))
    cat = w.detach()
    gs = torch.as_tensor(S[np.arange(nq), gold], device="cuda")
    assert call.counts(cat, gold, gs).cpu().tolist() == _want_counts(S, np.arange(n_cat), gold)
    excl = [{int(g + n_cat // 2) % n_cat} for g in gold]
    assert call.counts_ex(cat, gold, gs, excl).cpu().tolist() == _want_counts(S, np.arange(n_cat), gold, excl)
    # shards over shard_bounds, merged by k_merge_topk: equal to the one-call top-K, ties in ascending id order
    for world in (2, 3):
        for k in (5, 28):
            parts = []
            for g in range(world):
                lo, hi = KE.shard_bounds(n_cat, world, g)
                parts.append(call.topk(cat[lo:hi], k, id_base=lo))
            assert torch.equal(KE.merge_topk(torch.stack(parts)), call.topk(cat, k)), (world, k)
    # all-zero tables: every score 0, the top-K is ids 0 .. k-1 in every piece arrangement
    with torch.no_grad():
        w.zero_()
        m.rel_embeddings.weight.zero_()
    for k in (1, 11, 28):
        ids, sc = KE.keys_to_ids_scores(call.topk(cat, k))
        assert (ids.cpu().numpy() == np.arange(k)[None, :]).all() and (sc == 0).all(), k
    gs0 = torch.zeros(nq, dtype=torch.float32, device="cuda")
    assert call.counts(cat, gold, gs0).cpu().tolist() == gold.tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("name,d", [("transe", 100), ("transe", 128), ("transh", 64), ("transh", 252), ("transr", 100), ("transr", 128)])
def test_catalog_layouts_ids_and_filters(name, d):
    """Strided catalog (cat_ld > d: one bulk copy per row), tile_pitch unpadded (d / 4 odd) and padded (even), a shard
    with id_base > 0, cat_ids sub-catalogs, int32 and int64 ids, filters of length 0 / 1 / many (fewer than k
    survivors) and filters holding ids outside the shard."""
    rng = np.random.RandomState(d)
    E = 500
    m = _kg_model(name, d % 8 == 4, d, E)
    ent = m.ent_embeddings.weight.detach()
    nq = 70
    q, r = rng.randint(0, E, nq), rng.randint(0, 3, nq)
    lo, hi = 123, 431
    wide = torch.zeros((E, d + 12), dtype=torch.float32, device="cuda")
    wide[:, :d] = ent
    full = KGCall(m, name, "head", _lt(q), _lt(r)).scores(ent).cpu().numpy()
    for qdt in (torch.int64, torch.int32):
        for cat, base in ((ent, 0), (wide[:, :d], 0), (wide[lo:hi, :d], lo), (ent[lo:hi], lo)):
            n = cat.shape[0]
            S_full = full[:, base:base + n]
            filt = []
            for b in range(nq):
                kind = b % 5
                if kind == 0:
                    filt.append(set())
                elif kind == 1:
                    filt.append({int(base + S_full[b].argmin())})                 # length 1: the query's best row
                elif kind == 2:
                    filt.append(set((base + np.arange(n - 7)).tolist()))          # 7 survivors < k
                elif kind == 3:
                    filt.append(set(rng.randint(0, E, 40).tolist()) | {E + 5})    # ids outside the shard
                else:
                    filt.append(set((base + np.argsort(S_full[b])[:12]).tolist()) | {0, E - 1})
            gold = base + rng.randint(0, n, nq)
            excl = [set(rng.randint(base, base + n, 30).tolist()) - {int(g)} for g in gold]
            S = _kg_case(m, name, "head", _lt(q, qdt), _lt(r, qdt), (10, 64), cat=cat, id_base=base, filt=filt, gold=gold,
                         excl=excl, tag="%s d=%d %s base=%d ld=%d" % (name, d, qdt, base, cat.stride(0)))
            assert np.array_equal(S.view(np.uint32), S_full.view(np.uint32))     # the same bits wherever the row sits
    # cat_ids: gathered sub-catalog, scores bit-identical to the full catalog's columns
    sel = rng.choice(E, 77, replace=False)
    sub = KGCall(m, name, "head", _lt(q), _lt(r)).scores(ent[_lt(sel)].contiguous(), cat_ids=_lt(sel, torch.int32))
    assert np.array_equal(sub.cpu().numpy().view(np.uint32), full[:, sel].view(np.uint32))


# ---- GPU: evaluators, limits, switches ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,d", [("transe", 136), ("transh", 200), ("jtransup", 256), ("transr", 128),
                                    ("tup_soft_l2", 136), ("tup_soft_l1", 200), ("tup_gumbel_l2", 256), ("ktup_soft_l2", 256),
                                    ("ktup_gumbel_l2", 200)])
def test_evaluators_at_large_topn_and_wide_rows(name, d):
    from kgrec_b200 import metrics as KM
    rng = np.random.RandomState(d)
    if name.startswith(("tup", "ktup")):
        U, I = 90, 300
        m = _rec_model(name, d, U, I, 4)
        ev = {int(u): set(rng.choice(I, rng.randint(0, 8), replace=False).tolist()) for u in rng.choice(U, 60, replace=False)}
        train = {u: set(rng.choice(I, 40, replace=False).tolist()) for u in ev}
        u0 = [u for u in ev if ev[u]][0]
        train[u0] = set(range(I)) - set(list(ev[u0])[:1]) - {3, 4}
        seed = 0x51ED
        for topn in (1, 50, 128):
            rv = KM.RecEvaluator(m, ev, [train], topn=topn)
            got = rv.result(rv.run(seed=seed))
            m._next_seed = lambda: seed
            want = KM.evaluate_rec(m, ev, [train], topn=topn)
            assert got[3] == want[3]
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
        return
    E = 400
    m = _kg_model(name, d % 8 == 0, d, E)

    def dct(n):
        out = {}
        while len(out) < n:
            out[(int(rng.randint(0, E - 1)), int(rng.randint(0, 3)))] = set(rng.choice(E - 1, rng.randint(1, 9), replace=False).tolist())
        return out
    he, te = dct(30), dct(35)
    ha = [{k: set(rng.choice(E - 1, 50, replace=False).tolist()) for k in list(he)[::2]}]
    ta = [{k: {next(iter(te[k]))} for k in list(te)[::3]}]
    for topn in (1, 50, 128):
        ev = KM.KGEvaluator(m, he, te, ha, ta, topn=topn)
        assert ev.result(ev.run()) == KM.evaluate_kg(m, he, te, ha, ta, topn=topn), topn


@pytest.mark.gpu
def test_plain_rec_path_limit_is_stated():
    """TUP soft at d = 256: the augmented rows do not fit, the plain path serves n_pref <= 25 at topn 128 and rejects
    n_pref = 26 at topn 127 on the host with a message naming the limit."""
    rng = np.random.RandomState(3)
    m = _rec_model("tup_soft_l2", 256, 20, 140, 25)
    _rec_case(m, rng.choice(20, 9, replace=False), (128,), rng=rng, tag="P=25")
    m = _rec_model("tup_soft_l2", 256, 20, 140, 26)
    assert m.rec_eval_max_topn() == 126
    with pytest.raises(RuntimeError, match="kgrec_pref_eval_supported"):
        m.topk_items(_lt([1, 2]), k=127)
    _rec_case(m, rng.choice(20, 9, replace=False), (126,), rng=rng, tag="P=26 k=126")


_SWITCH_SCRIPT = r"""
import sys, numpy as np, torch
sys.path[:0] = [%(root)r, %(root)r + "/joint-kg-recommender_b200"]
import kgrec_b200 as K
torch.manual_seed(0)
out = {}
for name, d in (("transe", 32), ("transh", 200), ("tup", 64)):
    rng = np.random.RandomState(d)
    if name == "tup":
        m = K.TransUPModel(False, d, 3000, 700, 4, False)
        with torch.no_grad():
            m.item_embeddings.weight[350:] = m.item_embeddings.weight[:350]
        keys = m.topk_items(torch.as_tensor(rng.randint(0, 3000, 2000), device="cuda"), k=11)
        out[name] = [keys.cpu().numpy().tolist()]
        continue
    m = (K.TransEModel if name == "transe" else K.TransHModel)(False, d, 700, 3)
    with torch.no_grad():
        m.ent_embeddings.weight[350:] = m.ent_embeddings.weight[:350]
    q = torch.as_tensor(rng.randint(0, 700, 5000), device="cuda")
    r = torch.as_tensor(rng.randint(0, 3, 5000), device="cuda")
    g = torch.as_tensor(rng.randint(0, 700, 5000), device="cuda")
    out[name] = [m.topk("tail", q, r, k=11).cpu().numpy().tolist(), m.rank_counts("tail", q, r, g).cpu().numpy().tolist()]
import json
json.dump(out, open(sys.argv[1], "w"))
"""


@pytest.mark.gpu
def test_scheduling_switches_change_nothing(tmp_path):
    """KGREC_EVAL_SHARE=0 (no shared bound between pieces) and KGREC_EVAL_ROTATE=0 (warp 0 issues every tile) are
    read once per process: each runs in its own subprocess; keys and counts equal the default run's bit for bit."""
    script = tmp_path / "switch.py"
    script.write_text(_SWITCH_SCRIPT % {"root": ROOT})
    res = {}
    for tag, extra in (("default", {}), ("share0", {"KGREC_EVAL_SHARE": "0"}), ("rotate0", {"KGREC_EVAL_ROTATE": "0"})):
        env = dict(os.environ)
        env.pop("KGREC_EVAL_SHARE", None)
        env.pop("KGREC_EVAL_ROTATE", None)
        env.update(extra)
        out = tmp_path / (tag + ".json")
        subprocess.run([sys.executable, "-s", str(script), str(out)], env=env, check=True, timeout=600)
        res[tag] = json.loads(out.read_text())
    assert res["share0"] == res["default"]
    assert res["rotate0"] == res["default"]
