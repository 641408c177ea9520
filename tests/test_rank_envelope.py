"""The whole envelope of the rank-count entry points and the top-n helpers (csrc/eval.cu, csrc/eval_transr.cu), against
float64 and against the definitions restated here.

  * rec rank counts (kgrec_rec_gold_scores + kgrec_rec_rank_count through RecModelBase.gold_scores_items /
    rank_counts_items, and once through ctypes): exact against the definition applied to the score matrix of the path
    the call takes (the kernel's own scores, themselves within 8 (d + P) 2^-24 sum|terms| of float64), and between the
    float64 counts of the items surely below / possibly below the gold wherever the bounds allow (equal to the float64
    count when no bound straddles the gold);
  * dual link counts (kgrec_eval_rank_count_dual, kgrec_transr_eval_rank_count_dual): raw and filtered counts exact
    against the definition on the kgrec_eval_scores matrix (filtered: not in X_i; raw: not in X_i and G_i), and
    bracketed by float64 as above;
  * kgrec_rec_topk_metrics against a float64 restatement of getRecPerformance (utils/misc.py:213-248);
  * kgrec_merge_topk against evaluation.merge_topk_host;
  * ST-Gumbel L2 evaluation of pairs whose true score is 0: every path keeps them first.
Every score matrix, gold score and key the file reads back has its sign bit clear (make_key orders non-negative
floats only).

Which case covers which part of the envelope:
  every kernel of the rec rank mode, by name; golds 0 / 1 / 31 / 32 / 33 / 64 / 65 / all but three,
    filtered golds, ties, 3 and 5 shards, all-zero tables ....................... test_rec_rank_kernels
  d % 4 == 0 to 256 (TUP soft), stride 12 + named d (ST-Gumbel, KTUP) ............ test_rec_rank_d_sweep
  n_pref 1 / 4 / 20 / 32 / 64 / 65 / 128 ....................................... test_rec_rank_preference_counts
  nq 1 .. 129, int32 / int64 ids, a user twice, both noise sources, catalog tile edges, ctypes
                                                                                  test_rec_rank_queries_and_catalog_edges
  dual counts, every d % 4 == 0 to 256 (TransR 128): the 16- and 8-warp plans .... test_dual_d_sweep
  dual counts with CTA ranges across query tiles, twin rows, all-zero table ...... test_dual_pieces_ties_and_zero_table
  dual counts: int32 ids, qvec, strided catalog, 3 shards, a gold missing from X_i  test_dual_layouts_and_precondition
  kgrec_rec_topk_metrics at k 1 .. 128 and a second grid-stride pass ............. test_rec_topk_metrics_envelope
  kgrec_merge_topk: 1 / 2 / 3 x SM lists, k 1 .. 128 ............................. test_merge_topk_envelope
  ST-Gumbel L2 scores of true value 0 (TUP / KTUP, P = 1 / 4) .................... test_st_gumbel_l2_zero_scores_rank_first
On the CPU: the restated definitions on hand-computed examples and the zero-score construction in float64.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from test_eval_envelope import NAMED_D, _check_scores, _f64, _kg_model, _kg_ref, _rec_model, _rec_path, _rec_ref
from test_rec_rank_counts import oracle_counts

INF = np.uint64(0xFFFF_FFFF_FFFF_FFFF)
GOLD_SIZES = (0, 1, 31, 32, 33, 64, 65, -3)          # -3: the whole catalog but three


# ---- definitions, restated ------------------------------------------------------------------------------------------
def _nonneg(x, tag):
    """No score of a matrix / gold-score array has its sign bit set (-0.0 and negatives would key after +inf)."""
    bits = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    bad = (bits >> 31) != 0
    assert not bad.any(), "%s: %d scores with the sign bit set, first %r" % (tag, bad.sum(), x[bad].ravel()[0])


def _nonneg_keys(keys, tag):
    k = np.ascontiguousarray(keys).view(np.uint64)
    bad = (k != INF) & ((k >> np.uint64(63)) != 0)
    assert not bad.any(), "%s: %d keys with the score's sign bit set" % (tag, bad.sum())


def dual_counts(S, ids, gold, rows, X, G):
    """(raw, filtered) per query i: catalog columns with (S bits, id) < (gold's), filtered: id not in X[rows[i]], raw:
    id not in both X[rows[i]] and G[rows[i]] (the header's precondition G within X makes this "not in G"; a gold id
    outside X counts in raw, as documented)."""
    S = np.ascontiguousarray(S, dtype=np.float32)
    raw, filt = [], []
    for i, g in enumerate(gold):
        j = int(np.flatnonzero(ids == g)[0])
        below = (S[i] < S[i, j]) | ((S[i] == S[i, j]) & (ids < g))
        x, gs = X[rows[i]], G[rows[i]]
        in_x = np.isin(ids, list(x))
        filt.append(int((below & ~in_x).sum()))
        raw.append(int((below & ~(in_x & np.isin(ids, list(gs)))).sum()))
    return np.asarray(raw), np.asarray(filt)


def bracket(ref, B, ids, gold, skip, unknown=None):
    """float64 bounds on a count: (#items surely below the gold, #items possibly below it) among ~skip, where item e is
    surely below when ref_e + B_e < ref_g - B_g and surely above when ref_e - B_e > ref_g + B_g; `unknown` items
    (ST-Gumbel near ties) are only possibly below.  None when the gold itself is unknown."""
    j = int(np.flatnonzero(ids == gold)[0])
    if unknown is not None and unknown[j]:
        return None
    lo_g, hi_g = ref[j] - B[j], ref[j] + B[j]
    unk = unknown if unknown is not None else np.zeros(len(ids), bool)
    below = (ref + B < lo_g) & ~unk & ~skip
    above = (ref - B > hi_g) & ~unk & ~skip
    return int(below.sum()), int((~skip).sum() - above.sum())


def topk_metrics(lists, golds):
    """[n, 5] float64 (f1, precision, recall, hit, ndcg) of getRecPerformance on id lists (empty places dropped):
    precision = hits / list length, recall = hits / |gold|, ndcg_at_k method 0 (weights 1, 1, 1/log2(3), ...)."""
    out = np.zeros((len(lists), 5))
    for q, (ids, gold) in enumerate(zip(lists, golds)):
        hits = [i in gold for i in ids]
        n_hit = sum(hits)
        if not n_hit:
            continue
        w = [1.0 if p == 0 else 1.0 / np.log2(p + 1.0) for p in range(len(ids))]
        p, r = n_hit / len(ids), n_hit / len(gold)
        out[q] = (2 * p * r / (p + r), p, r, 1.0, sum(wi for wi, h in zip(w, hits) if h) / sum(w[:n_hit]))
    return out


def zero_items(user, Pm, Nm, ks):
    """float64 rows i with |proj(u) + r - proj(i)|^2 = 0 exactly in real arithmetic for preference k (r = Pm[k],
    w = Nm[k]): s = r.w / (|w|^2 - 1), a = -r + s w, i = u - a (then a . w = s and a + r - (a . w) w = 0)."""
    r, w = Pm[ks], Nm[ks]
    s = (r * w).sum(-1) / ((w * w).sum(-1) - 1.0)
    return user - (-r + s[:, None] * w)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_rec_count_definition_with_ties_zero_keys_and_filtered_golds():
    # all-zero scores: every key is its id.  Gold 0 has key 0, and so has the filtered gold 3 in the kernel's sorted
    # gold list; gold 0 counts nothing, gold 3 is -1, gold 5 counts 1, 2, 4 (3 is a gold, not counted)
    z = np.zeros((1, 8), np.float32)
    assert oracle_counts(z, [{0, 3, 5}], [{3}]).tolist() == [0, -1, 3]
    # ties between golds and non-golds: items 1 and 4 repeat gold 2's score; ids break the tie
    s = np.asarray([[0.5, 0.25, 0.25, 0.75, 0.25, 0.0]], np.float32)
    assert oracle_counts(s, [{2, 3}], [set()]).tolist() == [2, 4]        # gold 2: {5, 1}; gold 3: {5, 1, 4, 0}
    assert oracle_counts(s, [{2, 3}], [{5, 1}]).tolist() == [0, 2]
    assert oracle_counts(s, [{2, 3}], [{2, 3}]).tolist() == [-1, -1]      # every gold filtered
    # the float64 bracket: item 0 straddles the gold, item 2 is surely above, item 1 surely below
    ref, B = np.asarray([1.0, 0.0, 3.0, 1.05]), np.asarray([0.1, 0.1, 0.1, 0.1])
    assert bracket(ref, B, np.arange(4), 3, np.asarray([False, False, False, True])) == (1, 2)
    assert bracket(ref, B, np.arange(4), 3, np.zeros(4, bool), np.asarray([0, 0, 0, 1], bool)) is None


def test_dual_definition_on_a_hand_computed_example():
    S = np.asarray([[0.3, 0.1, 0.2, 0.2, 0.9, 0.0],
                    [0.3, 0.1, 0.2, 0.2, 0.9, 0.0]], np.float32)
    ids = np.arange(6)
    # query 0: gold 3 (0.2); below it by (score, id): 5, 1, 2.  X = {1, 2, 3}, G = {2, 3}:
    #   filtered skips 1, 2 -> {5}; raw skips only 2 -> {5, 1}
    # query 1: gold 0 (0.3); below it 5, 1, 2, 3.  X = {2, 3}, G = {1, 2, 3} holds 1, which X lacks (the documented
    #   case): filtered skips 2, 3 -> {5, 1}; raw skips only what both hold, 2 and 3 -> {5, 1}, not {5}
    X, G = [{1, 2, 3}, {2, 3}], [{2, 3}, {1, 2, 3}]
    raw, filt = dual_counts(S, ids, [3, 0], [0, 1], X, G)
    assert raw.tolist() == [2, 2] and filt.tolist() == [1, 2]
    raw, filt = dual_counts(np.zeros((1, 6), np.float32), ids, [4], [0], [set(range(6))], [{4}])
    assert raw.tolist() == [4] and filt.tolist() == [0]                    # whole-catalog exclusion row


def test_topk_metrics_restatement_on_hand_computed_lists():
    from kgrec_b200 import evaluation as KE
    lists = [[10, 11, 12, 13], [7, 8], [], [5]]
    golds = [{11, 13, 99}, {1}, {4}, {5, 6}]
    got = topk_metrics(lists, golds)
    # list 0: hits at places 1 and 3 of 4: p = 1/2, r = 2/3, dcg = 1 + 1/log2(4), idcg = 1 + 1
    assert got[0, :4].tolist() == pytest.approx([2 * 0.5 * (2 / 3) / (0.5 + 2 / 3), 0.5, 2 / 3, 1.0])
    assert got[0, 4] == pytest.approx((1 + 1 / np.log2(4)) / 2)
    assert got[1].tolist() == [0.0] * 5 and got[2].tolist() == [0.0] * 5
    assert got[3].tolist() == pytest.approx([2 * 0.5 / 1.5, 1.0, 0.5, 1.0, 1.0])
    np.testing.assert_allclose(got, np.asarray(KE.rec_metrics_from_topk(lists, golds), np.float64), rtol=1e-12, atol=0)


def test_merge_host_statement_keeps_equal_keys_and_empty_tails():
    from kgrec_b200 import evaluation as KE
    lists = np.asarray([[[1, 5, INF]], [[1, 2, 9]], [[INF, INF, INF]]], dtype=np.uint64)
    got = KE.merge_topk_host(torch.from_numpy(lists.view(np.int64))).numpy().view(np.uint64)
    assert got.tolist() == [[1, 1, 2]]


def test_zero_score_construction_in_float64():
    rng = np.random.RandomState(0)
    d, P, n = 64, 4, 500
    Pm, Nm = rng.uniform(-0.3, 0.3, (P, d)), rng.uniform(-0.3, 0.3, (P, d))
    u = rng.uniform(-0.3, 0.3, (n, d))
    ks = rng.randint(0, P, n)
    i = zero_items(u, Pm, Nm, ks).astype(np.float32).astype(np.float64)    # the fp32 table row
    w = Nm[ks]
    e = (u - (u * w).sum(-1, keepdims=True) * w) + Pm[ks] - (i - (i * w).sum(-1, keepdims=True) * w)
    score = (e * e).sum(-1)
    mag = (np.abs(u) + np.abs(i) + np.abs(Pm[ks])).max()
    assert score.max() < 1e-12 * mag * mag * d                           # only the fp32 rounding of the item rows


# ---- GPU helpers ----------------------------------------------------------------------------------------------------
def _lt(x, dtype=torch.int64):
    return torch.as_tensor(np.asarray(x), dtype=dtype, device="cuda")


def _csr(sets):
    ptr = np.concatenate([[0], np.cumsum([len(s) for s in sets])]).astype(np.int64)
    ids = np.concatenate([np.asarray(sorted(s), dtype=np.int32) for s in sets] + [np.zeros(0, np.int32)])
    return _lt(ptr), _lt(ids if ids.size else np.zeros(1, np.int32), torch.int32), int(ids.size)


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rec_sets(rng, nq, I, sizes=GOLD_SIZES):
    """Gold and filter sets per user: gold counts cycling through `sizes` (clipped to the catalog), filter rows that are
    empty, random, hold a gold, hold every gold of the user, or the whole catalog, and ids beyond the catalog."""
    golds, filts = [], []
    for q in range(nq):
        n = sizes[q % len(sizes)]
        n = max(0, min(I, I + n if n < 0 else n))
        g = set(int(x) for x in rng.choice(I, n, replace=False))
        kind = q % 5
        f = set() if kind == 0 else set(int(x) for x in rng.choice(I, min(I, int(rng.randint(1, 12))), replace=False))
        if kind == 2 and g:
            f.add(min(g))                                      # one filtered gold
        if kind == 3 and q % 3 == 0:
            f |= g                                             # every gold filtered
        if q % 11 == 7:
            f = set(range(I)) | {I + 4}                        # the whole catalog, and an id beyond it
        golds.append(g)
        filts.append(f)
    return golds, filts


def _dup_rows(m, rng, golds=()):
    """Duplicated item rows (equal scores, ties broken by id), some of them copies of golds, so golds tie with
    non-golds."""
    w = m.item_embeddings.weight
    I = w.shape[0]
    if I < 8:
        return
    src = list(rng.choice(I, I // 8, replace=False)) + [min(g) for g in golds if g][:4]
    src = torch.as_tensor(np.asarray(src, dtype=np.int64), device=w.device)
    with torch.no_grad():
        w[(src + 3) % I] = w[src]
        if m.MODEL == 4:
            m._item2ent[(src + 3) % I] = m._item2ent[src]


def _zero_tables(m):
    with torch.no_grad():
        for t in m._weights().values():
            t.zero_()


def _matrix(m, path, ut, gu=None, seed=0):
    """The score matrix of one rec path for the user list ut (same noise as the rank call: explicit uniforms or the
    hashed draws of `seed` at the same query positions)."""
    from kgrec_b200 import _lib
    users = m.user_embeddings.weight.detach()
    if path == "gumbel_aug":
        return m._eval(m.MODEL, _lib.SIDE_REC, None, None, "scores", catalog=m.gumbel_catalog(),
                       qvec=m._gumbel_rows(users, ids=ut, with_consts=True), gumbel_u=gu, seed=seed)
    if path == "soft_aug":
        return m._eval(m.MODEL, _lib.SIDE_REC, None, None, "scores", catalog=m.soft_catalog(), qvec=m._aug_rows(users, True, ids=ut))
    return m._eval(m.MODEL, _lib.SIDE_REC, ut, None, "scores", catalog=m._rec_catalog(), gumbel_u=gu, seed=seed)


def _kernel(m, topn):
    """The kernel launch_rec_rank takes for this model and topn."""
    from kgrec_b200 import _lib
    d = m.embedding_size
    path = _rec_path(m, topn)
    if path == "soft_aug":
        return "k_eval_soft_l1" if m.L1_flag else "k_eval_soft_l2"
    if path == "gumbel_aug":
        return "gumbel_tiled16" if d <= 128 else "gumbel_tiled8"
    assert _lib.load().kgrec_pref_eval_supported(d, m.pref_embeddings.weight.shape[0], int(m.use_st_gumbel), topn)
    return "%s_nch%d" % ("hard" if m.use_st_gumbel else "soft", 1 if d <= 128 else 2)


def _rec_rank_case(m, u, golds, filts, topn=0, gu=None, seed=0, shards=(), tag=""):
    """Rank counts and gold scores of one call against the definition on the path's own matrix; float64 checks when
    the noise is explicit (or there is none); shard sums for every entry of `shards` (a list of cut points)."""
    I = m.item_embeddings.weight.shape[0]
    un = np.asarray(u.cpu().numpy() if torch.is_tensor(u) else u, dtype=np.int64)
    ut = u if torch.is_tensor(u) else _lt(u)
    nq = len(un)
    S = _matrix(m, _rec_path(m, topn), ut, gu, seed).cpu().numpy()
    _nonneg(S, tag + " matrix")
    gptr, gids, n_gold = _csr(golds)
    fcsr = _csr(filts)[:2]
    kw = dict(gumbel_u=gu, seed=seed if gu is None else 0, topn=topn, n_gold=n_gold)
    want = oracle_counts(S, golds, filts)
    got = m.rank_counts_items(ut, (gptr, gids), fcsr, **kw).cpu().numpy()
    assert got.tolist() == want.tolist(), tag
    if n_gold:
        gs = m.gold_scores_items(ut, (gptr, gids), **kw).cpu().numpy()
        _nonneg(gs, tag + " gold scores")
        rows = np.repeat(np.arange(nq), [len(g) for g in golds])
        assert np.array_equal(gs.view(np.uint32), S[rows, gids.cpu().numpy()[:n_gold]].view(np.uint32)), tag
    if gu is not None or not m.use_st_gumbel:
        gu64 = gu.cpu().numpy().astype(np.float64) if gu is not None else None
        ref, B, near = _rec_ref(m, _f64(m), un, gu64)
        _check_scores(S, ref, B, tag, near)
        ids = np.arange(I)
        j = 0
        for q, (g, f) in enumerate(zip(golds, filts)):
            skip = np.isin(ids, list(g | f))
            for x in sorted(g):
                if got[j] >= 0:
                    br = bracket(ref[q], B[q], ids, x, skip, near[q] if m.use_st_gumbel else None)
                    if br is not None:
                        assert br[0] <= got[j] <= br[1], (tag, q, x, br, got[j])
                j += 1
    cat = m._rec_catalog()
    for cuts in shards:
        bounds = list(zip(cuts[:-1], cuts[1:]))
        assert bounds[0][0] == 0 and bounds[-1][1] == I
        skw = dict(kw)
        parts = []
        for lo, hi in bounds:
            if gu is not None:
                skw["gumbel_u"] = gu[:, lo:hi].contiguous()
            parts.append((lo, hi, dict(skw)))
        gs = sum(m.gold_scores_items(ut, (gptr, gids), catalog=cat[lo:hi], id_base=lo, **k) for lo, hi, k in parts)
        total = sum(m.rank_counts_items(ut, (gptr, gids), fcsr, catalog=cat[lo:hi], id_base=lo, gold_scores=gs, **k)
                    for lo, hi, k in parts)
        assert torch.where(total < 0, torch.full_like(total, -1), total).cpu().tolist() == want.tolist(), (tag, cuts)
    return S, got


# ---- GPU: rec rank counts -------------------------------------------------------------------------------------------
# (kernel, model name, d, P, topn): every kernel launch_rec_rank launches
REC_KERNELS = [
    ("k_eval_soft_l1", "tup_soft_l1", 100, 20, 0),
    ("k_eval_soft_l2", "ktup_soft_l2", 64, 20, 0),
    ("gumbel_tiled16", "tup_gumbel_l2", 128, 20, 0),
    ("gumbel_tiled8", "ktup_gumbel_l2", 200, 8, 0),
    ("hard_nch1", "tup_gumbel_l1", 100, 20, 0),                  # ST-Gumbel L1
    ("hard_nch2", "ktup_gumbel_l1", 200, 8, 0),
    ("hard_nch1", "tup_gumbel_l2", 64, 65, 0),                   # L2 with P = 65 > 64 augmented preferences
    ("hard_nch1", "ktup_gumbel_l2", 128, 4, 88),                 # L2 with topn past kgrec_gumbel_aug_supported
    ("hard_nch2", "tup_gumbel_l2", 256, 32, 128),
    ("soft_nch1", "tup_soft_l2", 128, 20, 62),                   # soft, topn >= 62 at d = 128
    ("soft_nch2", "tup_soft_l1", 148, 8, 0),                     # soft, d >= 148
    ("soft_nch2", "ktup_soft_l2", 200, 8, 10),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,name,d,P,topn", REC_KERNELS)
def test_rec_rank_kernels(kernel, name, d, P, topn):
    rng = np.random.RandomState(d * 7 + P + topn + len(name))
    torch.manual_seed(d + P)
    U, I = 120, 300
    m = _rec_model(name, d, U, I, P, seed=d + P)
    assert _kernel(m, topn) == kernel
    u = rng.choice(U, 48, replace=False)
    golds, filts = _rec_sets(rng, len(u), I)
    _dup_rows(m, rng, golds)
    gu = torch.rand(len(u), I, P, device="cuda") if m.use_st_gumbel else None
    S, got = _rec_rank_case(m, u, golds, filts, topn, gu=gu, shards=[(0, 100, 200, 300), (0, 60, 120, 180, 240, 300)],
                            tag="%s %s d=%d P=%d" % (kernel, name, d, P))
    assert (got == -1).any() and (got > 0).any()
    assert any((S[q] == S[q, x]).sum() > 1 for q, g in enumerate(golds) for x in g)         # golds tied with other items
    assert any(len(g) == 1 for g in golds)                       # so some shard holds none of that user's golds
    if m.use_st_gumbel:                                          # hashed noise: the matrix of the same call
        _rec_rank_case(m, u, golds, filts, topn, seed=0x5EED + d, shards=[(0, 100, 200, 300)], tag=kernel + " hashed")
    # all-zero tables: every key is its id; gold 0 (key 0) next to a filtered gold, whose sorted key is also 0
    _zero_tables(m)
    golds0 = [{0, 3, 5, 200}, {0, 7}, set(range(0, I, 2)), {1}]
    filts0 = [{3}, set(), {4, 6}, {1}]
    gu0 = gu[:4] if gu is not None else None
    S0, got0 = _rec_rank_case(m, u[:4], golds0, filts0, topn, gu=gu0, tag=kernel + " zero")
    assert not S0.view(np.uint32).any()
    # gold 200: ids 0..199 but golds 0, 3, 5; gold 2j of user 2: the j odd ids below it
    assert got0.tolist() == [0, -1, 3, 197] + [0, 6] + [-1 if j in (2, 3) else j for j in range(I // 2)] + [-1]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_soft_l1", "tup_soft_l2", "tup_gumbel_l2", "tup_gumbel_l1", "ktup_soft_l2", "ktup_gumbel_l2"])
def test_rec_rank_d_sweep(name):
    """TUP soft at every d % 4 == 0 up to 256, ST-Gumbel and KTUP at a stride of 12 plus the named widths."""
    rng = np.random.RandomState(len(name) * 13)
    U, I = 12, 140
    ds = range(4, 257, 4) if name.startswith("tup_soft") else sorted(set(range(4, 257, 12)) | set(NAMED_D))
    seen = set()
    for d in ds:
        m = _rec_model(name, d, U, I, 4, seed=d)
        u = rng.choice(U, 9, replace=False)
        golds, filts = _rec_sets(rng, 9, I)
        _dup_rows(m, rng, golds)
        gu = torch.rand(9, I, 4, device="cuda") if m.use_st_gumbel else None
        _rec_rank_case(m, u, golds, filts, gu=gu, tag="%s d=%d" % (name, d))
        seen.add(_kernel(m, 0))
    want = {"tup_soft_l1": {"k_eval_soft_l1", "soft_nch2"}, "tup_soft_l2": {"k_eval_soft_l2", "soft_nch2"},
            "tup_gumbel_l2": {"gumbel_tiled16", "gumbel_tiled8"}, "tup_gumbel_l1": {"hard_nch1", "hard_nch2"},
            "ktup_soft_l2": {"k_eval_soft_l2", "soft_nch2"}, "ktup_gumbel_l2": {"gumbel_tiled16", "gumbel_tiled8"}}[name]
    assert seen == want, seen


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_gumbel_l2", "tup_gumbel_l1", "tup_soft_l2", "ktup_gumbel_l2"])
@pytest.mark.parametrize("P", [1, 4, 20, 32, 64, 65, 128])
def test_rec_rank_preference_counts(name, P):
    from kgrec_b200 import _lib
    d = 64
    m = _rec_model(name, d, 30, 150, P, seed=P)
    if _rec_path(m, 10) == "plain" and not _lib.load().kgrec_pref_eval_supported(d, P, int(m.use_st_gumbel), 10):
        pytest.skip("outside kgrec_pref_eval_supported")
    rng = np.random.RandomState(P + 3)
    u = rng.choice(30, 14, replace=False)
    golds, filts = _rec_sets(rng, 14, 150)
    gu = torch.rand(14, 150, P, device="cuda") if m.use_st_gumbel else None
    _rec_rank_case(m, u, golds, filts, topn=10, gu=gu, tag="%s P=%d" % (name, P))
    if name == "tup_gumbel_l2":
        assert _kernel(m, 10) == ("gumbel_tiled16" if P <= 64 else "hard_nch1")


def _tile_rows(kernel, d):
    if kernel.startswith("k_eval_soft"):
        return 32
    if kernel.startswith("gumbel"):
        return 64 if d <= 128 else 32
    return max(4, min(64, (16 * 1024) // (d * 4))) & ~3        # plain_tile_rows(d)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,name,d,P,topn", [REC_KERNELS[i] for i in (0, 2, 3, 4, 7, 10)])
def test_rec_rank_queries_and_catalog_edges(kernel, name, d, P, topn):
    from kgrec_b200 import _lib, functional as KF
    rng = np.random.RandomState(d + 5 * P)
    U, I = 140, 70
    m = _rec_model(name, d, U, I, P, seed=d)
    assert _kernel(m, topn) == kernel
    sizes = (0, 1, 31, 32, 33, 64, 65, -3)
    for nq in (1, 7, 8, 9, 63, 64, 65, 127, 128, 129):
        u = rng.randint(0, U, nq)
        if nq > 1:
            u[-1] = u[0]                                         # one user listed twice in the call
        ut = _lt(u, torch.int32 if nq % 2 else torch.int64)
        golds, filts = _rec_sets(rng, nq, I, sizes)
        explicit = m.use_st_gumbel and nq % 3 == 0
        gu = torch.rand(nq, I, P, device="cuda") if explicit else None
        _rec_rank_case(m, ut, golds, filts, topn, gu=gu, seed=0 if explicit else 0xC0DE + nq,
                       tag="%s nq=%d %s" % (kernel, nq, ut.dtype))
    tn = _tile_rows(kernel, d)
    for n_cat in sorted({1, tn - 1, tn, tn + 1, 2 * tn + 1}):
        mc = _rec_model(name, d, U, n_cat, P, seed=n_cat)
        assert _kernel(mc, topn) == kernel
        u = rng.randint(0, U, 37)
        golds, filts = _rec_sets(rng, 37, n_cat, (0, 1, 2, -1))
        gu = torch.rand(37, n_cat, P, device="cuda") if mc.use_st_gumbel else None
        _rec_rank_case(mc, u, golds, filts, topn, gu=gu, tag="%s n_cat=%d" % (kernel, n_cat))
    # once straight through ctypes, int32 user ids, with a caller-built workspace (plain paths take ids, not rows)
    if kernel.startswith(("hard", "soft")):
        nq = 21
        u = rng.randint(0, U, nq)
        ut = _lt(u, torch.int32)
        golds, filts = _rec_sets(rng, nq, I, sizes)
        gptr, gids, n_gold = _csr(golds)
        fptr, fids, _ = _csr(filts)
        lib = _lib.load()
        T = KF.make_tables(m._weights(), m.embedding_size, m.L1_flag, m.use_st_gumbel, m._item2ent)
        cat = m._rec_catalog().contiguous()
        seed = 0xABCD
        head = (C.byref(T), m.MODEL, KF._ptr(ut), 4, None, nq, KF._ptr(cat), cat.stride(0), I, 0, KF._ptr(gptr), KF._ptr(gids))
        gs = torch.zeros(n_gold, dtype=torch.float32, device="cuda")
        _lib.check(lib.kgrec_rec_gold_scores(*head, None, seed, KF._ptr(gs), KF._stream()))
        ws = torch.empty(int(lib.kgrec_rec_rank_workspace_bytes(nq, n_gold)) // 8 + 1, dtype=torch.int64, device="cuda")
        counts = torch.zeros(n_gold, dtype=torch.int32, device="cuda")
        _lib.check(lib.kgrec_rec_rank_count(*head, n_gold, KF._ptr(gs), KF._ptr(fptr), KF._ptr(fids), None, seed, KF._ptr(counts),
                                            KF._ptr(ws), ws.numel() * 8, KF._stream()))
        S = _matrix(m, "plain", ut, None, seed).cpu().numpy()
        _nonneg(gs.cpu().numpy(), kernel + " ctypes gold scores")
        assert counts.cpu().tolist() == oracle_counts(S, golds, filts).tolist()


# ---- GPU: dual link counts ------------------------------------------------------------------------------------------
def _dual_call(m, name, side, q, r, gold, gs, row, X, G, cat, id_base=0, idx=torch.int64, qvec=None):
    """(raw, filtered) of kgrec_eval_rank_count_dual (kgrec_transr_eval_rank_count_dual for TransR: q / r sorted by r)."""
    from kgrec_b200 import _lib, functional as KF
    lib = _lib.load()
    d = m.embedding_size
    sd = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
    n = len(gold)
    qt, rt = _lt(q, idx), _lt(r, idx)
    g32, row_t = _lt(gold, torch.int32), _lt(row, torch.int32)
    gst = torch.as_tensor(np.asarray(gs, np.float32), device="cuda")
    xp, xi, _ = _csr(X)
    gp, gi, _ = _csr(G)
    raw = torch.zeros(n, dtype=torch.int32, device="cuda")
    filt = torch.zeros(n, dtype=torch.int32, device="cuda")
    st = KF._stream()
    if name == "transr":
        assert (np.diff(r) >= 0).all()
        T = KF.make_tables(m._weights(), d, m.L1_flag)
        cut = np.flatnonzero(np.diff(r)) + 1
        begin = torch.as_tensor(np.concatenate([[0], cut, [n]]).astype(np.int64))
        rels = torch.as_tensor(np.asarray(r)[np.concatenate([[0], cut])].astype(np.int64))
        ws = torch.empty(int(lib.kgrec_transr_workspace_floats(n, cat.shape[0], d)), dtype=torch.float32, device="cuda")
        _lib.check(lib.kgrec_transr_eval_rank_count_dual(
            C.byref(T), sd, KF._ptr(qt), KF._ptr(rt), qt.element_size(), n, C.c_void_p(begin.data_ptr()),
            C.c_void_p(rels.data_ptr()), rels.numel(), KF._ptr(cat), cat.stride(0), cat.shape[0], id_base, KF._ptr(ws),
            KF._ptr(gst), KF._ptr(g32), KF._ptr(filt), KF._ptr(row_t), KF._ptr(xp), KF._ptr(xi), KF._ptr(gp), KF._ptr(gi),
            KF._ptr(raw), KF._ptr(m._status_buf(torch.device("cuda"))), st))
    else:
        T = KF.make_tables(m._weights(), d, m.L1_flag, m.use_st_gumbel, m._item2ent)
        kg = _lib.TRANSH if name == "jtransup" else m.MODEL
        _lib.check(lib.kgrec_eval_rank_count_dual(
            C.byref(T), kg, sd, None if qvec is not None else KF._ptr(qt), None if qvec is not None else KF._ptr(rt),
            qt.element_size(), KF._ptr(qvec), n, KF._ptr(cat), cat.stride(0), cat.shape[0], id_base, KF._ptr(gst), KF._ptr(g32),
            KF._ptr(filt), KF._ptr(row_t), KF._ptr(xp), KF._ptr(xi), KF._ptr(gp), KF._ptr(gi), KF._ptr(raw), st))
    return raw.cpu().numpy(), filt.cpu().numpy()


def _kg_scores(m, name, side, q, r, cat, id_base=0, idx=torch.int64, qvec=None):
    from kgrec_b200 import _lib, evaluation as KE, functional as KF
    sd = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
    if qvec is not None:
        T = KF.make_tables(m._weights(), m.embedding_size, m.L1_flag, m.use_st_gumbel, m._item2ent)
        return KE.run(T, _lib.TRANSH if name == "jtransup" else m.MODEL, sd, None, None, "scores", cat, id_base=id_base, qvec=qvec)
    if name == "transr":
        return m._scores(sd, _lt(q, idx), _lt(r, idx), catalog=cat, id_base=id_base)
    kg = _lib.TRANSH if name == "jtransup" else m.MODEL
    return m._eval(kg, sd, _lt(q, idx), _lt(r, idx), "scores", catalog=cat, id_base=id_base)


def _dual_sets(rng, n_ent, n_rows, lo=0, hi=None):
    """Exclusion rows X and gold rows G (G within X): X empty / one id / the whole catalog / random, G of 0 / 1 / many
    ids."""
    hi = n_ent if hi is None else hi
    X, G = [], []
    for j in range(n_rows):
        k = (0, 1, int(rng.randint(2, 25)))[j % 3]
        g = set(int(x) for x in rng.choice(np.arange(lo, hi), min(k, hi - lo), replace=False))
        kind = j % 4
        x = set() if kind == 0 else {int(rng.randint(0, n_ent))} if kind == 1 else \
            set(range(n_ent)) if (kind == 2 and j % 8 == 2) else set(int(v) for v in rng.choice(n_ent, int(rng.randint(2, 40)), replace=False))
        X.append(x | g)
        G.append(g)
    return X, G


def _pick_gold(rng, rows, G, N):
    """Each pair's gold: mostly an id of its gold row, sometimes any id (a gold outside its gold row)."""
    return np.asarray([int(rng.choice(sorted(G[j]))) if G[j] and rng.rand() < 0.8 else int(rng.randint(0, N)) for j in rows])


def _dual_case(m, name, side, q, r, rows, X, G, gold, cat=None, id_base=0, idx=torch.int64, qvec=None, ref=True, tag=""):
    """One dual call against the definition on the kernel's own matrix (and float64 brackets); returns (raw, filt)."""
    cat = m.ent_embeddings.weight.detach() if cat is None else cat
    N = cat.shape[0]
    ids = id_base + np.arange(N)
    n = len(q)
    S = _kg_scores(m, name, side, q, r, cat, id_base, idx, qvec).cpu().numpy()
    _nonneg(S, tag + " matrix")
    gs = S[np.arange(n), gold - id_base]
    raw, filt = _dual_call(m, name, side, q, r, gold, gs, rows, X, G, cat, id_base, idx, qvec)
    want_raw, want_filt = dual_counts(S, ids, gold, rows, X, G)
    assert raw.tolist() == want_raw.tolist(), tag + " raw"
    assert filt.tolist() == want_filt.tolist(), tag + " filtered"
    if ref and qvec is None:
        W = _f64(m)
        rf, B = _kg_ref("transh" if name == "jtransup" else name, W, np.asarray(q, np.int64), np.asarray(r, np.int64), side,
                        cat.double().cpu().numpy(), m.L1_flag)
        _check_scores(S, rf, B, tag)
        for i in range(n):
            in_x = np.isin(ids, list(X[rows[i]]))
            for got, skip in ((filt[i], in_x), (raw[i], in_x & np.isin(ids, list(G[rows[i]])))):
                lo, hi = bracket(rf[i], B[i], ids, gold[i], skip)
                assert lo <= got <= hi, (tag, i, lo, got, hi)
    return raw, filt


@pytest.mark.gpu
@pytest.mark.parametrize("name,l1", [("transe", False), ("transe", True), ("transh", False), ("transh", True),
                                     ("jtransup", False), ("jtransup", True), ("transr", False), ("transr", True)])
def test_dual_d_sweep(name, l1):
    """Every d % 4 == 0 up to 256 (TransR 128): the 16-warp plans to d = 128, the 8-warp plans beyond."""
    rng = np.random.RandomState(len(name) * 3 + int(l1))
    E = 140
    for d in range(4, (128 if name == "transr" else 256) + 1, 4):
        m = _kg_model(name, l1, d, E, seed=d)
        n_ent = m.ent_embeddings.weight.shape[0]
        with torch.no_grad():                                  # twin rows: equal scores, ties broken by id
            w = m.ent_embeddings.weight
            src = _lt(rng.choice(n_ent, 20, replace=False))
            w[(src + 5) % n_ent] = w[src]
        X, G = _dual_sets(rng, n_ent, 12)
        n = 40
        rows = rng.randint(0, 12, n)                           # rows shared by several queries
        q, r = rng.randint(0, E - 1, n), rng.randint(0, 3, n)
        if name == "transr":
            o = np.argsort(r, kind="stable")
            q, r, rows = q[o], r[o], rows[o]
        _dual_case(m, name, "head" if d % 8 else "tail", q, r, rows, X, G, _pick_gold(rng, rows, G, n_ent),
                   idx=torch.int32 if d % 12 == 0 else torch.int64, tag="%s l1=%d d=%d" % (name, l1, d))


def _pieces(nq, n_cat, tn, tqt, sm):
    """eval_plan's tiling of a register-tiled call: (units_per_cta, n_tiles, does some CTA range cross a query tile)."""
    n_tiles, n_qt = -(-n_cat // tn), -(-nq // tqt)
    total = n_tiles * n_qt
    ctas = min(sm, total)
    upc = -(-total // ctas)
    grid = -(-total // upc)
    crosses = any((b * upc) // n_tiles != (min(total, (b + 1) * upc) - 1) // n_tiles for b in range(grid))
    return upc, n_tiles, crosses


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["transe", "transh", "jtransup"])
def test_dual_pieces_ties_and_zero_table(name):
    """Several CTAs per query tile, and CTA ranges that cross from one query tile into the next (end_qtile flushes the
    filtered counts mid-range while the raw count takes per-row atomics); rows i and i + n_cat / 2 identical, the gold
    among tied rows; then an all-zero table."""
    sm = _sm()
    d, n_cat = 32, 600
    tn, tqt = (128, 128) if name == "transe" else (64, 128)          # 16-warp plans at d = 32
    nq = 0
    for nqt in range(2, 400):
        upc, n_tiles, crosses = _pieces(nqt * tqt - 3, n_cat, tn, tqt, sm)
        if crosses and upc < n_tiles and nqt * n_tiles > sm:
            nq = nqt * tqt - 3
            break
    upc, n_tiles, crosses = _pieces(nq, n_cat, tn, tqt, sm)
    assert nq > 0 and crosses and upc < n_tiles
    rng = np.random.RandomState(11)
    m = _kg_model(name, False, d, n_cat + 1 if name == "jtransup" else n_cat)
    cat = m.ent_embeddings.weight.detach()[:n_cat]
    w = m.ent_embeddings.weight
    with torch.no_grad():
        w[n_cat // 2:n_cat] = w[:n_cat // 2]
    q, r = rng.randint(0, n_cat, nq), rng.randint(0, 3, nq)
    X, G = _dual_sets(rng, n_cat, 50)
    S = _kg_scores(m, name, "tail", q, r, cat).cpu().numpy()
    _nonneg(S, name + " pieces")
    # the gold: the query's best row or the row at a random place of its order, or the twin of either (tied keys)
    pick = np.argsort(S, axis=1, kind="stable")[np.arange(nq), np.where(np.arange(nq) % 4 == 0, 0, rng.randint(1, n_cat, nq))]
    gold = np.where(np.arange(nq) % 2, pick, (pick + n_cat // 2) % n_cat)
    twin = (gold + n_cat // 2) % n_cat
    Xs, Gs = [], []
    for i in range(nq):            # a row per query: G = a gold row + the gold (+ its twin); X = G + a filter (+ the twin)
        j = int(rng.randint(0, 50))
        Gs.append(G[j] | {int(gold[i])} | ({int(twin[i])} if i % 3 == 1 else set()))
        Xs.append(X[j] | Gs[-1] | ({int(twin[i])} if i % 3 == 2 else set()))
    rows1 = np.arange(nq)
    gs = S[np.arange(nq), gold]
    raw, filt = _dual_call(m, name, "tail", q, r, gold, gs, rows1, Xs, Gs, cat)
    want_raw, want_filt = dual_counts(S, np.arange(n_cat), gold, rows1, Xs, Gs)
    assert raw.tolist() == want_raw.tolist() and filt.tolist() == want_filt.tolist()
    assert (want_raw > want_filt).any() and (want_filt > 0).any()
    with torch.no_grad():
        for t in m._weights().values():
            t.zero_()
    S0 = _kg_scores(m, name, "tail", q, r, cat).cpu().numpy()
    assert not S0.view(np.uint32).any()
    raw, filt = _dual_call(m, name, "tail", q, r, gold, np.zeros(nq, np.float32), rows1, Xs, Gs, cat)
    want_raw = [sum(1 for e in range(g) if not (e in Xs[i] and e in Gs[i])) for i, g in enumerate(gold)]
    want_filt = [sum(1 for e in range(g) if e not in Xs[i]) for i, g in enumerate(gold)]
    assert raw.tolist() == want_raw and filt.tolist() == want_filt


@pytest.mark.gpu
@pytest.mark.parametrize("name,d", [("transe", 100), ("transe", 128), ("transh", 64), ("transh", 252), ("jtransup", 200),
                                    ("transr", 100)])
def test_dual_layouts_and_precondition(name, d):
    """int32 ids, explicit query vectors (qvec), a strided catalog (cat_ld > d), three shards with id_base, and a gold
    row holding an id its exclusion row lacks: that id counts in the raw count (the documented precondition)."""
    from kgrec_b200 import evaluation as KE
    rng = np.random.RandomState(d + len(name))
    E = 400
    m = _kg_model(name, d % 8 == 4, d, E)
    ent = m.ent_embeddings.weight.detach()
    n_ent = ent.shape[0]
    n = 70
    q, r = rng.randint(0, E - 1, n), rng.randint(0, 3, n)
    rows = rng.randint(0, 20, n)
    if name == "transr":
        o = np.argsort(r, kind="stable")
        q, r, rows = q[o], r[o], rows[o]
    X, G = _dual_sets(rng, n_ent, 20)
    gold = _pick_gold(rng, rows, G, n_ent)
    tag = "%s d=%d" % (name, d)
    whole = _dual_case(m, name, "head", q, r, rows, X, G, gold, idx=torch.int32, tag=tag + " int32")
    # strided catalog: the same counts
    wide = torch.zeros((n_ent, d + 12), dtype=torch.float32, device="cuda")
    wide[:, :d] = ent
    strided = _dual_case(m, name, "head", q, r, rows, X, G, gold, cat=wide[:, :d], ref=False, tag=tag + " strided")
    assert all(np.array_equal(a, b) for a, b in zip(whole, strided))
    # three shards with id_base: per-shard counts add up to the whole-catalog counts
    S = _kg_scores(m, name, "head", q, r, ent).cpu().numpy()
    gs = S[np.arange(n), gold]
    tot = [np.zeros(n, np.int64), np.zeros(n, np.int64)]
    for lo, hi in (KE.shard_bounds(n_ent, 3, g) for g in range(3)):
        part = _dual_call(m, name, "head", q, r, gold, gs, rows, X, G, ent[lo:hi], id_base=lo)
        tot[0] += part[0]
        tot[1] += part[1]
    assert tot[0].tolist() == whole[0].tolist() and tot[1].tolist() == whole[1].tolist()
    # the documented precondition case: G_i holds ids X_i lacks; below the gold they still count in raw
    Gx = [g | (set(int(v) for v in rng.choice(n_ent, 60, replace=False)) - x) for g, x in zip(G, X)]
    raw, _ = _dual_case(m, name, "head", q, r, rows, X, Gx, gold, ref=False, tag=tag + " G not in X")
    assert raw.tolist() == whole[0].tolist()
    lone = [sum(1 for e in Gx[rows[i]] - X[rows[i]] if (S[i, e], e) < (S[i, gold[i]], gold[i])) for i in range(n)]
    assert sum(lone) > 0
    # explicit query vectors [c | w] (KG kinds other than TransR)
    if name != "transr":
        qv = torch.randn(n, 2 * d, device="cuda") * 0.3
        _dual_case(m, name, "head", q, r, rows, X, G, gold, qvec=qv, tag=tag + " qvec")


# ---- GPU: top-n metrics, merge ----------------------------------------------------------------------------------------
def _lists_and_golds(rng, nq, k, n_ids=1000):
    """Key lists (ascending, UINT64_MAX tails) and gold sets: full and short lists, hits at places 0 / 31 / 32 / 127,
    gold sets larger than k, users with no hit."""
    keys = np.full((nq, k), INF, dtype=np.uint64)
    lists, golds = [], []
    for q in range(nq):
        kind = q % 6
        L = k if kind in (0, 1, 2) else int(rng.randint(0, k + 1))
        ids = rng.choice(n_ids, L, replace=False)
        g = set(int(x) for x in rng.choice(n_ids, int(rng.randint(1, 6)), replace=False))
        places = [p for p in (0, 31, 32, 127) if p < L]
        if kind == 1:
            g |= set(int(ids[p]) for p in places)
        elif kind == 2:
            g |= set(int(x) for x in ids[: min(L, max(1, 2 * k // 3))]) | set(range(n_ids, n_ids + k + 5))   # larger than k
        elif kind == 4:
            g -= set(int(x) for x in ids)                     # no hit
            g = g or {n_ids + 1}
        elif L:
            g.add(int(ids[int(rng.randint(0, L))]))
        bits = np.sort(rng.randint(0, 0x7F80_0000, L).astype(np.uint64))
        keys[q, :L] = (bits << np.uint64(32)) | ids.astype(np.uint64)
        lists.append([int(x) for x in ids])
        golds.append(g)
    return keys, lists, golds


@pytest.mark.gpu
def test_rec_topk_metrics_envelope():
    from kgrec_b200 import _lib, functional as KF
    lib = _lib.load()
    rng = np.random.RandomState(5)
    second_pass = 8 * 16 * _sm() + 37                            # past the grid cap: a second grid-stride pass
    for k in (1, 31, 32, 33, 64, 65, 127, 128):
        nq = second_pass if k == 33 else 96
        keys, lists, golds = _lists_and_golds(rng, nq, k)
        gptr, gids, _ = _csr(golds)
        out = torch.full((nq, 5), float("nan"), dtype=torch.float64, device="cuda")
        kt = torch.as_tensor(keys.view(np.int64), device="cuda")
        _lib.check(lib.kgrec_rec_topk_metrics(KF._ptr(kt), nq, k, KF._ptr(gptr), KF._ptr(gids), KF._ptr(out), KF._stream()))
        want = topk_metrics(lists, golds)
        got = out.cpu().numpy()
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, err_msg="k=%d" % k)
        assert (want[:, 3] == 0).any() and (want[:, 3] == 1).any()
        if k >= 33:
            assert (want[:, 4] < 1).any()                        # hits placed past the first 32 places


@pytest.mark.gpu
def test_merge_topk_envelope():
    from kgrec_b200 import evaluation as KE
    rng = np.random.RandomState(6)
    pool = ((np.arange(400, dtype=np.uint64) // np.uint64(3)) << np.uint64(32)) | np.arange(400, dtype=np.uint64) % np.uint64(50)
    for n_lists in (1, 2, 3 * _sm()):
        for k in (1, 32, 33, 128):
            for nq in (1, 7, 8, 9, 15, 16, 17):
                lists = np.full((n_lists, nq, k), INF, dtype=np.uint64)
                for l in range(n_lists):
                    for q in range(nq):
                        L = int(rng.randint(0, k + 1)) if (l + q) % 3 else k
                        lists[l, q, :L] = np.sort(rng.choice(pool, L, replace=False))     # equal keys across lists
                t = torch.as_tensor(lists.view(np.int64))
                got = KE.merge_topk(t.cuda()).cpu()
                want = KE.merge_topk_host(t)
                assert torch.equal(got, want), (n_lists, k, nq)
                if n_lists > 2 and k > 1:
                    v = lists[lists != INF]
                    assert np.unique(v).size < v.size            # equal keys across lists


# ---- GPU: ST-Gumbel L2 scores of true value 0 -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,P", [("tup_gumbel_l2", 1), ("tup_gumbel_l2", 4), ("ktup_gumbel_l2", 1), ("ktup_gumbel_l2", 4)])
def test_st_gumbel_l2_zero_scores_rank_first(name, P):
    """Items built so that a + r - (a . w) w = 0 for their user (float64 score ~1e-15): the expanded form of
    KIND_GUMBEL_L2 evaluates them to +-rounding noise, and a negative result keys after every other item.  Each must be
    its user's top-1, count 0 as a gold, and no score may carry the sign bit, through evaluate / evaluateRec,
    topk_items, rank_counts_items and RecEvaluator(ranks=True)."""
    from kgrec_b200 import evaluation as KE, metrics as KM
    d, U, I, nu = 64, 40, 200, 30
    m = _rec_model(name, d, U, I, P, seed=P)
    assert _rec_path(m, 0) == "gumbel_aug" and _rec_path(m, 10) == "gumbel_aug"
    ktup = m.MODEL == 4
    if not ktup:       # TUP's normal rows start at unit length, where only r orthogonal to w reaches 0: shorten them
        with torch.no_grad():
            m.pref_norm_embeddings.weight.mul_(0.7)
    W = {k: v.detach().double().cpu().numpy() for k, v in m._weights().items()}
    hf = 0.5 if ktup else 1.0
    Pm = hf * (W["pref"] + (W["rel"] if ktup else 0))
    Nm = hf * (W["pref_norm"] + (W["norm"] if ktup else 0))
    users = np.arange(nu)
    ks = users % P
    items = 100 + users                                          # item 100 + u is user u's zero-score item
    rows = zero_items(W["user"][users], Pm, Nm, ks)
    with torch.no_grad():
        if ktup:
            ent = m.ent_embeddings.weight.detach().double().cpu().numpy()[m.item2ent.cpu().numpy()[items]]
            rows = rows - ent
        m.item_embeddings.weight[_lt(items)] = torch.as_tensor(rows, dtype=torch.float32, device="cuda")
    # uniforms making k_u the certain arg-max of every constructed pair (P = 4); any draw does for P = 1
    gu = torch.rand(nu, I, P, device="cuda") * 0.98 + 0.01
    if P > 1:
        gu[torch.arange(nu), _lt(items)] = 1e-7
        gu[torch.arange(nu), _lt(items), _lt(ks)] = 1.0 - 1e-7
    ut = _lt(users)
    ref, B, near = _rec_ref(m, _f64(m), users, gu.cpu().numpy().astype(np.float64))
    assert not near[users, items].any()
    assert (np.abs(ref[users, items]) < 1e-9).all()
    others = ref.copy()
    others[users, items] = np.inf
    assert (others.min(1) > 1e-2).all()                         # every constructed item is its user's float64 top-1
    sources = [dict(gumbel_u=gu)] + ([dict(seed=0x2E80)] if P == 1 else [])
    gptr, gids, n_gold = _csr([{int(i)} for i in items])
    ev = KM.RecEvaluator(m, {int(u): {int(i)} for u, i in zip(users, items)}, None, topn=10, ranks=True)
    assert ev.users.cpu().tolist() == users.tolist()
    for src in sources:
        gu_s, seed = src.get("gumbel_u"), src.get("seed", 0)
        tag = "%s P=%d %s" % (name, P, "explicit" if gu_s is not None else "hashed")
        S = _matrix(m, "gumbel_aug", ut, gu_s, seed).cpu().numpy()
        m._next_seed = lambda: seed
        S2 = (m.evaluateRec(ut, None, gu_s) if ktup else m.evaluate(ut, gu_s)).cpu().numpy()
        assert np.array_equal(S.view(np.uint32), S2.view(np.uint32))
        _nonneg(S, tag + " matrix")
        if gu_s is not None:
            _check_scores(S, ref, B, tag, near)
        assert (S.argmin(1) == items).all(), tag
        keys = m.topk_items(ut, k=10, gumbel_u=gu_s).cpu().numpy()
        _nonneg_keys(keys, tag + " top-k")
        ids, _ = KE.keys_to_ids_scores(torch.as_tensor(keys))
        assert (ids[:, 0].numpy() == items).all(), tag + " top-1"
        counts = m.rank_counts_items(ut, (gptr, gids), gumbel_u=gu_s, seed=seed, n_gold=n_gold).cpu().numpy()
        assert (counts == 0).all(), tag + " rank counts"
        gs = m.gold_scores_items(ut, (gptr, gids), gumbel_u=gu_s, seed=seed, n_gold=n_gold).cpu().numpy()
        _nonneg(gs, tag + " gold scores")
        assert (ev.rank_counts(seed=seed, gumbel_u=gu_s).cpu().numpy() == 0).all(), tag + " evaluator ranks"
        res = ev.result(ev.run(seed=seed, gumbel_u=gu_s))
        assert res[3] == 1.0 and res[4] == 1.0 and res[5] == 0.0 and res[6] == 1.0, (tag, res)
