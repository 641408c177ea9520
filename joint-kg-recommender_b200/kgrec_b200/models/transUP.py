"""TUP (`-model_type transup`) on the CUDA engine.  Mirrors jTransUP/models/transUP.py
(constructor 19-67, forward 69-82, evaluate 84-102, getPreferences 105-115,
st_gumbel_softmax 143-170, reportPreference 172-180)."""
import torch

from .. import _lib
from .. import functional as KF
from .base import KGRecModule, _make_tables


def build_model(FLAGS, user_total, item_total, entity_total, relation_total, i_map=None, e_map=None, new_map=None):
    return TransUPModel(L1_flag=FLAGS.L1_flag, embedding_size=FLAGS.embedding_size, user_total=user_total,
                        item_total=item_total, preference_total=FLAGS.num_preferences,
                        use_st_gumbel=FLAGS.use_st_gumbel)


class RecModelBase(KGRecModule):
    """What TUP and KTUP share on the recommendation side."""

    def _rec_catalog(self):
        return self.item_embeddings.weight.detach()

    def _aug_rows(self, rows, is_query, ids=None):
        """Augmented rows of the soft-preference evaluation (kgrec_pref_aug_rows)."""
        import ctypes as C
        dev = self._require_cuda()
        lib = _lib.load()
        T = KF.make_tables(self._weights(), self.embedding_size, self.L1_flag, self.use_st_gumbel, self._item2ent)
        n = ids.numel() if ids is not None else rows.shape[0]
        lda = int(lib.kgrec_pref_aug_ld(self.embedding_size))
        out = torch.empty((n, lda), dtype=torch.float32, device=dev)
        _lib.check(lib.kgrec_pref_aug_rows(C.byref(T), self.MODEL, 1 if is_query else 0,
                                           KF._ptr(ids), ids.element_size() if ids is not None else 8,
                                           KF._ptr(rows), rows.stride(0), n, KF._ptr(out), lda, KF._stream()))
        KF.count_launches(1)
        return out

    def soft_catalog(self, catalog=None):
        """Augmented item catalog for repeated soft-mode evaluation calls (build once per table
        state: it depends on the item and preference tables)."""
        cat = self._rec_catalog() if catalog is None else catalog
        return self._aug_rows(cat.contiguous(), False)

    def _gumbel_rows(self, rows, ids=None, with_consts=False):
        """Augmented rows of the ST-Gumbel (squared-L2) evaluation: [x | x.P'_k / 2 | x.(hf N'_k) | pad]
        (kgrec_gumbel_aug_rows); with_consts: the [3 P] table constants are stored right behind the rows,
        where the evaluation kernels expect them for the QUERY rows."""
        import ctypes as C
        dev = self._require_cuda()
        lib = _lib.load()
        T = KF.make_tables(self._weights(), self.embedding_size, self.L1_flag, self.use_st_gumbel, self._item2ent)
        n = ids.numel() if ids is not None else rows.shape[0]
        P = self.pref_embeddings.weight.shape[0]
        ld = int(lib.kgrec_gumbel_aug_ld(self.embedding_size, P))
        buf = torch.empty(n * ld + (3 * P if with_consts else 0), dtype=torch.float32, device=dev)
        out = buf[:n * ld].view(n, ld)
        gconst = C.c_void_p(buf.data_ptr() + n * ld * 4) if with_consts else None
        _lib.check(lib.kgrec_gumbel_aug_rows(C.byref(T), self.MODEL, KF._ptr(ids), ids.element_size() if ids is not None else 8,
                                             KF._ptr(rows), rows.stride(0), n, KF._ptr(out), ld, gconst, KF._stream()))
        KF.count_launches(1)
        return out

    def gumbel_catalog(self, catalog=None):
        """Augmented item catalog for repeated ST-Gumbel evaluation calls (rebuild when the item or preference
        tables change)."""
        cat = self._rec_catalog() if catalog is None else catalog
        return self._gumbel_rows(cat.contiguous())

    def _gumbel_aug_ok(self, k=0):
        if not self.use_st_gumbel or self.L1_flag:
            return False
        return bool(_lib.load().kgrec_gumbel_aug_supported(self.embedding_size, self.pref_embeddings.weight.shape[0], k))

    def _pref_aug_ok(self, k=0):
        """Soft preferences on augmented rows (k_eval_soft); False -> the plain path on user / item ids."""
        if self.use_st_gumbel:
            return False
        return bool(_lib.load().kgrec_pref_aug_supported(self.embedding_size, k))

    def rec_eval_max_topn(self):
        """Largest topn (<= 128) that topk_items / RecEvaluator serve at this model's shape: 0 when only the score
        matrix (evaluate / evaluateRec) can be computed, -1 when not even that."""
        d, P = self.embedding_size, self.pref_embeddings.weight.shape[0]
        if d % 4 or d > self.EVAL_MAX_DIM:
            return -1
        lib = _lib.load()

        def ok(k):
            return self._gumbel_aug_ok(k) or self._pref_aug_ok(k) or bool(lib.kgrec_pref_eval_supported(d, P, int(self.use_st_gumbel), k))
        return max([k for k in range(0, 129) if ok(k)] or [-1])

    def _eval_envelope_warning(self):
        k = self.rec_eval_max_topn()
        if k < 128:
            what = "evaluate / evaluateRec / topk_items raise" if k < 0 else "topk_items / RecEvaluator need topn <= %d" % k
            return ("%s with embedding_size %d and preference_total %d: %s (the rec-side kernel stages both preference "
                    "tables in shared memory; see kgrec_pref_eval_supported)"
                    % (type(self).__name__, self.embedding_size, self.pref_embeddings.weight.shape[0], what))
        return None

    def _rec_call(self, mode, u_ids, gumbel_u, catalog, soft_catalog, **kw):
        dev = self._require_cuda()
        k = kw.get("k", 10) if mode == "topk" else 0
        if self._gumbel_aug_ok(k):
            # ST-Gumbel, squared L2: the tiled distance kernel on augmented rows + a per-pair arg-max epilogue
            u = KF.as_index(u_ids, dev)
            if u.numel() == 0:
                return self._eval(self.MODEL, _lib.SIDE_REC, u, None, mode, catalog=self._rec_catalog(), **kw)
            aug_cat = soft_catalog if soft_catalog is not None else self.gumbel_catalog(catalog)
            qrows = self._gumbel_rows(self.user_embeddings.weight.detach(), ids=u, with_consts=True)
            seed = self._next_seed() if gumbel_u is None else 0
            return self._eval(self.MODEL, _lib.SIDE_REC, None, None, mode, catalog=aug_cat, qvec=qrows, gumbel_u=gumbel_u,
                              seed=seed, **kw)
        if self._pref_aug_ok(k):
            u = KF.as_index(u_ids, dev)
            if u.numel() == 0:
                return self._eval(self.MODEL, _lib.SIDE_REC, u, None, mode, catalog=self._rec_catalog(), **kw)
            aug_cat = soft_catalog if soft_catalog is not None else self.soft_catalog(catalog)
            qrows = self._aug_rows(self.user_embeddings.weight.detach(), True, ids=u)
            return self._eval(self.MODEL, _lib.SIDE_REC, None, None, mode, catalog=aug_cat, qvec=qrows, **kw)
        seed = self._next_seed() if (self.use_st_gumbel and gumbel_u is None) else 0
        cat = self._rec_catalog() if catalog is None else catalog
        return self._eval(self.MODEL, _lib.SIDE_REC, u_ids, None, mode, catalog=cat, gumbel_u=gumbel_u, seed=seed, **kw)

    def _rec_scores(self, u_ids, gumbel_u=None):
        return self._rec_call("scores", u_ids, gumbel_u, None, None)

    def topk_items(self, u_ids, k=10, filter_csr=None, catalog=None, id_base=0, gumbel_u=None, soft_catalog=None):
        """K best items per user as uint64 keys (int64 storage): score bits << 32 | item id.
        catalog: a row shard of the item table (KTUP: of _rec_catalog()); soft_catalog: its
        augmented form from soft_catalog() (soft preferences) or gumbel_catalog() (ST-Gumbel, L2),
        reusable across calls while the tables are unchanged."""
        return self._rec_call("topk", u_ids, gumbel_u, catalog, soft_catalog, id_base=id_base, k=k,
                              filter_csr=filter_csr)

    def _rank_inputs(self, u, catalog, soft_catalog, topn):
        """(user ids or None, query rows or None, catalog rows) of the path topk_items(k=topn) takes, so that the
        rank pass scores a pair exactly as that list does."""
        users = self.user_embeddings.weight.detach()
        if self._gumbel_aug_ok(topn):
            cat = soft_catalog if soft_catalog is not None else self.gumbel_catalog(catalog)
            return None, self._gumbel_rows(users, ids=u, with_consts=True), cat
        if self._pref_aug_ok(topn):
            cat = soft_catalog if soft_catalog is not None else self.soft_catalog(catalog)
            return None, self._aug_rows(users, True, ids=u), cat
        return u, None, (self._rec_catalog() if catalog is None else catalog).contiguous()

    def _rank_call(self, u_ids, gold_csr, filter_csr, catalog, id_base, soft_catalog, gumbel_u, seed, topn, n_gold, gold_scores):
        import ctypes as C
        dev = self._require_cuda()
        lib = _lib.load()
        u = KF.as_index(u_ids, dev)
        gptr, gids = gold_csr
        n_gold = int(gids.numel()) if n_gold is None else int(n_gold)
        if gptr.dtype != torch.int64 or gids.dtype != torch.int32 or gptr.numel() != u.numel() + 1:
            raise ValueError("kgrec_b200: gold_csr is (int64 ptr [n_users + 1], int32 ascending ids)")
        if u.numel() == 0 or n_gold == 0:
            return None, n_gold, dev
        q, qrows, cat = self._rank_inputs(u, catalog, soft_catalog, topn)
        if gumbel_u is not None:
            gumbel_u = gumbel_u.to(dev, torch.float32).contiguous()
        if seed is None:
            seed = self._next_seed() if (self.use_st_gumbel and gumbel_u is None) else 0
        T = KF.make_tables(self._weights(), self.embedding_size, self.L1_flag, self.use_st_gumbel, self._item2ent)
        head = (C.byref(T), self.MODEL, KF._ptr(q), q.element_size() if q is not None else 8, KF._ptr(qrows), u.numel(),
                KF._ptr(cat), cat.stride(0), cat.shape[0], id_base, KF._ptr(gptr), KF._ptr(gids))
        if gold_scores is None:
            gold_scores = torch.zeros(n_gold, dtype=torch.float32, device=dev)
            _lib.check(lib.kgrec_rec_gold_scores(*head, KF._ptr(gumbel_u), seed, KF._ptr(gold_scores), KF._stream()))
            KF.count_launches(1)
        return (lib, head, gumbel_u, seed, gold_scores, (q, qrows, cat)), n_gold, dev     # head holds raw pointers into the last

    def gold_scores_items(self, u_ids, gold_csr, catalog=None, id_base=0, soft_catalog=None, gumbel_u=None, seed=0, topn=0,
                          n_gold=None):
        """float32 [n_gold]: score(user, gold) of every gold of gold_csr that lies in the catalog shard, 0 elsewhere,
        computed by the sweep rank_counts_items compares against.  Arrays of different shards add (one all-reduce);
        pass the sum as rank_counts_items(gold_scores=...) on every shard, with the same user list and seed."""
        call, n_gold, dev = self._rank_call(u_ids, gold_csr, None, catalog, id_base, soft_catalog, gumbel_u, seed, topn, n_gold, None)
        return call[4] if call else torch.zeros(n_gold, dtype=torch.float32, device=dev)

    def rank_counts_items(self, u_ids, gold_csr, filter_csr=None, catalog=None, id_base=0, soft_catalog=None, gumbel_u=None,
                          seed=None, gold_scores=None, topn=0, n_gold=None):
        """int32 [n_gold]: for every gold item of every user (gold_csr = (int64 ptr [n_users + 1], int32 ascending
        ids)), the number of catalog items ranked before it in the (score, id) order of topk_items, leaving out the
        user's filter row (filter_csr, as topk_items takes it) and the user's other golds; -1 for a gold that is itself
        filtered (kgrec_rec_rank_count).  One query per user: with hashed ST-Gumbel noise the scores are those
        topk_items sees for the same user list and seed.  topn selects the path topk_items(k=topn) takes.
        catalog / id_base / soft_catalog: a shard, as in topk_items; per-shard counts add (sharded_rank_counts; a
        skipped gold is then negative) once gold_scores holds the summed gold_scores_items of all shards."""
        call, n_gold, dev = self._rank_call(u_ids, gold_csr, filter_csr, catalog, id_base, soft_catalog, gumbel_u, seed, topn,
                                            n_gold, gold_scores)
        counts = torch.zeros(n_gold, dtype=torch.int32, device=dev)
        if call:
            lib, head, gumbel_u, seed, gs, _alive = call
            fptr, fids = filter_csr if filter_csr is not None else (None, None)
            ws = torch.empty(int(lib.kgrec_rec_rank_workspace_bytes(head[5], n_gold)) // 8 + 1, dtype=torch.int64, device=dev)
            _lib.check(lib.kgrec_rec_rank_count(*head, n_gold, KF._ptr(gs.contiguous().float()), KF._ptr(fptr), KF._ptr(fids),
                                                KF._ptr(gumbel_u), seed, KF._ptr(counts), KF._ptr(ws), ws.numel() * 8, KF._stream()))
            KF.count_launches(3)      # gold sort, catalog sweep, prefix sums
        return counts

    def rank_loss(self, pos, neg, target=-1.0, loss="bpr", batch_pos=None, gumbel_u=None):
        """Fused pos + K negatives + ranking loss: pos = (u, i), neg = (u repeated, ni)."""
        pos = (pos[0], pos[1], None)
        neg = (neg[0], neg[1], None)
        return self._rank_loss(self.MODEL, pos, neg, loss, target, batch_pos, gumbel_u)

    def loss_step(self, pos, neg, target=-1.0, loss="bpr", batch_pos=None, gumbel_u=None):
        """rank_loss(...) followed by loss.sum().backward(), as one kernel pass: returns
        (loss[batches], pos_scores, neg_scores) and leaves the gradients in .grad."""
        return self._loss_step(self.MODEL, (pos[0], pos[1], None), (neg[0], neg[1], None), loss, target, batch_pos,
                               gumbel_u)

    def _mix_tables(self):
        """(P, N, half): the preference tables the mixing uses."""
        return self.pref_embeddings.weight, self.pref_norm_embeddings.weight, 1.0

    def _pair_vectors(self, u_id, i_ids):
        dev = self._require_cuda()
        i_ids = KF.as_index(i_ids, dev).long()
        u = self.user_embeddings.weight[KF.as_index(u_id, dev).long().view(-1)[:1]].expand(i_ids.numel(), -1)
        return u, self.item_embeddings.weight[i_ids]

    def reportPreference(self, u_id, i_ids):
        """(pre_probs, r_e, norm) for logging (-is_report; item_recommendation.py:68).
        A diagnostics path, not the hot path: a handful of rows through library ops."""
        u_e, i_e = self._pair_vectors(u_id, i_ids)
        P, N, hf = self._mix_tables()
        with torch.no_grad():
            probs = (u_e + i_e) @ P.t() / 2
            if self.use_st_gumbel:
                g = -torch.log(-torch.log(torch.rand_like(probs) + 1e-20) + 1e-20)
                probs = torch.nn.functional.one_hot((probs + g).argmax(-1), probs.shape[-1]).float()
            return probs, probs @ P * hf, probs @ N * hf


class TransUPModel(RecModelBase):
    MODEL = _lib.TUP
    TABLES = {"user": "user_embeddings", "item": "item_embeddings",
              "pref": "pref_embeddings", "pref_norm": "pref_norm_embeddings"}

    def __init__(self, L1_flag, embedding_size, user_total, item_total, preference_total, use_st_gumbel):
        super().__init__()
        self.L1_flag = L1_flag
        self.embedding_size = embedding_size
        self.user_total = user_total
        self.item_total = item_total
        self.preference_total = preference_total
        self.use_st_gumbel = use_st_gumbel
        d = embedding_size
        _make_tables(self, [("user_embeddings", user_total, d, True), ("item_embeddings", item_total, d, True),
                            ("pref_embeddings", preference_total, d, True),
                            ("pref_norm_embeddings", preference_total, d, True)])
        self._finish_init()

    def forward(self, u_ids, i_ids, gumbel_u=None):
        """score[b] of the pairs (u_ids[b], i_ids[b]).  gumbel_u: optional [B, P] uniform draws
        replacing the in-kernel generator (parity runs)."""
        return self._score(self.MODEL, u_ids, i_ids, None, gumbel_u)

    def evaluate(self, u_ids, gumbel_u=None):
        """[B, item_total] scores of every (user, item) pair; gumbel_u optional [B, I, P]."""
        return self._rec_scores(u_ids, gumbel_u)
