"""TransE on the CUDA engine.  Mirrors jTransUP/models/transE.py (constructor 18-49,
forward 51-63, evaluateHead/Tail 65-105) with every method one kernel call."""
from .. import _lib
from .. import functional as KF
from .base import KGRecModule, _make_tables


def build_model(FLAGS, user_total, item_total, entity_total, relation_total, i_map=None, e_map=None, new_map=None):
    """Same dispatch hook as the reference (transE.py:8-15, called from base.py:165-166)."""
    return TransEModel(L1_flag=FLAGS.L1_flag, embedding_size=FLAGS.embedding_size,
                       ent_total=entity_total, rel_total=relation_total)


class KGModelBase(KGRecModule):
    """What TransE / TransH / TransR share: (h, t, r) scoring and entity-catalog evaluation."""

    TABLES = {"ent": "ent_embeddings", "rel": "rel_embeddings"}

    def __init__(self, L1_flag, embedding_size, ent_total, rel_total):
        super().__init__()
        self.L1_flag = L1_flag
        self.embedding_size = embedding_size
        self.ent_total = ent_total
        self.rel_total = rel_total
        _make_tables(self, self._table_specs())

    def _table_specs(self):
        d = self.embedding_size
        return [("ent_embeddings", self.ent_total, d, True), ("rel_embeddings", self.rel_total, d, True)]

    def forward(self, h, t, r):
        """score[b] of the triples (h[b], r[b], t[b]); argument order as the reference."""
        return self._score(self.MODEL, h, t, r)

    def rank_loss(self, pos, neg, margin=1.0, loss="margin", batch_pos=None):
        """Fused pos + K negatives + ranking loss: pos = (h, t, r), neg = (nh, nt, nr) with
        K * len(h) entries (negatives of positive j at [j*K, (j+1)*K)).
        Returns (loss per batch [n_batches], pos_scores, neg_scores)."""
        return self._rank_loss(self.MODEL, pos, neg, loss, margin, batch_pos)

    def rank_loss_corrupt(self, pos, corrupt, margin=1.0, loss="margin", batch_pos=None):
        """rank_loss with the negatives in the group-compact format: corrupt[j*K + k] >= 0 replaces
        the tail of positive j by that entity, < 0 replaces the head by ~corrupt (what the
        reference's corrupt_head/tail sampler draws; functional.encode_corrupt converts).
        Reads and writes (3 + K) rows per group instead of 3 (1 + K).  TransE / TransH."""
        return self._rank_loss_corrupt(self.MODEL, pos, corrupt, loss, margin, batch_pos)

    def loss_step_corrupt(self, pos, corrupt, margin=1.0, loss="margin", batch_pos=None, grad_loss=1.0, reg=False):
        """rank_loss_corrupt(...) followed by (grad_loss * loss.sum()).backward(), in ONE kernel:
        returns (loss per batch, pos_scores, neg_scores) and leaves the gradients in .grad
        (accumulating like autograd does).  Use when nothing else feeds the ranking-loss term's
        upstream -- the case in all the reference drivers, which call backward() on the loss.
        reg=True: the loss of knowledge_representation.py:189-204 in full -- the ranking loss plus
        normLoss over the gathered entity / relation rows (and orthogonalLoss for TransH) -- values
        and gradients from the same kernel pass.  For TransR the norms are those of the raw ent / rel
        rows, not the projected ones, and proj has no regulariser, as in the reference."""
        return self._loss_step_corrupt(self.MODEL, pos, corrupt, loss, margin, batch_pos, grad_loss, reg)

    def graphed_loss_step(self, n_pos, n_neg, margin=1.0, loss="margin", batch_pos=None, grad_loss=1.0, reg=False):
        """loss_step_corrupt for a fixed batch shape as a CUDA graph over static id buffers (the single-batch
        latency path): fill `.h / .t / .r / .corrupt` of the returned object, call `.replay()`."""
        return KF.GraphedCorruptStep(self, n_pos, n_neg, margin, loss, batch_pos, grad_loss, reg)

    # -- evaluation: [B, ent_total] matrices for the unchanged drivers ---------------------
    def _catalog(self):
        return self.ent_embeddings.weight.detach()

    def evaluateHead(self, t, r, all_e_ids=None):
        return self._eval(self.MODEL, _lib.SIDE_HEAD, t, r, "scores", catalog=self._catalog())

    def evaluateTail(self, h, r, all_e_ids=None):
        return self._eval(self.MODEL, _lib.SIDE_TAIL, h, r, "scores", catalog=self._catalog())

    # -- on-chip reductions of the same scores (extensions) ---------------------------------
    def topk(self, side, q, r, k=10, filter_csr=None, catalog=None, id_base=0):
        """K best entities per query as uint64 keys (int64 storage): score bits << 32 | id."""
        s = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
        cat = self._catalog() if catalog is None else catalog
        return self._eval(self.MODEL, s, q, r, "topk", catalog=cat, id_base=id_base, k=k, filter_csr=filter_csr)

    def rank_counts(self, side, q, r, gold_ids, gold_scores=None, catalog=None, id_base=0, out=None):
        """#entities ranked strictly before each query's gold id ((score, id) order)."""
        s = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
        cat = self._catalog() if catalog is None else catalog
        if gold_scores is None:
            gold_scores = self.gold_scores(side, q, r, gold_ids)
        return self._eval(self.MODEL, s, q, r, "rank", catalog=cat, id_base=id_base,
                          gold_scores=gold_scores, gold_ids=gold_ids, out=out)

    def gold_scores(self, side, q, r, gold_ids):
        """Scores of (query, gold) pairs computed by the evaluation kernel itself, so that they
        compare bit-exactly with the catalog scores in rank_counts."""
        import torch
        from .. import functional as KF
        dev = self._require_cuda()
        g = KF.as_index(gold_ids, dev).long()
        s = _lib.SIDE_HEAD if side == "head" else _lib.SIDE_TAIL
        rows = self._catalog()[g].contiguous()                 # [nq, d] gathered gold rows
        # score each query against its own gold row: diagonal of a [nq, nq] evaluation, done
        # in chunks so the temporary stays small
        out = torch.empty(g.numel(), dtype=torch.float32, device=dev)
        q, r = KF.as_index(q, dev), KF.as_index(r, dev)
        for lo in range(0, g.numel(), 512):
            hi = min(g.numel(), lo + 512)
            m = self._eval(self.MODEL, s, q[lo:hi], r[lo:hi], "scores", catalog=rows[lo:hi], cat_ids=g[lo:hi])
            out[lo:hi] = m.diagonal()
        return out


class TransEModel(KGModelBase):
    MODEL = _lib.TRANSE

    def __init__(self, L1_flag, embedding_size, ent_total, rel_total):
        super().__init__(L1_flag, embedding_size, ent_total, rel_total)
        self._finish_init()
