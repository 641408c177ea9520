"""Sparse-row training step: fused forward + loss + backward into persistent accumulators, then
a clip + optimizer update of exactly the rows the batch touched (SURVEY 8f, next row 1).

Replaces the reference's `trainer.optimizer_zero_grad(); losses.backward(); clip_grad_norm;
trainer.optimizer_step()` sequence (knowledge_representation.py:187-216, item_recommendation.py:
168-192, knowledgable_recommendation.py:320-402, utils/trainer.py:63-81), whose cost is O(table)
per step, with one whose cost is O(batch):

    step kernel (dense-accumulate gradients)      kgrec_corrupt_loss_step / kgrec_rank_loss_step
    [regularisers of the driver]                  fused (KG side) / kgrec_reg_* (rec side)
    epoch marks from the batch's id arrays        kgrec_rows_mark        1 launch
    clip_grad_norm's total norm                   kgrec_rows_sqnorm      1 launch, all tables
    SGD / Adagrad / Adam on the marked rows       kgrec_rows_update      1 launch, all tables

Update rules are torch.optim's SGD / Adagrad / Adam formulas; Adam is applied to the touched rows
only ("lazy"), which differs from dense Adam on untouched rows (SURVEY 7.3-3).  A table takes
part in a step when the step's loss reaches it -- as in the reference, where parameters whose
``.grad`` is None are skipped (KTUP: the rec branch moves user / item / aligned entities / pref /
pref_norm / rel / norm, the KG branch ent / rel / norm).

Exact trajectories (rows="all", kgrec_rows_update_ex): the reference's trainer steps a dense torch.optim optimizer over
nn.Embedding tables with dense gradients, so every row of every table the loss reaches moves on every step -- Adam
through m / v, SGD / RMSprop through their momentum buffers, any rule through weight decay -- including rows the batch
did not touch.  rows="all" does the same, at O(table) per step as the reference does; rows="touched" (the default)
stays the fast O(batch) mode that is not the reference's trajectory.  Also there: SGD with momentum, RMSprop (the
reference's "Rmsprop"), Adam's step count per table (torch keeps one per parameter), and reset(), the trainer's
optimizer_reset.  "A table takes part" is torch >= 2's zero_grad(set_to_none=True) rule above.  The reference was written
for torch 0.3, whose zero_grad zeroed gradients in place: there KTUP's rec tables, once they have a gradient, also take
part in KG steps (weight decay and Adam's m / v keep moving them).  That variant is not built.
"""
import ctypes as C

import torch

from . import _lib
from . import functional as KF

_KINDS = {"SGD": 0, "Adagrad": 1, "Adam": 2, "Rmsprop": 3, "RMSprop": 3}
_ROWS = {"touched": _lib.ROWS_TOUCHED, "all": _lib.ROWS_ALL}
# utils/trainer.py:63-78: the reference's -optimizer_type values; momentum = FLAGS.momentum for SGD and Rmsprop only
_FLAG_TYPES = ("Adam", "SGD", "Adagrad", "Rmsprop")
_ATTR = {"ent": "ent_embeddings", "rel": "rel_embeddings", "norm": "norm_embeddings", "proj": "proj_embeddings",
         "user": "user_embeddings", "item": "item_embeddings", "pref": "pref_embeddings",
         "pref_norm": "pref_norm_embeddings"}
# tables whose rows are gathered by id (the others are small and every row takes part)
_GATHERED = ("ent", "rel", "norm", "user", "item")


def flags_kwargs(FLAGS):
    """SparseRowOptimizer's keyword arguments for the reference's flags (see SparseRowOptimizer.from_flags)."""
    t = FLAGS.optimizer_type
    if t not in _FLAG_TYPES:
        raise ValueError("optimizer_type must be one of %s" % (_FLAG_TYPES,))
    momentum = float(FLAGS.momentum) if t in ("SGD", "Rmsprop") else 0.0
    return dict(optimizer_type=t, lr=float(FLAGS.learning_rate), l2_lambda=float(FLAGS.l2_lambda),
                clip=float(FLAGS.clipping_max_value), momentum=momentum, rows="all")


class SparseRowOptimizer:
    def __init__(self, model, optimizer_type="Adagrad", lr=0.01, l2_lambda=0.0, clip=None,
                 eps=None, betas=(0.9, 0.999), momentum=0.0, alpha=0.99, rows="touched"):
        """rows: "touched" updates the rows the batch touched (O(batch)); "all" updates every row of the tables the
        step's loss reaches, as torch.optim's dense step does (O(table)).  momentum: SGD and RMSprop.  alpha: RMSprop.
        Any setting other than the defaults runs through kgrec_rows_update_ex."""
        if optimizer_type not in _KINDS:
            raise ValueError("optimizer_type must be one of %s" % sorted(_KINDS))
        if rows not in _ROWS:
            raise ValueError("rows must be one of %s" % sorted(_ROWS))
        self.model, self.kind, self.lr, self.wd, self.clip = model, _KINDS[optimizer_type], lr, l2_lambda, clip
        self.momentum, self.alpha, self.rows = float(momentum), float(alpha), rows
        if self.momentum < 0.0 or (self.momentum and self.kind in (1, 2)):
            raise ValueError("momentum: >= 0, and for SGD and RMSprop only")
        self.eps = eps if eps is not None else (1e-10 if self.kind == 1 else 1e-8)
        self.betas = betas
        # the defaults run kgrec_rows_update as before; everything else kgrec_rows_update_ex
        self.exact = rows != "touched" or self.momentum != 0.0 or self.kind == 3
        self.t = 0
        dev = model._require_cuda()
        self.names = KF.MODEL_TABLES[model.MODEL]
        w = model._weights()
        self.acc = {k: torch.zeros_like(w[k]) for k in self.names}
        ktup = model.MODEL == _lib.KTUP
        self.marks = {k: torch.zeros(w[k].shape[0], dtype=torch.int32, device=dev)
                      for k in self.names if k in _GATHERED and not (ktup and k in ("rel", "norm"))}
        use_s1 = self.kind != 0 or self.momentum != 0.0         # Adagrad sum, Adam m, RMSprop square_avg, SGD's buffer
        use_s2 = self.kind == 2 or (self.kind == 3 and self.momentum != 0.0)      # Adam v, RMSprop's momentum buffer
        self.s1 = {k: torch.zeros_like(w[k]) if use_s1 else None for k in self.names}
        self.s2 = {k: torch.zeros_like(w[k]) if use_s2 else None for k in self.names}
        # Adam's step count per table (torch keeps one per parameter and advances it only when the parameter has a
        # gradient): slot i belongs to self.names[i]
        self.steps = torch.zeros(len(self.names), dtype=torch.int64, device=dev) if self.exact and self.kind == 2 else None
        self.sqnorm = torch.zeros(1, dtype=torch.float32, device=dev)
        self.reg_loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self._rows_ws = None          # work buffers of the row-factored soft rec step, allocated on first use

    @classmethod
    def from_flags(cls, model, FLAGS):
        """What the reference's ModelTrainer.optimizer_reset builds (utils/trainer.py:63-78) from -optimizer_type,
        -learning_rate, -l2_lambda and -momentum, with the drivers' clip_grad_norm at -clipping_max_value, as an exact
        (rows="all") optimizer: momentum for SGD and Rmsprop only, torch's default eps / betas / alpha."""
        return cls(model, **flags_kwargs(FLAGS))

    def reset(self, lr):
        """The trainer's optimizer_reset (utils/trainer.py:98-102, learning-rate decay): a fresh optimizer at `lr` --
        the rule's state and Adam's step counts are zeroed in place on the current stream (nothing is reallocated, so
        captured graphs stay valid)."""
        if self.kind == 2 and self.steps is None:
            raise ValueError("reset: Adam restarts its step count only with per-table step counts (rows='all')")
        for v in list(self.s1.values()) + list(self.s2.values()):
            if v is not None:
                v.zero_()
        if self.steps is not None:
            self.steps.zero_()
        self.lr = float(lr)

    # -- shared tail of every step: marks -> total norm -> update --------------------------------------
    def _seg(self, ids, table, compact=False, remap=None):
        m = self.marks[table]
        return _lib.MarkSeg(ids=ids.data_ptr(), n=ids.numel(), idx_bytes=ids.element_size(), compact=int(compact),
                            remap=remap.data_ptr() if remap is not None else None,
                            n_remap=remap.numel() if remap is not None else 0,
                            marks=m.data_ptr(), rows=m.numel())

    def _mark(self, segs, state=None):
        """Start a step: bump the epoch and mark the rows the step's id arrays name.  state: the epoch is the device
        step state's (which the caller has advanced for this step); self.t still counts the step."""
        m = self.model
        self.t += 1
        seg_arr = (_lib.MarkSeg * len(segs))(*segs)
        status = KF._ptr(m._status_buf(m.device))
        if state is None:
            _lib.check(_lib.load().kgrec_rows_mark(seg_arr, len(segs), self.t, status, KF._stream()))
        else:
            _lib.check(_lib.load().kgrec_rows_mark_dev(seg_arr, len(segs), state.ptr, status, KF._stream()))
        KF.count_launches(1)

    def _update(self, tables, state=None):
        """Finish a step: total norm (clip) and the optimizer update of the marked rows of `tables`."""
        m = self.model
        lib = _lib.load()
        stream = KF._stream()
        w = m._weights()
        entries = []
        for k in tables:
            mk = self.marks.get(k)
            entries.append(_lib.OptTable(
                table=w[k].data.data_ptr(), acc=self.acc[k].data_ptr(),
                state1=self.s1[k].data_ptr() if self.s1[k] is not None else None,
                state2=self.s2[k].data_ptr() if self.s2[k] is not None else None,
                marks=mk.data_ptr() if mk is not None else None, rows=w[k].shape[0], dim=w[k].shape[1], keep_acc=0))
        tab_arr = (_lib.OptTable * len(entries))(*entries)
        use_clip = self.clip is not None
        if use_clip:
            self.sqnorm.zero_()
            if state is None:
                _lib.check(lib.kgrec_rows_sqnorm(tab_arr, len(entries), self.t, KF._ptr(self.sqnorm), stream))
            else:
                _lib.check(lib.kgrec_rows_sqnorm_dev(tab_arr, len(entries), state.ptr, KF._ptr(self.sqnorm), stream))
        sq = KF._ptr(self.sqnorm) if use_clip else None
        if self.exact:
            self._update_ex(tables, tab_arr, len(entries), sq, state)
            KF.count_launches(1 + int(use_clip) + int(self.steps is not None))
            return
        if state is None:
            _lib.check(lib.kgrec_rows_update(tab_arr, len(entries), self.t, self.kind, self.lr, self.eps, self.betas[0],
                                             self.betas[1], self.t, self.wd, sq, float(self.clip or 0.0), stream))
        else:      # epoch, lr and Adam's step from the device step state
            _lib.check(lib.kgrec_rows_update_dev(tab_arr, len(entries), state.ptr, self.kind, self.eps, self.betas[0],
                                                 self.betas[1], self.wd, sq, float(self.clip or 0.0), stream))
        KF.count_launches(1 + int(use_clip))

    def _update_ex(self, tables, tab_arr, n, sq, state):
        steps = None
        if self.steps is not None:          # the call's tables are a run of self.names: its counters are a slice
            i = self.names.index(tables[0])
            if tuple(self.names[i:i + n]) != tuple(tables):
                raise AssertionError("tables of one update must be a run of the optimizer's tables")
            steps = self.steps.data_ptr() + 8 * i
        P = _lib.OptParams(kind=self.kind, rows=_ROWS[self.rows], lr=self.lr, eps=self.eps, beta1=self.betas[0],
                           beta2=self.betas[1], alpha=self.alpha, momentum=self.momentum, weight_decay=self.wd,
                           max_norm=float(self.clip or 0.0), step_counts=steps)
        lib = _lib.load()
        if state is None:
            _lib.check(lib.kgrec_rows_update_ex(tab_arr, n, self.t, C.byref(P), sq, KF._stream()))
        else:               # epoch and lr from the device step state
            _lib.check(lib.kgrec_rows_update_ex_dev(tab_arr, n, state.ptr, C.byref(P), sq, KF._stream()))

    def _apply(self, segs, tables, state=None):
        """segs: MarkSeg list of this step's id arrays; tables: names of the tables the step's loss reaches."""
        self._mark(segs, state)
        self._update(tables, state)

    def _grads(self, names):
        g = _lib.Grads()
        g.mode = 1
        for k in names:
            setattr(g, k, self.acc[k].data_ptr())
        return g

    # -- KG models: TransE / TransH / TransR, and the KG branch of KTUP ---------------------------------
    def step_corrupt(self, pos, corrupt, margin=1.0, loss="margin", batch_pos=None, reg=False, grad_loss=1.0, state=None):
        """One training step on positives (h, t, r) and group-compact negatives; returns the
        per-batch losses (device tensor; nothing synchronises).  reg=True adds the KG drivers'
        normLoss / orthogonalLoss regularisers inside the same kernel (kgrec_corrupt_loss_step), for
        TransE / TransH / TransR alike (TransR: normLoss of the raw ent / rel rows; proj has none).
        KTUP: the joint model's KG branch (TransH on ent / rel / norm), grad_loss = kg_lambda.
        state (kgrec_b200.train.StepState, advanced for this step): the optimizer reads its epoch mark, learning rate
        and step count on the device (the `_dev` entry points) -- the step a GraphedTrainLoop captures."""
        m = self.model
        if m.MODEL not in (_lib.TRANSE, _lib.TRANSH, _lib.TRANSR, _lib.KTUP):
            raise NotImplementedError("step_corrupt: KG models and the KG branch of KTUP")
        kmodel = _lib.TRANSH if m.MODEL == _lib.KTUP else m.MODEL
        names = KF.MODEL_TABLES[kmodel]
        dev = m._require_cuda()
        pos = tuple(KF.as_index(x, dev) for x in pos)
        idx_bytes = KF._idx_bytes(*pos)
        corrupt = corrupt.to(dev, torch.int32, non_blocking=True).contiguous().view(-1)
        n_pos = pos[0].numel()
        bp = batch_pos or max(1, n_pos)
        out = torch.zeros((n_pos + bp - 1) // bp if n_pos else 0, dtype=torch.float32, device=dev)
        if n_pos == 0:
            return out
        if corrupt.numel() % n_pos:
            raise ValueError("corrupt ids must be a whole multiple of the positives")
        n_neg = corrupt.numel() // n_pos
        w = m._weights()
        lib = _lib.load()
        ptr = KF._ptr
        T = KF.make_tables({k: w[k] for k in names}, m.embedding_size, m.L1_flag)
        g = self._grads(names)
        pos_s = torch.empty(n_pos, dtype=torch.float32, device=dev)
        neg_s = torch.empty(n_pos * n_neg, dtype=torch.float32, device=dev)
        ws = torch.empty(lib.kgrec_corrupt_loss_step_workspace_bytes(C.byref(T), kmodel, n_pos) // 4, dtype=torch.float32, device=dev)
        kind = {"margin": _lib.LOSS_MARGIN, "bpr": _lib.LOSS_BPR}[loss]
        _lib.check(lib.kgrec_corrupt_loss_step(
            C.byref(T), kmodel, ptr(pos[0]), ptr(pos[1]), ptr(pos[2]), idx_bytes, n_pos, ptr(corrupt),
            n_neg, bp, kind, float(margin), float(grad_loss), 1 if reg else 0, ptr(pos_s), ptr(neg_s), ptr(out),
            C.byref(g), None, None, ptr(ws), ptr(m._status_buf(dev)), KF._stream()))
        KF.count_launches(2)
        segs = [self._seg(pos[0], "ent"), self._seg(pos[1], "ent"), self._seg(corrupt, "ent", compact=True)]
        segs += [self._seg(pos[2], k) for k in ("rel", "norm") if k in names and k in self.marks]   # KTUP: small tables, all rows
        self._apply(segs, names, state)
        return out

    # -- recommendation models: TUP, and the rec branch of KTUP -----------------------------------------------
    def step_pairs(self, pos, neg, target=-1.0, loss="bpr", batch_pos=None, gumbel_u=None, reg=False, state=None):
        """One training step on (u, i) positives and (u repeated, ni) negatives: forward + ranking
        loss + backward in the tile kernel (kgrec_rank_loss_step), then clip + update.  reg=True adds
        the driver's regularisers: TUP (item_recommendation.py:177-180) orthogonalLoss(pref, pref_norm) +
        normLoss(user rows) + normLoss(item rows of cat[pos, neg]) + normLoss(pref); KTUP rec branch
        (knowledgable_recommendation.py:343-344) orthogonalLoss(pref, pref_norm).
        Returns (loss per batch, regulariser value) as device tensors.
        state: as step_corrupt; the Gumbel seed is then state.gumbel_seed + state.step, read on the device, instead of
        the model's next seed."""
        m = self.model
        if m.MODEL not in (_lib.TUP, _lib.KTUP):
            raise NotImplementedError("step_pairs: TUP / KTUP")
        dev = m._require_cuda()
        pu, pi = (KF.as_index(x, dev) for x in pos)
        nu, ni = (KF.as_index(x, dev) for x in neg)
        idx_bytes = KF._idx_bytes(pu, pi, nu, ni)
        n_pos = pu.numel()
        bp = batch_pos or max(1, n_pos)
        out = torch.zeros((n_pos + bp - 1) // bp if n_pos else 0, dtype=torch.float32, device=dev)
        self.reg_loss.zero_()
        if n_pos == 0:
            return out, self.reg_loss
        if ni.numel() % n_pos:
            raise ValueError("negatives must be a whole multiple of the positives")
        n_neg = ni.numel() // n_pos
        names = self.names
        w = m._weights()
        lib = _lib.load()
        ptr = KF._ptr
        stream = KF._stream()
        T = KF.make_tables({k: w[k] for k in names}, m.embedding_size, m.L1_flag, m.use_st_gumbel, m._item2ent)
        ktup = m.MODEL == _lib.KTUP
        g = self._grads([k for k in names if not (ktup and k in ("rel", "norm"))])   # KTUP: rel / norm share pref / pref_norm's
        pos_s = torch.empty(n_pos, dtype=torch.float32, device=dev)
        neg_s = torch.empty(n_pos * n_neg, dtype=torch.float32, device=dev)
        ws = torch.empty(max(1, n_pos), dtype=torch.float32, device=dev)
        kind = {"margin": _lib.LOSS_MARGIN, "bpr": _lib.LOSS_BPR}[loss]
        if gumbel_u is not None:
            gumbel_u = gumbel_u.to(dev, torch.float32).contiguous()
        seed = m._next_seed() if (m.use_st_gumbel and gumbel_u is None and state is None) else 0
        segs = [self._seg(pu, "user"), self._seg(pi, "item"), self._seg(ni, "item")]
        if ktup:
            segs += [self._seg(pi, "ent", remap=m._item2ent), self._seg(ni, "ent", remap=m._item2ent)]
        self._mark(segs, state)
        rows_path = self._use_rows_path(n_pos, n_neg, nu, pu)
        if rows_path:
            # soft preferences: the [P x d] contractions once per distinct row of the step (csrc/train_rec_rows.cu)
            if self._rows_ws is None:
                n_fl = lib.kgrec_rec_rows_workspace_floats(w["user"].shape[0], w["item"].shape[0], m.embedding_size,
                                                           w["pref"].shape[0], 1 if ktup else 0)
                # device-state steps start from a zeroed workspace instead of first_use: a captured first_use would
                # clear the accumulators again on every replay
                self._rows_ws = (torch.empty if state is None else torch.zeros)(int(n_fl), dtype=torch.float32, device=dev)
                first = int(state is None)
            else:
                first = 0
            head = (C.byref(T), m.MODEL, ptr(pu), ptr(pi), ptr(ni), idx_bytes, n_pos, n_neg, bp, kind, float(target), 1.0,
                    ptr(self.marks["user"]), ptr(self.marks["item"]))
            tail = (ptr(self._rows_ws), first, C.byref(g), ptr(pos_s), ptr(neg_s), ptr(out), ptr(ws),
                    ptr(self.reg_loss) if (reg and not ktup) else None, ptr(gumbel_u))
            if state is None:
                _lib.check(lib.kgrec_rec_rows_step(*head, self.t, *tail, seed, ptr(m._status_buf(dev)), stream))
            else:
                _lib.check(lib.kgrec_rec_rows_step_dev(*head, state.ptr, *tail, ptr(m._status_buf(dev)), stream))
            KF.count_launches(8)
        else:
            head = (C.byref(T), m.MODEL, ptr(pu), ptr(pi), None, ptr(nu), ptr(ni), None, idx_bytes, n_pos, n_neg, bp, kind,
                    float(target), 1.0, ptr(gumbel_u))
            tail = (ptr(pos_s), ptr(neg_s), ptr(out), C.byref(g), None, None, None, ptr(ws), ptr(m._status_buf(dev)), stream)
            if state is None:
                _lib.check(lib.kgrec_rank_loss_step(*head, seed, *tail))
            else:
                _lib.check(lib.kgrec_rank_loss_step_dev(*head, state.ptr, *tail))
            KF.count_launches(2)
        if ktup:      # (pref + rel) and (pref_norm + norm) enter the score as sums (jTransUP.py:253-258): equal gradients
            self.acc["rel"].copy_(self.acc["pref"])
            self.acc["norm"].copy_(self.acc["pref_norm"])
        if reg:
            d = m.embedding_size
            pw, nw = w["pref"], w["pref_norm"]
            _lib.check(lib.kgrec_reg_orth_tables(ptr(pw), ptr(nw), pw.shape[0], d, 1.0, ptr(self.reg_loss),
                                                 ptr(self.acc["pref"]), ptr(self.acc["pref_norm"]), stream))
            KF.count_launches(1)
            if not ktup:
                status = ptr(m._status_buf(dev))
                fused = rows_path                                  # rows path: normLoss of the gathered rows is fused into its pair kernel
                for tab, ids in (() if fused else (("user", pu), ("item", pi), ("item", ni))):
                    _lib.check(lib.kgrec_reg_norm_rows(ptr(w[tab]), w[tab].shape[0], d, ptr(ids), ids.element_size(),
                                                       ids.numel(), 1.0, ptr(self.reg_loss), ptr(self.acc[tab]), status, stream))
                _lib.check(lib.kgrec_reg_norm_rows(ptr(pw), pw.shape[0], d, None, 8, pw.shape[0], 1.0, ptr(self.reg_loss),
                                                   ptr(self.acc["pref"]), None, stream))
                KF.count_launches(4)
        self._update(names, state)
        return out, self.reg_loss

    def _use_rows_path(self, n_pos, n_neg, nu, pu):
        """Row-factored step (train_rec_rows.cu) when the step re-uses rows enough: its per-row kernels cost more than
        a pair of the pair kernel per DISTINCT row, its pair stage less.  KGREC_REC_ROWS=0 | force overrides."""
        import os
        m = self.model
        env = os.environ.get("KGREC_REC_ROWS", "")
        d, P = m.embedding_size, m.pref_embeddings.weight.shape[0]
        ok = d % 4 == 0 and d <= 128 and P <= 32 and 1 <= n_neg <= 31 and not (m.use_st_gumbel and m.L1_flag)
        if not ok or env == "0":
            return False
        # the row path scores negative k of positive j as (pu[j], ni[j, k]): the (u repeated, ni) contract of this
        # method (what getNegRatings produces); nu itself is not read
        if env == "force":
            return True
        pairs = n_pos * (1 + n_neg)
        rows = min(m.user_embeddings.weight.shape[0], n_pos) + min(m.item_embeddings.weight.shape[0], pairs)
        # crossover measured on an H100 (TUP d=100 P=20, 262144 positives + 1 negative, full optimizer step): soft
        # rows / pairs 0.095 -> 1.35 vs 1.39 ms, 0.19 -> 1.79 vs 1.54; ST-Gumbel 0.29 -> 1.50 vs 1.78, 0.38 -> 1.72 vs 1.77
        return rows <= (0.35 if m.use_st_gumbel else 0.1) * pairs
