"""Shared machinery of the drop-in model classes.

The five classes in this package keep the constructors, attribute modules,
method names and ``state_dict`` keys of the reference classes
(jTransUP/models/{transE,transH,transR,transUP,jTransUP}.py; SURVEY.md 8b) so the
reference's drivers can call them unchanged, but every method body is one call
into the CUDA library: there are no torch ops on the scoring path.

Extensions over the reference (all optional, defaults reproduce the reference):
  * ``grad_mode``  'dense' (default: ``param.grad`` exactly as the reference's
    autograd lays it out, works with the unchanged ModelTrainer) or 'sparse'
    (row gradients as uncoalesced sparse COO tensors, no O(table) work);
  * ``rank_loss`` the fused positive + K-negative + margin/BPR loss;
  * ``topk`` / ``rank_counts`` on-chip reductions of the evaluate* matrices;
  * explicit Gumbel noise (``gumbel_u=``) for bit-reproducible parity runs.
"""
import contextlib
import math
import os

import torch
import torch.nn as nn

from .. import _lib
from .. import functional as KF
from .. import evaluation as KE


def _init_table(rows, dim, normalize=True):
    """xavier_uniform then row-wise L2 normalisation (transE.py:31-46 and peers)."""
    w = torch.empty(rows, dim, dtype=torch.float32)
    nn.init.xavier_uniform_(w)
    if normalize:
        w = torch.nn.functional.normalize(w, p=2, dim=1)
    return w


def _embedding(weight, **kw):
    emb = nn.Embedding(weight.shape[0], weight.shape[1], **kw)
    emb.weight = nn.Parameter(weight)
    return emb


_DEVICE_INIT = [None]


@contextlib.contextmanager
def device_init(device="cuda"):
    """Construct models with their tables drawn directly on `device` (same distribution: xavier-uniform
    bound, rows L2-normalised) instead of through the reference's CPU generator stream.  For large
    catalogs (millions of rows: seconds on the host, milliseconds on the GPU) and benchmarks; the
    tables are then NOT the ones the reference would draw for the same seed."""
    prev = _DEVICE_INIT[0]
    _DEVICE_INIT[0] = torch.device(device)
    try:
        yield
    finally:
        _DEVICE_INIT[0] = prev


def _make_tables_on_device(module, specs, dev):
    for s in specs:
        attr, rows, dim, normalize = s[:4]
        pad_rows = s[4] if len(s) > 4 else 0
        kw = s[5] if len(s) > 5 else {}
        bound = math.sqrt(6.0 / (rows + dim))
        w = torch.empty(rows + pad_rows, dim, dtype=torch.float32, device=dev)
        w[:rows].uniform_(-bound, bound)
        if normalize:
            w[:rows] = torch.nn.functional.normalize(w[:rows], p=2, dim=1)
        if pad_rows:
            w[rows:].zero_()
        emb = nn.Embedding(rows + pad_rows, dim, device="meta", **kw)
        emb.weight = nn.Parameter(w)
        setattr(module, attr, emb)


def _make_tables(module, specs):
    """Create the attribute ``nn.Embedding``s of a model the way the reference constructors
    consume torch's global generator: every ``xavier_uniform`` draw of the group first, in the
    listed order, then the ``nn.Embedding`` constructors (whose own normal init is discarded)
    -- transE.py:31-38, transH.py:31-40, transR.py:36-51, transUP.py:36-49, jTransUP.py:52-66,
    83-94.  With the same ``torch.manual_seed`` the tables therefore start bit-identical to the
    reference's, which is what lets a driver run be compared step for step.

    specs: (attribute, rows, dim, normalize[, extra zero rows, Embedding kwargs])."""
    if _DEVICE_INIT[0] is not None:
        return _make_tables_on_device(module, specs, _DEVICE_INIT[0])
    raw = [_init_table(s[1], s[2], normalize=False) for s in specs]
    for s, w in zip(specs, raw):
        attr, rows, dim, normalize = s[:4]
        pad_rows = s[4] if len(s) > 4 else 0
        kw = s[5] if len(s) > 5 else {}
        emb = nn.Embedding(rows + pad_rows, dim, **kw)
        if normalize:
            w = torch.nn.functional.normalize(w, p=2, dim=1)
        if pad_rows:
            w = torch.cat([w, torch.zeros(pad_rows, dim)], dim=0)
        emb.weight = nn.Parameter(w)
        setattr(module, attr, emb)


class KGRecModule(nn.Module):
    """Common base: table registry, grad switches, device handling, counters."""

    MODEL = None            # _lib.TRANSE ...
    TABLES = {}             # kernel table name -> attribute name of the nn.Embedding

    def __init__(self):
        super().__init__()
        self.is_pretrained = False
        self.grad_mode = os.environ.get("KGREC_GRAD_MODE", "dense")
        self.use_st_gumbel = False
        self._seed_counter = 0
        self._status = None
        self._item2ent = None

    @property
    def kernel_launches(self):
        """Kernels of the CUDA library enqueued so far by this process (all modules)."""
        return KF.LAUNCHES[0]

    # -- reference API --------------------------------------------------------
    def disable_grad(self):
        for _, param in self.named_parameters():
            param.requires_grad = False

    def enable_grad(self):
        for _, param in self.named_parameters():
            param.requires_grad = True

    # -- plumbing -------------------------------------------------------------
    # full-catalog evaluation kernels: embedding_size % 4 == 0 and <= 256 (TransR: <= 128); the training
    # kernels take any embedding_size <= 512
    EVAL_MAX_DIM = 256

    def _finish_init(self):
        """The reference moves every table to the GPU when one is visible (misc.py:11-16)."""
        d = self.embedding_size
        import warnings
        if d % 4 or d > self.EVAL_MAX_DIM:
            # the reference's drivers call evaluate* eval_interval_steps into a run: say so now, not there
            warnings.warn("kgrec_b200: %s with embedding_size %d can be trained but not evaluated: evaluate* / topk need a "
                          "multiple of 4, <= %d (the call will raise)" % (type(self).__name__, d, self.EVAL_MAX_DIM),
                          stacklevel=3)
        else:
            msg = self._eval_envelope_warning()
            if msg:
                warnings.warn("kgrec_b200: " + msg, stacklevel=3)
        self._check_every = int(os.environ.get("KGREC_CHECK_EVERY", "0"))
        self._calls = 0
        if torch.cuda.is_available():
            self.cuda()

    def _eval_envelope_warning(self):
        """A shape-dependent limit of the evaluation kernels inside the embedding_size rule, or None."""
        return None

    def _maybe_check(self):
        """Out-of-range ids: the kernels clamp them to row 0 and raise a device status word (the reference's
        nn.Embedding would assert).  It is read back -- a device sync -- at the evaluate* calls, which the
        drivers follow with a .cpu() anyway, and every KGREC_CHECK_EVERY-th scoring call when that is set."""
        if self._check_every:
            self._calls += 1
            if self._calls % self._check_every == 0:
                self.check_indices()

    def _weights(self):
        return {k: getattr(self, attr).weight for k, attr in self.TABLES.items()}

    @property
    def device(self):
        return next(self.parameters()).device

    def _require_cuda(self):
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError(
                "kgrec_b200: %s lives on %s.  The scoring engine is CUDA-only (sm_90a); "
                "there is no CPU or PyTorch fallback." % (type(self).__name__, dev))
        return dev

    def _status_buf(self, dev):
        if self._status is None or self._status.device != dev:
            self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        return self._status

    def check_indices(self):
        """Raise if any kernel since the last check saw an out-of-range id (device sync)."""
        if self._status is not None and int(self._status.item()) != 0:
            self._status.zero_()
            raise IndexError("kgrec_b200: an index was out of range for its table")

    def _next_seed(self):
        self._seed_counter += 1
        return (int(torch.initial_seed()) * 1000003 + self._seed_counter) & 0xFFFFFFFFFFFFFFFF

    def _cfg(self, model=None, seed=0):
        return KF._Ctx(self.MODEL if model is None else model, self.embedding_size, self.L1_flag,
                       self.use_st_gumbel, self._item2ent, self.grad_mode, seed)

    def _tables_for(self, model):
        w = self._weights()
        return [w[name] for name in KF.MODEL_TABLES[model]]

    def _score(self, model, a, b, c, gumbel_u=None):
        dev = self._require_cuda()
        a, b = KF.as_index(a, dev), KF.as_index(b, dev)
        c = KF.as_index(c, dev) if c is not None else None
        if a.numel() == 0:                       # empty batch: the reference returns an empty score vector
            return torch.zeros(0, dtype=torch.float32, device=dev) + 0 * sum(w.sum() for w in self._tables_for(model))
        if gumbel_u is not None:
            gumbel_u = gumbel_u.to(dev, torch.float32).contiguous()
        seed = self._next_seed() if (self.use_st_gumbel and gumbel_u is None) else 0
        out = KF.ScoreFunction.apply(self._cfg(model, seed), a, b, c, gumbel_u, self._status_buf(dev),
                                     *self._tables_for(model))
        self._maybe_check()
        return out

    def _rank_loss(self, model, pos, neg, loss, param, batch_pos=None, gumbel_u=None):
        dev = self._require_cuda()
        pos = tuple(KF.as_index(x, dev) if x is not None else None for x in pos)
        neg = tuple(KF.as_index(x, dev) if x is not None else None for x in neg)
        n_pos = pos[0].numel()
        if n_pos == 0 or neg[0].numel() % n_pos:
            raise ValueError("negatives must be a whole multiple of the positives")
        n_neg = neg[0].numel() // n_pos
        kind = {"margin": _lib.LOSS_MARGIN, "bpr": _lib.LOSS_BPR}[loss]
        if gumbel_u is not None:
            gumbel_u = gumbel_u.to(dev, torch.float32).contiguous()
        seed = self._next_seed() if (self.use_st_gumbel and gumbel_u is None) else 0
        return KF.RankLossFunction.apply(self._cfg(model, seed), pos, neg, n_neg, batch_pos or n_pos, kind, param,
                                         gumbel_u, self._status_buf(dev), *self._tables_for(model))

    def _rank_loss_corrupt(self, model, pos, corrupt, loss, param, batch_pos=None):
        dev = self._require_cuda()
        pos = tuple(KF.as_index(x, dev) for x in pos)
        corrupt = corrupt.to(dev, torch.int32, non_blocking=True).contiguous().view(-1)
        n_pos = pos[0].numel()
        if n_pos == 0 or corrupt.numel() % n_pos:
            raise ValueError("corrupt ids must be a whole multiple of the positives")
        kind = {"margin": _lib.LOSS_MARGIN, "bpr": _lib.LOSS_BPR}[loss]
        return KF.CorruptLossFunction.apply(self._cfg(model, 0), pos, corrupt, corrupt.numel() // n_pos,
                                            batch_pos or n_pos, kind, param, self._status_buf(dev),
                                            *self._tables_for(model))

    def _loss_step_corrupt(self, model, pos, corrupt, loss, param, batch_pos=None, grad_loss=1.0, reg=False):
        dev = self._require_cuda()
        pos = tuple(KF.as_index(x, dev) for x in pos)
        corrupt = corrupt.to(dev, torch.int32, non_blocking=True).contiguous().view(-1)
        n_pos = pos[0].numel()
        if n_pos == 0 or corrupt.numel() % n_pos:
            raise ValueError("corrupt ids must be a whole multiple of the positives")
        kind = {"margin": _lib.LOSS_MARGIN, "bpr": _lib.LOSS_BPR}[loss]
        names = KF.MODEL_TABLES[model]
        w = self._weights()
        out, ps, ns, grads = KF.corrupt_loss_step(self._cfg(model, 0), {k: w[k] for k in names}, pos, corrupt,
                                                  corrupt.numel() // n_pos, batch_pos or n_pos, kind, param,
                                                  self._status_buf(dev), grad_loss, reg)
        for k in names:          # what loss.sum().backward() would have left in .grad
            p = w[k]
            if p.requires_grad:
                p.grad = grads[k] if p.grad is None else p.grad + grads[k]
        return out, ps, ns

    def _loss_step(self, model, pos, neg, loss, param, batch_pos=None, gumbel_u=None, grad_loss=1.0):
        """Forward + ranking loss + backward in one call; leaves the gradients in .grad."""
        dev = self._require_cuda()
        pos = tuple(KF.as_index(x, dev) if x is not None else None for x in pos)
        neg = tuple(KF.as_index(x, dev) if x is not None else None for x in neg)
        n_pos = pos[0].numel()
        if n_pos == 0 or neg[0].numel() % n_pos:
            raise ValueError("negatives must be a whole multiple of the positives")
        kind = {"margin": _lib.LOSS_MARGIN, "bpr": _lib.LOSS_BPR}[loss]
        if gumbel_u is not None:
            gumbel_u = gumbel_u.to(dev, torch.float32).contiguous()
        seed = self._next_seed() if (self.use_st_gumbel and gumbel_u is None) else 0
        names = KF.MODEL_TABLES[model]
        w = self._weights()
        out, ps, ns, grads = KF.rank_loss_step(self._cfg(model, seed), {k: w[k] for k in names}, pos, neg,
                                               neg[0].numel() // n_pos, batch_pos or n_pos, kind, param, gumbel_u,
                                               self._status_buf(dev), grad_loss)
        for k in names:
            p = w[k]
            if p.requires_grad and grads[k] is not None:
                g = grads[k].clone() if (model == _lib.KTUP and k in ("rel", "norm")) else grads[k]   # shared buffer
                p.grad = g if p.grad is None else p.grad + g
        return out, ps, ns

    # -- evaluation helpers ------------------------------------------------------
    def _eval(self, model, side, q, r, mode, **kw):
        dev = self._require_cuda()
        q = KF.as_index(q, dev) if q is not None else None
        r = KF.as_index(r, dev) if r is not None else None
        nq = q.numel() if q is not None else kw["qvec"].shape[0]
        if nq == 0:                              # no queries: empty results of the right shape
            if mode == "scores":
                return torch.zeros((0, kw["catalog"].shape[0]), dtype=torch.float32, device=dev)
            if mode == "topk":
                return torch.zeros((0, kw.get("k", 10)), dtype=torch.int64, device=dev)
            return torch.zeros(0, dtype=torch.int32, device=dev)
        T = KF.make_tables(self._weights(), self.embedding_size, self.L1_flag, self.use_st_gumbel, self._item2ent)
        out = KE.run(T, model, side, q, r, mode, **kw)
        if mode == "scores":                     # the drivers' full-matrix path: its caller copies to the host next
            self.check_indices()
        return out
