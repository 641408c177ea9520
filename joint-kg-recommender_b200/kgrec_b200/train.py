"""Complete training steps replayed from CUDA graphs: the reference's one optimizer update per batch
(knowledge_representation.py:187-216, item_recommendation.py:168-192, knowledgable_recommendation.py:320-402) without
per-step host work.

One step is the loop of INTEGRATION section 6 on the device:

    kgrec_batch_gather        the batch's id columns from DeviceTrainIterator's shuffled order at the device cursor
    kgrec_step_advance        step += 1, epoch += 1, cursor += batch_size       (the device step state)
    kgrec_sample_*_dev        negatives, seed = sample_seed + step
    loss step                 kgrec_corrupt_loss_step (KG) / kgrec_rank_loss_step_dev | kgrec_rec_rows_step_dev (rec)
    kgrec_rows_*_dev          marks, clip norm, SGD / Adagrad / Adam with lr and Adam's t read from the state
                              (kgrec_rows_update_ex_dev for the optimizer's exact / momentum / RMSprop settings)

Every scalar that changes from step to step is read from the device step state, so a graph of S such steps can be
replayed as it is.  Epoch boundaries are kept on the host: run() knows from DeviceTrainIterator's rule how many batches
are left in each iterator's epoch, replays the S-step graph only while its batches fit, runs the rest through 1-step
graphs, and reshuffles (with the iterator's own generator, into the same static order buffer) between replays.  The
batches are therefore the eager iterator's, and the results bit-for-bit those of the same steps run eagerly through
the `_dev` entry points (steps_per_graph=0 runs exactly that).
"""
import ctypes as C

import torch

from . import _lib
from . import functional as KF

_MASK = 0xFFFFFFFFFFFFFFFF


def _as_int64(v):
    """The int64 with the bits of the uint64 v."""
    v = int(v) & _MASK
    return v - (1 << 64) if v >= (1 << 63) else v


def _as_int32(v):
    return ((int(v) + (1 << 31)) % (1 << 32)) - (1 << 31)


class StepState:
    """struct kgrec_step_state (include/kgrec_b200.h) in device memory.  Fields are written with fill kernels on the
    current stream: nothing synchronises."""

    def __init__(self, device, step=0, epoch=None, gumbel_seed=0, sample_seed=0, lr=0.0):
        self.buf = torch.zeros(C.sizeof(_lib.StepState) // 8, dtype=torch.int64, device=device)
        self.buf[0].fill_(int(step))
        self.buf[1].fill_(_as_int64(gumbel_seed))
        self.buf[2].fill_(_as_int64(sample_seed))
        self.buf.view(torch.int32)[_lib.StepState.epoch.offset // 4].fill_(_as_int32(step if epoch is None else epoch))
        self.set_lr(lr)

    @property
    def ptr(self):
        return C.c_void_p(self.buf.data_ptr())

    def set_lr(self, lr):
        self.buf.view(torch.float32)[_lib.StepState.lr.offset // 4].fill_(float(lr))

    def advance(self, cursor=None, batch=0):
        """kgrec_step_advance: begin the next step (and move `cursor`, an int64 device scalar, by `batch`)."""
        _lib.check(_lib.load().kgrec_step_advance(self.ptr, KF._ptr(cursor), int(batch), KF._stream()))
        KF.count_launches(1)

    def read(self):
        """The fields as a dict (device sync)."""
        raw = _lib.StepState.from_buffer_copy(self.buf.cpu().numpy().tobytes())
        return {k: getattr(raw, k) for k, _ in _lib.StepState._fields_}


def replay_plan(kinds, starts, n, batch_size, n_steps, steps_per_graph, step0=0):
    """The host schedule of GraphedTrainLoop.run, without a device.

    kinds(g) -> name of the iterator step g draws from; starts: {name: DeviceTrainIterator.start}; n / batch_size:
    {name: rows / batch size}.  Returns [(reshuffle, steps)]: `reshuffle` lists the iterators that start a new epoch
    before the replay, `steps` is steps_per_graph (the S-step graph) or 1.  Mirrors DeviceTrainIterator.__next__: a
    new epoch begins when start + batch_size > n - batch_size."""
    starts = dict(starts)
    left = lambda k: max(0, (n[k] - batch_size[k] - starts[k]) // batch_size[k])
    plan, g, S = [], step0, steps_per_graph

    def fits(steps):
        """(the steps' batches fit the iterators' epochs, the iterators that must start a new epoch first)"""
        cnt = {}
        for i in range(steps):
            cnt[kinds(g + i)] = cnt.get(kinds(g + i), 0) + 1
        new = [k for k in cnt if left(k) == 0]
        return all((n[k] // batch_size[k] if k in new else left(k)) >= c for k, c in cnt.items()), new
    while n_steps > 0:
        ok, new = fits(S) if (S > 1 and n_steps >= S) else (False, None)
        steps = S if ok else 1
        if not ok:
            _, new = fits(1)
        for k in new:
            starts[k] = -batch_size[k]
        for i in range(steps):
            starts[kinds(g + i)] += batch_size[kinds(g + i)]
        plan.append((new, steps))
        g += steps
        n_steps -= steps
    return plan


class _Source:
    """One DeviceTrainIterator on the device: a static copy of its order, the batch cursor and the gathered batch."""

    def __init__(self, it, sampler, n_neg):
        if it.n < it.batch_size:
            raise ValueError("GraphedTrainLoop: every batch must be a full batch (batch_size <= rows of the data)")
        if len(it.cols) > 4:
            raise ValueError("GraphedTrainLoop: at most 4 id columns")
        self.it, self.sampler, self.n_neg = it, sampler, int(n_neg)
        dev = it.device
        self.order = it.order.to(torch.int64).clone()
        self.cursor = torch.zeros(1, dtype=torch.int64, device=dev)
        self.cursor.fill_(it.start + it.batch_size)
        self.batch = [torch.empty(it.batch_size, dtype=c.dtype, device=dev) for c in it.cols]
        self._cols = (C.c_void_p * len(it.cols))(*[c.data_ptr() for c in it.cols])
        self._outs = (C.c_void_p * len(self.batch))(*[b.data_ptr() for b in self.batch])

    def gather(self, status):
        it = self.it
        _lib.check(_lib.load().kgrec_batch_gather(
            KF._ptr(self.order), self.order.numel(), KF._ptr(self.cursor), self._cols, self._outs, len(self.batch),
            self.batch[0].element_size(), it.n, it.batch_size, KF._ptr(status), KF._stream()))
        KF.count_launches(1)

    def new_epoch(self):
        """DeviceTrainIterator.__next__'s epoch boundary, enqueued between replays."""
        it = self.it
        it.start = -it.batch_size
        it.epoch += 1
        it._shuffle()
        self.order.copy_(it.order)
        self.cursor.fill_(0)


class GraphedTrainLoop:
    """N complete training steps (gather -> negatives -> forward + loss + backward -> clip -> optimizer update) per call
    of run(N), replayed from CUDA graphs of `steps_per_graph` steps.

    model / optimizer: a kgrec_b200 model and its SparseRowOptimizer.  iterator / sampler / n_neg: the training
    DeviceTrainIterator (int32 ids), its negative sampler and the negatives per positive -- for KTUP the rec side's, with
    the KG side's in kg_iterator / kg_sampler / kg_n_neg.
      KG models (TransE / TransH / TransR): sample_corrupt -> step_corrupt(margin, loss, reg)
      TUP: sample_neg_items -> step_pairs(target, loss="bpr", reg) (the row-factored or the pair kernel, chosen by
           SparseRowOptimizer's rule when the step is captured)
      KTUP: step g is a rec step when g % 10 < 10 * joint_ratio, else a KG step with grad_loss = kg_lambda
           (knowledgable_recommendation.py:320-402); steps_per_graph must then be a multiple of 10.
    Seeds: the sampler seed of step s is sample_seed + s, the Gumbel seed continues the model's own sequence (that of
    model._next_seed()), s counting the optimizer's steps.  steps_per_graph=0 runs the same `_dev` launches eagerly.
    The tables, the optimizer's state and the iterators' positions are those the same steps run eagerly leave."""

    def __init__(self, model, optimizer, iterator, sampler, n_neg, steps_per_graph=10, margin=1.0, loss="margin",
                 reg=False, target=-1.0, kg_iterator=None, kg_sampler=None, kg_n_neg=1, joint_ratio=0.5,
                 kg_lambda=1.0, sample_seed=0):
        m = model
        self.dev = m._require_cuda()
        self.model, self.opt = m, optimizer
        self.S = int(steps_per_graph)
        self.ktup = m.MODEL == _lib.KTUP
        self.kg_model = m.MODEL in (_lib.TRANSE, _lib.TRANSH, _lib.TRANSR)
        if not (self.kg_model or m.MODEL in (_lib.TUP, _lib.KTUP)):
            raise NotImplementedError("GraphedTrainLoop: TransE / TransH / TransR / TUP / KTUP")
        if self.S < 0 or (self.ktup and self.S > 1 and self.S % 10):
            raise ValueError("steps_per_graph: >= 0, and a multiple of 10 for KTUP (the joint schedule's cycle)")
        self.margin, self.loss, self.reg, self.target = float(margin), loss, bool(reg), float(target)
        self.joint_ratio, self.kg_lambda = float(joint_ratio), float(kg_lambda)
        self.src = {}
        if self.ktup:
            if kg_iterator is None or kg_sampler is None:
                raise ValueError("GraphedTrainLoop: KTUP needs kg_iterator and kg_sampler")
            self.src["rec"] = _Source(iterator, sampler, n_neg)
            self.src["kg"] = _Source(kg_iterator, kg_sampler, kg_n_neg)
        else:
            self.src["kg" if self.kg_model else "rec"] = _Source(iterator, sampler, n_neg)
        if "rec" in self.src and self.src["rec"].batch[0].dtype != torch.int32:
            raise ValueError("GraphedTrainLoop: the rec iterator must yield int32 ids (the sampler's width)")
        t0 = optimizer.t
        self.step = 0                # steps this loop has run
        self.state = StepState(self.dev, step=t0, gumbel_seed=(int(torch.initial_seed()) * 1000003 + m._seed_counter - t0),
                               sample_seed=sample_seed, lr=optimizer.lr)
        self._status = m._status_buf(self.dev)
        self._graphs = {}

    # -- schedule -------------------------------------------------------------------------------------------------
    def kind(self, g):
        """Which iterator step g (counted from this loop's first step) draws from."""
        if not self.ktup:
            return next(iter(self.src))
        return "rec" if (g % 10) < 10 * self.joint_ratio else "kg"

    # -- one step, as launches on the current stream ------------------------------------------------------------
    def _enqueue(self, kind):
        s = self.src[kind]
        s.gather(self._status)
        self.state.advance(s.cursor, s.it.batch_size)
        opt = self.opt
        if kind == "kg":
            pos = tuple(s.batch[:3])
            corrupt = s.sampler.sample(pos, s.n_neg, state=self.state)
            gl = self.kg_lambda if self.ktup else 1.0
            return opt.step_corrupt(pos, corrupt, margin=self.margin, loss=self.loss, reg=self.reg, grad_loss=gl,
                                    state=self.state)
        u, i = s.batch[:2]
        ni = s.sampler.sample(u, i, s.n_neg, state=self.state)
        nu = u if s.n_neg == 1 else u.repeat_interleave(s.n_neg)
        out, _ = opt.step_pairs((u, i), (nu, ni), target=self.target, loss="bpr", reg=self.reg, state=self.state)
        return out

    def _mutable(self):
        m, opt = self.model, self.opt
        ts = list(m.parameters()) + list(opt.acc.values()) + list(opt.marks.values()) + [opt.sqnorm, opt.reg_loss]
        ts += [v for v in list(opt.s1.values()) + list(opt.s2.values()) if v is not None]
        ts += [opt.steps] if opt.steps is not None else []
        ts += [self.state.buf, self._status] + [s.cursor for s in self.src.values()]
        ts += [s.sampler._status() for s in self.src.values()]
        return ts

    def _graph(self, g0, steps):
        kinds = tuple(self.kind(g0 + i) for i in range(steps))
        if kinds in self._graphs:
            return self._graphs[kinds]
        opt = self.opt
        if not self._graphs:
            # one eager pass over every step kind loads the kernels before the first capture; its effects are undone
            saved = [(t, t.detach().clone()) for t in self._mutable()]
            t0 = opt.t
            for k in self.src:
                self._enqueue(k)
            for t, c in saved:
                t.detach().copy_(c)
            if opt._rows_ws is not None:
                opt._rows_ws.zero_()
            opt.t = t0
        t0 = opt.t
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            losses = torch.cat([self._enqueue(k).view(-1) for k in kinds])
        opt.t = t0
        self._graphs[kinds] = (graph, losses)
        return self._graphs[kinds]

    # -- public ---------------------------------------------------------------------------------------------------
    def run(self, n_steps):
        """Run n_steps training steps; returns their losses, one per step, as a device tensor (nothing synchronises).
        The iterators' host positions (start, epoch, generator) advance as the eager loop's would."""
        n_steps = int(n_steps)
        out = torch.empty(n_steps, dtype=torch.float32, device=self.dev)
        plan = replay_plan(self.kind, {k: s.it.start for k, s in self.src.items()},
                           {k: s.it.n for k, s in self.src.items()}, {k: s.it.batch_size for k, s in self.src.items()},
                           n_steps, self.S, self.step)
        done = 0
        for reshuffle, steps in plan:
            for k in reshuffle:
                self.src[k].new_epoch()
            if self.S == 0:
                for i in range(steps):
                    out[done + i:done + i + 1].copy_(self._enqueue(self.kind(self.step + i)).view(-1)[:1])
            else:
                graph, losses = self._graph(self.step, steps)
                graph.replay()
                out[done:done + steps].copy_(losses)
                self.opt.t += steps
            for i in range(steps):
                s = self.src[self.kind(self.step + i)]
                s.it.start += s.it.batch_size
            self.step += steps
            done += steps
        if self.model.use_st_gumbel:
            self.model._seed_counter += n_steps
        return out

    def set_lr(self, lr):
        """Learning rate of the following steps (the trainer's optimizer_reset decay): written on the device, no
        recapture."""
        self.opt.lr = float(lr)
        self.state.set_lr(lr)

    def reset_optimizer(self, lr):
        """The trainer's optimizer_reset between replays: SparseRowOptimizer.reset(lr) (state and Adam's per-table step
        counts zeroed in place) and set_lr(lr).  No recapture: the buffers keep their addresses and the step counts are
        read on the device."""
        self.opt.reset(lr)
        self.set_lr(lr)

    def check(self):
        """Raise if an id was out of range or a sampler key had no valid negative since the last check (device sync)."""
        self.model.check_indices()
        for s in self.src.values():
            s.sampler.check()
