"""Exact torch.optim trajectories from the sparse-row optimizer (kgrec_rows_update_ex / _ex_dev, SparseRowOptimizer with
rows="all", momentum, RMSprop, per-table Adam step counts, reset, from_flags) and GraphedTrainLoop.reset_optimizer.

The reference's trainer (utils/trainer.py:63-102) steps a dense torch.optim optimizer over dense-gradient nn.Embedding
tables, so every row of every table the loss reaches moves on every step.  rows="all" must reproduce that trajectory:
  - rule level: the entry point itself on fixed accumulators and marks (no atomics anywhere), >= 50 steps, against
    torch.optim on the GPU (row mode ALL) or the numpy restatement of the rules (row mode TOUCHED);
  - model level: full training steps against grad_mode="dense" copies driven by torch.optim + clip_grad_norm_, with the
    launch scripts' settings.  The dense gradient accumulators are atomic sums on both sides, so these agree to float
    rounding, as the existing parity tests do;
  - CUDA graphs: the same `_dev` steps replayed and run eagerly.
CPU tests: symbols, struct layout, host-side argument validation, from_flags' mapping, and the numpy restatement of the
four rules pinned against torch.optim on the CPU."""
import copy
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

FAKE = 0x7000_0000_1000
KINDS = {"SGD": 0, "Adagrad": 1, "Adam": 2, "RMSprop": 3}


# ---- numpy restatement of torch.optim's rules (float32) ------------------------------------------------------------
def np_rule(kind, p, g, s1, s2, t, lr, wd=0.0, momentum=0.0, alpha=0.99, eps=1e-8, betas=(0.9, 0.999)):
    """One step of torch.optim.<kind> on float32 arrays, in torch's order of operations (single-tensor path); s1 / s2
    are updated in place; returns the new p.  t: the step count after this step (Adam's bias terms)."""
    f = np.float32
    if wd:
        g = g + f(wd) * p
    if kind == "SGD":
        if not momentum:
            return p - f(lr) * g
        s1[...] = f(momentum) * s1 + g                 # a zero buffer gives torch's first-step buf = g
        return p - f(lr) * s1
    if kind == "Adagrad":
        s1[...] = s1 + g * g
        return p - f(lr) * (g / (np.sqrt(s1) + f(eps)))
    if kind == "Adam":
        b1, b2 = betas
        s1[...] = s1 + f(1 - b1) * (g - s1)            # lerp: m + (1 - b1) (g - m)
        s2[...] = s2 * f(b2) + f(1 - b2) * g * g
        bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
        return p - f(lr / bc1) * (s1 / (np.sqrt(s2) / f(math.sqrt(bc2)) + f(eps)))
    if kind == "RMSprop":
        s1[...] = f(alpha) * s1 + f(1 - alpha) * g * g
        q = g / (np.sqrt(s1) + f(eps))
        if not momentum:
            return p - f(lr) * q
        s2[...] = f(momentum) * s2 + q
        return p - f(lr) * s2
    raise ValueError(kind)


def torch_opt(kind, params, lr, wd=0.0, momentum=0.0, **kw):
    """What ModelTrainer.optimizer_reset builds (momentum for SGD / RMSprop only)."""
    if kind == "SGD":
        return torch.optim.SGD(params, lr=lr, weight_decay=wd, momentum=momentum, **kw)
    if kind == "RMSprop":
        return torch.optim.RMSprop(params, lr=lr, weight_decay=wd, momentum=momentum, **kw)
    return getattr(torch.optim, kind)(params, lr=lr, weight_decay=wd, **kw)


STATE_KEYS = {"SGD": ("momentum_buffer", None), "Adagrad": ("sum", None), "Adam": ("exp_avg", "exp_avg_sq"),
              "RMSprop": ("square_avg", "momentum_buffer")}


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_exact_optimizer_symbols_are_exported():
    from kgrec_b200 import _lib
    lib = _lib.load()
    for name in ("kgrec_rows_update_ex", "kgrec_rows_update_ex_dev"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


def test_opt_params_layout_matches_header():
    from kgrec_b200 import _lib
    P = _lib.OptParams
    # int32 kind, int32 rows, float lr, eps, beta1, beta2, alpha, momentum, weight_decay, max_norm, int64* step_counts
    assert C.sizeof(P) == 48
    offs = [getattr(P, k).offset for k in ("kind", "rows", "lr", "eps", "beta1", "beta2", "alpha", "momentum",
                                           "weight_decay", "max_norm", "step_counts")]
    assert offs == [0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 40]
    assert (_lib.ROWS_TOUCHED, _lib.ROWS_ALL) == (0, 1)


def test_c_abi_exact_update_argument_validation_without_a_gpu():
    from kgrec_b200 import _lib
    lib = _lib.load()

    def err():
        return lib.kgrec_last_error().decode()

    def tab(**kw):
        d = dict(table=FAKE, acc=FAKE, state1=FAKE, state2=FAKE, marks=FAKE, rows=100, dim=100, keep_acc=0)
        d.update(kw)
        return (_lib.OptTable * 1)(_lib.OptTable(**d))

    def params(**kw):
        d = dict(kind=2, rows=1, lr=1e-3, eps=1e-8, beta1=0.9, beta2=0.999, alpha=0.99, momentum=0.0, weight_decay=0.0,
                 max_norm=5.0, step_counts=FAKE)
        d.update(kw)
        return _lib.OptParams(**d)

    def ex(tabs=None, n=1, p=None, null_params=False):
        return lib.kgrec_rows_update_ex(tabs or tab(), n, 1, None if null_params else C.byref(p or params()), None, None)

    def ex_dev(state=FAKE, p=None):
        return lib.kgrec_rows_update_ex_dev(tab(), 1, state, C.byref(p or params()), None, None)
    assert ex(null_params=True) != 0 and "params is NULL" in err()
    assert ex(p=params(kind=4)) != 0 and "unknown kind 4" in err()
    assert ex(p=params(kind=-1)) != 0 and "unknown kind" in err()
    assert ex(p=params(rows=2)) != 0 and "unknown row mode 2" in err()
    assert ex(tabs=tab(state1=None), p=params(kind=0, momentum=0.9)) != 0 and "state missing" in err()   # SGD buffer
    assert ex(tabs=tab(state1=None), p=params(kind=1)) != 0 and "state missing" in err()                 # Adagrad sum
    assert ex(tabs=tab(state2=None), p=params(kind=2)) != 0 and "state missing" in err()                 # Adam v
    assert ex(tabs=tab(state1=None), p=params(kind=3)) != 0 and "state missing" in err()                 # RMSprop sq
    assert ex(tabs=tab(state2=None), p=params(kind=3, momentum=0.9)) != 0 and "state missing" in err()   # its buffer
    assert ex(p=params(kind=2, step_counts=None)) != 0 and "step_counts is NULL" in err()
    assert ex(tabs=(_lib.OptTable * 9)(*([tab()[0]] * 9)), n=9) != 0 and "tables per call" in err()
    assert ex(tabs=tab(acc=None)) != 0 and "no accumulator" in err()
    assert ex(tabs=tab(rows=0)) != 0
    assert ex_dev(state=None) != 0 and "step state is NULL" in err()
    assert ex_dev(p=params(kind=7)) != 0 and "unknown kind 7" in err()
    # the existing entry point keeps its four rules
    assert lib.kgrec_rows_update(tab(), 1, 1, 3, 0.01, 1e-10, 0.9, 0.999, 1, 0.0, None, 0.0, None) != 0
    assert "unknown kind" in err()


def _flags(**kw):
    d = dict(optimizer_type="Adagrad", learning_rate=0.005, l2_lambda=1e-5, momentum=0.9, clipping_max_value=5.0)
    d.update(kw)
    return types.SimpleNamespace(**d)


def test_from_flags_follows_the_trainer():
    """ModelTrainer.optimizer_reset (utils/trainer.py:63-78): momentum only for SGD and Rmsprop, rows="all"."""
    from kgrec_b200.optim import flags_kwargs, SparseRowOptimizer
    want = {"Adam": ("Adam", 0.0), "SGD": ("SGD", 0.9), "Adagrad": ("Adagrad", 0.0), "Rmsprop": ("Rmsprop", 0.9)}
    for t, (kind, mom) in want.items():
        kw = flags_kwargs(_flags(optimizer_type=t, learning_rate=0.01, l2_lambda=2e-5, clipping_max_value=3.0))
        assert kw == dict(optimizer_type=kind, lr=0.01, l2_lambda=2e-5, clip=3.0, momentum=mom, rows="all"), t
    for bad in ("RMSprop", "adam", "Adadelta", ""):
        with pytest.raises(ValueError):
            flags_kwargs(_flags(optimizer_type=bad))
        with pytest.raises(ValueError):
            SparseRowOptimizer.from_flags(None, _flags(optimizer_type=bad))


@pytest.mark.parametrize("kind,wd,momentum,clip", [
    ("SGD", 0.0, 0.0, None), ("SGD", 1e-2, 0.9, 0.5), ("Adagrad", 0.0, 0.0, None), ("Adagrad", 1e-2, 0.0, 0.5),
    ("Adam", 0.0, 0.0, None), ("Adam", 1e-2, 0.0, 0.5), ("RMSprop", 0.0, 0.0, None), ("RMSprop", 1e-2, 0.0, 0.5),
    ("RMSprop", 1e-2, 0.9, 0.5)])
def test_numpy_rules_match_torch_optim_on_cpu(kind, wd, momentum, clip):
    """The restatement the GPU tests use for TOUCHED mode, against torch.optim (CPU, float32) over 30 steps with zero
    and non-zero gradient entries, weight decay and clip_grad_norm_: eps placement, first-step momentum, bias terms."""
    rng = np.random.RandomState(5)
    p0 = rng.randn(6, 5).astype(np.float32)
    lr = 0.01
    w = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch_opt(kind, [w], lr, wd, momentum, foreach=False)
    p, s1, s2 = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
    for t in range(1, 31):
        g = (rng.randn(6, 5) * (rng.rand(6, 5) < 0.4)).astype(np.float32)     # most entries zero
        gt = torch.from_numpy(g.copy())
        if clip is not None:      # clip_grad_norm_'s coefficient, from its own norm
            coef = torch.clamp(clip / (torch.linalg.vector_norm(gt) + 1e-6), max=1.0)
            g = g * coef.numpy()
            w.grad = gt
            torch.nn.utils.clip_grad_norm_([w], clip)
        else:
            w.grad = gt
        opt.step()
        p = np_rule(kind, p, g, s1, s2, t, lr, wd, momentum)
    # float rounding over 30 steps on entries of order 1 (torch's CPU kernels fuse some multiply-adds)
    np.testing.assert_allclose(p, w.detach().numpy(), rtol=1e-6, atol=2e-6)
    k1, k2 = STATE_KEYS[kind]
    st = opt.state[w]
    for mine, key in ((s1, k1), (s2, k2)):
        if key and key in st:
            want = st[key].numpy()
            np.testing.assert_allclose(mine, want, rtol=1e-5, atol=1e-6 * float(np.abs(want).max()))


# ---- GPU: rule level -----------------------------------------------------------------------------------------------
# (rows, dim, marked): vec rows, the scalar path (dim % 4 != 0), a TransR-shaped wide table (d x d = 4096 floats a row,
# swept in segments) and tables without marks ("every row")
SPECS = [(700, 32, True), (90, 10, True), (6, 4096, False), (24, 36, False)]


class _Tabs:
    def __init__(self, kind, momentum, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        use_s1 = kind != "SGD" or momentum
        use_s2 = kind == "Adam" or (kind == "RMSprop" and momentum)
        self.p, self.acc, self.s1, self.s2, self.marks = [], [], [], [], []
        for rows, dim, marked in SPECS:
            self.p.append(torch.randn(rows, dim, device="cuda", generator=g) * 0.3)
            self.acc.append(torch.zeros(rows, dim, device="cuda"))
            self.s1.append(torch.zeros(rows, dim, device="cuda") if use_s1 else None)
            self.s2.append(torch.zeros(rows, dim, device="cuda") if use_s2 else None)
            self.marks.append(torch.zeros(rows, dtype=torch.int32, device="cuda") if marked else None)
        self.counts = torch.zeros(len(SPECS), dtype=torch.int64, device="cuda")
        self.sq = torch.zeros(1, device="cuda")

    def entries(self, n):
        from kgrec_b200 import _lib
        ptr = lambda x: x.data_ptr() if x is not None else None  # noqa: E731
        return (_lib.OptTable * n)(*[_lib.OptTable(table=self.p[t].data_ptr(), acc=self.acc[t].data_ptr(), state1=ptr(self.s1[t]),
                                                  state2=ptr(self.s2[t]), marks=ptr(self.marks[t]), rows=SPECS[t][0],
                                                  dim=SPECS[t][1], keep_acc=0) for t in range(n)])


def _fill_step(T, e, n, gen, max_norm):
    """Marks ~10% of the marked tables' rows with epoch e and writes their accumulators; tables without marks get an
    accumulator on every row (some rows zero).  Writes the total norm into T.sq; returns (marked row masks, clip scale)."""
    masks = []
    for t in range(n):
        rows, dim, marked = SPECS[t]
        if marked:
            idx = torch.randperm(rows, generator=gen)[:max(1, rows // 10)].cuda()
            T.marks[t][idx] = e
            T.acc[t][idx] = (torch.randn(idx.numel(), dim, generator=gen) * 0.5).cuda()
            masks.append(T.marks[t] == e)
        else:
            a = torch.randn(rows, dim, generator=gen) * 0.5
            a[rows // 2:rows // 2 + 1] = 0
            T.acc[t].copy_(a.cuda())
            masks.append(torch.ones(rows, dtype=torch.bool, device="cuda"))
    T.sq.copy_(sum((T.acc[t].double() ** 2).sum() for t in range(n)).float().view(1))
    scale = torch.clamp(max_norm / (T.sq.sqrt() + 1e-6), max=1.0)
    return masks, scale


def _run_rule(kind, rows_mode, wd, momentum, steps=50, max_norm=2.0, seed=0):
    """(our tables and state, the reference's) after `steps` steps; every third step updates only the first two tables
    (per-table Adam counts).  rows_mode "all": torch.optim on the GPU; "touched": np_rule on the marked rows."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    lr = {"SGD": 0.05, "Adagrad": 0.02, "Adam": 0.01, "RMSprop": 1e-3}[kind]
    ours, ref = _Tabs(kind, momentum, seed), _Tabs(kind, momentum, seed)
    params = [torch.nn.Parameter(p.clone()) for p in ref.p]
    topt = torch_opt(kind, params, lr, wd, momentum)
    ref_s1 = [x.cpu().numpy() if x is not None else None for x in ref.s1]
    ref_s2 = [x.cpu().numpy() if x is not None else None for x in ref.s2]
    ref_p = [p.cpu().numpy() for p in ref.p]
    counts = [0] * len(SPECS)
    gen = torch.Generator().manual_seed(seed + 100)
    P = _lib.OptParams(kind=KINDS[kind], rows=_lib.ROWS_ALL if rows_mode == "all" else _lib.ROWS_TOUCHED, lr=lr,
                       eps=1e-10 if kind == "Adagrad" else 1e-8, beta1=0.9, beta2=0.999, alpha=0.99, momentum=momentum,
                       weight_decay=wd, max_norm=max_norm, step_counts=ours.counts.data_ptr())
    for e in range(1, steps + 1):
        n = 2 if e % 3 == 0 else len(SPECS)
        state = gen.get_state()
        masks, scale = _fill_step(ours, e, n, gen, max_norm)
        grads = [(ours.acc[t] * scale) for t in range(n)]
        _lib.check(lib.kgrec_rows_update_ex(ours.entries(n), n, e, C.byref(P), ours.sq.data_ptr(), None))
        gen.set_state(state)
        _fill_step(ref, e, n, gen, max_norm)            # the same draws; ref.acc is not consumed by anything
        if rows_mode == "all":
            for t, w in enumerate(params):
                w.grad = grads[t] if t < n else None
            topt.step()
        else:
            for t in range(n):
                counts[t] += 1
                m = masks[t].cpu().numpy()
                g = grads[t].cpu().numpy()[m]
                s1 = ref_s1[t][m] if ref_s1[t] is not None else None
                s2 = ref_s2[t][m] if ref_s2[t] is not None else None
                ref_p[t][m] = np_rule(kind, ref_p[t][m], g, s1, s2, counts[t], lr, wd, momentum,
                                      eps=1e-10 if kind == "Adagrad" else 1e-8)
                if s1 is not None:
                    ref_s1[t][m] = s1
                if s2 is not None:
                    ref_s2[t][m] = s2
    torch.cuda.synchronize()
    for t in range(len(SPECS)):
        assert not ours.acc[t].any(), t                     # every consumed accumulator row is clear again
    if rows_mode == "all":
        k1, k2 = STATE_KEYS[kind]
        want = [(w.detach(), topt.state[w].get(k1), topt.state[w].get(k2) if k2 else None) for w in params]
    else:
        dev = lambda x: torch.from_numpy(x).cuda() if x is not None else None  # noqa: E731
        want = [(dev(ref_p[t]), dev(ref_s1[t]), dev(ref_s2[t])) for t in range(len(SPECS))]
    got = [(ours.p[t], ours.s1[t], ours.s2[t]) for t in range(len(SPECS))]
    return got, want, ours.counts.cpu().tolist()


RULES = [("SGD", 0.0, 0.0), ("SGD", 1e-2, 0.0), ("SGD", 0.0, 0.9), ("SGD", 1e-2, 0.9), ("Adagrad", 0.0, 0.0),
         ("Adagrad", 1e-2, 0.0), ("Adam", 0.0, 0.0), ("Adam", 1e-2, 0.0), ("RMSprop", 0.0, 0.0), ("RMSprop", 1e-2, 0.0),
         ("RMSprop", 0.0, 0.9), ("RMSprop", 1e-2, 0.9)]


@pytest.mark.gpu
@pytest.mark.parametrize("rows_mode", ["all", "touched"])
@pytest.mark.parametrize("kind,wd,momentum", RULES)
def test_rule_level_trajectory_matches_torch(kind, wd, momentum, rows_mode):
    """50 steps of kgrec_rows_update_ex on fixed accumulators / marks (no atomics on either side; the clip norm is
    written, not summed by the kernel).  Bound: |ours - torch| <= 2e-5 (1 + |torch|) on tables and state -- fp32
    re-association (fma contraction, powf, lerp vs the two-term mean) over 50 steps; any wrong rule, eps, bias term,
    momentum start or row semantics is orders of magnitude larger."""
    got, want, counts = _run_rule(kind, rows_mode, wd, momentum)
    for t, ((p, s1, s2), (wp, w1, w2)) in enumerate(zip(got, want)):
        torch.testing.assert_close(p, wp, rtol=2e-5, atol=2e-5, msg=lambda m: "table %d: %s" % (t, m))
        for a, b in ((s1, w1), (s2, w2)):
            if a is not None and b is not None:
                tol = 2e-5 * max(1.0, float(b.abs().max()))
                torch.testing.assert_close(a, b, rtol=2e-5, atol=tol, msg=lambda m: "state of table %d: %s" % (t, m))
    if kind == "Adam":
        assert counts == [50, 50, 34, 34]                     # two tables skip every third call
    if rows_mode == "all" and (wd or momentum or kind in ("Adam", "RMSprop")):
        # the dense semantics: rows keep moving after their last touch; with weight decay every row moves
        moved = (got[0][0] != _Tabs(kind, momentum, 0).p[0]).any(dim=1)
        assert moved.all() if wd else moved.float().mean() > 0.9


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["SGD", "Adagrad", "Adam"])
def test_touched_mode_without_momentum_is_bit_identical_to_the_existing_entry_point(kind):
    """kgrec_rows_update_ex in TOUCHED mode with momentum 0 runs the kernel of kgrec_rows_update: tables and state are
    bit-identical.  Adam is compared with kgrec_rows_update_dev, whose bias terms are formed on the device as the
    per-table counts' are (kgrec_rows_update forms them on the host, with the host's powf)."""
    from kgrec_b200 import _lib
    from kgrec_b200.train import StepState
    lib = _lib.load()
    a, b = _Tabs(kind, 0.0, 3), _Tabs(kind, 0.0, 3)
    lr, eps, wd = 0.02, (1e-10 if kind == "Adagrad" else 1e-8), 1e-2
    gen = torch.Generator().manual_seed(7)
    state = StepState("cuda", step=0, lr=lr)
    n = len(SPECS)
    for e in range(1, 21):
        st = gen.get_state()
        _fill_step(a, e, n, gen, 2.0)
        gen.set_state(st)
        _fill_step(b, e, n, gen, 2.0)
        P = _lib.OptParams(kind=KINDS[kind], rows=_lib.ROWS_TOUCHED, lr=lr, eps=eps, beta1=0.9, beta2=0.999, alpha=0.99,
                           momentum=0.0, weight_decay=wd, max_norm=2.0, step_counts=a.counts.data_ptr())
        _lib.check(lib.kgrec_rows_update_ex(a.entries(n), n, e, C.byref(P), a.sq.data_ptr(), None))
        if kind == "Adam":
            state.advance()
            _lib.check(lib.kgrec_rows_update_dev(b.entries(n), n, state.ptr, KINDS[kind], eps, 0.9, 0.999, wd,
                                                 b.sq.data_ptr(), 2.0, None))
        else:
            _lib.check(lib.kgrec_rows_update(b.entries(n), n, e, KINDS[kind], lr, eps, 0.9, 0.999, e, wd, b.sq.data_ptr(),
                                             2.0, None))
    torch.cuda.synchronize()
    for t in range(n):
        assert torch.equal(a.p[t], b.p[t]), t
        for x, y in ((a.s1[t], b.s1[t]), (a.s2[t], b.s2[t])):
            assert (x is None and y is None) or torch.equal(x, y), t


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["SGD", "Adagrad"])
def test_all_mode_leaves_untouched_rows_bit_unchanged_where_the_rule_does(kind):
    """Plain SGD and Adagrad without weight decay: a zero-gradient row is bit-unchanged, and ALL does not touch it."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    T = _Tabs(kind, 0.0, 4)
    before = [p.clone() for p in T.p]
    gen = torch.Generator().manual_seed(9)
    P = _lib.OptParams(kind=KINDS[kind], rows=_lib.ROWS_ALL, lr=0.05, eps=1e-10, momentum=0.0, weight_decay=0.0,
                       max_norm=2.0, step_counts=None)
    untouched = [torch.ones(r, dtype=torch.bool, device="cuda") for r, _, _ in SPECS]
    for e in range(1, 6):
        masks, _ = _fill_step(T, e, len(SPECS), gen, 2.0)
        for u, m in zip(untouched, masks):
            u &= ~m
        _lib.check(lib.kgrec_rows_update_ex(T.entries(len(SPECS)), len(SPECS), e, C.byref(P), T.sq.data_ptr(), None))
    torch.cuda.synchronize()
    for t in (0, 1):
        assert untouched[t].any()
        assert torch.equal(T.p[t][untouched[t]], before[t][untouched[t]])
        assert not torch.equal(T.p[t], before[t])


# ---- GPU: model trajectories ---------------------------------------------------------------------------------------
D = 32
E_, R_, U_, I_, P_ = 1500, 9, 300, 250, 5
SETTINGS = {       # the launch scripts': transe.sh / transh.sh / transr.sh / ktup.sh, transup.sh, -optimizer_type SGD / Rmsprop
    "Adam": dict(lr=1e-3, wd=0.0, momentum=0.0),
    "Adagrad": dict(lr=5e-3, wd=1e-5, momentum=0.0),
    "SGD": dict(lr=1e-2, wd=1e-5, momentum=0.9),
    "RMSprop": dict(lr=1e-3, wd=1e-5, momentum=0.9),
}


def _model(name, seed):
    import kgrec_b200 as K
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed)
    if name in ("transe_l1", "transe_l2", "transh", "transr"):
        cls = {"transe_l1": K.TransEModel, "transe_l2": K.TransEModel, "transh": K.TransHModel, "transr": K.TransRModel}[name]
        return cls(name == "transe_l1", 16 if name == "transr" else D, E_, R_)
    if name.startswith("tup"):
        return K.TransUPModel(False, D, U_, I_, P_, False)
    ents = rng.permutation(E_)[:I_]
    new_map = {i: ((int(ents[i]) if i % 10 < 7 else -1), i) for i in range(I_)}
    return K.jTransUPModel(True, D, U_, I_, E_, P_, {i: i for i in range(I_)}, new_map, False, False)


def _batch(kind, gen, B=48, KN=2, n_rel=R_):
    if kind == "kg":
        pos = tuple(torch.randint(0, n, (B,), generator=gen).cuda() for n in (E_, E_, n_rel))
        cid = torch.randint(0, E_, (B * KN,), generator=gen, dtype=torch.int32)
        return pos, torch.where(torch.rand(B * KN, generator=gen) < 0.5, ~cid, cid).cuda()
    u = torch.randint(0, U_, (B,), generator=gen).cuda()
    return (u, torch.randint(0, I_, (B,), generator=gen).cuda()), (u, torch.randint(0, I_, (B,), generator=gen).cuda())


def _dense_step(m2, ref, kind, batch, clip, reg, ktup):
    """The reference's step on the dense copy: zero_grad (set_to_none), backward, clip_grad_norm_, step."""
    ref.zero_grad()
    if kind == "kg":
        pos, corrupt = batch
        if ktup:
            m2.kg_loss_step_corrupt(pos, corrupt, margin=1.0, grad_loss=0.5, reg=reg)
        else:
            m2.loss_step_corrupt(pos, corrupt, margin=1.0, reg=reg)
    else:
        l2_, _, _ = m2.rank_loss(batch[0], batch[1], target=-1.0)
        l2_.sum().backward()
    torch.nn.utils.clip_grad_norm_(m2.parameters(), clip)
    ref.step()


def _sparse_step(opt, kind, batch, reg, ktup):
    if kind == "kg":
        opt.step_corrupt(batch[0], batch[1], margin=1.0, grad_loss=0.5 if ktup else 1.0, reg=reg)
    else:
        opt.step_pairs(batch[0], batch[1], target=-1.0)


def _step_kind(name, g):
    if name.startswith("ktup"):
        return "rec" if g % 10 < 5 else "kg"
    return "rec" if name.startswith("tup") else "kg"


def _assert_models_close(m1, m2, tol=1e-4):
    for (n1, p1), (n2, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        assert n1 == n2
        torch.testing.assert_close(p1.detach(), p2.detach(), rtol=tol, atol=tol / 4, msg=lambda m: "%s: %s" % (n1, m))


TRAJ = [("transe_l1", "Adam", 5.0), ("transe_l1", "SGD", 5.0), ("transe_l2", "Adam", 0.5), ("transe_l2", "RMSprop", 5.0),
        ("transh", "Adam", 5.0), ("transh", "Adagrad", 5.0), ("transr", "Adam", 5.0), ("transr", "SGD", 0.5),
        ("tup_pairs", "Adagrad", 5.0), ("tup_pairs", "Adam", 0.5), ("tup_pairs", "RMSprop", 5.0), ("tup_rows", "Adagrad", 5.0),
        ("tup_rows", "SGD", 5.0), ("ktup_pairs", "Adam", 5.0), ("ktup_pairs", "Adagrad", 0.5), ("ktup_rows", "Adam", 5.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,clip", TRAJ)
def test_model_trajectory_matches_dense_torch_optim(monkeypatch, name, kind, clip):
    """rows="all" training steps against a grad_mode="dense" copy driven by torch.optim + clip_grad_norm_, every table
    compared (most rows are never touched: small batches on 1500 entities / 300 users / 250 items).  KTUP alternates 5 rec
    and 5 KG steps a cycle, so its user / item / pref tables skip the KG steps (per-table Adam counts).  The clip norm and
    the dense accumulators are atomic sums on both sides: the bound is float rounding, as in the existing parity tests."""
    from kgrec_b200.optim import SparseRowOptimizer
    monkeypatch.setenv("KGREC_REC_ROWS", "force" if name.endswith("_rows") else "0")
    st = SETTINGS[kind]
    steps = 6 if kind == "RMSprop" else 20
    m1 = _model(name, 11)
    m2 = copy.deepcopy(m1)
    m2.grad_mode = "dense"
    ref = torch_opt(kind, list(m2.parameters()), st["lr"], st["wd"], st["momentum"])
    opt = SparseRowOptimizer(m1, optimizer_type=kind, lr=st["lr"], l2_lambda=st["wd"], clip=clip,
                             momentum=st["momentum"], rows="all")
    ktup = name.startswith("ktup")
    reg = name == "transh" or ktup
    before = {n: p.detach().clone() for n, p in m1.named_parameters()}
    gen = torch.Generator().manual_seed(17)
    for g in range(steps):
        k = _step_kind(name, g)
        batch = _batch(k, gen, n_rel=P_ if ktup else R_)
        _dense_step(m2, ref, k, batch, clip, reg, ktup)
        _sparse_step(opt, k, batch, reg, ktup)
    torch.cuda.synchronize()
    _assert_models_close(m1, m2)
    for k in opt.acc:
        assert not opt.acc[k].any(), k
    if ktup:
        assert not m1.ent_embeddings.weight[-1].any()            # the padding row stays exactly zero
        assert opt.steps.tolist() == [10, 10, 20, 20, 20, 10, 10] if kind == "Adam" else True
    if SETTINGS[kind]["wd"]:    # the dense semantics: weight decay moves the rows no batch touched as well
        big = "item_embeddings.weight" if name.startswith("tup") else "ent_embeddings.weight"
        assert (dict(m1.named_parameters())[big].detach() != before[big]).any(dim=1).float().mean() > 0.99
    m1.check_indices()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["Adam", "Adagrad"])
def test_reset_mid_run_equals_a_fresh_torch_optimizer(kind):
    """SparseRowOptimizer.reset(lr) is ModelTrainer.optimizer_reset: a fresh torch optimizer at the new lr from the
    current tables (Adam's step count starts again)."""
    from kgrec_b200.optim import SparseRowOptimizer
    st = SETTINGS[kind]
    m1 = _model("transh", 12)
    m2 = copy.deepcopy(m1)
    m2.grad_mode = "dense"
    ref = torch_opt(kind, list(m2.parameters()), st["lr"], st["wd"])
    opt = SparseRowOptimizer(m1, optimizer_type=kind, lr=st["lr"], l2_lambda=st["wd"], clip=5.0, rows="all")
    gen = torch.Generator().manual_seed(23)
    for g in range(16):
        if g == 8:
            ref = torch_opt(kind, list(m2.parameters()), st["lr"] * 0.5, st["wd"])
            opt.reset(st["lr"] * 0.5)
        batch = _batch("kg", gen)
        _dense_step(m2, ref, "kg", batch, 5.0, True, False)
        _sparse_step(opt, "kg", batch, True, False)
    torch.cuda.synchronize()
    _assert_models_close(m1, m2)
    if kind == "Adam":
        assert opt.steps.tolist() == [8, 8, 8]


# ---- GPU: CUDA graphs ----------------------------------------------------------------------------------------------
N_TRIPLES, N_RATINGS, BATCH = 2600, 2600, 256          # 10 batches an epoch


def _loop_env(name, kind, S, seed=0):
    from kgrec_b200.data import DeviceTrainIterator
    from kgrec_b200.optim import SparseRowOptimizer
    from kgrec_b200.sampling import RatingNegativeSampler, TripleNegativeSampler
    from kgrec_b200.train import GraphedTrainLoop
    rng = np.random.RandomState(seed)
    model = _model(name, seed)
    kg = np.stack([rng.randint(0, E_, N_TRIPLES), rng.randint(0, E_, N_TRIPLES), rng.randint(0, R_, N_TRIPLES)], 1)
    st = SETTINGS[kind]
    opt = SparseRowOptimizer(model, optimizer_type=kind, lr=st["lr"], l2_lambda=st["wd"], clip=5.0,
                             momentum=st["momentum"], rows="all")
    kw = dict(steps_per_graph=S, sample_seed=5, reg=True)
    if name.startswith("ktup"):
        kg[:, 2] %= P_
        ratings = np.stack([rng.randint(0, U_, N_RATINGS), rng.randint(0, I_, N_RATINGS)], 1)
        it = DeviceTrainIterator(ratings, BATCH, device="cuda", seed=seed + 1)
        kw.update(kg_iterator=DeviceTrainIterator(kg, 200, device="cuda", seed=seed + 2),
                  kg_sampler=TripleNegativeSampler(E_, P_, known_triples=kg), joint_ratio=0.5, kg_lambda=0.5)
        loop = GraphedTrainLoop(model, opt, it, RatingNegativeSampler(I_, known_ratings=ratings), 1, **kw)
    else:
        it = DeviceTrainIterator(kg, BATCH, device="cuda", seed=seed + 1)
        loop = GraphedTrainLoop(model, opt, it, TripleNegativeSampler(E_, R_, known_triples=kg), 2, **kw)
    return model, opt, loop


def _state(model, opt):
    out = {"w." + k: v.detach().clone() for k, v in model.named_parameters()}
    for nm, d in (("s1", opt.s1), ("s2", opt.s2)):
        out.update({nm + "." + k: v.clone() for k, v in d.items() if v is not None})
    if opt.steps is not None:
        out["steps"] = opt.steps.clone()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,S", [("transh", "Adam", 1), ("transh", "Adam", 10), ("transe_l2", "Adagrad", 10),
                                         ("transh", "SGD", 10), ("ktup_pairs", "Adam", 10)])
def test_graphed_loop_with_exact_rows_matches_eager(monkeypatch, name, kind, S):
    """GraphedTrainLoop over rows="all" optimizers (S = 1 and 10, KTUP S = 10) against the same `_dev` steps run eagerly
    (steps_per_graph=0): 27 steps over 2.7 epochs with a reset_optimizer between replays.  2e-5: the atomic order of the
    accumulators and the clip norm.  reset_optimizer captures nothing: no new graph, the same graph objects."""
    monkeypatch.setenv("KGREC_REC_ROWS", "0")
    res = []
    for mode in (S, 0):
        model, opt, loop = _loop_env(name, kind, mode)
        loop.run(15)
        graphs = dict(loop._graphs)
        loop.reset_optimizer(SETTINGS[kind]["lr"] * 0.5)
        assert set(loop._graphs) == set(graphs)                     # nothing captured
        loop.run(12)
        torch.cuda.synchronize()
        assert all(loop._graphs[k] is graphs[k] for k in graphs)    # and nothing recaptured
        assert loop.state.read()["lr"] == pytest.approx(SETTINGS[kind]["lr"] * 0.5)
        res.append(_state(model, opt))
    g, e = res
    assert g.keys() == e.keys()
    for k in g:
        if k == "steps":
            assert torch.equal(g[k], e[k])
            continue
        torch.testing.assert_close(g[k], e[k], rtol=2e-5, atol=2e-5, msg=lambda m: "%s: %s" % (k, m))


# ---- GPU: against the reference's own trainer ----------------------------------------------------------------------
def _reference_trainer():
    import sys
    from oracle import make_ref
    if not make_ref.available():
        pytest.skip("oracle/_ref not built (oracle/make_ref.py needs a checkout of the reference)")
    for p in reversed(make_ref.env_paths()):
        if p not in sys.path:
            sys.path.insert(0, p)
    import gflags  # noqa: F401
    from jTransUP.utils.trainer import ModelTrainer
    return ModelTrainer


@pytest.mark.gpu
@pytest.mark.parametrize("name,flags", [
    ("transh", dict(optimizer_type="Adam", learning_rate=0.001, l2_lambda=0.0)),            # transh.sh
    ("tup_pairs", dict(optimizer_type="Adagrad", learning_rate=0.005, l2_lambda=1e-5)),     # transup.sh
    ("transh", dict(optimizer_type="SGD", learning_rate=0.01, l2_lambda=1e-5)),              # -optimizer_type SGD
    ("tup_pairs", dict(optimizer_type="Rmsprop", learning_rate=0.001, l2_lambda=1e-5))])     # -optimizer_type Rmsprop
def test_from_flags_reproduces_the_reference_trainer(monkeypatch, name, flags):
    """The torch side is built by the reference's own ModelTrainer.optimizer_reset (utils/trainer.py:63-78) called on a
    stand-in trainer; SparseRowOptimizer.from_flags from the same flags reproduces its trajectory."""
    ModelTrainer = _reference_trainer()
    from kgrec_b200.optim import SparseRowOptimizer
    monkeypatch.setenv("KGREC_REC_ROWS", "0")
    F = _flags(momentum=0.9, clipping_max_value=5.0, **flags)
    m1 = _model(name, 13)
    m2 = copy.deepcopy(m1)
    m2.grad_mode = "dense"
    stand = types.SimpleNamespace(parameters=[p for _, p in m2.named_parameters()], optimizer_type=F.optimizer_type,
                                  l2_lambda=F.l2_lambda, momentum=F.momentum)
    ModelTrainer.optimizer_reset(stand, F.learning_rate)
    opt = SparseRowOptimizer.from_flags(m1, F)
    assert opt.rows == "all" and opt.clip == 5.0
    gen = torch.Generator().manual_seed(29)
    steps = 6 if F.optimizer_type == "Rmsprop" else 12
    for g in range(steps):
        k = _step_kind(name, g)
        batch = _batch(k, gen)
        _dense_step(m2, stand.optimizer, k, batch, F.clipping_max_value, False, False)
        _sparse_step(opt, k, batch, False, False)
    torch.cuda.synchronize()
    _assert_models_close(m1, m2)
