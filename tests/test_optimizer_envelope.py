"""The whole envelope of the kernels around every training step, against float64 or exact restatements.

Kernels, and what picks them (restated in `update_kernel`, `vec_rule` and `div_rule` below):
  kgrec_rows_update / _dev / _ex / _ex_dev (csrc/optim.cu)
    k_rows_update       the marked rows of every table of the call, 32 rows a warp, kRowsInFlight = 4 at a time
    k_rows_update_all   row mode ALL: every row, a flat grid-stride walk over 128-bit (vec) or 32-bit units,
                        unless the rule leaves a zero-gradient row bit-unchanged (plain SGD / Adagrad without
                        weight decay): those run k_rows_update
    k_step_counts       Adam's per-table step counts (the _ex entry points)
    vec                 dim % 4 == 0 and the table, accumulator and state pointers 16-byte aligned
    div                 dim > 512 is swept as div = dim / seg rows of seg floats, seg the largest multiple of 4 in
                        64..512 dividing dim (4096 -> 8, 10000 -> 20; 513, 524, 1028 keep div = 1)
  kgrec_rows_sqnorm / _dev       k_rows_sqnorm, the same sweep
  kgrec_rows_mark / _dev         k_rows_mark
  kgrec_reg_norm_rows            k_reg_norm_rows (vec: d % 4 == 0, table and accumulator 16-byte aligned)
  kgrec_reg_orth_tables          k_reg_orth
  kgrec_hashset_build            k_hashset_insert
  kgrec_sample_corrupt / _dev    k_sample_corrupt
  kgrec_sample_neg_items / _dev  k_sample_items
  kgrec_batch_gather             k_batch_gather
  kgrec_step_advance             k_step_advance

Bounds.  Every optimizer output element (parameter and state) satisfies
    |kernel - ref| <= C_BOUND (k 2^-24 twin + adam)
where ref is the rule in float64 on the kernel's own float32 inputs of that call (parameters, accumulator, state and
the sqnorm the test writes), k the number of rounded operations on the element's path, twin the same computation with
every operand replaced by its magnitude and every subtraction by an addition (`T` below carries value, twin and k), and
`adam` the conditioning of Adam's bias terms: |update| times powf's error (POWF_ULPS ulp of beta^t, beta the float32
value) over 1 - beta^t, halved for the second moment's square root.  The clip norm is bounded by C_BOUND (longest
addition chain) 2^-24 sum; the regularisers by the twin bound, each atomic addition counted on the chain.  Rows of
reg_norm_rows whose |x|^2 lies within the bound of 1 are redrawn.

C_BOUND = 1 is the smallest integer constant every case passes with.  Largest measured ratio to the C_BOUND = 1
bound on an H100: optimizer rules 0.63, clip norm 0.015, regularisers 0.65 (pytest -s prints them).

Exact requirements: rows an update does not reach keep their table, state and accumulator bits; an updated marked row's
accumulator is exactly 0; unmarked accumulator rows hold NaN before the call and after it (neither sweep reads or writes
them); NaN guards before and after every table, accumulator and state buffer keep their bits; Adam's step counts move
by exactly 1.  Marks, samplers, hash set, batch gather and step advance are compared bit for bit with restatements
(Philox4x32-10 and splitmix64 in numpy).

Which case covers which part of the envelope:
  every dim 1..16, dim % 4 == 0 up to 512, 513, 524, 1028, 4096, 10000; 1..8 tables a call, marked and unmarked,
    vec and scalar reached by dim % 4 and by a pointer one float off, rows 1 / 31 / 32 / 33, every rule with and
    without weight decay and clip (scale < 1 and == 1), both row modes, Adam tables at different step counts ........
    ................................................................................... test_update_dims
  rows past sm_count 8 8 32 (a second grid-stride pass of the sweep) and ALL units past sm_count 8 256 4 ...........
    ................................................................................... test_update_grid_stride
  three calls in a row, each measured on its own inputs (Adam at t = 1, 2, 3) ......... test_update_three_calls
  kgrec_rows_update_dev / _ex_dev with a StepState, the legacy host bias terms ........ test_update_entry_points
  ALL past 2^32 units (64-bit quotient; about 38 GB) .................................. test_update_all_past_32_bits
  keep_acc across two calls, and its rejection in one call ............................ test_keep_acc_*
  clip norm: the shapes above, NaN unmarked rows, a nonzero start, no marked row ...... test_sqnorm_*
  marks: 1..8 segments (empty ones among them), shared and separate marks, compact + remap, int32 / int64, out of
    range, past sm_count 16 256 ids, _dev ............................................. test_rows_mark
  regularisers: d 1..300, vec / scalar both ways, ids NULL / int32 / int64, repeats, out of range, NULL outputs,
    scale != 1, n past sm_count 8 8 ................................................... test_reg_*
  samplers: unfiltered / filtered, scans and keys with no valid negative, n_cat 2 and 2^31 - 1, int32 / int64, past
    sm_count 16 256 draws, _dev seeds ................................................ test_sample_*
  hash set with repeated keys ......................................................... test_hashset_build
  batch gather (1..4 columns, int32 / int64, bad positions and rows, past sm_count 4 256) and step advance ........
    ................................................................................... test_batch_gather, test_step_advance
On the CPU: the restated dispatch rules, and the keep_acc rejection with its message.
Profiles name the kernel each case was meant to reach (the union of a test's captures; a capture that lost its kernel
records is taken again).  When no capture of a test delivers any kernel record -- seen after other profiled tests in
the same process -- the test warns that its dispatch was not checked; every other check still runs.
Run time on one H100 80GB HBM3 at a 700 W power limit: about 36 s for the GPU cases, the 38 GB case included.
"""
import ctypes as C
import re
import time
import warnings

import numpy as np
import pytest
import torch

U24 = 2.0 ** -24
C_BOUND = 1
POWF_ULPS = 4
FAKE = 0x7000_0000_1000
INVALID = 1                                   # KGREC_ERR_INVALID
SGD, ADAGRAD, ADAM, RMSPROP = 0, 1, 2, 3
TOUCHED, ALL = 0, 1
GUARD = 4                                     # NaN floats before and after every optimizer buffer (16 bytes)
f32 = np.float32
KEEP_MSG = ("sparse row optimizer: table %d reads the accumulator that table %d of the same call clears (keep_acc = 0); "
            "an accumulator cleared by one entry is read by no other entry of the call")


# ---- the dispatch, restated ------------------------------------------------------------------------------------------
def update_kernel(kind, mode, momentum, wd):
    """rows_update_ex: ROWS_ALL runs k_rows_update_all, except for plain SGD and Adagrad without weight decay."""
    plain = (kind == SGD and momentum == 0) or kind == ADAGRAD
    return "k_rows_update_all" if mode == ALL and not (plain and wd == 0) else "k_rows_update"


def vec_rule(dim, ptrs):
    """sweep_args: the 128-bit path takes dim % 4 == 0 and every non-NULL pointer 16-byte aligned."""
    return dim % 4 == 0 and all(p is None or p % 16 == 0 for p in ptrs)


def div_rule(dim):
    """sweep_args: rows wider than 512 floats are swept as dim / seg rows of seg floats, seg the largest multiple of 4
    in 64..512 dividing dim."""
    if dim > 512:
        for seg in range(512, 63, -4):
            if dim % seg == 0:
                return dim // seg
    return 1


DIMS = list(range(1, 17)) + list(range(20, 513, 4)) + [513, 524, 1028, 4096, 10000]


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_dispatch_rules_restated():
    """The restated rules on the shapes this file uses: the segmentation the sweeps apply to the wide dims, the vec
    rule's two routes off the 128-bit path, and the row-mode rule for every rule setting."""
    assert {d: div_rule(d) for d in DIMS if div_rule(d) != 1} == {4096: 8, 10000: 20}
    assert [div_rule(d) for d in (512, 513, 516, 524, 1028, 1024, 2048)] == [1, 1, 3, 1, 1, 2, 4]
    assert vec_rule(8, (256, 512, None, None)) and vec_rule(4096, (16, 32, 48, 64))
    assert not vec_rule(6, (256, 512, None, None)) and not vec_rule(8, (256, 516, None, None))
    assert not vec_rule(8, (256, 512, 260, None)) and not vec_rule(8, (256, 512, 272, 4))
    want = {(SGD, 0, 0): "k_rows_update", (SGD, 0.9, 0): "k_rows_update_all", (SGD, 0, 1e-2): "k_rows_update_all",
            (ADAGRAD, 0, 0): "k_rows_update", (ADAGRAD, 0, 1e-2): "k_rows_update_all",
            (ADAM, 0, 0): "k_rows_update_all", (RMSPROP, 0, 0): "k_rows_update_all",
            (RMSPROP, 0.9, 1e-2): "k_rows_update_all"}
    for (kind, mom, wd), name in want.items():
        assert update_kernel(kind, ALL, mom, wd) == name
        assert update_kernel(kind, TOUCHED, mom, wd) == "k_rows_update"


def test_keep_acc_rejected_in_one_call_without_a_gpu():
    """Every update entry point refuses a call in which one entry clears an accumulator another entry reads: the
    entries share it (keep_acc = 1 on either side, or on neither) or overlap it by one row; the message names the rule.
    (test_keep_acc_shared_in_one_call runs the calls this rule lets through.)"""
    from kgrec_b200 import _lib
    lib = _lib.load()

    def tabs(*es):
        return (_lib.OptTable * len(es))(*[_lib.OptTable(table=FAKE + 0x100000 * (i + 1), acc=acc, state1=FAKE,
                                                         state2=FAKE, marks=None, rows=rows, dim=8, keep_acc=keep)
                                           for i, (acc, rows, keep) in enumerate(es)])
    P = _lib.OptParams(kind=0, rows=ALL, lr=0.1, eps=1e-8, beta1=0.9, beta2=0.999, alpha=0.99, momentum=0.0,
                       weight_decay=1e-2, max_norm=1.0, step_counts=None)
    calls = [lambda t, n: lib.kgrec_rows_update_ex(t, n, 1, C.byref(P), None, None),
             lambda t, n: lib.kgrec_rows_update_ex_dev(t, n, FAKE, C.byref(P), None, None),
             lambda t, n: lib.kgrec_rows_update(t, n, 1, 0, 0.1, 1e-8, 0.9, 0.999, 1, 0.0, None, 0.0, None),
             lambda t, n: lib.kgrec_rows_update_dev(t, n, FAKE, 0, 1e-8, 0.9, 0.999, 0.0, None, 0.0, None)]
    A, B = FAKE, FAKE + 0x40000
    cases = [((A, 10, 1), (A, 10, 0), (0, 1)),                     # keep, then the entry that clears it
             ((A, 10, 0), (A, 10, 1), (1, 0)),                     # the clearing entry first
             ((A, 10, 0), (A, 10, 0), (0, 1)),                     # both clear
             ((A, 10, 1), (A + 9 * 32, 4, 0), (0, 1)),             # overlap by one row
             ((B, 3, 0), (A, 10, 1), (A + 9 * 32, 4, 0), (1, 2))]
    for call in calls:
        for *es, (t, o) in cases:
            assert call(tabs(*es), len(es)) == INVALID, es
            assert lib.kgrec_last_error().decode() == KEEP_MSG % (t, o), es
    # the clip norm reads accumulators only: the rule is not the sqnorm sweep's
    rc = lib.kgrec_rows_sqnorm(tabs((A, 10, 1), (A, 10, 0)), 2, 1, None, None)
    assert rc == INVALID and lib.kgrec_last_error().decode() == "sqnorm is NULL"


# ---- float64 values with their twin and operation count --------------------------------------------------------------
class T:
    """A value of the kernel's computation in float64 (v), its absolute-value twin (w) and a count k of rounded
    operations such that |kernel - v| <= k 2^-24 w to first order: sums take the larger count plus one, products
    and quotients the sum plus one."""
    __slots__ = ("v", "w", "k")

    def __init__(self, v, w=None, k=0):
        self.v = np.asarray(v, np.float64)
        self.w = np.abs(self.v) if w is None else np.asarray(w, np.float64)
        self.k = k


def add(a, b):
    return T(a.v + b.v, a.w + b.w, max(a.k, b.k) + 1)


def sub(a, b):
    return T(a.v - b.v, a.w + b.w, max(a.k, b.k) + 1)


def mul(a, b):
    return T(a.v * b.v, a.w * b.w, a.k + b.k + 1)


def div(a, b):
    return T(a.v / b.v, a.w * b.w / (b.v * b.v), a.k + b.k + 1)


def sqrt(a):
    s = np.sqrt(a.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        w = np.where(s > 0, a.w / np.where(s > 0, s, 1.0), np.sqrt(a.w))
    return T(s, w, a.k + 1)


def fma(a, b, c):
    return T(a.v * b.v + c.v, a.w * b.w + c.w, max(a.k + b.k, c.k) + 1)


def K(x):
    """A float32 constant of the call, exact."""
    return T(float(f32(x)))


# ---- the rules, restated (opt_elem) ----------------------------------------------------------------------------------
class Rule:
    def __init__(self, kind, momentum=0.0, wd=0.0, clip=None, lr=0.05):
        self.kind, self.momentum, self.wd, self.clip, self.lr = kind, momentum, wd, clip, lr
        self.eps = 1e-10 if kind == ADAGRAD else 1e-8
        self.beta1, self.beta2, self.alpha = 0.9, 0.999, 0.99
        for c in (self.beta1, self.beta2, self.alpha):
            assert float(f32(1) - f32(c)) == 1.0 - float(f32(c))          # 1 - c is exact in float32
        self.use_s1 = kind != SGD or momentum != 0
        self.use_s2 = kind == ADAM or (kind == RMSPROP and momentum != 0)

    def __repr__(self):
        return "%s%s%s%s" % (["sgd", "adagrad", "adam", "rmsprop"][self.kind], "-mom" if self.momentum else "",
                             "-wd" if self.wd else "", {None: "", "lt1": "-clip", "eq1": "-clip1"}[self.clip])

    def bias(self, t):
        """(1 - beta1^t, sqrt(1 - beta2^t)) as T, and the relative error powf's result brings into the update."""
        out, cond = [], 0.0
        for beta, half in ((self.beta1, 1.0), (self.beta2, 0.5)):
            bt = float(f32(beta)) ** t
            out.append(1.0 - bt)
            cond += half * POWF_ULPS * float(np.spacing(f32(bt))) / (1.0 - bt)
        return T(out[0], k=1), sqrt(T(out[1], k=1)), cond

    def apply(self, p, g, s1, s2, t, lr=None):
        """opt_elem on T values: (p', s1', s2', Adam's conditioning term per element or 0)."""
        lr = K(self.lr if lr is None else lr)
        if self.wd:
            g = fma(K(self.wd), p, g)
        if self.kind == SGD:
            if not self.momentum:
                return sub(p, mul(lr, g)), None, None, 0.0
            b = add(mul(K(self.momentum), s1), g)
            return sub(p, mul(lr, b)), b, None, 0.0
        if self.kind == ADAGRAD:
            s = fma(g, g, s1)
            return sub(p, div(mul(lr, g), add(sqrt(s), K(self.eps)))), s, None, 0.0
        if self.kind == RMSPROP:
            sq = fma(mul(K(f32(1) - f32(self.alpha)), g), g, mul(K(self.alpha), s1))
            q = div(g, add(sqrt(sq), K(self.eps)))
            if not self.momentum:
                return sub(p, mul(lr, q)), sq, None, 0.0
            b = add(mul(K(self.momentum), s2), q)
            return sub(p, mul(lr, b)), sq, b, 0.0
        m = add(mul(K(self.beta1), s1), mul(K(f32(1) - f32(self.beta1)), g))
        v = add(mul(K(self.beta2), s2), mul(mul(K(f32(1) - f32(self.beta2)), g), g))
        b1, b2, cond = self.bias(t)
        upd = div(mul(div(lr, b1), m), add(div(sqrt(v), b2), K(self.eps)))
        return sub(p, upd), m, v, np.abs(upd.v) * cond


def clip_scale(sq, max_norm):
    """k_rows_update's clip coefficient from the float32 *sqnorm: min(1, max_norm / (sqrt(sq) + 1e-6))."""
    if sq is None:
        return T(1.0)
    s = float(f32(max_norm)) / (np.sqrt(float(f32(sq))) + float(f32(1e-6)))
    assert abs(s - 1.0) > 1e-3, "clip coefficient on the kink of fminf"
    return T(1.0) if s >= 1.0 else T(s, s, 3)


# ---- GPU helpers -----------------------------------------------------------------------------------------------------
def _lib_():
    from kgrec_b200 import _lib
    return _lib, _lib.load()


def _kernels(fn, seen):
    """fn() under a CUDA profile; the kernel names are appended to seen (a short capture can lose records, so a test
    asserts on the union of its profiles)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
        time.sleep(0.02)            # lets the activity buffers of a microsecond-long capture arrive
    keys = [e.key for e in prof.key_averages()]
    _RAW[:] = (_RAW + [k for k in keys if "k_" in k])[-8:]
    seen.append(_kernel_names(keys))
    return out


_RAW = []          # the last raw kernel keys, for a failure message


def _kernel_names(keys):
    """The kgrec kernel identifiers in profiler keys, demangled ("kgrec::k_rows_update(kgrec::SweepArgs)") or mangled
    ("_ZN5kgrec13k_rows_updateENS_9SweepArgsE": the identifier after its length)."""
    out = set()
    for key in keys:
        out.update(re.findall(r"(?<![\w])k_\w+", key))
        for m in re.finditer(r"(\d+)(k_\w+)", key):
            out.add(m.group(2)[:int(m.group(1))])
    return out


def _again(fn, seen, names):
    """Profile fn() again (its results were checked already) while the captures lack one of names: now and then a
    capture loses its kernel records."""
    for _ in range(6):
        if all(nm in set().union(*seen) for nm in names):
            return
        _kernels(fn, seen)


def _want(seen, names, absent=()):
    got = set().union(*seen) if seen else set()
    if not got:
        # no capture of the test delivered a kernel record at all (the profiler can lose every record of a short
        # capture, more often after other profiled tests in the same process): the dispatch is not checked this time
        warnings.warn("the profiler delivered no kernel records: %s not checked" % (names,))
        return
    for nm in names:
        assert nm in got, (nm, sorted(got), _RAW)
    for nm in absent:
        assert nm not in got, (nm, sorted(got))


def _sms():
    return _lib_()[1].kgrec_sm_count()


def _p(x):
    return None if x is None else C.c_void_p(x if isinstance(x, int) else x.data_ptr())


class Guarded:
    """A float32 device buffer of host's values between NaN guards of GUARD floats, `off` floats past a 16-byte
    boundary (torch's allocations are 512-byte aligned)."""

    def __init__(self, host, off=0):
        host = np.ascontiguousarray(host, f32).ravel()
        self.n, self.off = host.size, off
        full = np.full(GUARD + off + self.n + GUARD, np.nan, f32)
        full[GUARD + off:GUARD + off + self.n] = host
        self.full0 = full.view(np.int32).copy()
        self.base = torch.from_numpy(full).cuda()
        self.ptr = self.base.data_ptr() + 4 * (GUARD + off)
        assert (self.ptr % 16 == 0) == (off == 0)

    def get(self):
        full = self.base.cpu().numpy()
        bits = full.view(np.int32)
        lo, hi = GUARD + self.off, GUARD + self.off + self.n
        assert np.array_equal(bits[:lo], self.full0[:lo]) and np.array_equal(bits[hi:], self.full0[hi:]), "guard"
        return full[lo:hi].copy()


def _same_bits(a, b):
    return np.array_equal(np.asarray(a, f32).view(np.int32), np.asarray(b, f32).view(np.int32))


class Ratio:
    """The largest measured |kernel - ref| / bound of a group of checks (reported with -s)."""
    worst = {}

    @classmethod
    def note(cls, group, r):
        cls.worst[group] = max(cls.worst.get(group, 0.0), float(r))


def _check_bound(got, ref, bound, tag, group="optimizer"):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    assert np.all(np.isfinite(got)), tag
    bad = err > C_BOUND * bound
    if bad.any():
        i = int(np.flatnonzero(bad.ravel())[0])
        raise AssertionError("%s: %d elements over the bound; first at %d: got %r ref %r bound %r" % (
            tag, int(bad.sum()), i, got.ravel()[i], ref.ravel()[i], (C_BOUND * bound).ravel()[i]))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), 0.0)
    Ratio.note(group, r.max() if r.size else 0.0)


# ---- optimizer tables ------------------------------------------------------------------------------------------------
class Tab:
    """One table entry: parameters, accumulator, state in guarded device buffers, and the marks (NULL: every row).
    Unmarked accumulator rows hold NaN.  offs: floats off 16-byte alignment of (table, acc, state1, state2)."""

    def __init__(self, rng, rule, rows, dim, marked, epoch, offs=(0, 0, 0, 0), frac=0.6):
        self.rows, self.dim, self.rule, self.offs, self.marked = rows, dim, rule, offs, marked
        self.p = (rng.randn(rows, dim) * 0.5).astype(f32)
        pos = rule.kind in (ADAGRAD, RMSPROP)
        self.s1 = ((rng.rand(rows, dim) * 0.02 if pos else rng.randn(rows, dim) * 0.05).astype(f32)
                   if rule.use_s1 else None)
        self.s2 = ((rng.rand(rows, dim) * 1e-3 if rule.kind == ADAM else rng.randn(rows, dim) * 0.05).astype(f32)
                   if rule.use_s2 else None)
        self.renew(rng, epoch, frac)

    def renew(self, rng, epoch, frac=0.6, outs=None):
        """Fresh marks and accumulator (and, from outs, the last call's parameters and state), uploaded."""
        rows, dim = self.rows, self.dim
        if outs is not None:
            self.p, _, self.s1, self.s2 = outs
        self.mk = (rng.rand(rows) < frac) if self.marked else np.ones(rows, bool)
        if self.marked and rows > 1:
            self.mk[rng.randint(rows)] = False
        self.acc = np.where(self.mk[:, None], rng.randn(rows, dim) * 0.1, np.nan).astype(f32)
        self.marks = None
        if self.marked:
            other = epoch - 1 - rng.randint(0, 1 << 20, rows)
            self.marks = torch.as_tensor(np.where(self.mk, epoch, other).astype(np.int32), device="cuda")
        self.b = [Guarded(x, o) if x is not None else None
                  for x, o in zip((self.p, self.acc, self.s1, self.s2), self.offs)]

    def ptrs(self):
        return tuple(None if b is None else b.ptr for b in self.b)

    def vec(self):
        return vec_rule(self.dim, self.ptrs())

    def entry(self, keep=0):
        from kgrec_b200 import _lib
        t, a, s1, s2 = self.ptrs()
        return _lib.OptTable(table=t, acc=a, state1=s1, state2=s2, marks=_p(self.marks), rows=self.rows, dim=self.dim,
                             keep_acc=keep)

    def read(self):
        return [None if b is None else b.get().reshape(self.rows, self.dim) for b in self.b]

    def check(self, mode, scale, t, tag, lr=None, acc_seen=None, keep=False):
        """The table after one update against the rule on its inputs; the exact requirements on every row."""
        rule = self.rule
        p1, a1, s11, s21 = self.read()
        every = mode == ALL and update_kernel(rule.kind, mode, rule.momentum, rule.wd) == "k_rows_update_all"
        upd = np.ones(self.rows, bool) if every else self.mk
        acc_in = self.acc if acc_seen is None else acc_seen
        g0 = np.where(self.mk[:, None], acc_in, 0.0)
        g = mul(T(g0, np.abs(g0)), scale)
        z = np.zeros_like(self.p, np.float64)
        s1 = T(self.s1) if self.s1 is not None else T(z)
        s2 = T(self.s2) if self.s2 is not None else T(z)
        pr, r1, r2, cond = rule.apply(T(self.p), g, s1, s2, t, lr)
        u = upd
        for got, old, ref, extra, what in ((p1, self.p, pr, cond, "table"), (s11, self.s1, r1, 0.0, "state1"),
                                           (s21, self.s2, r2, 0.0, "state2")):
            if old is None:
                continue
            bound = pr.k * U24 * ref.w + extra if what == "table" else ref.k * U24 * ref.w
            bound = np.broadcast_to(bound, ref.v.shape)
            _check_bound(got[u], ref.v[u], bound[u], "%s %s" % (tag, what))
            assert _same_bits(got[~u], old[~u]), "%s %s: a row the update does not reach moved" % (tag, what)
        if keep:
            assert _same_bits(a1, acc_in), "%s: keep_acc changed the accumulator" % tag
        else:
            assert np.all(a1[self.mk] == 0) and not np.signbit(a1[self.mk]).any(), "%s: acc not cleared" % tag
            assert np.all(np.isnan(a1[~self.mk])), "%s: an unmarked accumulator row was written" % tag
        return p1, a1, s11, s21


def _params(rule, mode, steps):
    from kgrec_b200 import _lib
    return _lib.OptParams(kind=rule.kind, rows=mode, lr=rule.lr, eps=rule.eps, beta1=rule.beta1, beta2=rule.beta2,
                          alpha=rule.alpha, momentum=rule.momentum, weight_decay=rule.wd,
                          max_norm=1.0 if rule.clip == "lt1" else 1e3, step_counts=_p(steps))


def _sqnorm(rule):
    """(device *sqnorm, its value): 25 with max_norm 1 (scale about 0.2) or 1e3 (scale 1); None without clip."""
    if rule.clip is None:
        return None, None
    return torch.full((1,), 25.0, device="cuda"), 25.0


def _run_update(rule, tabs, mode, epoch, tag, seen=None, entry="ex", steps0=None, state=None, legacy_step=None):
    """One update call of tabs; every table checked.  Returns the tables' outputs."""
    _lib, lib = _lib_()
    n = len(tabs)
    arr = (_lib.OptTable * n)(*[t.entry() for t in tabs])
    sq, sqv = _sqnorm(rule)
    max_norm = 1.0 if rule.clip == "lt1" else 1e3
    steps = None
    if entry in ("ex", "ex_dev") and rule.kind == ADAM:
        steps0 = np.asarray(steps0 if steps0 is not None else [0] * n, np.int64)
        steps = torch.as_tensor(steps0, device="cuda")

    def call():
        if entry == "ex":
            P = _params(rule, mode, steps)
            _lib.check(lib.kgrec_rows_update_ex(arr, n, epoch, C.byref(P), _p(sq), None))
        elif entry == "ex_dev":
            P = _params(rule, mode, steps)
            P.lr = 123.0                                   # _ex_dev reads the state's
            _lib.check(lib.kgrec_rows_update_ex_dev(arr, n, state.ptr, C.byref(P), _p(sq), None))
        elif entry == "legacy":
            _lib.check(lib.kgrec_rows_update(arr, n, epoch, rule.kind, rule.lr, rule.eps, rule.beta1, rule.beta2,
                                             legacy_step, rule.wd, _p(sq), max_norm, None))
        else:
            _lib.check(lib.kgrec_rows_update_dev(arr, n, state.ptr, rule.kind, rule.eps, rule.beta1, rule.beta2,
                                                 rule.wd, _p(sq), max_norm, None))
    if seen is not None:
        _kernels(call, seen)
    else:
        call()
        torch.cuda.synchronize()
    scale = clip_scale(sqv, max_norm)
    if steps is not None:
        assert np.array_equal(steps.cpu().numpy(), steps0 + 1), tag + " step counts"
    outs = []
    for i, tb in enumerate(tabs):
        t = steps0[i] + 1 if steps is not None else (legacy_step if legacy_step is not None else 1)
        if entry == "dev" and state is not None:
            t = state.read()["step"]
        lr = state.read()["lr"] if entry in ("ex_dev", "dev") else None
        outs.append(tb.check(mode if entry in ("ex", "ex_dev") else TOUCHED, scale, t,
                             "%s table %d (%d x %d)" % (tag, i, tb.rows, tb.dim), lr=lr))
    if seen is not None:
        ex = entry in ("ex", "ex_dev")
        _again(call, seen, [update_kernel(rule.kind, mode, rule.momentum, rule.wd) if ex else "k_rows_update"] +
               (["k_step_counts"] if steps is not None else []))
    return outs


def _dim_specs(rng, rule):
    """(rows, dim, marked, offs) for every dim of DIMS: rows 1 / 31 / 32 / 33 and others, marks on two tables in three,
    every third dim % 4 == 0 table with one pointer a float off (the ones the rule has)."""
    out = []
    rows_cycle = [33, 1, 31, 32, 7, 64, 45, 100]
    live = [0, 1] + ([2] if rule.use_s1 else []) + ([3] if rule.use_s2 else [])
    for i, d in enumerate(DIMS):
        rows = rows_cycle[i % len(rows_cycle)]
        if d >= 1028:
            rows = min(rows, 33 if d < 10000 else 13)
        offs = [0, 0, 0, 0]
        if d % 4 == 0 and i % 3 == 0:
            offs[live[(i // 3) % len(live)]] = 1
        out.append((rows, d, i % 3 != 2, tuple(offs)))
    return out


RULES = [Rule(SGD), Rule(SGD, wd=1e-2, clip="eq1"), Rule(SGD, 0.9, clip="lt1"), Rule(SGD, 0.9, 1e-2, "lt1"),
         Rule(ADAGRAD, clip="lt1"), Rule(ADAGRAD, wd=1e-2),
         Rule(ADAM), Rule(ADAM, wd=1e-2, clip="lt1"),
         Rule(RMSPROP, clip="eq1"), Rule(RMSPROP, wd=1e-2, clip="lt1"), Rule(RMSPROP, 0.9), Rule(RMSPROP, 0.9, 1e-2, "lt1")]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [TOUCHED, ALL], ids=["touched", "all"])
@pytest.mark.parametrize("rule", RULES, ids=repr)
def test_update_dims(rule, mode):
    """Every dim of DIMS through kgrec_rows_update_ex, 1..8 tables a call (marked and unmarked, both paths each way),
    Adam tables at step counts 0, 1, 4, 99, ... in one call; the intended sweep from the profile."""
    rng = np.random.RandomState(1000 + 10 * RULES.index(rule) + mode)
    specs = _dim_specs(rng, rule)
    seen, routes, i, size, epoch = [], set(), 0, 1, 11
    while i < len(specs):
        group = specs[i:i + size]
        tabs = [Tab(rng, rule, r, d, m, epoch, o) for r, d, m, o in group]
        routes |= {(tb.vec(), tb.dim % 4 == 0) for tb in tabs}
        steps0 = [0, 1, 4, 99, 0, 2, 9, 1000][:len(tabs)]
        _run_update(rule, tabs, mode, epoch, "%r dims %s" % (rule, [d for _, d, _, _ in group]),
                    seen if i == 0 else None, steps0=steps0)
        i += size
        size = size % 8 + 1
        epoch += 1
    assert routes == {(True, True), (False, True), (False, False)}
    name = update_kernel(rule.kind, mode, rule.momentum, rule.wd)
    other = "k_rows_update_all" if name == "k_rows_update" else "k_rows_update"
    _want(seen, [name] + (["k_step_counts"] if rule.kind == ADAM else []), absent=[other])


@pytest.mark.gpu
@pytest.mark.parametrize("rule", [Rule(ADAM, wd=1e-2, clip="lt1"), Rule(SGD, wd=1e-2)], ids=repr)
@pytest.mark.parametrize("mode", [TOUCHED, ALL], ids=["touched", "all"])
def test_update_grid_stride(rule, mode):
    """Rows past sm_count 8 8 32 in one table (the sweep's second grid-stride pass), and in ALL past sm_count 8 256 4
    units (k_rows_update_all's second pass): a marked vec table, a marked scalar one and a small unmarked one."""
    rng = np.random.RandomState(7 + mode)
    rows = _sms() * 8 * 8 * 32 + 1000
    assert rows * 5 > _sms() * 8 * 256 * 4
    tabs = [Tab(rng, rule, rows, 4, True, 3), Tab(rng, rule, rows, 5, True, 3, frac=0.3), Tab(rng, rule, 33, 12, False, 3)]
    seen = []
    _run_update(rule, tabs, mode, 3, "%r grid stride" % rule, seen, steps0=[2, 0, 7])
    name = update_kernel(rule.kind, mode, rule.momentum, rule.wd)
    _want(seen, [name])


@pytest.mark.gpu
@pytest.mark.parametrize("rule", [Rule(ADAM, clip="lt1"), Rule(RMSPROP, 0.9, 1e-2), Rule(SGD, 0.9, 1e-2, "lt1")],
                         ids=repr)
def test_update_three_calls(rule):
    """Three calls in a row on the same tables; each call's outputs are the next call's inputs, with a fresh
    accumulator and fresh marks: errors are measured per call (Adam at t = 1, 2, 3, where powf's error is largest)."""
    rng = np.random.RandomState(3)
    specs = [(40, 8, True, (0, 0, 0, 0)), (33, 7, True, (0, 0, 0, 0)), (20, 4096, False, (0, 0, 0, 0)),
             (31, 12, True, (0, 1, 0, 0))]
    tabs = [Tab(rng, rule, r, d, m, 1, o) for r, d, m, o in specs]
    steps = np.zeros(len(tabs), np.int64)
    for call in range(3):
        epoch = 1 + call
        if call:
            for tb, out in zip(tabs, outs):
                tb.renew(rng, epoch, outs=out)
        outs = _run_update(rule, tabs, ALL, epoch, "%r call %d" % (rule, call), steps0=steps)
        steps = steps + 1


@pytest.mark.gpu
def test_update_entry_points():
    """kgrec_rows_update_ex_dev and kgrec_rows_update_dev with epoch, lr and (for _dev) Adam's step read from a
    StepState; the legacy kgrec_rows_update with Adam's bias terms formed on the host, at steps 1, 2 and 1000."""
    from kgrec_b200.train import StepState
    rng = np.random.RandomState(21)
    specs = [(33, 16, True, (0, 0, 0, 0)), (31, 6, True, (0, 0, 0, 0)), (5, 10000, True, (0, 0, 0, 0)),
             (32, 20, False, (0, 0, 1, 0))]
    seen = []
    for rule in (Rule(ADAM, wd=1e-2, clip="lt1"), Rule(RMSPROP, 0.9, 1e-2, "lt1"), Rule(SGD, wd=1e-2)):
        for mode in (TOUCHED, ALL):
            state = StepState("cuda", step=5, epoch=77, lr=0.03)
            tabs = [Tab(rng, rule, r, d, m, 77, o) for r, d, m, o in specs]
            _run_update(rule, tabs, mode, 0, "%r ex_dev" % rule, seen, entry="ex_dev", steps0=[3, 0, 1, 8],
                        state=state)
    for rule in (Rule(ADAM, wd=1e-2, clip="lt1"), Rule(ADAGRAD, clip="lt1"), Rule(SGD, wd=1e-2)):
        for step in (1, 2, 1000):
            state = StepState("cuda", step=step, epoch=9, lr=0.02)
            tabs = [Tab(rng, rule, r, d, m, 9, o) for r, d, m, o in specs]
            _run_update(rule, tabs, TOUCHED, 0, "%r dev step %d" % (rule, step), seen, entry="dev", state=state)
            tabs = [Tab(rng, rule, r, d, m, 4, o) for r, d, m, o in specs]
            _run_update(rule, tabs, TOUCHED, 4, "%r legacy step %d" % (rule, step), seen, entry="legacy",
                        legacy_step=step)
    _want(seen, ["k_rows_update", "k_rows_update_all", "k_step_counts"])


@pytest.mark.gpu
def test_update_all_past_32_bits():
    """One scalar-path ALL call (SGD with weight decay, no state) over a single table of more than 2^32 units, so
    k_rows_update_all takes its 64-bit quotient for the units past 2^32 - 1: a wrong row there reads a wrong mark.
    Marks every third row; checked in chunks on the device against the rule in float64."""
    dim = 5
    rows = (1 << 32) // dim + 300_000
    units = rows * dim
    need = units * 8 + rows * 4 + (5 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
    _lib, lib = _lib_()
    epoch, lr, wd = 5, f32(0.25), f32(0.125)
    table = torch.empty(units, device="cuda")
    acc = torch.empty(units, device="cuda")
    marks = torch.empty(rows, dtype=torch.int32, device="cuda")
    CH = 1 << 26

    def chunk(a, b):
        u = torch.arange(a, b, device="cuda", dtype=torch.int64)
        r = u // dim
        mk = (r % 3) == 0
        p = ((u % 13) - 6).float() * 0.125
        g = ((u % 11) - 5).float() * 0.0625
        return u, r, mk, p, g
    for a in range(0, units, CH):
        b = min(units, a + CH)
        u, r, mk, p, g = chunk(a, b)
        table[a:b] = p
        acc[a:b] = torch.where(mk, g, torch.full_like(g, float("nan")))
        del u, r, mk, p, g
    for a in range(0, rows, CH):
        b = min(rows, a + CH)
        r = torch.arange(a, b, device="cuda", dtype=torch.int64)
        marks[a:b] = torch.where(r % 3 == 0, epoch, epoch - 1).int()
    arr = (_lib.OptTable * 1)(_lib.OptTable(table=table.data_ptr(), acc=acc.data_ptr(), marks=marks.data_ptr(),
                                            rows=rows, dim=dim))
    P = _lib.OptParams(kind=SGD, rows=ALL, lr=float(lr), eps=1e-8, weight_decay=float(wd), max_norm=1.0)
    seen = []
    _kernels(lambda: _lib.check(lib.kgrec_rows_update_ex(arr, 1, epoch, C.byref(P), None, None)), seen)
    for a in range(0, units, CH):
        b = min(units, a + CH)
        u, r, mk, p, g = chunk(a, b)
        g = torch.where(mk, g, torch.zeros_like(g)).double()
        p = p.double()
        ref = p - float(lr) * (float(wd) * p + g)
        bound = 3 * U24 * (p.abs() + float(lr) * (float(wd) * p.abs() + g.abs()))
        err = (table[a:b].double() - ref).abs()
        assert bool((err <= C_BOUND * bound).all()), "units %d..%d" % (a, b)
        got = acc[a:b]
        assert bool((got[mk] == 0).all()) and bool(got[~mk].isnan().all()), "acc, units %d..%d" % (a, b)
        del u, r, mk, p, g, ref, bound, err, got
    _again(lambda: _lib.check(lib.kgrec_rows_update_ex(arr, 1, epoch, C.byref(P), None, None)), seen,
           ["k_rows_update_all"])
    _want(seen, ["k_rows_update_all"])


# ---- keep_acc ------------------------------------------------------------------------------------------------------
def _shared_pair(rng, rule, rows, dim, epoch):
    """Two table entries with their own parameters and state and one accumulator."""
    a, b = Tab(rng, rule, rows, dim, True, epoch), Tab(rng, rule, rows, dim, True, epoch)
    b.mk, b.marks, b.acc, b.b[1] = a.mk, a.marks, a.acc, a.b[1]
    return a, b


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [TOUCHED, ALL], ids=["touched", "all"])
def test_keep_acc_across_two_calls(mode):
    """Entry A keeps the shared accumulator in one call, entry B clears it in the next: both step with the same
    gradient, and A's call leaves the accumulator bit for bit."""
    _lib, lib = _lib_()
    rule = Rule(RMSPROP, 0.9, 1e-2)
    rng = np.random.RandomState(5)
    for rows, dim in ((_sms() * 64 * 32, 4), (100, 7)):
        a, b = _shared_pair(rng, rule, rows, dim, 2)
        P = _params(rule, mode, None)
        _lib.check(lib.kgrec_rows_update_ex((_lib.OptTable * 1)(a.entry(keep=1)), 1, 2, C.byref(P), None, None))
        a.check(mode, T(1.0), 1, "keep", keep=True)
        _lib.check(lib.kgrec_rows_update_ex((_lib.OptTable * 1)(b.entry()), 1, 2, C.byref(P), None, None))
        b.check(mode, T(1.0), 1, "clear")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [TOUCHED, ALL], ids=["touched", "all"])
def test_keep_acc_shared_in_one_call(mode):
    """The same two entries in one call.  With the clearing entry first and sm_count 64 chunks of 32 rows a table,
    warp w of the touched-row sweep updates row block w of the clearing entry and then the same block of the keeping
    entry, which would read the accumulator already cleared and step with a zero gradient (in other layouts, and in
    the ALL sweep, the two race).  The call is refused instead, whatever the order of the entries, and nothing moves;
    entries that both keep a shared accumulator run as before."""
    _lib, lib = _lib_()
    rule = Rule(RMSPROP, 0.9, 1e-2)
    rng = np.random.RandomState(6)
    a, b = _shared_pair(rng, rule, _sms() * 64 * 32, 4, 2)
    P = _params(rule, mode, None)
    for order, msg in (((b.entry(), a.entry(keep=1)), KEEP_MSG % (1, 0)), ((a.entry(keep=1), b.entry()),
                                                                           KEEP_MSG % (0, 1))):
        with pytest.raises(RuntimeError) as e:
            _lib.check(lib.kgrec_rows_update_ex((_lib.OptTable * 2)(*order), 2, 2, C.byref(P), None, None))
        assert msg in str(e.value)
    torch.cuda.synchronize()
    for tb in (a, b):
        p1, a1, s1, s2 = tb.read()
        assert _same_bits(p1, tb.p) and _same_bits(a1, tb.acc) and _same_bits(s1, tb.s1) and _same_bits(s2, tb.s2)
    _lib.check(lib.kgrec_rows_update_ex((_lib.OptTable * 2)(a.entry(keep=1), b.entry(keep=1)), 2, 2, C.byref(P),
                                        None, None))
    a.check(mode, T(1.0), 1, "keep a", keep=True)
    b.check(mode, T(1.0), 1, "keep b", keep=True)


# ---- clip norm -------------------------------------------------------------------------------------------------------
def _sqnorm_chain(tabs, sms):
    """The longest addition chain of k_rows_sqnorm for these tables: one warp's fmas over the 32-row chunks it
    sweeps (vec rows in batches of kRowsInFlight = 4, padding included), warp_sum, the CTA's 8 partials, one atomic
    per CTA, the initial value."""
    costs = []
    for tb in tabs:
        div = div_rule(tb.dim)
        rows, dim = tb.rows * div, tb.dim // div
        mk = np.repeat(tb.mk, div)
        nchunk = (rows + 31) // 32
        m = np.bincount(np.arange(rows) // 32, weights=mk, minlength=nchunk).astype(np.int64)
        per = ((dim + 3) // 4 + 31) // 32
        costs.append(per * (((m + 3) // 4) * 16 if tb.vec() else m * 4))
    cost = np.concatenate(costs)
    grid = max(1, min((cost.size + 7) // 8, sms * 8))
    per_warp = np.bincount(np.arange(cost.size) % (grid * 8), weights=cost)
    return int(per_warp.max()) + 5 + 8 + grid + 1


def _run_sqnorm(tabs, epoch, init, seen=None, state=None):
    _lib, lib = _lib_()
    arr = (_lib.OptTable * len(tabs))(*[t.entry() for t in tabs])
    sq = torch.full((1,), init, device="cuda")
    if state is None:
        fn = lambda: _lib.check(lib.kgrec_rows_sqnorm(arr, len(tabs), epoch, _p(sq), None))       # noqa: E731
    else:
        fn = lambda: _lib.check(lib.kgrec_rows_sqnorm_dev(arr, len(tabs), state.ptr, _p(sq), None))  # noqa: E731
    if seen is not None:
        _kernels(fn, seen)
    else:
        fn()
    got = float(sq.item())
    for tb in tabs:
        p1, a1, s1, s2 = tb.read()
        assert _same_bits(a1, tb.acc) and _same_bits(p1, tb.p), "the clip norm wrote a table"
    if seen is not None:
        _again(fn, seen, ["k_rows_sqnorm"])
    ref = float(f32(init)) + sum(float(np.sum(np.square(tb.acc[tb.mk].astype(np.float64)))) for tb in tabs)
    return got, ref


@pytest.mark.gpu
def test_sqnorm_dims():
    """Every dim of DIMS in 1..8 tables a call (NaN in every unmarked row), rows past sm_count 8 8 32, a nonzero
    start, and the _dev entry point's epoch: against the float64 sum of squares of the marked rows."""
    from kgrec_b200.train import StepState
    rng = np.random.RandomState(31)
    rule = Rule(SGD)
    specs = _dim_specs(rng, rule) + [(_sms() * 2048 + 77, 4, True, (0, 0, 0, 0)), (_sms() * 2048 + 5, 3, True,
                                                                                     (0, 0, 0, 0))]
    seen, i, size, sms = [], 0, 1, _sms()
    while i < len(specs):
        group = specs[i:i + size]
        epoch = 40 + i
        tabs = [Tab(rng, rule, r, d, m, epoch, o) for r, d, m, o in group]
        init = float(rng.rand() * 3)
        state = StepState("cuda", step=3, epoch=epoch) if size % 2 else None
        got, ref = _run_sqnorm(tabs, epoch, init, seen if i == 0 else None, state)
        bound = _sqnorm_chain(tabs, sms) * U24 * ref
        _check_bound(np.array([got]), np.array([ref]), np.array([bound]), "sqnorm %s" % [t.dim for t in tabs],
                     "sqnorm")
        i += size
        size = size % 8 + 1
    _want(seen, ["k_rows_sqnorm"])


@pytest.mark.gpu
def test_sqnorm_no_marked_row():
    """A call whose tables have no marked row (every accumulator row NaN) leaves *sqnorm bit for bit."""
    rng = np.random.RandomState(32)
    tabs = [Tab(rng, Rule(SGD), r, d, True, 9, o, frac=0.0) for r, d, o in ((33, 8, (0, 0, 0, 0)),
                                                                            (40, 5, (0, 0, 0, 0)),
                                                                            (3, 4096, (0, 1, 0, 0)))]
    assert not any(tb.mk.any() for tb in tabs)
    got, ref = _run_sqnorm(tabs, 9, 1.5)
    assert got == 1.5 and ref == 1.5


# ---- marks -----------------------------------------------------------------------------------------------------------
def mark_ref(segs, marks, epoch):
    """k_rows_mark restated: compact (~v), then the remap, then the range check; out of range marks row 0."""
    bad = False
    for s in segs:
        v = np.asarray(s["ids"], np.int64).copy()
        if s["compact"]:
            v = np.where(v < 0, ~v, v)
        if s["remap"] is not None:
            out = (v < 0) | (v >= len(s["remap"]))
            bad |= bool(out.any())
            v = np.asarray(s["remap"], np.int64)[np.where(out, 0, v)]
        out = (v < 0) | (v >= s["rows"])
        bad |= bool(out.any())
        marks[s["marks"]][np.where(out, 0, v)] = epoch
    return bad


def _mark_case(rng, lib, _lib, segs_spec, epoch, seen=None, state=None):
    """segs_spec: (n, ib, compact, remap_len or 0, marks key, rows, out-of-range ids); one call, compared exactly."""
    keys = {}
    for *_, mk, rows, _ in segs_spec:
        keys.setdefault(mk, rows)
    marks_h = {k: rng.randint(-5, epoch, rows).astype(np.int32) for k, rows in keys.items()}
    marks_d = {k: torch.as_tensor(v, device="cuda") for k, v in marks_h.items()}
    segs, host, keep = [], [], []
    for n, ib, compact, n_remap, mk, rows, n_bad in segs_spec:
        hi = n_remap if n_remap else rows
        ids = rng.randint(0, hi, n).astype(np.int64)
        if compact:
            ids = np.where(rng.rand(n) < 0.5, ~ids, ids)
        remap = rng.randint(0, rows, n_remap).astype(np.int32) if n_remap else None
        if remap is not None:
            remap[:2] = [0, rows - 1]
        if n_bad:
            pos = rng.choice(n, n_bad, replace=False)
            big = (1 << 40) if ib == 8 else (1 << 30)
            ids[pos] = rng.choice([hi, hi + 7, big, -1 if not compact else ~big], n_bad)
            if remap is not None:
                remap[2], ids[pos[0]] = rows, 2       # an id the remap sends out of the table's range
        dt = torch.int64 if ib == 8 else torch.int32
        idd = torch.as_tensor(ids, dtype=dt, device="cuda") if n else None
        rd = torch.as_tensor(remap, device="cuda") if remap is not None else None
        keep += [idd, rd]
        segs.append(_lib.MarkSeg(ids=_p(idd), n=n, idx_bytes=ib, compact=int(compact), remap=_p(rd),
                                 n_remap=n_remap, marks=marks_d[mk].data_ptr(), rows=rows))
        host.append(dict(ids=ids, compact=compact, remap=remap, rows=rows, marks=mk))
    status = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    arr = (_lib.MarkSeg * len(segs))(*segs)
    if state is None:
        fn = lambda: _lib.check(lib.kgrec_rows_mark(arr, len(segs), epoch, _p(status), None))          # noqa: E731
    else:
        fn = lambda: _lib.check(lib.kgrec_rows_mark_dev(arr, len(segs), state.ptr, _p(status), None))  # noqa: E731
    if seen is not None:
        _kernels(fn, seen)
    else:
        fn()
    bad = mark_ref(host, marks_h, epoch)
    for k in marks_h:
        assert np.array_equal(marks_d[k].cpu().numpy(), marks_h[k]), (segs_spec, k)
    assert int(status.item()) == (1 if bad else 7), segs_spec
    if seen is not None:
        _again(fn, seen, ["k_rows_mark"])
    return bad


@pytest.mark.gpu
def test_rows_mark():
    """1..8 segments with empty ones among them, shared and separate marks arrays, compact ids with and without a
    remap, int32 and int64 ids, out-of-range ids (of the remap and of the table), more than sm_count 16 256 ids, and
    the _dev entry point's epoch: marks and status exactly as restated."""
    from kgrec_b200.train import StepState
    _lib, lib = _lib_()
    rng = np.random.RandomState(41)
    seen, n_bad_calls = [], 0
    for n_segs in range(1, 9):
        for trial in range(4):
            spec = []
            for s in range(n_segs):
                n = 0 if (s % 3 == 1 and trial % 2) else int(rng.randint(1, 300))
                ib = (4, 8)[(s + trial) % 2]
                compact = bool((s + trial) % 3 == 0)
                n_remap = int(rng.randint(5, 60)) if (s + trial) % 4 == 1 else 0
                mk = "shared" if s % 2 == 0 else "own%d" % s
                rows = 500 if mk == "shared" else int(rng.randint(1, 400))
                bad = int(rng.randint(1, 4)) if (trial == 3 and n > 10 and s == 0) else 0
                spec.append((n, ib, compact, n_remap, mk, rows, bad))
            state = StepState("cuda", step=2, epoch=1000 + trial) if trial == 2 else None
            n_bad_calls += _mark_case(rng, lib, _lib, spec, 1000 + trial, seen if n_segs == 8 and trial == 0 else None,
                                      state)
    assert n_bad_calls >= 6
    big = _sms() * 16 * 256 + 1234
    _mark_case(rng, lib, _lib, [(big, 8, True, 0, "m", 100_000, 5), (big // 3, 4, False, 3000, "m", 100_000, 0)],
               77, seen)
    _want(seen, ["k_rows_mark"])


# ---- regularisers ----------------------------------------------------------------------------------------------------
def _reg_rows(rng, rows, d):
    """Rows with |x|^2 in [0.5, 1.5], redrawn while within the bound of the kink at 1."""
    x = rng.randn(rows, d)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x = (x * np.sqrt(rng.uniform(0.5, 1.5, rows))[:, None]).astype(f32)
    k = max(_n2_k(d, True), _n2_k(d, False))
    for _ in range(10):
        n2 = np.sum(np.square(x.astype(np.float64)), 1)
        near = np.abs(n2 - 1.0) <= 2 * k * U24 * n2
        if not near.any():
            return x
        x[near] *= f32(1.01)
    raise AssertionError("rows stay near the kink")


def _n2_k(d, vec):
    """Rounded operations of a row's |x|^2: a lane's fma chain, then warp_sum's 5 additions."""
    return ((((d + 3) // 4) + 31) // 32 * 4 if vec else (d + 31) // 32) + 5


def _reg_norm_case(rng, lib, _lib, d, rows, n, ib, off_t, off_a, scale, seen=None, no_loss=False, no_acc=False,
                   n_bad=0):
    x = _reg_rows(rng, rows, d)
    a0 = (rng.randn(rows, d) * 0.01).astype(f32)
    tb, ab = Guarded(x, off_t), Guarded(a0, off_a)
    vec = vec_rule(d, (tb.ptr, None if no_acc else ab.ptr))
    if ib:
        ids = rng.randint(0, rows, n).astype(np.int64)
        ids[:min(n, 5)] = ids[0]                                  # repeats
        if n_bad:
            ids[rng.choice(n, n_bad, replace=False)] = rng.choice([-1, rows, rows + 5, 1 << 33 if ib == 8 else -7], n_bad)
        idd = torch.as_tensor(ids, dtype=torch.int64 if ib == 8 else torch.int32, device="cuda")
    else:
        ids, idd = np.arange(n), None
    loss0 = 0.375
    loss = torch.full((1,), loss0, device="cuda")
    status = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    fn = lambda: _lib.check(lib.kgrec_reg_norm_rows(                                          # noqa: E731
        tb.ptr, rows, d, _p(idd), ib or 8, n, scale, None if no_loss else _p(loss), None if no_acc else ab.ptr,
        _p(status), None))
    _kernels(fn, seen) if seen is not None else fn()
    ok = (ids >= 0) & (ids < rows)
    r = ids[ok]
    n2 = np.sum(np.square(x.astype(np.float64)), 1)
    on = n2[r] > 1.0
    cnt = np.bincount(r[on], minlength=rows)
    s = float(f32(scale))
    k_n2 = _n2_k(d, vec)
    grid = max(1, min((n + 7) // 8, _sms() * 8))
    per_warp = (n + grid * 8 - 1) // (grid * 8)
    lref = loss0 + s * np.sum(n2[r][on] - 1.0)
    ltw = loss0 + s * np.sum(n2[r][on] + 1.0)
    lk = k_n2 + 1 + per_warp + 8 + 1 + grid + 1
    got_l = float(loss.item())
    if no_loss:
        assert got_l == loss0
    else:
        _check_bound(np.array([got_l]), np.array([lref]), np.array([lk * U24 * ltw]), "norm d %d loss" % d, "reg")
    acc = ab.get().reshape(rows, d)
    xg = x.astype(np.float64)
    aref = a0 + cnt[:, None] * 2 * s * xg
    atw = np.abs(a0) + cnt[:, None] * 2 * abs(s) * np.abs(xg)
    ak = 1 + cnt.max(initial=0)
    if no_acc:
        assert _same_bits(acc, a0)
    else:
        _check_bound(acc, aref, ak * U24 * atw, "norm d %d acc" % d, "reg")
        assert _same_bits(acc[cnt == 0], a0[cnt == 0])
    assert int(status.item()) == (1 if n_bad else 5)
    if seen is not None:
        _again(fn, seen, ["k_reg_norm_rows"])
    return vec


@pytest.mark.gpu
def test_reg_norm_rows():
    """kgrec_reg_norm_rows at every d in 1..300 (vec and scalar; scalar also by a table or accumulator a float off),
    ids NULL / int32 / int64 with repeats, out-of-range ids, NULL loss or accumulator, scale != 1, and n past
    sm_count 8 8 rows: loss and accumulator against float64."""
    _lib, lib = _lib_()
    rng = np.random.RandomState(51)
    seen, paths = [], set()
    for d in range(1, 301):
        off_t, off_a = (1, 0) if d % 12 == 4 else ((0, 1) if d % 12 == 8 else (0, 0))
        ib = (0, 4, 8)[d % 3]
        rows = 40 if d > 50 else 70
        n = rows if ib == 0 else 90
        vec = _reg_norm_case(rng, lib, _lib, d, rows, n, ib, off_t, off_a, (1.0, 0.37, 2.5)[d % 3],
                             seen if d == 1 else None, no_loss=d % 17 == 0, no_acc=d % 19 == 0,
                             n_bad=3 if (ib and d % 5 == 0) else 0)
        paths.add((vec, d % 4 == 0))
    assert paths == {(True, True), (False, True), (False, False)}
    big = _sms() * 8 * 8 + 500
    _reg_norm_case(rng, lib, _lib, 64, big, big, 0, 0, 0, 0.5, seen)
    _reg_norm_case(rng, lib, _lib, 33, 2000, big * 2, 8, 0, 0, 1.0, seen, n_bad=4)
    _want(seen, ["k_reg_norm_rows"])


def _reg_orth_case(rng, lib, _lib, d, rows, scale, seen=None, no=()):
    x = (rng.randn(rows, d) * 0.5).astype(f32)
    w = (rng.randn(rows, d) * 0.5).astype(f32)
    ar0, an0 = (rng.randn(rows, d) * 0.01).astype(f32), (rng.randn(rows, d) * 0.01).astype(f32)
    xb, wb, arb, anb = Guarded(x), Guarded(w, d % 2), Guarded(ar0, int(d % 3 == 1)), Guarded(an0)
    loss0 = -0.25
    loss = torch.full((1,), loss0, device="cuda")
    fn = lambda: _lib.check(lib.kgrec_reg_orth_tables(                                        # noqa: E731
        xb.ptr, wb.ptr, rows, d, scale, None if "loss" in no else _p(loss), None if "rel" in no else arb.ptr,
        None if "norm" in no else anb.ptr, None))
    _kernels(fn, seen) if seen is not None else fn()
    X, Wt = x.astype(np.float64), w.astype(np.float64)
    kl = (d + 31) // 32 + 5
    wr = T(np.sum(X * Wt, 1), np.sum(np.abs(X * Wt), 1), kl)
    n2 = T(np.sum(X * X, 1), None, kl)
    q = div(wr, n2)
    term = div(mul(wr, wr), n2)
    s = K(scale)
    grid = max(1, min((rows + 7) // 8, _sms() * 8))
    per_warp = (rows + grid * 8 - 1) // (grid * 8)
    lk = term.k + per_warp + 8 + 1 + grid + 1
    ltw = abs(loss0) + abs(float(s.v)) * np.sum(term.w)
    lref = loss0 + float(s.v) * np.sum(term.v)
    got_l = float(loss.item())
    if "loss" in no:
        assert got_l == loss0
    else:
        _check_bound(np.array([got_l]), np.array([lref]), np.array([lk * U24 * ltw]), "orth d %d loss" % d, "reg")
    Q, two = T(q.v[:, None], q.w[:, None], q.k), K(2.0)
    grel = mul(s, sub(mul(mul(two, Q), T(Wt)), mul(mul(mul(two, Q), Q), T(X))))
    gnrm = mul(mul(mul(s, two), Q), T(X))
    for b, a0, g, nm in ((arb, ar0, grel, "rel"), (anb, an0, gnrm, "norm")):
        got = b.get().reshape(rows, d)
        if nm in no:
            assert _same_bits(got, a0)
            continue
        ref = add(T(a0), g)
        _check_bound(got, ref.v, ref.k * U24 * ref.w, "orth d %d acc %s" % (d, nm), "reg")
    if seen is not None:
        _again(fn, seen, ["k_reg_orth"])


@pytest.mark.gpu
def test_reg_orth_tables():
    """kgrec_reg_orth_tables at every d in 1..300 (tables and accumulators on and off 16-byte alignment), NULL loss or
    accumulators, scale != 1, and rows past sm_count 8 8: loss and both accumulators against float64."""
    _lib, lib = _lib_()
    rng = np.random.RandomState(61)
    seen = []
    nos = [(), ("loss",), ("rel",), ("norm",)]
    for d in range(1, 301):
        _reg_orth_case(rng, lib, _lib, d, 30 if d > 50 else 60, (1.0, 0.37, 2.5)[d % 3], seen if d == 1 else None,
                       nos[d % 4] if d % 7 == 0 else ())
    _reg_orth_case(rng, lib, _lib, 50, _sms() * 8 * 8 + 300, 0.5, seen)
    _want(seen, ["k_reg_orth"])


# ---- samplers and hash set -------------------------------------------------------------------------------------------
M32 = np.uint64(0xFFFFFFFF)


def philox_bits(seed, pair, k):
    """philox_uniform_bits (csrc/common.cuh): Philox4x32-10, counter (pair, k, 0x4b47), key seed; word 0."""
    pair = np.asarray(pair, np.uint64)
    c0, c1 = pair & M32, pair >> np.uint64(32)
    c2 = np.full_like(pair, np.uint64(k & 0xFFFFFFFF))
    c3 = np.full_like(pair, np.uint64(0x4B47))
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = c0 * np.uint64(0xD2511F53), c2 * np.uint64(0xCD9E8D57)
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & M32,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & M32)
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0


def mix64(x):
    x = np.asarray(x, np.uint64).copy()
    x ^= x >> np.uint64(30)
    x *= np.uint64(0xBF58476D1CE4E5B9)
    x ^= x >> np.uint64(27)
    x *= np.uint64(0x94D049BB133111EB)
    x ^= x >> np.uint64(31)
    return x


def sample_ref(kind, cols, n_neg, n_cat, n_rel, keys, seed):
    """k_sample_corrupt / k_sample_items restated: the coin (corrupt), up to 64 multiply-shift draws, the scan on from
    the last draw, the last draw emitted when no id is valid.  Returns (int32 output, status raised)."""
    seed &= (1 << 64) - 1
    n_pos = len(cols[0])
    total = n_pos * n_neg
    m = np.arange(total, dtype=np.uint64)
    j = (m // np.uint64(n_neg)).astype(np.int64)
    a, b = (np.asarray(c, np.int64)[j].astype(np.uint64) for c in cols[:2])
    r = np.asarray(cols[2], np.int64)[j].astype(np.uint64) if kind == "corrupt" else None
    N, R = np.uint64(n_cat), np.uint64(n_rel)
    head = (philox_bits(seed, m, 0xFFFFFFFF) & np.uint64(1)) == 1 if kind == "corrupt" else np.zeros(total, bool)
    orig = np.where(head, a, b)

    def valid(idx, e):
        ok = e != orig[idx]
        if keys is not None:
            if kind == "corrupt":
                key = np.where(head[idx], (e * R + r[idx]) * N + b[idx], (a[idx] * R + r[idx]) * N + e)
            else:
                key = a[idx] * N + e
            ok &= ~np.isin(key, keys)
        return ok
    ent = np.zeros(total, np.uint64)
    found = np.zeros(total, bool)
    for att in range(64):
        idx = np.flatnonzero(~found)
        if not idx.size:
            break
        e = (philox_bits(seed, m[idx], att) * N) >> np.uint64(32)
        ent[idx] = e
        found[idx] = valid(idx, e)
    bad = False
    for i in np.flatnonzero(~found):
        es = (ent[i] + np.arange(1, n_cat, dtype=np.uint64)) % N
        v = valid(np.full(es.size, i), es)
        if v.any():
            ent[i] = es[np.argmax(v)]
        else:
            bad = True
    out = ent.astype(np.int64)
    out = np.where(head, ~out, out).astype(np.int32)
    return out, bad, int((~found).sum())


def _hashset(lib, _lib, keys):
    cap = int(lib.kgrec_hashset_capacity(len(keys)))
    table = torch.empty(cap, dtype=torch.int64, device="cuda")
    kd = torch.as_tensor(np.asarray(keys, np.uint64).view(np.int64), device="cuda")
    _lib.check(lib.kgrec_hashset_build(_p(kd), len(keys), _p(table), cap, None))
    return table, cap


def _sample(lib, _lib, kind, cols, ib, n_neg, n_cat, n_rel, table, cap, seed, state=None):
    dt = torch.int64 if ib == 8 else torch.int32
    d = [torch.as_tensor(np.asarray(c, np.int64), dtype=dt, device="cuda") for c in cols]
    out = torch.empty(len(cols[0]) * n_neg, dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    tp = _p(table)
    if kind == "corrupt":
        args = (_p(d[0]), _p(d[1]), _p(d[2]), ib, len(cols[0]), n_neg, n_cat, n_rel, tp, cap)
        if state is None:
            _lib.check(lib.kgrec_sample_corrupt(*args, seed & ((1 << 64) - 1), _p(out), _p(status), None))
        else:
            _lib.check(lib.kgrec_sample_corrupt_dev(*args, state.ptr, _p(out), _p(status), None))
    else:
        args = (_p(d[0]), _p(d[1]), ib, len(cols[0]), n_neg, n_cat, tp, cap)
        if state is None:
            _lib.check(lib.kgrec_sample_neg_items(*args, seed & ((1 << 64) - 1), _p(out), _p(status), None))
        else:
            _lib.check(lib.kgrec_sample_neg_items_dev(*args, state.ptr, _p(out), _p(status), None))
    return out.cpu().numpy(), int(status.item())


def _dense_kg(rng, n_ent, n_rel):
    """Known triples: 30 % of all, plus (h, r) keys with all tails known but one, and with all tails known; the same
    for (r, t) heads.  Positives: known triples, the dense keys among them."""
    keys = set(int(k) for k in rng.choice(n_ent * n_rel * n_ent, n_ent * n_rel * n_ent * 3 // 10, replace=False))
    tk = lambda h, r, t: (h * n_rel + r) * n_ent + t          # noqa: E731
    pos = []
    for i, (h, r) in enumerate([(1, 0), (2, 1), (3, 2), (4, 0)]):
        skip = [5] if i % 2 == 0 else []
        keys |= {tk(h, r, t) for t in range(n_ent) if t not in skip}
        pos += [(h, (7 + i) % n_ent, r)] * 6
        keys.add(tk(h, r, (7 + i) % n_ent))
    for i, (r, t) in enumerate([(1, 9), (2, 11)]):
        keys |= {tk(h, r, t) for h in range(n_ent) if not (i == 0 and h == 6)}
        pos += [(13 + i, t, r)] * 6
    arr = np.array(sorted(keys), np.int64)
    for k in rng.choice(arr, 200):
        h, rest = divmod(int(k), n_rel * n_ent)
        r, t = divmod(rest, n_ent)
        pos.append((h, t, r))
    pos = np.array(pos, np.int64)
    return np.array(sorted(keys), np.uint64), [pos[:, 0], pos[:, 1], pos[:, 2]]


def _dense_rec(rng, n_user, n_item):
    keys = set(int(k) for k in rng.choice(n_user * n_item, n_user * n_item * 3 // 10, replace=False))
    pos = []
    for u, skip in ((0, [4]), (1, []), (2, [9, 10])):
        keys |= {u * n_item + i for i in range(n_item) if i not in skip}
        pos += [(u, 3)] * 8
    arr = np.array(sorted(keys), np.int64)
    for k in rng.choice(arr, 200):
        pos.append(divmod(int(k), n_item))
    pos = np.array(pos, np.int64)
    return np.array(sorted(keys), np.uint64), [pos[:, 0], pos[:, 1]]


@pytest.mark.gpu
def test_hashset_build():
    """kgrec_hashset_build on keys with repeats: the non-empty slots hold exactly the distinct keys, each once, and
    each is reachable from its home slot mix64(key) & mask without an empty slot between (the probe's invariant)."""
    _lib, lib = _lib_()
    rng = np.random.RandomState(71)
    seen = []
    for n in (1, 300, _sms() * 16 * 256 + 999):
        base = rng.randint(0, 1 << 62, max(1, n * 2 // 3), dtype=np.int64).astype(np.uint64)
        keys = np.concatenate([base, rng.choice(base, n - base.size)]) if n > base.size else base
        rng.shuffle(keys)
        table, cap = _kernels(lambda: _hashset(lib, _lib, keys), seen)
        t = table.cpu().numpy().view(np.uint64)
        full = t != np.uint64(0xFFFFFFFFFFFFFFFF)
        assert np.array_equal(np.sort(t[full]), np.unique(keys)), n
        home = (mix64(t[full]) & np.uint64(cap - 1)).astype(np.int64)
        slot = np.flatnonzero(full)
        empty = np.flatnonzero(~full)
        # the first empty slot at or after home (cyclically) must come after the key's slot
        nxt = empty[np.searchsorted(empty, home) % empty.size]
        dist_key = (slot - home) % cap
        dist_empty = (nxt - home) % cap
        assert np.all(dist_key < dist_empty), n
    _again(lambda: _hashset(lib, _lib, keys), seen, ["k_hashset_insert"])
    _want(seen, ["k_hashset_insert"])


@pytest.mark.gpu
@pytest.mark.parametrize("ib", [4, 8])
def test_sample_corrupt(ib):
    """kgrec_sample_corrupt bit for bit against the restatement: unfiltered (n_ent 2, 1000, 2^31 - 1), filtered on a
    dense known set (draws that reach the scan, keys without any valid negative: status 2 and the last draw), and more
    than sm_count 16 256 draws."""
    _lib, lib = _lib_()
    rng = np.random.RandomState(81 + ib)
    seen = []
    keys, cols = _dense_kg(rng, 30, 3)
    table, cap = _hashset(lib, _lib, keys)
    seed = 0x1234_5678_9ABC_DEF0 + ib
    got, st = _kernels(lambda: _sample(lib, _lib, "corrupt", cols, ib, 16, 30, 3, table, cap, seed), seen)
    want, bad, scanned = sample_ref("corrupt", cols, 16, 30, 3, keys, seed)
    assert scanned > 10 and bad
    assert np.array_equal(got, want) and st == 2
    for n_cat in (2, 1000, (1 << 31) - 1):
        n = 700
        c = [rng.randint(0, n_cat, n), rng.randint(0, n_cat, n), rng.randint(0, 5, n)]
        got, st = _sample(lib, _lib, "corrupt", c, ib, 3, n_cat, 5, None, 0, seed + n_cat)
        want, bad, _ = sample_ref("corrupt", c, 3, n_cat, 5, None, seed + n_cat)
        assert np.array_equal(got, want) and st == 0 and not bad, n_cat
    n_pos, n_neg, n_ent = _sms() * 16 * 256 // 4 + 1000, 4, 100_000
    c = [rng.randint(0, n_ent, n_pos), rng.randint(0, n_ent, n_pos), rng.randint(0, 7, n_pos)]
    k = ((c[0][:50_000] * 7 + c[2][:50_000]) * n_ent + rng.randint(0, n_ent, 50_000)).astype(np.uint64)
    table, cap = _hashset(lib, _lib, k)
    got, st = _kernels(lambda: _sample(lib, _lib, "corrupt", c, ib, n_neg, n_ent, 7, table, cap, 99), seen)
    want, bad, _ = sample_ref("corrupt", c, n_neg, n_ent, 7, np.unique(k), 99)
    assert np.array_equal(got, want) and st == 0
    _again(lambda: _sample(lib, _lib, "corrupt", c, ib, n_neg, n_ent, 7, table, cap, 99), seen, ["k_sample_corrupt"])
    _want(seen, ["k_sample_corrupt"])


@pytest.mark.gpu
@pytest.mark.parametrize("ib", [4, 8])
def test_sample_neg_items(ib):
    """kgrec_sample_neg_items bit for bit against the restatement, as test_sample_corrupt."""
    _lib, lib = _lib_()
    rng = np.random.RandomState(91 + ib)
    seen = []
    keys, cols = _dense_rec(rng, 20, 25)
    table, cap = _hashset(lib, _lib, keys)
    seed = (1 << 63) + 12345 + ib
    got, st = _kernels(lambda: _sample(lib, _lib, "items", cols, ib, 16, 25, 1, table, cap, seed), seen)
    want, bad, scanned = sample_ref("items", cols, 16, 25, 1, keys, seed)
    assert scanned > 10 and bad
    assert np.array_equal(got, want) and st == 2
    for n_cat in (2, 1000, (1 << 31) - 1):
        n = 700
        c = [rng.randint(0, 50, n), rng.randint(0, n_cat, n)]
        got, st = _sample(lib, _lib, "items", c, ib, 3, n_cat, 1, None, 0, seed + n_cat)
        want, bad, _ = sample_ref("items", c, 3, n_cat, 1, None, seed + n_cat)
        assert np.array_equal(got, want) and st == 0 and not bad, n_cat
    n_pos, n_neg, n_item = _sms() * 16 * 256 // 4 + 1000, 4, 50_000
    c = [rng.randint(0, 3000, n_pos), rng.randint(0, n_item, n_pos)]
    k = (c[0][:60_000] * n_item + rng.randint(0, n_item, 60_000)).astype(np.uint64)
    table, cap = _hashset(lib, _lib, k)
    got, st = _kernels(lambda: _sample(lib, _lib, "items", c, ib, n_neg, n_item, 1, table, cap, 5), seen)
    want, bad, _ = sample_ref("items", c, n_neg, n_item, 1, np.unique(k), 5)
    assert np.array_equal(got, want) and st == 0
    _again(lambda: _sample(lib, _lib, "items", c, ib, n_neg, n_item, 1, table, cap, 5), seen, ["k_sample_items"])
    _want(seen, ["k_sample_items"])


@pytest.mark.gpu
def test_sample_dev_seed():
    """The _dev samplers draw with seed state.sample_seed + state.step (mod 2^64): bit for bit the by-value call with
    that seed, and the restatement."""
    from kgrec_b200.train import StepState
    _lib, lib = _lib_()
    rng = np.random.RandomState(101)
    kg_keys, kg_cols = _dense_kg(rng, 30, 3)
    kt, kc = _hashset(lib, _lib, kg_keys)
    rec_keys, rec_cols = _dense_rec(rng, 20, 25)
    rt, rc = _hashset(lib, _lib, rec_keys)
    for sample_seed, step in ((0, 1), (987654321, 41), ((1 << 64) - 3, 5)):
        state = StepState("cuda", step=step - 1, sample_seed=sample_seed)
        state.advance()
        seed = (sample_seed + step) & ((1 << 64) - 1)
        for kind, cols, t, cap, n_cat, n_rel, keys in (("corrupt", kg_cols, kt, kc, 30, 3, kg_keys),
                                                        ("items", rec_cols, rt, rc, 25, 1, rec_keys)):
            dev, st_dev = _sample(lib, _lib, kind, cols, 8, 5, n_cat, n_rel, t, cap, 0, state=state)
            val, st_val = _sample(lib, _lib, kind, cols, 8, 5, n_cat, n_rel, t, cap, seed)
            want, bad, _ = sample_ref(kind, cols, 5, n_cat, n_rel, keys, seed)
            assert np.array_equal(dev, val) and np.array_equal(dev, want) and st_dev == st_val == (2 if bad else 0)


# ---- step state ------------------------------------------------------------------------------------------------------
def gather_ref(order, cursor, cols, n_rows, batch):
    p = cursor + np.arange(batch)
    okp = (p >= 0) & (p < len(order))
    row = np.where(okp, np.asarray(order)[np.clip(p, 0, len(order) - 1)], 0)
    okr = (row >= 0) & (row < n_rows)
    row = np.where(okr, row, 0)
    return [np.asarray(c)[row] for c in cols], bool((~okp).any() or (~okr).any())


@pytest.mark.gpu
def test_batch_gather():
    """kgrec_batch_gather exactly as restated: 1..4 columns of int32 / int64, cursors inside the order, running past
    its end and before its start, order entries outside [0, n_rows) (row 0, status 1), batches past sm_count 4 256."""
    _lib, lib = _lib_()
    rng = np.random.RandomState(111)
    seen = []
    big = _sms() * 4 * 256 + 3000
    cases = [(n_cols, ib, n_rows, n_order, cursor, batch, n_bad)
             for n_cols in (1, 2, 3, 4) for ib in (4, 8)
             for (n_rows, n_order, cursor, batch, n_bad) in ((500, 500, 0, 128, 0), (500, 700, 650, 128, 0),
                                                             (300, 300, -5, 64, 0), (400, 400, 10, 200, 3))]
    cases += [(4, 8, big + 10, big + 10, 5, big, 0), (2, 4, big, big, 0, big, 7)]
    for i, (n_cols, ib, n_rows, n_order, cursor, batch, n_bad) in enumerate(cases):
        order = rng.permutation(max(n_order, n_rows))[:n_order].astype(np.int64) % n_rows
        if n_bad:
            window = np.arange(max(cursor, 0), min(n_order, cursor + batch))
            order[rng.choice(window, n_bad, replace=False)] = rng.choice([-1, n_rows, n_rows + 9, 1 << 40], n_bad)
        dt = torch.int64 if ib == 8 else torch.int32
        cols = [rng.randint(-(1 << 30), 1 << 30, n_rows).astype(np.int64) for _ in range(n_cols)]
        cd = [torch.as_tensor(c, dtype=dt, device="cuda") for c in cols]
        outs = [torch.full((batch,), -99, dtype=dt, device="cuda") for _ in range(n_cols)]
        od = torch.as_tensor(order, device="cuda")
        cur = torch.tensor([cursor], dtype=torch.int64, device="cuda")
        status = torch.full((1,), 3, dtype=torch.int32, device="cuda")
        ca = (C.c_void_p * n_cols)(*[c.data_ptr() for c in cd])
        oa = (C.c_void_p * n_cols)(*[o.data_ptr() for o in outs])
        fn = lambda: _lib.check(lib.kgrec_batch_gather(_p(od), n_order, _p(cur), ca, oa, n_cols, ib, n_rows,  # noqa
                                                       batch, _p(status), None))
        _kernels(fn, seen) if i in (0, len(cases) - 1) else fn()
        want, bad = gather_ref(order, cursor, cols, n_rows, batch)
        for o, w in zip(outs, want):
            assert np.array_equal(o.cpu().numpy().astype(np.int64), w), (n_cols, ib, cursor, batch)
        assert int(status.item()) == (1 if bad else 3), (n_cols, ib, cursor, batch, n_bad)
        assert int(cur.item()) == cursor
        _again(fn, seen, ["k_batch_gather"])
    _want(seen, ["k_batch_gather"])


@pytest.mark.gpu
def test_step_advance():
    """kgrec_step_advance: step and epoch + 1, the cursor + batch when given; the seeds and lr keep their bits."""
    from kgrec_b200.train import StepState
    _lib, lib = _lib_()
    seen = []
    state = StepState("cuda", step=41, epoch=-3, gumbel_seed=(1 << 64) - 1, sample_seed=12345, lr=0.1)
    before = state.read()
    cur = torch.tensor([1000], dtype=torch.int64, device="cuda")
    _kernels(lambda: _lib.check(lib.kgrec_step_advance(state.ptr, _p(cur), 256, None)), seen)
    _lib.check(lib.kgrec_step_advance(state.ptr, None, 77, None))
    _lib.check(lib.kgrec_step_advance(state.ptr, _p(cur), 0, None))
    after = state.read()
    assert after == dict(before, step=44, epoch=0)
    assert int(cur.item()) == 1256
    _again(lambda: _lib.check(lib.kgrec_step_advance(state.ptr, None, 0, None)), seen, ["k_step_advance"])
    _want(seen, ["k_step_advance"])


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    """Prints (pytest -s) the largest measured ratio to the C_BOUND = 1 bound of each group of checks."""
    yield
    for k, v in sorted(Ratio.worst.items()):
        print("\nlargest ratio to the bound, %s: %.3g" % (k, v / C_BOUND))
