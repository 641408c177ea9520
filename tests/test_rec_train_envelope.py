"""The whole envelope the TUP / KTUP training entry points accept, against float64.

Three engines train the recommendation models, chosen on the host by shape and data rules:
  row-factored step   kgrec_rec_rows_step (csrc/train_rec_rows.cu), taken by SparseRowOptimizer.step_pairs
  tile engine         k_rec_tile<PT, GUM, MODE> behind kgrec_score_fwd / _bwd, kgrec_rank_loss_fwd / _step
  one warp per pair   k_score_fwd / k_rank_loss_fwd / k_score_bwd<FAM_REC, NCH, VEC, PR> (csrc/train_dev.cuh)
Each case pins one engine (KGREC_REC_ROWS / KGREC_REC_TILE) and checks, at every element of the scores, the per-batch
losses and the gradient tables,
    |kernel - ref| <= C_BOUND (d + P) 2^-24 twin
where ref is the oracle (oracle/kg_oracle.py) on float64 copies of the tables, and twin is the same computation with
every operand replaced by its magnitude and every subtraction by an addition (through the ST-Gumbel softmax
y (|gp| + sum y |gp|)), scattered exactly like the gradients.  The bound follows each element's own cancellation; an
element whose twin is 0 (a row the step did not touch, the padding entity) must be exactly 0.  Kinks are screened out
before the call: the ids (or uniforms) of a group with a pair within its bound of a hinge, of an L1 residual component
e_k = 0, or of an ST-Gumbel arg-max tie are redrawn (at most 3 % of the first draw, or 3 pairs of a small batch,
may need it: L1 rows of d >= 100 put 1-3 % of the pairs within the bound of e_k = 0; L2 cases need almost none), and the rows under the
fused normLoss keep |x|^2 away from 1.  Profiles name the kernels each family runs.

Which case covers which part of the envelope:
  row-factored step (SparseRowOptimizer.step_pairs, KGREC_REC_ROWS=force; gradients read from opt.acc)
    every d % 4 == 0 in 4..128 (TUP soft L2, TUP ST-Gumbel L2) ....... test_rows_d_sweep
    d in {4, 12, 36, 68, 100, 116, 128} for the other four models ..... test_rows_d_short
    P in {1, 2, 7, 8, 9, 19, 20, 21, 31, 32} (PT = 8 / 20 / 32), all
      six models, profile of k_soft_rows_* / k_gumbel_rows_*<PT> ...... test_rows_preference_counts
    n_neg in {1, 2, 15, 16, 30, 31}, BPR / margin, batch_pos not
      dividing n_pos and batch_pos = 1, int32 / int64 ids, ids 0 and
      n - 1, heavy reuse and none, KTUP padding and shared entities ... test_rows_negatives_losses_ids
    fused normLoss (reg=True, TUP) with duplicate rows ................ test_rows_fused_norm_loss
    two steps on one optimizer, rows shared between them ............. test_rows_two_steps
    hashed ST-Gumbel noise: one preference per pair, bit-for-bit repeat test_rows_hashed_noise
  tile engine (KGREC_REC_TILE=force)
    PT 8 / 20 / 32 x soft / ST-Gumbel x FWD / BWD / STEP, n_neg 1 / 7 /
      15 and the fallback at 16, ragged last tile, several tiles per
      CTA, d in {4, 52, 100, 128}, dense and sparse grad_mode + slots . test_tile_engine
  one warp per pair (KGREC_REC_TILE=0)
    d in {4, 50, 100, 128, 130, 132, 200, 255, 256, 300, 511, 512}, P up
      to the backward limit of each band, NCH 1 / 2 / 4 x VEC ......... test_pair_engine
    forward-only P up to the largest the host accepts ................. test_pair_engine_forward_limit
On the CPU: _use_rows_path against the host checks of kgrec_rec_rows_step, and the accepted (d, P) region of
kgrec_rank_loss_step with its messages.
Run time on one H100 (80 GB HBM3): about 80 s for the GPU cases.
"""
import ctypes as C
import re

import numpy as np
import pytest
import torch

from oracle import kg_oracle as O

U24 = 2.0 ** -24
C_BOUND = 2             # the smallest integer constant the cases pass with (the evaluation envelope needs 8)
PREF_SCALE = 0.15       # preference-side rows (pref, pref_norm, KTUP rel, norm) at norm 0.15: see _model
FAKE = 0x7000_0000_1000
UNSUPPORTED = 2          # KGREC_ERR_UNSUPPORTED
MODELS = {   # name: (ktup, gumbel, l1)
    "tup_soft_l1": (False, False, True), "tup_soft_l2": (False, False, False), "tup_gumbel_l2": (False, True, False),
    "ktup_soft_l1": (True, False, True), "ktup_soft_l2": (True, False, False), "ktup_gumbel_l2": (True, True, False),
}


# ---- CPU ------------------------------------------------------------------------------------------------------------
class _Stub:
    """What SparseRowOptimizer._use_rows_path reads of its model."""
    def __init__(self, d, P, gumbel, l1):
        self.embedding_size, self.use_st_gumbel, self.L1_flag = d, gumbel, l1
        self.pref_embeddings = torch.nn.Embedding(P, 1)
        self.user_embeddings = torch.nn.Embedding(10, 1)
        self.item_embeddings = torch.nn.Embedding(10, 1)


def test_rows_gate_agrees_with_the_host_checks(monkeypatch):
    """_use_rows_path (with KGREC_REC_ROWS=force) takes the row-factored step exactly where kgrec_rec_rows_step accepts
    the shape, over a (d, P, n_neg, ST-Gumbel, L1) grid; n_pos = 0 with fake pointers, so nothing reaches a device."""
    from types import SimpleNamespace
    from kgrec_b200 import _lib
    from kgrec_b200.optim import SparseRowOptimizer
    lib = _lib.load()
    monkeypatch.setenv("KGREC_REC_ROWS", "force")
    g = _lib.Grads(mode=1, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE, ent=FAKE)
    seen = {True: 0, False: 0}
    for model in (_lib.TUP, _lib.KTUP):
        for d in (4, 8, 50, 64, 100, 124, 128, 130, 132, 256):
            for P in (1, 8, 20, 31, 32, 33, 64):
                for n_neg in (1, 15, 31, 32):
                    for gumbel, l1 in ((0, 0), (0, 1), (1, 0), (1, 1)):
                        t = _lib.Tables(dim=d, ld=d, n_user=10, n_item=10, n_ent=10, n_rel=P, n_pref=P, l1=l1,
                                        use_gumbel=gumbel, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE, ent=FAKE,
                                        rel=FAKE, norm=FAKE, item2ent=FAKE)
                        rc = lib.kgrec_rec_rows_step(C.byref(t), model, FAKE, FAKE, FAKE, 4, 0, n_neg, 8, _lib.LOSS_BPR,
                                                     -1.0, 1.0, FAKE, FAKE, 1, FAKE, 0, C.byref(g), FAKE, FAKE, FAKE, FAKE,
                                                     None, None, 0, None, None)
                        host = rc == 0
                        if not host:
                            assert rc == UNSUPPORTED, lib.kgrec_last_error().decode()
                        opt = SimpleNamespace(model=_Stub(d, P, bool(gumbel), bool(l1)))
                        gate = SparseRowOptimizer._use_rows_path(opt, 4, n_neg, None, None)
                        assert gate == host, (model, d, P, n_neg, gumbel, l1, lib.kgrec_last_error().decode())
                        seen[host] += 1
    assert seen[True] > 100 and seen[False] > 100


def _step_rc(lib, _lib, model, d, P):
    t = _lib.Tables(dim=d, ld=d, n_user=10, n_item=10, n_ent=10, n_rel=P, n_pref=P, user=FAKE, item=FAKE, pref=FAKE,
                    pref_norm=FAKE, ent=FAKE, rel=FAKE, norm=FAKE, item2ent=FAKE)
    g = _lib.Grads(mode=1, user=FAKE, item=FAKE, pref=FAKE, pref_norm=FAKE, ent=FAKE)
    rc = lib.kgrec_rank_loss_step(C.byref(t), model, FAKE, FAKE, None, FAKE, FAKE, None, 4, 0, 1, 8, _lib.LOSS_BPR, -1.0,
                                  1.0, None, 0, FAKE, FAKE, FAKE, C.byref(g), None, None, None, FAKE, None, None)
    return rc, lib.kgrec_last_error().decode()


def _fwd_rc(lib, _lib, model, d, P):
    t = _lib.Tables(dim=d, ld=d, n_user=10, n_item=10, n_ent=10, n_rel=P, n_pref=P, user=FAKE, item=FAKE, pref=FAKE,
                    pref_norm=FAKE, ent=FAKE, rel=FAKE, norm=FAKE, item2ent=FAKE)
    return lib.kgrec_score_fwd(C.byref(t), model, FAKE, FAKE, None, 4, 0, None, 0, FAKE, None, None)


def _max_p(fn, d):
    return max([P for P in range(1, 129) if fn(d, P)] or [0])


def test_rank_loss_step_accepted_region_is_pinned():
    """kgrec_rank_loss_step for TUP / KTUP over (d, P): the backward limit P <= 64 / 32 / 16 for d <= 128 / 256 / 512 (16
    from d = 129 when d % 4 != 0: the scalar path is built for NCH 1 and 4 only), the
    forward entry points' own limit (the staged preference tables and the backward scratch in 220 KB of shared memory),
    nothing past d = 512 or P = 128 -- each rejection with the message that names it."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    fwd_max = {4: 128, 100: 128, 128: 128, 130: 128, 200: 112, 255: 75, 256: 87, 300: 64, 511: 37, 512: 37}
    for model in (_lib.TUP, _lib.KTUP):
        fwd = lambda d, P: _fwd_rc(lib, _lib, model, d, P) == 0     # noqa: E731
        assert {d: _max_p(fwd, d) for d in fwd_max} == fwd_max
        for d, pf in fwd_max.items():
            band = 64 if d <= 128 else (32 if d <= 256 and d % 4 == 0 else 16)     # d % 4 != 0: the scalar rows, NCH 4
            assert all(fwd(d, P) for P in range(1, pf + 1))
            for P in sorted({1, band, band + 1, pf, pf + 1, 128, 129}):
                rc, msg = _step_rc(lib, _lib, model, d, P)
                if P <= band:
                    assert rc == 0, (d, P, msg)
                    continue
                assert rc == UNSUPPORTED, (d, P)
                if P > 128:
                    assert "preference_total %d outside [1, 128]" % P in msg
                elif P > pf:
                    assert msg == "preference tables do not fit in shared memory"
                else:
                    assert "backward: preference_total %d > %d is not built for embedding_size %d" % (P, band, d) in msg
        rc, msg = _step_rc(lib, _lib, model, 516, 4)
        assert rc == UNSUPPORTED and "embedding_size 516 > 512 is not built" in msg
        rc, msg = _step_rc(lib, _lib, model, 100, 0)
        assert rc == UNSUPPORTED and "preference_total 0 outside [1, 128]" in msg


# ---- float64 reference and its absolute-value twin -------------------------------------------------------------------
class Ref:
    """float64 copies of a TUP / KTUP model's tables, the oracle's scores and gradients, and the twin."""

    def __init__(self, m):
        from kgrec_b200 import _lib
        self.W = {k: v.detach().double().cpu().numpy() for k, v in m._weights().items()}
        self.ktup = m.MODEL == _lib.KTUP
        self.gumbel, self.l1 = bool(m.use_st_gumbel), bool(m.L1_flag)
        W = self.W
        self.d = W["user"].shape[1]
        self.P = W["pref"].shape[0]
        if self.ktup:
            self.i2e = m.item2ent.cpu().numpy().astype(np.int64)
            self.X = W["item"] + W["ent"][self.i2e]
            self.aX = np.abs(W["item"]) + np.abs(W["ent"][self.i2e])
            self.Pm, self.Nm = W["pref"] + W["rel"], W["pref_norm"] + W["norm"]
            self.aP = np.abs(W["pref"]) + np.abs(W["rel"])
            self.aN = np.abs(W["pref_norm"]) + np.abs(W["norm"])
        else:
            self.X, self.aX = W["item"], np.abs(W["item"])
            self.Pm, self.Nm, self.aP, self.aN = W["pref"], W["pref_norm"], np.abs(W["pref"]), np.abs(W["pref_norm"])
        self.hf = 0.5 if self.ktup else 1.0
        self.tau = C_BOUND * (self.d + self.P) * U24

    def _args(self):
        W = self.W
        if self.ktup:
            return (W["user"], W["item"], W["ent"], W["rel"], W["norm"], W["pref"], W["pref_norm"], self.i2e)
        return (W["user"], W["item"], W["pref"], W["pref_norm"])

    def score(self, u, i, noise):
        f = O.ktup_rec_score if self.ktup else O.tup_score
        return f(*self._args(), u, i, self.l1, noise)

    def grads(self, u, i, noise, g):
        f = O.ktup_rec_grads if self.ktup else O.tup_grads
        return f(*self._args(), u, i, self.l1, g, noise)

    def pairs(self, u, i, noise):
        """Per pair: the magnitudes the twin needs, the residual e, and the ST-Gumbel top-two gap with its bound."""
        uu, x = self.W["user"][u], self.X[i]
        au, ax = np.abs(uu), self.aX[i]
        sa = au + ax
        za = sa @ self.aP.T / 2
        out = {"sa": sa, "za": za}
        if self.gumbel:
            v = (uu + x) @ self.Pm.T / 2 + _gumbel(noise)
            ks = v.argmax(-1)
            pa = np.zeros_like(za)
            pa[np.arange(len(ks)), ks] = 1.0
            y = O.softmax_last(v)
            top = np.sort(v, axis=-1)
            out["gap"] = (top[:, -1] - top[:, -2]) if self.P > 1 else np.full(len(u), np.inf)
            out["gap_bound"] = 2 * self.tau * (np.abs(za).max(-1) + np.abs(_gumbel(noise)).max(-1) + 1.0)
            out["y"] = y
        else:
            pa = za
            _, r, w, _ = O.tup_preferences(uu + x, self.Pm, self.Nm, None, self.ktup)
        ra, wa = self.hf * pa @ self.aP, self.hf * pa @ self.aN
        if self.gumbel:
            _, r, w, _ = O.tup_preferences(uu + x, self.Pm, self.Nm, noise, self.ktup)
        xa = au + ax
        swa = (xa * wa).sum(-1)
        mm = xa + ra + swa[:, None] * wa
        out.update(pa=pa, wa=wa, xa=xa, swa=swa, mm=mm)
        out["e"] = O.proj_hyperplane(uu, w) + r - O.proj_hyperplane(x, w)
        out["twin"] = mm.sum(-1) if self.l1 else (mm * mm).sum(-1)
        return out

    def twin_grads(self, u, i, q, tg):
        """Gradient tables of the twin, given per-pair magnitudes q (from pairs) and upstream magnitudes tg."""
        epsa = tg[:, None] * (np.ones_like(q["mm"]) if self.l1 else 2 * q["mm"])
        ewa = (epsa * q["wa"]).sum(-1)
        gxa = epsa + ewa[:, None] * q["wa"]
        gwa = ewa[:, None] * q["xa"] + q["swa"][:, None] * epsa
        gpa = self.hf * (epsa @ self.aP.T + gwa @ self.aN.T)
        gpref = self.hf * (q["pa"].T @ epsa)
        gpn = self.hf * (q["pa"].T @ gwa)
        if self.gumbel:
            y = q["y"]
            gza = y * (gpa + (y * gpa).sum(-1, keepdims=True))
        else:
            gza = gpa
        gsa = gza @ self.aP / 2
        gpref = gpref + gza.T @ q["sa"] / 2
        gr = gxa + gsa
        W, d = self.W, self.d
        out = {"user": _scatter(W["user"].shape[0], u, gr), "item": _scatter(W["item"].shape[0], i, gr),
               "pref": gpref, "pref_norm": gpn}
        if self.ktup:
            ge = _scatter(W["ent"].shape[0], self.i2e[i], gr)
            ge[-1] = 0
            out.update(ent=ge, rel=gpref.copy(), norm=gpn.copy())
        return out


def _gumbel(u):
    return -np.log(-np.log(u + O.EPS_GUMBEL) + O.EPS_GUMBEL)


def _scatter(rows, idx, vals):
    out = np.zeros((rows, vals.shape[1]))
    np.add.at(out, idx, vals)
    return out


def _add(a, b):
    for k, v in b.items():
        a[k] = a.get(k, 0) + v
    return a


class Step:
    """float64 step of a (user, positive, negatives) batch: scores, per-batch losses, upstream gradients, and every
    table gradient, each with its bound."""

    def __init__(self, R, pu, pi, ni, noise, loss, param, bp):
        self.R, self.loss, self.param, self.bp = R, loss, param, bp
        n_pos, K = len(pu), len(ni) // len(pu)
        self.n_pos, self.K = n_pos, K
        un = np.repeat(pu, K)
        self.uid, self.iid = np.concatenate([pu, un]), np.concatenate([pi, ni])
        self.noise = noise
        self.q = R.pairs(self.uid, self.iid, noise)
        s = R.score(self.uid, self.iid, noise)
        self.sp, self.sn = s[:n_pos], s[n_pos:]
        t = self.q["twin"]
        self.tp, self.tn = t[:n_pos], t[n_pos:]

    def kinks(self):
        """Per pair: within its bound of a kink (hinge, L1 residual component, ST-Gumbel arg-max)."""
        R, q = self.R, self.q
        bad = np.zeros(len(self.uid), dtype=bool)
        if R.l1:
            bad |= (np.abs(q["e"]) <= R.tau * q["mm"]).any(-1)
        if R.gumbel:
            bad |= q["gap"] <= q["gap_bound"]
        if self.loss == "margin":
            h = self.param + np.repeat(self.sp, self.K) - self.sn
            hb = R.tau * (np.repeat(self.tp, self.K) + self.tn + abs(self.param))
            near = np.abs(h) <= hb
            bad[:self.n_pos] |= near.reshape(self.n_pos, self.K).any(-1)
            bad[self.n_pos:] |= near
        return bad

    def backward(self):
        """Per-batch losses and the upstream dLoss / dscore of every pair, with their twins; then the tables."""
        R, K, n_pos, t = self.R, self.K, self.n_pos, self.param
        spr = np.repeat(self.sp, K)
        tpr = np.repeat(self.tp, K)
        nb = (n_pos + self.bp - 1) // self.bp
        loss, tloss = np.zeros(nb), np.zeros(nb)
        gn, tgn = np.zeros(n_pos * K), np.zeros(n_pos * K)
        for b in range(nb):
            sl = slice(b * self.bp * K, min(n_pos, (b + 1) * self.bp) * K)
            if self.loss == "bpr":
                loss[b] = O.bpr_loss(spr[sl], self.sn[sl], t)
                gp_, _ = O.bpr_loss_grads(spr[sl], self.sn[sl], t)
                x = t * (spr[sl] - self.sn[sl])
                cnt = sl.stop - sl.start
                sig = 1 / (1 + np.exp(x))
                h = t * t * sig * (1 - sig) / cnt
                gn[sl] = -gp_
                tgn[sl] = np.abs(gp_) + h * (tpr[sl] + self.tn[sl])
                sp_ = np.maximum(-x, 0) + np.log1p(np.exp(-np.abs(x)))
                tloss[b] = (np.abs(sp_) + abs(t) * sig * (tpr[sl] + self.tn[sl]) + 1.0).sum() / cnt
            else:
                loss[b] = O.margin_loss(spr[sl], self.sn[sl], t)
                act, _ = O.margin_loss_grads(spr[sl], self.sn[sl], t)
                gn[sl] = -act
                tgn[sl] = act
                tloss[b] = (act * (tpr[sl] + self.tn[sl] + np.abs(spr[sl]) + np.abs(self.sn[sl]) + abs(t))).sum()
        gp = -gn.reshape(n_pos, K).sum(-1)
        tgp = tgn.reshape(n_pos, K).sum(-1)
        self.loss_ref, self.loss_twin = loss, tloss
        g, tg = np.concatenate([gp, gn]), np.concatenate([tgp, tgn])
        self.grads_ref = R.grads(self.uid, self.iid, self.noise, g)
        self.grads_twin = R.twin_grads(self.uid, self.iid, self.q, tg)
        return self


def _check(got, ref, twin, tau, tag):
    got = np.asarray(got, dtype=np.float64)
    B = tau * np.asarray(twin)
    err = np.abs(got - ref)
    bad = err > B
    assert not bad.any(), "%s: %d of %d elements over the bound, first %s: kernel %r ref %r bound %r" % (
        tag, bad.sum(), bad.size, np.argwhere(bad)[0], got[bad][0], np.asarray(ref)[bad][0], B[bad][0])


def _check_step(S, ps, ns, loss, grads, tag):
    R = S.R
    _check(ps, S.sp, S.tp, R.tau, tag + " pos scores")
    _check(ns, S.sn, S.tn, R.tau, tag + " neg scores")
    _check(loss, S.loss_ref, S.loss_twin, R.tau, tag + " loss")
    for k in (S.grads_ref if grads is not None else ()):
        _check(grads[k], S.grads_ref[k], S.grads_twin[k], R.tau, tag + " grad " + k)


# ---- batches with the kinks screened out ----------------------------------------------------------------------------
def _batch(R, rng, n_pos, K, U, I, loss="bpr", param=-1.0, bp=None, reuse=True, max_frac=0.03, lo=(0, 0)):
    """(pu, pi, ni, noise, Step) with ids in [lo, n) and the ends lo and n - 1 of both ranges present; groups with a
    pair near a kink are redrawn."""
    P = R.P
    if reuse:
        pu, pi, ni = rng.randint(lo[0], U, n_pos), rng.randint(lo[1], I, n_pos), rng.randint(lo[1], I, n_pos * K)
    else:
        assert U >= n_pos and I >= n_pos * (1 + K)
        pu = rng.permutation(U)[:n_pos]
        it = rng.permutation(I)[:n_pos * (1 + K)]
        pi, ni = it[:n_pos], it[n_pos:]
    noise = rng.rand(n_pos * (1 + K), P) if R.gumbel else None
    bp = bp or n_pos
    redrawn = None
    for _ in range(30):
        for ids, a, n in ((pu, lo[0], U), (pi, lo[1], I)):     # the range ends appear (screened like any other id)
            for e in (a, n - 1):
                if not ((ids == e).any() or (ids is pi and (ni == e).any())):
                    ids[rng.randint(0, len(ids))] = e
        if noise is not None:
            noise = noise.astype(np.float32).astype(np.float64)
        S = Step(R, pu, pi, ni, noise, loss, param, bp)
        bad = S.kinks()
        if redrawn is None:         # the pairs of the first draw that had to be redrawn
            redrawn = int(bad.sum())
            assert redrawn <= max(max_frac * len(bad), 3), "%d of %d pairs near a kink" % (redrawn, len(bad))
        if not bad.any():
            return pu, pi, ni, noise, S
        grp = bad[:n_pos] | bad[n_pos:].reshape(n_pos, K).any(-1)
        j = np.nonzero(grp)[0]
        if reuse:
            pi[j] = rng.randint(lo[1], I, len(j))
            ni.reshape(n_pos, K)[j] = rng.randint(lo[1], I, (len(j), K))
        else:      # keep the ids distinct: swap in unused ones
            free = np.setdiff1d(np.arange(I), np.concatenate([pi, ni]))
            new = rng.permutation(free)[:len(j) * (1 + K)]
            if len(new) == len(j) * (1 + K):
                pi[j] = new[:len(j)]
                ni.reshape(n_pos, K)[j] = new[len(j):].reshape(len(j), K)
        if noise is not None:
            noise[j] = rng.rand(len(j), P)
            noise[n_pos:].reshape(n_pos, K, P)[j] = rng.rand(len(j), K, P)
    raise AssertionError("kinks left after 30 redraws")


# ---- GPU helpers ------------------------------------------------------------------------------------------------------
def _model(name, d, P, U, I, seed=0, shared=True):
    """TUP or KTUP; KTUP: a fifth of the items unaligned (padding entity), the aligned ones on E = I / 3 entities, so
    several items share one.  Rows are scaled to norms in [0.8, 0.95] u [1.05, 1.2]: the fused normLoss is active on
    about half of them and no row sits near its kink.  The preference-side rows are scaled by PREF_SCALE on top: with
    unit rows the soft mixing r = sum_k z_k P'_k is a sum of random-sign terms whose magnitudes are ~100 times r
    itself, and a bound on that sum says little about the rest of the score."""
    import kgrec_b200 as K
    ktup, gumbel, l1 = MODELS[name]
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed + 1)
    if ktup:
        E = max(2, I // 3) if shared else 2 * I
        ents = rng.randint(0, E, I) if shared else rng.permutation(E)[:I]
        new_map = {i: ((int(ents[i]) if rng.rand() < 0.8 else -1), i) for i in range(I)}
        new_map[0] = (int(ents[0]), 0)
        new_map[I - 1] = (-1, I - 1)
        m = K.jTransUPModel(l1, d, U, I, E, P, {i: i for i in range(I)}, new_map, False, gumbel)
    else:
        m = K.TransUPModel(l1, d, U, I, P, gumbel)
    with torch.no_grad():
        for p in m.parameters():
            n = p.shape[0]
            f = torch.from_numpy(np.where(rng.rand(n) < 0.5, rng.uniform(0.8, 0.95, n), rng.uniform(1.05, 1.2, n)))
            p.mul_(f.float().to(p.device).view(-1, 1))
        for k, w in m._weights().items():
            if k in ("pref", "pref_norm", "rel", "norm"):
                w.mul_(PREF_SCALE)
    return m


def _kernels(fn, seen=None):
    """fn() under a CUDA profile: (its result, the kernel names); seen collects the names across calls (a short
    profile can miss records that the next one then shows, so one test checks the union of its profiles)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = " ".join(e.key for e in prof.key_averages())
    if seen is not None:
        seen.append(names)
    return out, names


class _Capture:
    """torch as the optimizer module sees it, recording the tensors torch.empty makes (step_pairs's score buffers)."""

    def __init__(self):
        self.made = []

    def __getattr__(self, k):
        return getattr(torch, k)

    def empty(self, *a, **kw):
        t = torch.empty(*a, **kw)
        self.made.append(t)
        return t


def _rows_opt(m):
    from kgrec_b200.optim import SparseRowOptimizer
    opt = SparseRowOptimizer(m, optimizer_type="SGD", lr=0.01)
    opt._update = lambda *a, **kw: None          # keep the accumulated gradients in opt.acc
    return opt


def _rows_step(opt, monkeypatch, pu, pi, ni, noise, loss="bpr", param=-1.0, bp=None, idx=torch.int64, reg=False):
    """One row-factored step: (pos scores, neg scores, per-batch loss, reg value, {table: gradient})."""
    from kgrec_b200 import optim as KO
    monkeypatch.setenv("KGREC_REC_ROWS", "force")
    cap = _Capture()
    monkeypatch.setattr(KO, "torch", cap)
    for v in opt.acc.values():
        v.zero_()
    K = len(ni) // len(pu)
    u, i, n = (torch.as_tensor(x, dtype=idx, device="cuda") for x in (pu, pi, ni))
    gu = torch.as_tensor(noise, dtype=torch.float32, device="cuda") if noise is not None else None
    out, reg_v = opt.step_pairs((u, i), (u.repeat_interleave(K), n), target=param, loss=loss, batch_pos=bp,
                                gumbel_u=gu, reg=reg)
    monkeypatch.setattr(KO, "torch", torch)
    assert opt._rows_ws is not None
    ps, ns = cap.made[0], cap.made[1]
    assert ps.numel() == len(pu) and ns.numel() == len(ni)
    g = {k: v.double().cpu().numpy() for k, v in opt.acc.items()}
    opt.model.check_indices()
    return ps.cpu().numpy(), ns.cpu().numpy(), out.cpu().numpy(), float(reg_v.item()), g


def _rows_case(name, d, P, n_pos, K, U, I, monkeypatch, seed=0, loss="bpr", param=-1.0, bp=None, idx=torch.int64,
               reuse=True, shared=True, seen=None):
    m = _model(name, d, P, U, I, seed, shared)
    R = Ref(m)
    rng = np.random.RandomState(seed + 7)
    pu, pi, ni, noise, S = _batch(R, rng, n_pos, K, U, I, loss, param, bp, reuse)
    opt = _rows_opt(m)
    run = lambda: _rows_step(opt, monkeypatch, pu, pi, ni, noise, loss, param, bp, idx)     # noqa: E731
    res = _kernels(run, seen)[0] if seen is not None else run()
    ps, ns, lo, _, g = res
    S.backward()
    _check_step(S, ps, ns, lo, g, "%s d=%d P=%d K=%d" % (name, d, P, K))
    return m, R, S


# ---- row-factored step -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_soft_l2", "tup_gumbel_l2"])
def test_rows_d_sweep(name, monkeypatch):
    for d in range(4, 129, 4):
        _rows_case(name, d, 20, 300, 2, 40, 60, monkeypatch, seed=d)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_soft_l1", "ktup_soft_l1", "ktup_soft_l2", "ktup_gumbel_l2"])
def test_rows_d_short(name, monkeypatch):
    for d in (4, 12, 36, 68, 100, 116, 128):
        _rows_case(name, d, 20, 300, 2, 40, 60, monkeypatch, seed=d)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS))
def test_rows_preference_counts(name, monkeypatch):
    """Every PT edge (P = 8 / 20 / 32 fill their instantiation, 9 / 21 start the next) and P % 4 != 0 for the (k & 3) == q
    stores of zx / cb; at d = 124 every unrolled chunk is in use."""
    seen = []
    for P in (1, 2, 7, 8, 9, 19, 20, 21, 31, 32):
        _rows_case(name, 124 if P in (8, 20, 32) else 36, P, 300, 3, 40, 60, monkeypatch, seed=P, seen=seen)
    names = " ".join(seen)
    fam = "gumbel" if MODELS[name][1] else "soft"
    for pt in (8, 20, 32):
        for k in ("fwd", "bwd", "tables"):
            assert "k_%s_rows_%s<%d>" % (fam, k, pt) in names, (pt, k)
    assert ("k_%s_pairs" % fam) in names


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS))
@pytest.mark.parametrize("K", [1, 2, 15, 16, 30, 31])
def test_rows_negatives_losses_ids(name, K, monkeypatch):
    """n_neg across the accepted range (ST-Gumbel's shared memory grows with (n_neg + 1) P); BPR with batch_pos not
    dividing n_pos, margin with batch_pos 1; int32 ids with heavy reuse, int64 ids with none."""
    loss, param, bp = ("bpr", -1.0, 37) if K % 2 else ("margin", 1.0, 1)
    _rows_case(name, 100, 20, 211, K, 30, 50, monkeypatch, seed=K, loss=loss, param=param, bp=bp, idx=torch.int32)
    n_pos = 40
    _rows_case(name, 68, 9, n_pos, K, n_pos + 7, 2 * n_pos * (K + 1) + 11, monkeypatch, seed=100 + K, loss=loss,
               param=param, bp=bp if bp == 1 else 13, idx=torch.int64, reuse=False, shared=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_soft_l1", "tup_soft_l2", "tup_gumbel_l2"])
def test_rows_fused_norm_loss(name, monkeypatch):
    """reg=True on TUP: the normLoss over the batch's user rows and the cat[pos, neg] item rows (duplicates counted
    each time) is fused into the pair kernel; the value and the accumulated gradient, with the orthogonal and
    preference-row terms the optimizer adds around it."""
    d, P, U, I, n_pos, K = 100, 20, 30, 40, 400, 3
    m = _model(name, d, P, U, I, seed=5)
    R = Ref(m)
    W = R.W
    for t in ("user", "item", "pref"):        # no row near the normLoss kink
        n2 = (W[t] ** 2).sum(1)
        assert (np.abs(n2 - 1) > 4 * R.tau * n2).all()
    rng = np.random.RandomState(5)
    pu, pi, ni, noise, S = _batch(R, rng, n_pos, K, U, I)
    opt = _rows_opt(m)
    ps, ns, lo, reg, g = _rows_step(opt, monkeypatch, pu, pi, ni, noise, reg=True)
    S.backward()
    rows = {"user": pu, "item": np.concatenate([pi, ni])}
    val = O.orthogonal_loss(W["pref"], W["pref_norm"]) + O.norm_loss(W["pref"])
    tval = ((np.abs(W["pref_norm"]) * np.abs(W["pref"])).sum(1) ** 2 / (W["pref"] ** 2).sum(1)).sum() + (W["pref"] ** 2).sum()
    go, gn = O.orthogonal_loss_grads(W["pref"], W["pref_norm"])
    qa = (np.abs(W["pref_norm"]) * np.abs(W["pref"])).sum(1, keepdims=True) / (W["pref"] ** 2).sum(1, keepdims=True)
    ref = {"pref": go + O.norm_loss_grads(W["pref"]), "pref_norm": gn}
    twin = {"pref": 2 * qa * np.abs(W["pref_norm"]) + 2 * qa * qa * np.abs(W["pref"]) + 2 * np.abs(W["pref"]),
            "pref_norm": 2 * qa * np.abs(W["pref"])}
    for t, ids in rows.items():
        x = W[t][ids]
        val += O.norm_loss(x)
        tval += (x ** 2).sum()
        ref[t] = _scatter(W[t].shape[0], ids, O.norm_loss_grads(x))
        twin[t] = _scatter(W[t].shape[0], ids, 2 * np.abs(x))
    _check([reg], [val], [tval], R.tau, name + " reg value")
    S.grads_ref = _add(dict(S.grads_ref), ref)
    S.grads_twin = _add(dict(S.grads_twin), twin)
    _check_step(S, ps, ns, lo, g, name + " reg")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS))
def test_rows_two_steps(name, monkeypatch):
    """Two steps on one optimizer with different batches over a shared subset of rows: the second step's accumulators
    hold that step's gradient alone (the backward left G_RA / G_WB, GZ / CK and KTUP's item work buffer clean)."""
    if name.endswith("l1") and "gumbel" in name:
        pytest.skip("not built")
    d, P, U, I = 128, 20, 50, 80
    m = _model(name, d, P, U, I, seed=9)
    R = Ref(m)
    opt = _rows_opt(m)
    rng = np.random.RandomState(9)
    for step, (lo_u, lo_i) in enumerate(((0, 0), (15, 25))):       # users 15..34 and items 25..54 are in both
        pu, pi, ni, noise, S = _batch(R, rng, 500, 3, U - 15 + lo_u, I - 25 + lo_i, bp=128, lo=(lo_u, lo_i))
        S.backward()
        ps, ns, lo, _, g = _rows_step(opt, monkeypatch, pu, pi, ni, noise, bp=128)
        _check_step(S, ps, ns, lo, g, "%s step %d" % (name, step))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tup_gumbel_l2", "ktup_gumbel_l2"])
def test_rows_hashed_noise(name, monkeypatch):
    """gumbel_u=None: the rows engine draws its own noise (Philox keyed by seed, positive, block).  Every pair's score
    is, within its bound, the float64 score with exactly one preference selected; two calls with one seed repeat bit
    for bit."""
    d, P, U, I, n_pos, K = 100, 20, 40, 60, 400, 3
    m = _model(name, d, P, U, I, seed=13)
    R = Ref(m)
    rng = np.random.RandomState(13)
    pu, pi, ni = rng.randint(0, U, n_pos), rng.randint(0, I, n_pos), rng.randint(0, I, n_pos * K)
    opt = _rows_opt(m)
    runs = []
    for _ in range(2):
        torch.manual_seed(77)
        m._seed_counter = 0
        runs.append(_rows_step(opt, monkeypatch, pu, pi, ni, None))
    assert np.array_equal(runs[0][0].view(np.uint32), runs[1][0].view(np.uint32))
    assert np.array_equal(runs[0][1].view(np.uint32), runs[1][1].view(np.uint32))
    got = np.concatenate([runs[0][0], runs[0][1]]).astype(np.float64)
    uid, iid = np.concatenate([pu, np.repeat(pu, K)]), np.concatenate([pi, ni])
    hit = np.zeros(len(uid), dtype=bool)
    for k in range(P):       # force preference k: the uniforms of k at 1, every other at 0
        nz = np.full((len(uid), P), 1e-30)
        nz[:, k] = 1.0 - 1e-7
        one = R.score(uid, iid, nz)
        q = R.pairs(uid, iid, nz)
        hit |= np.abs(got - one) <= R.tau * q["twin"]
    assert hit.all(), "%d pairs match no single preference" % (~hit).sum()


# ---- tile engine and one warp per pair (the model API) --------------------------------------------------------------
def _call(m, R, u, i, noise):
    nz = torch.as_tensor(noise, dtype=torch.float32, device="cuda") if noise is not None else None
    u, i = torch.as_tensor(u, device="cuda"), torch.as_tensor(i, device="cuda")
    if R.ktup:
        return m((u, i), None, is_rec=True, gumbel_u=nz)
    return m(u, i, gumbel_u=nz)


def _dense_grads(m, R):
    out = {}
    for k, w in m._weights().items():
        g = w.grad
        out[k] = np.zeros(w.shape) if g is None else (g.to_dense() if g.is_sparse else g).double().cpu().numpy()
    return out


def _flat_case(m, R, rng, n, gm, tag, check_slots=False):
    """score_fwd then score_bwd on n flat pairs with explicit noise and a random upstream gradient."""
    U, I = R.W["user"].shape[0], R.W["item"].shape[0]
    pu, pi, ni, noise, S = _batch(R, rng, n, 1, U, I)
    u, i = np.concatenate([pu, pu]), np.concatenate([pi, ni])
    nz = noise
    q = R.pairs(u, i, nz)
    ref = R.score(u, i, nz)
    up = rng.randn(len(u)) / 4
    up = up.astype(np.float32).astype(np.float64)
    m.grad_mode = gm
    m.zero_grad()
    s = _call(m, R, u, i, nz)
    _check(s.detach().cpu().numpy(), ref, q["twin"], R.tau, tag + " scores")
    s.backward(torch.as_tensor(up, dtype=torch.float32, device="cuda"))
    got = _dense_grads(m, R)
    want = R.grads(u, i, nz, up)
    twin = R.twin_grads(u, i, q, np.abs(up))
    for k in want:
        _check(got[k], want[k], twin[k], R.tau, tag + " grad " + k)
    if check_slots:
        w = m._weights()
        assert torch.equal(w["user"].grad._indices().view(-1).cpu(), torch.as_tensor(u))
        assert torch.equal(w["item"].grad._indices().view(-1).cpu(), torch.as_tensor(i))
        if R.ktup:
            assert torch.equal(w["ent"].grad._indices().view(-1).cpu(), torch.as_tensor(R.i2e[i]))
    m.check_indices()


def _group_case(m, R, rng, n_pos, K, tag, loss, param, bp, step=True):
    U, I = R.W["user"].shape[0], R.W["item"].shape[0]
    pu, pi, ni, noise, S = _batch(R, rng, n_pos, K, U, I, loss, param, bp)
    S.backward()
    dev = lambda x: torch.as_tensor(x, device="cuda")      # noqa: E731
    nz = torch.as_tensor(noise, dtype=torch.float32, device="cuda") if noise is not None else None
    pos, neg = (dev(pu), dev(pi)), (dev(np.repeat(pu, K)), dev(ni))
    m.grad_mode = "dense"
    m.zero_grad()
    if step:
        lo, ps, ns = m.loss_step(pos, neg, target=param, loss=loss, batch_pos=bp, gumbel_u=nz)
        _check_step(S, ps.detach().cpu().numpy(), ns.detach().cpu().numpy(), lo.detach().cpu().numpy(),
                    _dense_grads(m, R), tag + " step")
    else:
        lo, ps, ns = m.rank_loss(pos, neg, target=param, loss=loss, batch_pos=bp, gumbel_u=nz)
        _check_step(S, ps.detach().cpu().numpy(), ns.detach().cpu().numpy(), lo.detach().cpu().numpy(), None,
                    tag + " rank_loss")
    m.check_indices()


@pytest.mark.gpu
@pytest.mark.parametrize("P,pt", [(5, 8), (20, 20), (27, 32)])
@pytest.mark.parametrize("gumbel", [False, True])
def test_tile_engine(P, pt, gumbel, monkeypatch):
    """k_rec_tile<PT, GUM, MODE> forced for every mode: flat forward (several tiles per CTA, a ragged last tile), flat
    backward in dense and sparse grad_mode (slot ids checked), the fused rank loss forward, and the single-pass step
    for n_neg 1 / 7 / 15; n_neg = 16 has no room in the 16 pair slots and falls back to forward + backward."""
    monkeypatch.setenv("KGREC_REC_TILE", "force")
    monkeypatch.setenv("KGREC_REC_ROWS", "0")
    gum = "true" if gumbel else "false"
    seen = []
    for j, d in enumerate((4, 52, 100, 128)):
        name = ("ktup_" if j % 2 else "tup_") + ("gumbel_l2" if gumbel else ("soft_l1" if d == 52 else "soft_l2"))
        m = _model(name, d, P, 300, 400, seed=d + P)
        R = Ref(m)
        rng = np.random.RandomState(d * P)
        tag = "%s d=%d P=%d" % (name, d, P)
        n = 4500 + 13 * j            # > 132 SMs x 2 warps x 16 slots: several tiles per CTA, ragged last tile
        _kernels(lambda: _flat_case(m, R, rng, n, "dense", tag + " dense"), seen)
        _flat_case(m, R, rng, 3001, "sparse", tag + " sparse", check_slots=True)
        _kernels(lambda: _group_case(m, R, rng, 1500, 3, tag, "bpr", -1.0, 100, step=False), seen)
        def groups():
            for K in (1, 7, 15, 16):
                loss, param = ("margin", 1.0) if K == 7 else ("bpr", -1.0)
                _group_case(m, R, rng, 700, K, tag + " K=%d" % K, loss, param, 64)
        _kernels(groups, seen)
    names = " ".join(seen)
    for mode in (0, 1, 2):          # FWD, BWD (flat backward, and the fallback of n_neg = 16), STEP
        assert "k_rec_tile<%d, %s, %d>" % (pt, gum, mode) in names, (mode, names)


PAIR_CASES = [   # (d, P for the backward, NCH, VEC, PR)
    (4, 7, 1, True, 4), (50, 33, 1, False, 8), (100, 64, 1, True, 8), (128, 33, 1, True, 8), (130, 16, 4, False, 2),
    (132, 32, 2, True, 4), (200, 20, 2, True, 4), (255, 16, 4, False, 2), (256, 32, 2, True, 4), (300, 16, 4, True, 2),
    (511, 16, 4, False, 2), (512, 16, 4, True, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("d,P,nch,vec,pr", PAIR_CASES)
def test_pair_engine(d, P, nch, vec, pr, monkeypatch):
    """The one-warp-per-pair kernels at every (NCH, VEC) build, P at the backward limit of each d band, TUP and KTUP,
    soft L1 / L2 and ST-Gumbel: flat forward + backward, the fused rank loss, and the step (forward + backward)."""
    monkeypatch.setenv("KGREC_REC_TILE", "0")
    monkeypatch.setenv("KGREC_REC_ROWS", "0")
    v = "true" if vec else "false"
    seen = []
    l1 = "ktup_soft_l1" if d <= 200 else "ktup_soft_l2"     # wider L1 rows put too many residuals within the bound of 0
    for j, name in enumerate(("tup_soft_l2", l1, "tup_gumbel_l2", "ktup_gumbel_l2")):
        m = _model(name, d, P, 120, 150, seed=d + j)
        R = Ref(m)
        rng = np.random.RandomState(d + 31 * j)
        tag = "%s d=%d P=%d" % (name, d, P)
        _kernels(lambda: _flat_case(m, R, rng, 150, "dense", tag), seen)
        _kernels(lambda: _group_case(m, R, rng, 90, 3, tag, "bpr", -1.0, 32, step=False), seen)
        _group_case(m, R, rng, 90, 2, tag, "margin", 1.0, 1)
    names = " ".join(seen)
    assert re.search(r"k_score_fwd<3, %d, %s>" % (nch, v), names)           # FAM_REC = 3
    assert re.search(r"k_score_bwd<3, %d, %s, %d>" % (nch, v, pr), names)
    assert re.search(r"k_rank_loss_fwd<3, %d, %s>" % (nch, v), names)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [4, 128, 200, 256, 300, 512])
def test_pair_engine_forward_limit(d, monkeypatch):
    """Forward-only shapes: the largest P the host accepts at d (the step's backward is refused there)."""
    from kgrec_b200 import _lib
    monkeypatch.setenv("KGREC_REC_TILE", "0")
    lib = _lib.load()
    P = _max_p(lambda dd, pp: _fwd_rc(lib, _lib, _lib.TUP, dd, pp) == 0, d)
    for name in ("tup_soft_l2", "ktup_gumbel_l2"):
        m = _model(name, d, P, 60, 80, seed=d)
        R = Ref(m)
        rng = np.random.RandomState(d)
        pu, pi, ni, noise, S = _batch(R, rng, 100, 2, 60, 80)
        _check(_call(m, R, pu, pi, noise[:100] if noise is not None else None).detach().cpu().numpy(), S.sp, S.tp,
               R.tau, "%s d=%d P=%d fwd" % (name, d, P))
        _group_case(m, R, rng, 100, 2, "%s d=%d P=%d" % (name, d, P), "bpr", -1.0, 40, step=False)
