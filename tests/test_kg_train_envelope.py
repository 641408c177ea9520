"""The whole envelope the TransE / TransH / TransR training entry points accept, against float64.

Kernels, and what picks them (restated in `dispatch` below):
  kgrec_corrupt_loss_step / _fwd / _bwd (csrc/train_group.cu), negatives in the corrupt format
    k_group_step_e / _h        TransE / TransH, d <= 128, K <= 32, slot offsets and score indices in 32 bits
    k_group_step_e_tma         TransE STEP with slot gradients, no fused regulariser, K <= 29, ld == dim, its ring in
                               225 KB of shared memory and at least 2 groups per warp of every SM
    k_group_step<FAM, NCH>     every other TransE / TransH shape (+ k_group_slot_ids for the slot row ids)
    k_run_step_r               TransR STEP, d >= 32 and n_pos >= 4 n_rel (groups sorted by relation: k_rel_*)
    k_group_step_r<NVT>        TransR STEP otherwise
  kgrec_score_fwd / _bwd, kgrec_rank_loss_fwd / _bwd / _step (csrc/train_dev.cuh), expanded triples
    k_score_fwd / k_rank_loss_fwd / k_score_bwd<FAM, NCH, VEC>
Each case checks, at every element of the scores, the per-batch losses and the gradient tables (dense tables and
sparse slots),
    |kernel - ref| <= C_BOUND (d + K + 2 + m) 2^-24 twin
where ref is the oracle (oracle/kg_oracle.py) on float64 copies of the tables, m the number of contributions summed
into the element (0 for a slot, the number of slots scattered into a row under dense accumulation, the groups of a
batch for its loss), and twin the same computation with every operand replaced by its magnitude and every subtraction
by an addition, scattered exactly like the gradients.  An element whose twin is 0 must be exactly 0: rows the step did
not touch, and padding columns of strided tables (filled with NaN) that must not reach a gradient.  Sparse slot ids
must equal [h, t, c_1 .. c_K] and r per group exactly.  Kinks are screened out before the call: a group with a triple
within its bound of the hinge or of an L1 residual component e_k = 0 is redrawn (at most 3 % of the first draw's
triples, or 3 triples of a small batch, may need it; L1 stops at d = 200, d = 64 for TransR, where wider rows put more
residual components within the bound of 0); rows are scaled to norms in [0.8, 0.95] u [1.05, 1.2], away from the kink of the fused
normLoss.  The upstream twin is |g|: 0 / 1 for the margin loss; for BPR the coefficient (with its 1 / (cnt K)) plus
its sensitivity to the scores' own rounding, as in the recommendation envelope.  Profiles name the kernel each case
was meant to reach.

C_BOUND = 1 is the smallest integer constant the cases pass with: half the recommendation-training envelope's 2
(tests/test_rec_train_envelope.py) and an eighth of the evaluation envelope's 8 (tests/test_eval_envelope.py).

Which case covers which part of the envelope:
  register step kernels, every d % 4 == 0 in 4..128 (L2) and a short L1 list, K in {1, 2, 15, 16, 31, 32}, margin /
    BPR, dense / sparse, int32 / int64, ragged batches and batch_pos 1, fused reg, ids 0 and n - 1, heavy reuse
    and none ...................................................................... test_register_step
  FWD / BWD through rank_loss_corrupt + autograd, a different weight per batch ...... test_fwd_bwd_modes
  general kernel k_group_step<FAM, NCH> in STEP / FWD / BWD, NCH 2 / 4, K 33..64 ..... test_general_kernel
  TMA kernel: NS 16 / 32, K = 29, the ring-fit edges, the smallest launch ............ test_tma_kernel
  TransR run kernel at every d % 4 == 0 in 32..128, warp kernel nvt edges, the run /
    warp boundary, n_rel around 1024 (k_rel_scan's per > 1), reg, BPR, sparse ....... test_transr_*
  expanded-triple kernels at 17 widths, VEC false three ways ......................... test_expanded_kernels
  strided tables (ld = d + 4 / d + 1), and ld != dim keeps TransE off the TMA kernel .. test_strided_*
  slot offsets either side of the 32-bit limit (about 5 GB) ......................... test_slot_offsets_near_32_bits
On the CPU: the accepted region of every entry point with its messages, and the fused-regulariser rule at n_pos = 0.
Run time on one H100 80GB HBM3 at a 700 W power limit: about 90 s for the GPU cases.
"""
import ctypes as C
import math
import re

import numpy as np
import pytest
import torch

from oracle import kg_oracle as O

U24 = 2.0 ** -24
C_BOUND = 1
FAKE = 0x7000_0000_1000
INVALID, UNSUPPORTED = 1, 2          # KGREC_ERR_* (include/kgrec_b200.h)
STEP, FWD, BWD = "step", "fwd", "bwd"
TRANSE, TRANSH, TRANSR = 0, 1, 2     # kgrec model ids, and the FAM_* template values of the kernels
TMA_WARPS, TMA_STAGES = 16, 2


# ---- the dispatch, restated --------------------------------------------------------------------------------------------
def tma_smem(d, K):
    """group_step_tma_smem: the per-warp barriers and id slots, rounded to 128 bytes, and the row ring."""
    return ((TMA_WARPS * TMA_STAGES * (8 + 128) + 127) & ~127) + TMA_WARPS * TMA_STAGES * (3 + K) * d * 4


def on_registers(model, d, K, n_pos):
    """group_on_registers: TransE / TransH, NCH 1, K <= 32, slot offsets and score indices in 32 bits."""
    return model in (TRANSE, TRANSH) and d <= 128 and K <= 32 and n_pos * (2 + K) * d * 4 < 4.0e9 and n_pos * K < 2.0e9


def _b(x):
    return "true" if x else "false"


def dispatch(model, d, K, n_pos, mode, dense, reg, ld_eq, sms, l1=False, margin=True, n_rel=1):
    """The kernels kgrec_corrupt_loss_step / _fwd / _bwd launch for a shape, as profile names."""
    if model == TRANSR:
        assert mode == STEP
        if d >= 32 and n_pos >= 4 * n_rel:
            NC, qf = d // 4, d // 32
            if NC <= 16:
                qa, qb, qf, rb = 1, 1, (1 if qf <= 1 else 2), 2
            elif NC <= 27:
                qa, qb, qf, rb = 1, 3, (2 if qf <= 2 else 3), 2
            else:
                qa, qb, qf, rb = 2, 2, (3 if qf <= 3 else 4), 1
            return ["k_run_step_r<%d, %d, %d, %d, %s, %s>" % (qa, qb, qf, rb, _b(margin or reg), _b(reg))]
        nvt = 4 if K <= 2 else (12 if K <= 10 else 16)
        return ["k_group_step_r<%d, %s, %s>" % (nvt, _b(margin or reg), _b(reg))]
    reg_ok = on_registers(model, d, K, n_pos)
    if (mode == STEP and model == TRANSE and reg_ok and not dense and not reg and K <= 29 and ld_eq
            and tma_smem(d, K) <= 225 * 1024 and n_pos >= TMA_STAGES * TMA_WARPS * sms):
        return ["k_group_step_e_tma<%s, %s, 16, %d>" % (_b(l1), _b(margin), 16 if K < 16 else 32)]
    if reg_ok:
        name = "k_group_step_e" if model == TRANSE else "k_group_step_h"
        if mode == FWD:
            f = (l1, False, margin, False, False, True)
        elif mode == BWD:
            f = (l1, dense, margin, False, True, False)
        else:
            f = (l1, dense, True, True, False, False) if reg else (l1, dense, margin, False, False, False)
        return ["%s<%s>" % (name, ", ".join(_b(x) for x in f))]
    nch = 1 if d <= 128 else (2 if d <= 256 else 4)
    out = ["k_group_step<%d, %d, %s, %s, %s>" % (model, nch, _b(l1), _b(mode == BWD), _b(mode == FWD))]
    if not dense and mode != FWD:
        out.append("k_group_slot_ids")
    return out


def expanded_build(d, ld, aligned):
    """(NCH, VEC) of k_score_fwd / k_rank_loss_fwd / k_score_bwd (make_plan, KGREC_DISPATCH_ROW)."""
    vec = aligned and d % 4 == 0 and ld % 4 == 0
    nch = 1 if d <= 128 else (2 if d <= 256 else 4)
    if not vec and nch == 2:
        nch = 4
    return nch, vec


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_tma_ring_edges():
    """The ring-fit edges the TMA cases use, derived from the restated group_step_tma_smem."""
    fits = lambda d, K: tma_smem(d, K) <= 225 * 1024        # noqa: E731
    assert fits(128, 10) and not fits(128, 11)
    assert fits(100, 14) and not fits(100, 15)
    assert fits(96, 15) and not fits(100, 15)
    assert fits(92, 16) and not fits(96, 16)
    assert fits(52, 29) and not fits(56, 29)


def _tables(lib, _lib, model, d, ld, off):
    p = FAKE + off
    return _lib.Tables(dim=d, ld=ld, n_ent=50, n_rel=7, ent=p, rel=p, norm=p, proj=p)


def _corrupt_rc(lib, _lib, entry, model, d, K, reg, ld, off, ib, loss, n_pos=0):
    t = _tables(lib, _lib, model, d, ld, off)
    g = _lib.Grads(mode=1, ent=FAKE, rel=FAKE, norm=FAKE, proj=FAKE)
    if entry == STEP:
        rc = lib.kgrec_corrupt_loss_step(C.byref(t), model, FAKE, FAKE, FAKE, ib, n_pos, FAKE, K, 4, loss, 1.0, 1.0, reg,
                                         FAKE, FAKE, FAKE, C.byref(g), None, None, FAKE, None, None)
    elif entry == FWD:
        rc = lib.kgrec_corrupt_loss_fwd(C.byref(t), model, FAKE, FAKE, FAKE, ib, n_pos, FAKE, K, 4, loss, 1.0, FAKE, FAKE,
                                        FAKE, FAKE, None, None)
    else:
        rc = lib.kgrec_corrupt_loss_bwd(C.byref(t), model, FAKE, FAKE, FAKE, ib, n_pos, FAKE, K, 4, loss, 1.0, FAKE, FAKE,
                                        1.0, None, C.byref(g), None, None, None)
    return rc, lib.kgrec_last_error().decode()


def _corrupt_expect(entry, model, d, K, reg, ld, off, ib, loss):
    """(rc, message) the host checks of kgrec_corrupt_loss_* give, in their order."""
    if ld < d:
        return INVALID, "bad dim/ld (%d/%d)" % (d, ld)
    if d > 512:
        return UNSUPPORTED, "embedding_size %d > 512 is not built" % d
    if model == TRANSR and entry != STEP:
        return UNSUPPORTED, "corrupt-format ranking loss is built for TransE / TransH (model 2)"
    if not (off == 0 and d % 4 == 0 and ld % 4 == 0):
        return UNSUPPORTED, "corrupt-format ranking loss needs embedding_size % 4 == 0 and 16-byte aligned tables"
    if ib not in (4, 8):
        return INVALID, "idx_bytes must be 4 or 8"
    if entry != STEP:
        return 0, None
    if reg and loss != 0:
        return UNSUPPORTED, "fused regularisers go with the margin loss (the KG drivers' loss)"
    if model == TRANSR and (d > 128 or K > 14):
        return UNSUPPORTED, "TransR step kernel: embedding_size <= 128 and at most 14 negatives per positive"
    if reg and model != TRANSR and not (d <= 128 and K <= 32):
        return UNSUPPORTED, "fused regularisers are built for the d <= 128 margin-loss step kernels only"
    return 0, None


def test_corrupt_format_accepted_region_is_pinned():
    """kgrec_corrupt_loss_step / _fwd / _bwd for TransE / TransH / TransR over d up to 516, K in {1, 14, 15, 29, 32,
    33}, reg, ld in {d, d + 1, d + 4}, a table base off by one float, idx_bytes in {2, 4, 8} and both losses: each
    call is accepted or refused exactly where the restated checks say, with their message."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    seen = {}
    for entry in (STEP, FWD, BWD):
        for model in (TRANSE, TRANSH, TRANSR):
            for d in (4, 6, 32, 100, 128, 130, 132, 256, 512, 516):
                for K in (1, 14, 15, 29, 32, 33):
                    for reg in ((0, 1) if entry == STEP else (0,)):
                        for ld, off in ((d, 0), (d + 1, 0), (d + 4, 0), (d, 4), (d - 1, 0)):
                            for ib in (2, 4, 8):
                                for loss in (0, 1):
                                    want = _corrupt_expect(entry, model, d, K, reg, ld, off, ib, loss)
                                    rc, msg = _corrupt_rc(lib, _lib, entry, model, d, K, reg, ld, off, ib, loss)
                                    key = (entry, model, d, K, reg, ld - d, off, ib, loss)
                                    assert rc == want[0], (key, want, msg)
                                    if rc:
                                        assert msg == want[1], (key, msg)
                                    kind = re.sub(r"\d+", "#", want[1] or "accepted")
                                    seen[kind] = seen.get(kind, 0) + 1
    assert len(seen) == 9 and all(v > 10 for v in seen.values()), seen


def test_fused_regulariser_rule_at_zero_positives():
    """An empty call accepts exactly the shapes a real call does: the fused-regulariser rule for TransE / TransH (d
    <= 128 and K <= 32, the register step kernels) is checked before the n_pos == 0 return."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    for model in (TRANSE, TRANSH):
        for d, K in ((128, 32), (132, 1), (256, 10), (512, 1), (128, 33), (100, 64), (4, 1)):
            rc, msg = _corrupt_rc(lib, _lib, STEP, model, d, K, 1, d, 0, 4, 0)
            if d <= 128 and K <= 32:
                assert rc == 0, (model, d, K, msg)
            else:
                assert rc == UNSUPPORTED and msg == "fused regularisers are built for the d <= 128 margin-loss step " \
                                                     "kernels only", (model, d, K, msg)
            rc, _ = _corrupt_rc(lib, _lib, STEP, model, d, K, 0, d, 0, 4, 0)
            assert rc == 0


def test_expanded_accepted_region_is_pinned():
    """kgrec_score_fwd / _bwd and kgrec_rank_loss_fwd / _bwd / _step for TransE / TransH / TransR: every d up to 512,
    any ld >= d and any alignment (the scalar rows take what the 128-bit rows cannot), idx_bytes 4 or 8."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    g = _lib.Grads(mode=1, ent=FAKE, rel=FAKE, norm=FAKE, proj=FAKE)
    for model in (TRANSE, TRANSH, TRANSR):
        for d in (1, 3, 4, 127, 129, 130, 255, 257, 511, 512, 513, 516):
            for ld, off in ((d, 0), (d + 1, 0), (d, 4), (d - 1, 0)):
                for ib in (2, 4, 8):
                    t = _tables(lib, _lib, model, d, ld, off)
                    rcs = [
                        lib.kgrec_score_fwd(C.byref(t), model, FAKE, FAKE, FAKE, ib, 0, None, 0, FAKE, None, None),
                        lib.kgrec_score_bwd(C.byref(t), model, FAKE, FAKE, FAKE, ib, 0, None, 0, FAKE, C.byref(g), None),
                        lib.kgrec_rank_loss_fwd(C.byref(t), model, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, ib, 0, 14, 4, 0,
                                                1.0, None, 0, FAKE, FAKE, FAKE, FAKE, None, None),
                        lib.kgrec_rank_loss_bwd(C.byref(t), model, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, ib, 0, 33, 4, 1,
                                                -1.0, None, 0, FAKE, FAKE, 1.0, None, C.byref(g), None),
                        lib.kgrec_rank_loss_step(C.byref(t), model, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, ib, 0, 29, 4, 0,
                                                 1.0, 1.0, None, 0, FAKE, FAKE, FAKE, C.byref(g), None, None, None, FAKE,
                                                 None, None)]
                    if ld < d:
                        want = (INVALID, "bad dim/ld (%d/%d)" % (d, ld))
                    elif d > 512:
                        want = (UNSUPPORTED, "embedding_size %d > 512 is not built" % d)
                    elif ib not in (4, 8):
                        want = (INVALID, "idx_bytes must be 4 or 8")
                    else:
                        want = (0, None)
                    assert rcs == [want[0]] * 5, (model, d, ld, off, ib, rcs)
                    if want[0]:
                        assert lib.kgrec_last_error().decode() == want[1]


# ---- float64 reference and its absolute-value twin --------------------------------------------------------------------
def _norms(rng, n):
    return np.where(rng.rand(n) < 0.5, rng.uniform(0.8, 0.95, n), rng.uniform(1.05, 1.2, n))


class Tabs:
    """A TransE / TransH / TransR model's tables on the device, rows of pitch ld at a base `off` floats into their
    buffer (padding and the gap filled with NaN), and their float64 copies."""

    NAMES = {TRANSE: ("ent", "rel"), TRANSH: ("ent", "rel", "norm"), TRANSR: ("ent", "rel", "proj")}

    def __init__(self, model, d, E, R, seed, l1=False, ld=None, off=0):
        from kgrec_b200 import _lib
        rng = np.random.RandomState(seed)
        self.model, self.d, self.E, self.R, self.l1 = model, d, E, R, l1
        self.ld, self.off = ld or d, off
        self.W, self.buf, ptr = {}, {}, {}
        for nm in self.NAMES[model]:
            rows = E if nm == "ent" else R
            if nm == "proj":
                x = rng.randn(rows, d * d) / math.sqrt(d)
                b = torch.as_tensor(x.astype(np.float32), device="cuda").contiguous()
                ptr[nm] = b.data_ptr()
            else:
                x = rng.randn(rows, d)
                x *= (_norms(rng, rows) / np.linalg.norm(x, axis=1))[:, None]
                b = torch.full((rows * self.ld + off + 4,), float("nan"), dtype=torch.float32, device="cuda")
                b[off:off + rows * self.ld].view(rows, self.ld)[:, :d] = torch.as_tensor(x.astype(np.float32),
                                                                                        device="cuda")
                ptr[nm] = b.data_ptr() + 4 * off
            self.W[nm] = x.astype(np.float32).astype(np.float64)
            self.buf[nm] = b
        self.T = _lib.Tables(dim=d, ld=self.ld, l1=int(l1), n_ent=E, n_rel=R, ent=ptr["ent"], rel=ptr["rel"],
                             norm=ptr.get("norm", 0), proj=ptr.get("proj", 0))

    def terms(self, h, t, r, g, tg):
        """Per triple: the score and its twin, and the gradients of g * score with respect to the head row (the tail's
        is its negative), the relation row, the normal (TransH) and the matrix (TransR), each with its twin."""
        W, l1, d = self.W, self.l1, self.d
        xh, xt, rr = W["ent"][h], W["ent"][t], W["rel"][r]
        ah, at, ar = np.abs(xh), np.abs(xt), np.abs(rr)
        out = {}
        if self.model == TRANSE:
            e, a = xh + rr - xt, ah + ar + at
        elif self.model == TRANSH:
            w = W["norm"][r]
            aw = np.abs(w)
            e = O.proj_hyperplane(xh, w) + rr - O.proj_hyperplane(xt, w)
            a = ah + (ah * aw).sum(-1, keepdims=True) * aw + ar + at + (at * aw).sum(-1, keepdims=True) * aw
        else:
            M = W["proj"][r].reshape(-1, d, d)
            aM = np.abs(M)
            e = np.einsum("bij,bj->bi", M, xh - xt) + rr
            a = np.einsum("bij,bj->bi", aM, ah + at) + ar
        out["e"], out["a"] = e, a
        out["s"] = O.dist(e, l1)
        out["st"] = a.sum(-1) if l1 else (a * a).sum(-1)
        if g is None:
            return out
        eps = g[:, None] * O.ddist(e, l1)
        epsa = tg[:, None] * (np.ones_like(a) if l1 else 2 * a)
        out["eps"], out["epsa"] = eps, epsa
        if self.model == TRANSE:
            out["gx"], out["gxa"] = eps, epsa
        elif self.model == TRANSH:
            ew = (eps * w).sum(-1, keepdims=True)
            ewa = (epsa * aw).sum(-1, keepdims=True)
            x, xa = xh - xt, ah + at
            xw, xwa = (x * w).sum(-1, keepdims=True), (xa * aw).sum(-1, keepdims=True)
            out["gx"], out["gxa"] = eps - ew * w, epsa + ewa * aw
            out["gw"], out["gwa"] = -(ew * x + xw * eps), ewa * xa + xwa * epsa
        else:
            out["gx"], out["gxa"] = np.einsum("bij,bi->bj", M, eps), np.einsum("bij,bi->bj", aM, epsa)
            out["gM"] = np.einsum("bi,bj->bij", eps, xh - xt).reshape(len(r), -1)
            out["gMa"] = np.einsum("bi,bj->bij", epsa, ah + at).reshape(len(r), -1)
        return out


def _scatter(rows, idx, vals):
    out = np.zeros((rows, vals.shape[1]))
    np.add.at(out, idx, vals)
    return out


def _upstream(sp, sn, tp, tn, K, loss, param, bp, wb):
    """Per-batch losses with their twins, and dLoss/dscore of every positive and negative with its twin; batch b's
    upstream is wb[b]."""
    n_pos = len(sp)
    spr, tpr = np.repeat(sp, K), np.repeat(tp, K)
    nb = (n_pos + bp - 1) // bp
    lo, tlo, cnts = np.zeros(nb), np.zeros(nb), np.zeros(nb)
    gn, tgn = np.zeros(n_pos * K), np.zeros(n_pos * K)
    for b in range(nb):
        sl = slice(b * bp * K, min(n_pos, (b + 1) * bp) * K)
        cnt = sl.stop - sl.start
        cnts[b] = cnt // K
        if loss == "bpr":
            lo[b] = O.bpr_loss(spr[sl], sn[sl], param)
            gp_, _ = O.bpr_loss_grads(spr[sl], sn[sl], param)
            x = param * (spr[sl] - sn[sl])
            sig = 1 / (1 + np.exp(x))
            hh = param * param * sig * (1 - sig) / cnt
            gn[sl] = -gp_ * wb[b]
            tgn[sl] = (np.abs(gp_) + hh * (tpr[sl] + tn[sl])) * abs(wb[b])
            soft = np.maximum(-x, 0) + np.log1p(np.exp(-np.abs(x)))
            tlo[b] = (soft + abs(param) * sig * (tpr[sl] + tn[sl]) + 1.0).sum() / cnt
        else:
            lo[b] = O.margin_loss(spr[sl], sn[sl], param)
            act, _ = O.margin_loss_grads(spr[sl], sn[sl], param)
            gn[sl] = -act * wb[b]
            tgn[sl] = act * abs(wb[b])
            tlo[b] = (act * (tpr[sl] + tn[sl] + np.abs(spr[sl]) + np.abs(sn[sl]) + abs(param))).sum()
    gp = -gn.reshape(n_pos, K).sum(-1)
    tgp = tgn.reshape(n_pos, K).sum(-1)
    return lo, tlo, cnts, gp, gn, tgp, tgn


class Groups:
    """n_pos groups (h, t, r, K corrupted ids) and their float64 step: scores, per-batch losses (+ the fused
    regularisers), and the gradients as per-group slots (ent [n_pos, 2 + K], rel / norm [n_pos], dense proj) with
    twins."""

    def __init__(self, tabs, h, t, r, c, K, loss="margin", param=1.0, bp=None):
        self.tabs, self.K, self.loss, self.param = tabs, K, loss, param
        self.h, self.t, self.r, self.c = h, t, r, c
        n = self.n = len(h)
        self.bp = bp or n
        cc = c.reshape(n, K)
        self.head = cc < 0
        self.cid = np.where(self.head, ~cc, cc)
        nh = np.where(self.head, self.cid, h[:, None]).ravel()
        nt = np.where(self.head, t[:, None], self.cid).ravel()
        self.TH, self.TT = np.concatenate([h, nh]), np.concatenate([t, nt])
        self.TR = np.concatenate([r, np.repeat(r, K)])
        q = tabs.terms(self.TH, self.TT, self.TR, None, None)
        self.q = q
        self.sp, self.sn, self.tp, self.tn = q["s"][:n], q["s"][n:], q["st"][:n], q["st"][n:]
        self.slot_ids = np.concatenate([h[:, None], t[:, None], self.cid], 1)

    def tau(self, m=0):
        return C_BOUND * (self.tabs.d + self.K + 2 + np.asarray(m)) * U24

    def kinks(self):
        """Per triple (positives, then negatives): within its bound of the hinge or of an L1 residual component."""
        n, K, q = self.n, self.K, self.q
        bad = np.zeros(n * (1 + K), dtype=bool)
        if self.tabs.l1:
            bad |= (np.abs(q["e"]) <= self.tau() * q["a"]).any(-1)
        if self.loss == "margin":
            hv = self.param + np.repeat(self.sp, K) - self.sn
            near = np.abs(hv) <= self.tau() * (np.repeat(self.tp, K) + self.tn + abs(self.param))
            bad[:n] |= near.reshape(n, K).any(-1)
            bad[n:] |= near
        return bad

    def kink_groups(self):
        bad = self.kinks()
        return bad[:self.n] | bad[self.n:].reshape(self.n, self.K).any(-1)

    def backward(self, up=1.0, wb=None, reg=False):
        n, K, tabs = self.n, self.K, self.tabs
        nb = (n + self.bp - 1) // self.bp
        wb = up * (np.ones(nb) if wb is None else np.asarray(wb, dtype=np.float64))
        lo, tlo, self.cnts, gp, gn, tgp, tgn = _upstream(self.sp, self.sn, self.tp, self.tn, K, self.loss, self.param,
                                                         self.bp, wb)
        q = tabs.terms(self.TH, self.TT, self.TR, np.concatenate([gp, gn]), np.concatenate([tgp, tgn]))
        self.xq = q
        d = tabs.d
        hd = self.head
        slot, twin = {}, {}
        gx, gxa = q["gx"], q["gxa"]
        ngx, ngxa = gx[n:].reshape(n, K, d), gxa[n:].reshape(n, K, d)
        tl = (~hd)[:, :, None]
        slot_e = np.zeros((n, 2 + K, d))
        twin_e = np.zeros((n, 2 + K, d))
        slot_e[:, 0] = gx[:n] + (ngx * tl).sum(1)            # the head row: the positive, and negatives with a new tail
        twin_e[:, 0] = gxa[:n] + (ngxa * tl).sum(1)
        slot_e[:, 1] = -gx[:n] - (ngx * ~tl).sum(1)
        twin_e[:, 1] = gxa[:n] + (ngxa * ~tl).sum(1)
        slot_e[:, 2:] = np.where(~tl, ngx, -ngx)
        twin_e[:, 2:] = ngxa
        slot["ent"], twin["ent"] = slot_e, twin_e
        s1 = lambda v: v[:n] + v[n:].reshape(n, K, -1).sum(1)     # noqa: E731
        slot["rel"], twin["rel"] = s1(q["eps"]), s1(q["epsa"])
        if tabs.model == TRANSH:
            slot["norm"], twin["norm"] = s1(q["gw"]), s1(q["gwa"])
        if tabs.model == TRANSR:
            self.proj = _scatter(tabs.R, self.TR, q["gM"])
            self.proj_twin = _scatter(tabs.R, self.TR, q["gMa"])
            self.proj_m = np.bincount(self.TR, minlength=tabs.R)[:, None]
        if reg:      # normLoss over cat[h, t, nh, nt] and cat[r, nr] per batch (+ orthogonalLoss for TransH)
            W = tabs.W
            gb = wb[np.arange(n) // self.bp][:, None]
            mult = np.concatenate([1 + (~hd).sum(1, keepdims=True), 1 + hd.sum(1, keepdims=True),
                                   np.ones((n, K), dtype=np.int64)], 1)
            x = W["ent"][self.slot_ids]
            on = (x ** 2).sum(-1) > 1
            slot["ent"] = slot["ent"] + (gb * mult)[:, :, None] * 2 * x * on[:, :, None]
            twin["ent"] = twin["ent"] + (np.abs(gb) * mult)[:, :, None] * 2 * np.abs(x)
            rr = W["rel"][self.r]
            rv = O.norm_loss_grads(rr)
            slot["rel"] = slot["rel"] + gb * (1 + K) * rv
            twin["rel"] = twin["rel"] + np.abs(gb) * (1 + K) * 2 * np.abs(rr)
            per = (mult[:, :, None] * np.maximum((x ** 2).sum(-1, keepdims=True) - 1, 0)).sum((1, 2)) + \
                (1 + K) * np.maximum((rr ** 2).sum(-1) - 1, 0)
            tper = (mult[:, :, None] * (x ** 2).sum(-1, keepdims=True)).sum((1, 2)) + (1 + K) * (rr ** 2).sum(-1)
            if tabs.model == TRANSH:
                w = W["norm"][self.r]
                go, gw = O.orthogonal_loss_grads(rr, w)
                qa = (np.abs(w) * np.abs(rr)).sum(1, keepdims=True) / (rr ** 2).sum(1, keepdims=True)
                slot["rel"] = slot["rel"] + gb * (1 + K) * go
                twin["rel"] = twin["rel"] + np.abs(gb) * (1 + K) * (2 * qa * np.abs(w) + 2 * qa * qa * np.abs(rr))
                slot["norm"] = slot["norm"] + gb * (1 + K) * gw
                twin["norm"] = twin["norm"] + np.abs(gb) * (1 + K) * 2 * qa * np.abs(rr)
                per = per + (1 + K) * ((w * rr).sum(1) ** 2 / (rr ** 2).sum(1))
                tper = tper + (1 + K) * qa[:, 0] * (np.abs(w) * np.abs(rr)).sum(1)
            for b in range(nb):
                lo[b] += per[b * self.bp:(b + 1) * self.bp].sum()
                tlo[b] += tper[b * self.bp:(b + 1) * self.bp].sum()
        self.loss_ref, self.loss_twin = lo, tlo
        self.slot, self.twin = slot, twin
        return self

    def dense(self, name):
        """(gradient table, twin, contributions per row) under dense accumulation."""
        rows = self.tabs.E if name == "ent" else self.tabs.R
        ids = self.slot_ids.ravel() if name == "ent" else self.r
        d = self.tabs.d
        v, tw = self.slot[name].reshape(-1, d), self.twin[name].reshape(-1, d)
        return _scatter(rows, ids, v), _scatter(rows, ids, tw), np.bincount(ids, minlength=rows)[:, None]


def _check(got, ref, twin, tau, tag):
    got = np.asarray(got, dtype=np.float64)
    B = np.asarray(tau) * np.asarray(twin)
    err = np.abs(got - ref)
    bad = ~(err <= B)                    # NaN fails
    assert not bad.any(), "%s: %d of %d elements over the bound, first %s: kernel %r ref %r bound %r" % (
        tag, bad.sum(), bad.size, np.argwhere(bad)[0], got[bad][0], np.asarray(ref)[bad][0], B[bad][0])


def _draw(tabs, rng, n_pos, K, loss="margin", param=1.0, bp=None, reuse=True, max_frac=0.03, redraws=None):
    """(h, t, r, corrupt, Groups): ids 0 and n - 1 present; with reuse=False no entity appears twice; groups near a
    kink are redrawn."""
    E, R = tabs.E, tabs.R
    if reuse:
        h, t = rng.randint(0, E, n_pos), rng.randint(0, E, n_pos)
        ce = rng.randint(0, E, n_pos * K)
    else:
        assert E >= n_pos * (2 + K) + 8
        p = rng.permutation(E)[:n_pos * (2 + K)]
        h, t, ce = p[:n_pos], p[n_pos:2 * n_pos], p[2 * n_pos:]
    for ids, hi in ((h, E), (ce, E)):
        for e in (0, hi - 1):
            if not (np.concatenate([h, t, ce]) == e).any():
                ids[rng.randint(0, len(ids))] = e
    r = rng.randint(0, R, n_pos)
    r[rng.randint(0, n_pos)], r[rng.randint(0, n_pos)] = 0, R - 1
    head = rng.rand(n_pos * K) < 0.45
    c = np.where(head, ~ce, ce).astype(np.int32)
    first = None
    for _ in range(30):
        G = Groups(tabs, h, t, r, c, K, loss, param, bp)
        tri = G.kinks()
        bad = G.kink_groups()
        if first is None:       # the triples of the first draw that have to be redrawn
            first = int(tri.sum())
            assert first <= max(max_frac * len(tri), 3), "%d of %d triples near a kink" % (first, len(tri))
            if redraws is not None:
                redraws.append((first, len(tri)))
        if not bad.any():
            return h, t, r, c, G
        j = np.nonzero(bad)[0]
        if reuse:
            t[j] = rng.randint(0, E, len(j))
            ce2 = rng.randint(0, E, (len(j), K))
        else:
            free = np.setdiff1d(np.arange(E), np.concatenate([h, t, np.where(c < 0, ~c, c)]))
            new = rng.permutation(free)[:len(j) * (1 + K)]
            t[j] = new[:len(j)]
            ce2 = new[len(j):].reshape(len(j), K)
        cc = c.reshape(n_pos, K)
        cc[j] = np.where(cc[j] < 0, ~ce2, ce2)
    raise AssertionError("kinks left after 30 redraws")


# ---- GPU helpers ------------------------------------------------------------------------------------------------------
def _kernels(fn, seen):
    """fn() under a CUDA profile; the kernel names are appended to seen (a short capture can lose records, so a test
    asserts on the union of its profiles)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    seen.append(" ".join(e.key for e in prof.key_averages()))
    return out


def _again(fn, seen, names):
    """Profile fn() again (its results were checked already) while the last capture lacks one of names: now and then
    a capture loses its kernel records."""
    for _ in range(4):
        if all(nm in seen[-1] for nm in names):
            return
        _kernels(fn, seen)


def _want(seen, names):
    got = " ".join(seen)
    for nm in names:
        assert nm in got, (nm, sorted({k for k in got.split() if k.startswith("k")})[:40])


def _sms():
    from kgrec_b200 import _lib
    return _lib.load().kgrec_sm_count()


def _dev(x, ib):
    return torch.as_tensor(np.asarray(x), dtype=torch.int64 if ib == 8 else torch.int32, device="cuda")


class Call:
    """Device buffers of one corrupt-format call: ids, outputs, gradient tables (dense: zeros of the table's rows x d;
    slots: NaN, so a slot left unwritten fails its check)."""

    def __init__(self, tabs, G, ib, dense):
        from kgrec_b200 import _lib
        self.lib, self._lib = _lib.load(), _lib
        n, K, d = G.n, G.K, tabs.d
        self.tabs, self.G, self.ib, self.dense = tabs, G, ib, dense
        self.ids = [_dev(x, ib) for x in (G.h, G.t, G.r)]
        self.c = torch.as_tensor(G.c, dtype=torch.int32, device="cuda")
        self.ps = torch.empty(n, device="cuda")
        self.ns = torch.empty(n * K, device="cuda")
        self.lo = torch.empty((n + G.bp - 1) // G.bp, device="cuda")
        self.ws = torch.empty(self.lib.kgrec_corrupt_loss_step_workspace_bytes(C.byref(tabs.T), tabs.model, n) // 4,
                              device="cuda")
        self.g = {}
        for nm in Tabs.NAMES[tabs.model]:
            if nm == "proj":
                self.g[nm] = torch.zeros(tabs.R, d * d, device="cuda")
            elif dense:
                self.g[nm] = torch.zeros(tabs.E if nm == "ent" else tabs.R, d, device="cuda")
            else:
                self.g[nm] = torch.full((n * (2 + K) if nm == "ent" else n, d), float("nan"), device="cuda")
        self.sid = None if dense else (torch.full((n * (2 + K),), -7, dtype=torch.int64, device="cuda"),
                                       torch.full((n,), -7, dtype=torch.int64, device="cuda"))
        self.G_ = self._lib.Grads(mode=1 if dense else 0, **{k: v.data_ptr() for k, v in self.g.items()})

    def _p(self, x):
        return C.c_void_p(x.data_ptr()) if x is not None else None

    def _common(self):
        G = self.G
        return (C.byref(self.tabs.T), self.tabs.model, *[self._p(x) for x in self.ids], self.ib, G.n, self._p(self.c),
                G.K, G.bp, 1 if G.loss == "bpr" else 0, G.param)

    def step(self, up=1.0, reg=False):
        sid = self.sid or (None, None)
        rc = self.lib.kgrec_corrupt_loss_step(*self._common(), up, int(reg), self._p(self.ps), self._p(self.ns),
                                              self._p(self.lo), C.byref(self.G_), self._p(sid[0]), self._p(sid[1]),
                                              self._p(self.ws), None, None)
        assert rc == 0, self.lib.kgrec_last_error().decode()
        torch.cuda.synchronize()

    def fwd(self):
        rc = self.lib.kgrec_corrupt_loss_fwd(*self._common(), self._p(self.ps), self._p(self.ns), self._p(self.lo),
                                             self._p(self.ws), None, None)
        assert rc == 0, self.lib.kgrec_last_error().decode()
        torch.cuda.synchronize()

    def bwd(self, up, wb):
        sid = self.sid or (None, None)
        self.wb = torch.as_tensor(np.asarray(wb, dtype=np.float32), device="cuda")
        rc = self.lib.kgrec_corrupt_loss_bwd(*self._common(), self._p(self.ps), self._p(self.ns), up, self._p(self.wb),
                                             C.byref(self.G_), self._p(sid[0]), self._p(sid[1]), None)
        assert rc == 0, self.lib.kgrec_last_error().decode()
        torch.cuda.synchronize()

    def check(self, tag, grads=True, outputs=True):
        G, K, d = self.G, self.G.K, self.tabs.d
        if outputs:
            _check(self.ps.cpu().numpy(), G.sp, G.tp, G.tau(), tag + " pos scores")
            _check(self.ns.cpu().numpy(), G.sn, G.tn, G.tau(), tag + " neg scores")
            _check(self.lo.cpu().numpy(), G.loss_ref, G.loss_twin, G.tau(G.cnts), tag + " loss")
        if not grads:
            return
        for nm, buf in self.g.items():
            got = buf.double().cpu().numpy()
            if nm == "proj":
                _check(got, G.proj, G.proj_twin, G.tau(G.proj_m), tag + " grad proj")
            elif self.dense:
                ref, tw, m = G.dense(nm)
                _check(got, ref, tw, G.tau(m), tag + " dense grad " + nm)
            else:
                _check(got, G.slot[nm].reshape(-1, d), G.twin[nm].reshape(-1, d), G.tau(), tag + " slot grad " + nm)
        if not self.dense:
            assert np.array_equal(self.sid[0].cpu().numpy(), G.slot_ids.ravel()), tag + " slot ent ids"
            assert np.array_equal(self.sid[1].cpu().numpy(), G.r), tag + " slot rel ids"


def _step_case(model, d, K, n_pos, seed, seen, redraws=None, l1=False, loss="margin", bp=None, dense=True, ib=4,
               reg=False, reuse=True, E=None, R=7, ld=None, up=1.0):
    param = 1.0 if loss == "margin" else -1.0
    E = E or (2 * n_pos * (2 + K) + 17 if not reuse else max(8, n_pos // 4))
    tabs = Tabs(model, d, E, R, seed, l1=l1, ld=ld)
    rng = np.random.RandomState(seed + 1)
    _, _, _, _, G = _draw(tabs, rng, n_pos, K, loss, param, bp, reuse, redraws=redraws)
    call = Call(tabs, G, ib, dense)
    _kernels(lambda: call.step(up, reg), seen)
    G.backward(up=up, reg=reg)
    tag = "model %d d=%d K=%d n=%d l1=%d %s bp=%s dense=%d ib=%d reg=%d ld=%s" % (model, d, K, n_pos, l1, loss, bp, dense,
                                                                               ib, reg, ld)
    call.check(tag)
    names = dispatch(model, d, K, n_pos, STEP, dense, reg, (ld or d) == d, _sms(), l1, loss == "margin", R)
    _again(lambda: call.step(up, reg), seen, names)
    return names


# ---- register step kernels ----------------------------------------------------------------------------------------
KS = (1, 2, 15, 16, 31, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [TRANSE, TRANSH])
def test_register_step(model):
    """k_group_step_e / _h in STEP mode at every d % 4 == 0 in 4..128 (L2) and d in {4, 20, 64, 100, 128} (L1); K, the
    loss, dense / sparse, int32 / int64, batch_pos, the fused regulariser and row reuse vary with d so that each
    takes all its values several times."""
    seen, want, redraws = [], set(), []
    cases = [(d, False) for d in range(4, 129, 4)] + [(d, True) for d in (4, 20, 64, 100, 128)]
    for i, (d, l1) in enumerate(cases):
        K = KS[i % 6]
        loss = "margin" if i % 2 == 0 else "bpr"
        n_pos = 61
        bp = 1 if i % 5 == 0 else 23                # 23 does not divide 61: a ragged last batch
        reg = loss == "margin" and i % 4 == 0
        reuse = i % 3 != 2
        want.update(_step_case(model, d, K, n_pos, 100 * model + i, seen, redraws, l1=l1, loss=loss, bp=bp,
                               dense=(i // 2) % 2 == 0, ib=8 if (i // 3) % 2 else 4, reg=reg, reuse=reuse))
    _want(seen, want)
    print("triples redrawn: %d of %d" % (sum(a for a, _ in redraws), sum(b for _, b in redraws)))


# ---- FWD / BWD through the module and autograd --------------------------------------------------------------------------
def _module(tabs):
    import kgrec_b200 as K
    cls = {TRANSE: K.TransEModel, TRANSH: K.TransHModel}[tabs.model]
    m = cls(tabs.l1, tabs.d, tabs.E, tabs.R)
    with torch.no_grad():
        for nm in Tabs.NAMES[tabs.model]:
            getattr(m, nm + "_embeddings").weight.copy_(torch.as_tensor(tabs.W[nm], dtype=torch.float32))
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("model", [TRANSE, TRANSH])
@pytest.mark.parametrize("d,K", [(100, 10), (32, 32), (64, 40), (200, 5), (512, 3)])
def test_fwd_bwd_modes(model, d, K):
    """rank_loss_corrupt (kgrec_corrupt_loss_fwd) and (loss * w).sum().backward() (kgrec_corrupt_loss_bwd) with a
    different weight per batch, so that the upstream up_dev[j / batch_pos] is read per group; on the register kernels
    (d <= 128, K <= 32) and the general kernel; BPR with a ragged last batch; dense and sparse gradients."""
    seen, want = [], set()
    for j, (loss, gm) in enumerate((("margin", "dense"), ("bpr", "sparse"), ("bpr", "dense"), ("margin", "sparse"))):
        n_pos, bp = 150, 32
        param = 1.0 if loss == "margin" else -1.0
        tabs = Tabs(model, d, 60, 5, seed=d + K + j, l1=(j == 3))
        rng = np.random.RandomState(d * K + j)
        h, t, r, c, G = _draw(tabs, rng, n_pos, K, loss, param, bp)
        m = _module(tabs)
        m.grad_mode = gm
        m.zero_grad()
        wb = np.round(rng.uniform(-2, 2, (n_pos + bp - 1) // bp), 3)
        pos = tuple(_dev(x, 8) for x in (h, t, r))
        cd = torch.as_tensor(c, device="cuda")

        def run():
            lo, ps, ns = m.rank_loss_corrupt(pos, cd, margin=param, loss=loss, batch_pos=bp)
            (lo * torch.as_tensor(wb, dtype=torch.float32, device="cuda")).sum().backward()
            return lo, ps, ns
        lo, ps, ns = _kernels(run, seen)
        G.backward(wb=wb.astype(np.float32).astype(np.float64))
        tag = "model %d d=%d K=%d %s %s" % (model, d, K, loss, gm)
        _check(ps.detach().cpu().numpy(), G.sp, G.tp, G.tau(), tag + " pos")
        _check(ns.detach().cpu().numpy(), G.sn, G.tn, G.tau(), tag + " neg")
        _check(lo.detach().cpu().numpy(), G.loss_ref, G.loss_twin, G.tau(G.cnts), tag + " loss")
        for nm in Tabs.NAMES[model]:
            g = getattr(m, nm + "_embeddings").weight.grad
            if gm == "sparse" and g.is_coalesced():
                ref, tw, mm = G.dense(nm)
                _check(g.to_dense().double().cpu().numpy(), ref, tw, G.tau(mm), tag + " coalesced " + nm)
            elif gm == "sparse":
                ids = g._indices().view(-1).cpu().numpy()
                assert np.array_equal(ids, G.slot_ids.ravel() if nm == "ent" else G.r), tag + " COO ids " + nm
                _check(g._values().double().cpu().numpy(), G.slot[nm].reshape(-1, d), G.twin[nm].reshape(-1, d),
                       G.tau(), tag + " slots " + nm)
            else:
                ref, tw, mm = G.dense(nm)
                _check(g.double().cpu().numpy(), ref, tw, G.tau(mm), tag + " dense " + nm)
        names = [nm for mode in (FWD, BWD)
                 for nm in dispatch(model, d, K, n_pos, mode, gm == "dense", False, True, _sms(), j == 3, loss == "margin")]
        _again(run, seen, names)
        want.update(names)
    _want(seen, want)


# ---- the general kernel ---------------------------------------------------------------------------------------------
GENERAL = [(132, 3), (200, 10), (252, 1), (256, 5), (260, 2), (384, 1), (508, 4), (512, 1), (512, 10),
           (64, 33), (100, 40), (128, 64), (4, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("model", [TRANSE, TRANSH])
@pytest.mark.parametrize("d,K", GENERAL)
def test_general_kernel(model, d, K):
    """k_group_step<FAM, NCH> (+ k_group_slot_ids) in STEP, then FWD and BWD (with per-batch upstream weights) on the
    same groups: NCH 2 / 4 with full and partial last chunks, and K > 32 at d <= 128."""
    seen = []
    n_pos, bp = 45, 13
    i = d + K
    l1 = i % 3 == 0 and d <= 200 and K <= 32      # wider L1 groups put too many residual components near 0
    loss = "margin" if i % 2 else "bpr"
    param = 1.0 if loss == "margin" else -1.0
    want = set(_step_case(model, d, K, n_pos, i, seen, l1=l1, loss=loss, bp=bp, dense=i % 4 < 2, ib=4 + 4 * (i % 2)))
    tabs = Tabs(model, d, 40, 6, seed=i + 5, l1=l1)
    rng = np.random.RandomState(i)
    _, _, _, _, G = _draw(tabs, rng, n_pos, K, loss, param, bp)
    for dense in (True, False):
        call = Call(tabs, G, 8, dense)
        _kernels(call.fwd, seen)
        wb = np.round(rng.uniform(0.25, 2, (n_pos + bp - 1) // bp), 3)
        _kernels(lambda: call.bwd(0.5, wb), seen)
        G.backward(up=0.5, wb=wb.astype(np.float32))
        call.check("model %d d=%d K=%d fwd/bwd dense=%d" % (model, d, K, dense))
        for mode, fn in ((FWD, call.fwd), (BWD, lambda: call.bwd(0.5, wb))):
            names = dispatch(model, d, K, n_pos, mode, dense, False, True, _sms(), l1, loss == "margin")
            _again(fn, seen, names)
            want.update(names)
    _want(seen, want)


# ---- the TMA kernel -------------------------------------------------------------------------------------------------
TMA = [(96, 15, False, "margin"), (92, 16, True, "bpr"), (52, 29, False, "bpr"), (128, 10, True, "margin"),
       (128, 11, False, "margin"), (100, 14, False, "bpr"), (100, 15, True, "margin")]


@pytest.mark.gpu
@pytest.mark.parametrize("d,K,l1,loss", TMA)
def test_tma_kernel(d, K, l1, loss):
    """k_group_step_e_tma against float64 directly: NS 16 / 32 (K = 15 / 16), K = 29, and both sides of the ring-fit
    edges (d = 128 fits K = 10, not 11; d = 100 fits 14, not 15: those run the register kernel); n_pos at the
    smallest TMA launch (2 groups per warp of every SM) and one fewer (the register kernel)."""
    seen, want = [], set()
    n_min = TMA_STAGES * TMA_WARPS * _sms()
    for j, n_pos in enumerate((n_min, n_min - 1)):
        want.update(_step_case(TRANSE, d, K, n_pos, d * K + j, seen, l1=l1, loss=loss, bp=1000, dense=False,
                               ib=4 + 4 * j, E=3000))
    _want(seen, want)
    if tma_smem(d, K) <= 225 * 1024:
        assert any("k_group_step_e_tma" in w for w in want)


# ---- TransR ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 3, 14])
def test_transr_run_kernel(K):
    """k_run_step_r at every d % 4 == 0 in 32..128 (each QA / QB / QF / RB tile, d % 32 remainders), reg, margin and
    BPR, dense and sparse."""
    seen, want = [], set()
    for i, d in enumerate(range(32, 129, 4)):
        loss = "bpr" if i % 3 == 1 else "margin"
        want.update(_step_case(TRANSR, d, K, 40, 1000 * K + d, seen, l1=(i % 4 == 3 and d <= 64), loss=loss, bp=17,
                               dense=(i % 2 == 0), ib=4 + 4 * (i % 2), reg=(loss == "margin" and i % 3 == 0), R=5,
                               E=50))
    _want(seen, want)
    assert all("k_run_step_r" in w for w in want)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 3, 10, 11, 14])
def test_transr_warp_kernel(K):
    """k_group_step_r at its nvt edges (K <= 2: 4, <= 10: 12, else 16), d in {4, 20, 28, 32, 64, 128}; d < 32 always
    takes it, wider rows when n_pos < 4 n_rel."""
    seen, want = [], set()
    for i, d in enumerate((4, 20, 28, 32, 64, 128)):
        loss = "bpr" if (i + K) % 3 == 1 else "margin"
        n_pos, R = 37, 13
        want.update(_step_case(TRANSR, d, K, n_pos, 77 * K + d, seen, l1=(i % 3 == 2 and d <= 64), loss=loss, bp=11,
                               dense=(i + K) % 2 == 0, ib=4 + 4 * (i % 2), reg=(loss == "margin" and i % 2 == 0), R=R,
                               E=60))
    _want(seen, want)
    assert all("k_group_step_r" in w for w in want)


@pytest.mark.gpu
@pytest.mark.parametrize("n_rel", [1, 1023, 1024, 1025, 2500])
def test_transr_relation_counts(n_rel):
    """The run / warp boundary at n_pos = 4 n_rel - 1 and 4 n_rel, for n_rel around k_rel_scan's 1024 threads (its
    per > 1 branch from 1025), with relations that have no positive."""
    seen, want = [], set()
    d = 32
    for j, n_pos in enumerate((4 * n_rel - 1, 4 * n_rel)):
        tabs = Tabs(TRANSR, d, 300, n_rel, seed=n_rel + j)
        rng = np.random.RandomState(n_rel + j)
        K = 2 + j
        _, _, r, _, G = _draw(tabs, rng, n_pos, K, "margin", 1.0, 512)
        used = np.zeros(n_rel, bool)
        used[G.r] = True
        assert n_rel == 1 or not used.all()         # relations with no positive (the draw's n_pos is ~4 n_rel)
        call = Call(tabs, G, 4 + 4 * j, dense=(j == 0))
        _kernels(lambda: call.step(1.0, j == 1), seen)
        G.backward(reg=(j == 1))
        call.check("TransR n_rel=%d n_pos=%d" % (n_rel, n_pos))
        names = dispatch(TRANSR, d, K, n_pos, STEP, j == 0, j == 1, True, _sms(), False, True, n_rel) + ["k_rel_scan"]
        _again(lambda: call.step(1.0, j == 1), seen, names)
        want.update(names)
    _want(seen, want)
    assert "k_rel_scan" in " ".join(seen)


# ---- expanded-triple kernels ----------------------------------------------------------------------------------------
def _expanded_case(model, d, ld, off, seed, seen, want):
    """kgrec_score_fwd + kgrec_score_bwd with a random upstream (sparse slots), kgrec_rank_loss_fwd + _bwd with per
    batch weights (dense), kgrec_rank_loss_step (sparse)."""
    from kgrec_b200 import _lib
    lib = _lib.load()
    l1 = seed % 3 == 0 and d <= (64 if model == TRANSR else 200)
    tabs = Tabs(model, d, 40, 4, seed, l1=l1, ld=ld, off=off)
    rng = np.random.RandomState(seed)
    n_pos, K, bp = (24, 3, 10) if model != TRANSR or d <= 256 else (8, 3, 5)   # the float64 d x d matrices per triple
    loss = "margin" if seed % 2 else "bpr"
    param = 1.0 if loss == "margin" else -1.0
    _, _, _, _, G = _draw(tabs, rng, n_pos, K, loss, param, bp)
    tag = "expanded model %d d=%d ld=%d off=%d" % (model, d, tabs.ld, off)
    n = n_pos * (1 + K)
    TH, TT, TR = G.TH, G.TT, G.TR
    p = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None      # noqa: E731
    ib = 4 + 4 * (seed % 2)
    a, b, c = (_dev(x, ib) for x in (TH, TT, TR))
    pa, pb, pc = (_dev(x[:n_pos], ib) for x in (TH, TT, TR))
    na, nb, nc = (_dev(x[n_pos:], ib) for x in (TH, TT, TR))

    def grads(dense, nn):
        g = {}
        for nm in Tabs.NAMES[model]:
            if nm == "proj":
                g[nm] = torch.zeros(tabs.R, d * d, device="cuda")
            elif dense:
                g[nm] = torch.zeros(tabs.E if nm == "ent" else tabs.R, d, device="cuda")
            else:
                g[nm] = torch.full((2 * nn if nm == "ent" else nn, d), float("nan"), device="cuda")
        return g, _lib.Grads(mode=1 if dense else 0, **{k: v.data_ptr() for k, v in g.items()})

    def expect(g, tg, dense, got, what):
        q = tabs.terms(TH, TT, TR, g, tg)
        m_e = np.bincount(np.concatenate([TH, TT]), minlength=tabs.E)[:, None]
        m_r = np.bincount(TR, minlength=tabs.R)[:, None]
        ref = {"ent": (np.concatenate([q["gx"], -q["gx"]]), np.concatenate([q["gxa"], q["gxa"]]),
                       np.concatenate([TH, TT]), tabs.E, m_e),
               "rel": (q["eps"], q["epsa"], TR, tabs.R, m_r)}
        if model == TRANSH:
            ref["norm"] = (q["gw"], q["gwa"], TR, tabs.R, m_r)
        tau = lambda m: C_BOUND * (d + K + 2 + m) * U24      # noqa: E731
        for nm, (v, tw, ids, rows, m) in ref.items():
            if dense:
                _check(got[nm].double().cpu().numpy(), _scatter(rows, ids, v), _scatter(rows, ids, tw), tau(m),
                       tag + " " + what + " dense " + nm)
            else:
                _check(got[nm].double().cpu().numpy(), v, tw, tau(0), tag + " " + what + " slots " + nm)
        if model == TRANSR:
            _check(got["proj"].double().cpu().numpy(), _scatter(tabs.R, TR, q["gM"]), _scatter(tabs.R, TR, q["gMa"]),
                   tau(m_r), tag + " " + what + " proj")

    # flat scores, and their backward with a random upstream into slots
    s = torch.empty(n, device="cuda")
    _kernels(lambda: _lib.check(lib.kgrec_score_fwd(C.byref(tabs.T), model, p(a), p(b), p(c), ib, n, None, 0, p(s),
                                                    None, None)), seen)
    torch.cuda.synchronize()
    _check(s.cpu().numpy(), np.concatenate([G.sp, G.sn]), np.concatenate([G.tp, G.tn]), G.tau(), tag + " score_fwd")
    up = np.round(rng.randn(n) / 4, 4).astype(np.float32).astype(np.float64)
    upd = torch.as_tensor(up, dtype=torch.float32, device="cuda")
    gt, Gs = grads(False, n)
    _kernels(lambda: _lib.check(lib.kgrec_score_bwd(C.byref(tabs.T), model, p(a), p(b), p(c), ib, n, None, 0, p(upd),
                                                    C.byref(Gs), None)), seen)
    torch.cuda.synchronize()
    expect(up, np.abs(up), False, gt, "score_bwd")
    # the fused ranking loss, and its backward with a weight per batch into dense tables
    ps, ns = torch.empty(n_pos, device="cuda"), torch.empty(n_pos * K, device="cuda")
    nbat = (n_pos + bp - 1) // bp
    lo, ws = torch.empty(nbat, device="cuda"), torch.empty(n_pos, device="cuda")
    lk = 1 if loss == "bpr" else 0
    _kernels(lambda: _lib.check(lib.kgrec_rank_loss_fwd(C.byref(tabs.T), model, p(pa), p(pb), p(pc), p(na), p(nb), p(nc),
                                                        ib, n_pos, K, bp, lk, param, None, 0, p(ps), p(ns), p(lo), p(ws),
                                                        None, None)), seen)
    torch.cuda.synchronize()
    wb = np.round(rng.uniform(-1.5, 1.5, nbat), 3).astype(np.float32).astype(np.float64)
    G.backward(wb=wb)
    _check(ps.cpu().numpy(), G.sp, G.tp, G.tau(), tag + " rank_loss pos")
    _check(ns.cpu().numpy(), G.sn, G.tn, G.tau(), tag + " rank_loss neg")
    _check(lo.cpu().numpy(), G.loss_ref, G.loss_twin, G.tau(G.cnts), tag + " rank_loss loss")
    wbd = torch.as_tensor(wb, dtype=torch.float32, device="cuda")
    gd, Gd = grads(True, n)
    _kernels(lambda: _lib.check(lib.kgrec_rank_loss_bwd(C.byref(tabs.T), model, p(pa), p(pb), p(pc), p(na), p(nb), p(nc),
                                                        ib, n_pos, K, bp, lk, param, None, 0, p(ps), p(ns), 1.0, p(wbd),
                                                        C.byref(Gd), None)), seen)
    torch.cuda.synchronize()
    _, _, _, gp, gn, tgp, tgn = _upstream(G.sp, G.sn, G.tp, G.tn, K, loss, param, bp, wb)
    expect(np.concatenate([gp, gn]), np.concatenate([tgp, tgn]), True, gd, "rank_loss_bwd")
    # the single call: forward + backward with grad_loss 0.75 into slots
    gs2, Gs2 = grads(False, n)
    ps2, ns2, lo2 = torch.empty_like(ps), torch.empty_like(ns), torch.empty_like(lo)
    _kernels(lambda: _lib.check(lib.kgrec_rank_loss_step(C.byref(tabs.T), model, p(pa), p(pb), p(pc), p(na), p(nb),
                                                         p(nc), ib, n_pos, K, bp, lk, param, 0.75, None, 0, p(ps2),
                                                         p(ns2), p(lo2), C.byref(Gs2), None, None, None, p(ws), None,
                                                         None)), seen)
    torch.cuda.synchronize()
    _check(ps2.cpu().numpy(), G.sp, G.tp, G.tau(), tag + " rank_loss_step pos")
    _check(lo2.cpu().numpy(), G.loss_ref, G.loss_twin, G.tau(G.cnts), tag + " rank_loss_step loss")
    _, _, _, gp, gn, tgp, tgn = _upstream(G.sp, G.sn, G.tp, G.tn, K, loss, param, bp, np.full(nbat, 0.75))
    expect(np.concatenate([gp, gn]), np.concatenate([tgp, tgn]), False, gs2, "rank_loss_step")
    nch, vec = expanded_build(d, tabs.ld, off == 0)
    want.update(["k_score_fwd<%d, %d, %s>" % (model, nch, _b(vec)), "k_score_bwd<%d, %d, %s, 1>" % (model, nch, _b(vec)),
                 "k_rank_loss_fwd<%d, %d, %s>" % (model, nch, _b(vec))])


EXPANDED_D = (1, 3, 4, 50, 100, 127, 128, 129, 130, 132, 200, 255, 256, 257, 300, 511, 512)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [TRANSE, TRANSH, TRANSR])
def test_expanded_kernels(model):
    """k_score_fwd / k_rank_loss_fwd / k_score_bwd<FAM, NCH, VEC> at 17 widths across NCH 1 / 2 / 4, with VEC false
    reached three ways: d % 4 != 0, a table base one float off 16 bytes, and ld = d + 1."""
    seen, want = [], set()
    for i, d in enumerate(EXPANDED_D):
        if model == TRANSR and d > 256 and i % 2:
            continue                                 # the d x d matrices make the float64 side slow; 300 and 512 stay
        _expanded_case(model, d, d, 0, 10 * d + model, seen, want)
    for d in (100, 128, 256, 512):
        _expanded_case(model, d, d, 1, 3 * d + model, seen, want)
        _expanded_case(model, d, d + 1, 0, 5 * d + model, seen, want)
    _want(seen, want)
    assert any("false>" in w for w in want)


# ---- strided tables -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("model", [TRANSE, TRANSH, TRANSR])
def test_strided_step_tables(model):
    """ld = d + 4 for the step families (register, general and both TransR kernels), the padding columns NaN: no
    gradient or score may read them.  ld != dim keeps TransE off the TMA kernel even where it would fit."""
    seen, want = [], set()
    shapes = [(100, 10, 60), (128, 3, 200), (36, 2, 400)] if model == TRANSR else [(100, 10, 60), (256, 5, 50),
                                                                                    (4, 32, 40)]
    for i, (d, K, n_pos) in enumerate(shapes):
        want.update(_step_case(model, d, K, n_pos, 9 * d + K, seen, l1=(i == 2), loss="margin" if i != 1 else "bpr",
                               bp=16, dense=(i % 2 == 0), ib=4 + 4 * (i % 2), reg=(i == 0), R=3, ld=d + 4, E=90))
    if model == TRANSE:
        n_pos = TMA_STAGES * TMA_WARPS * _sms()
        names = _step_case(TRANSE, 100, 10, n_pos, 3, seen, dense=False, ld=104, E=3000, bp=1024)
        assert names and "tma" not in names[0]
        want.update(names)
        assert "k_group_step_e_tma" not in " ".join(seen)
    _want(seen, want)


@pytest.mark.gpu
@pytest.mark.parametrize("model", [TRANSE, TRANSH, TRANSR])
def test_strided_expanded_tables(model):
    """ld = d + 4 (the 128-bit rows) and ld = d + 1 (the scalar rows) for the expanded-triple kernels."""
    seen, want = [], set()
    for d in (4, 64, 200, 300):
        _expanded_case(model, d, d + 4, 0, 7 * d + model, seen, want)
        _expanded_case(model, d, d + 1, 0, 11 * d + model, seen, want)
    _want(seen, want)


# ---- slot offsets near the 32-bit limit ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_slot_offsets_near_32_bits():
    """Sparse TransE at d = 128, K = 10: n_pos (2 + K) d 4 just under 4e9 bytes of slots (the register-side kernels;
    here the TMA kernel) and just over (the general kernel, 64-bit slot offsets).  Every slot id of every group, and
    the scores, losses and slot values of whole batches (the first, the last, three random ones) against float64."""
    d, K, bp = 128, 10, 1024
    n_under = int(4.0e9 // ((2 + K) * d * 4))
    if (n_under * (2 + K) * d * 4) >= 4.0e9:
        n_under -= 1
    n_over = n_under + 1
    need = n_over * ((2 + K) * d * 4 + (2 + K) * 8 * 2 + 64) + (1 << 28)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
    from kgrec_b200 import _lib
    lib = _lib.load()
    tabs = Tabs(TRANSE, d, 5000, 50, seed=4)
    rng = np.random.RandomState(4)
    seen = []
    for n_pos in (n_under, n_over):
        assert on_registers(TRANSE, d, K, n_pos) == (n_pos == n_under)
        h = torch.randint(0, tabs.E, (n_pos,), device="cuda", dtype=torch.int32)
        t = torch.randint(0, tabs.E, (n_pos,), device="cuda", dtype=torch.int32)
        r = torch.randint(0, tabs.R, (n_pos,), device="cuda", dtype=torch.int32)
        ce = torch.randint(0, tabs.E, (n_pos * K,), device="cuda", dtype=torch.int32)
        c = torch.where(torch.rand(n_pos * K, device="cuda") < 0.45, ~ce, ce)
        h[0], t[-1], ce[-1] = 0, tabs.E - 1, 0
        ps, ns = torch.empty(n_pos, device="cuda"), torch.empty(n_pos * K, device="cuda")
        nb = (n_pos + bp - 1) // bp
        lo, ws = torch.empty(nb, device="cuda"), torch.empty(n_pos, device="cuda")
        ge = torch.empty(n_pos * (2 + K), d, device="cuda")
        gr = torch.empty(n_pos, d, device="cuda")
        sid = torch.empty(n_pos * (2 + K), dtype=torch.int64, device="cuda")
        sidr = torch.empty(n_pos, dtype=torch.int64, device="cuda")
        Gr = _lib.Grads(mode=0, ent=ge.data_ptr(), rel=gr.data_ptr())
        p = lambda x: C.c_void_p(x.data_ptr())        # noqa: E731
        _kernels(lambda: _lib.check(lib.kgrec_corrupt_loss_step(
            C.byref(tabs.T), TRANSE, p(h), p(t), p(r), 4, n_pos, p(c), K, bp, 0, 1.0, 1.0, 0, p(ps), p(ns), p(lo),
            C.byref(Gr), p(sid), p(sidr), p(ws), None, None)), seen)
        want = torch.cat([h.long().view(-1, 1), t.long().view(-1, 1), torch.where(c < 0, ~c, c).long().view(-1, K)], 1)
        assert torch.equal(sid, want.view(-1)), "slot ent ids, n_pos %d" % n_pos
        assert torch.equal(sidr, r.long()), "slot rel ids, n_pos %d" % n_pos
        del want
        hc, tc, rc_, cc = (x.cpu().numpy() for x in (h, t, r, c))
        for b in sorted({0, nb - 1, *rng.randint(1, nb - 1, 3).tolist()}):
            j0, j1 = b * bp, min(n_pos, (b + 1) * bp)
            G = Groups(tabs, hc[j0:j1], tc[j0:j1], rc_[j0:j1], cc[j0 * K:j1 * K], K, "margin", 1.0, bp)
            G.backward()
            tag = "n_pos %d batch %d" % (n_pos, b)
            _check(ps[j0:j1].cpu().numpy(), G.sp, G.tp, G.tau(), tag + " pos")
            _check(ns[j0 * K:j1 * K].cpu().numpy(), G.sn, G.tn, G.tau(), tag + " neg")
            _check(lo[b:b + 1].cpu().numpy(), G.loss_ref, G.loss_twin, G.tau(G.cnts), tag + " loss")
            ok = ~G.kink_groups()                  # the ids are drawn on the device: a group on the hinge is left out
            assert ok.mean() > 0.97
            _check(ge[j0 * (2 + K):j1 * (2 + K)].double().cpu().numpy().reshape(-1, 2 + K, d)[ok], G.slot["ent"][ok],
                   G.twin["ent"][ok], G.tau(), tag + " ent slots")
            _check(gr[j0:j1].double().cpu().numpy()[ok], G.slot["rel"][ok], G.twin["rel"][ok], G.tau(),
                   tag + " rel slots")
        del ge, gr, sid, sidr, h, t, r, ce, c, ps, ns
        torch.cuda.empty_cache()
    names = " ".join(seen)
    assert "k_group_step_e_tma<false, true, 16, 16>" in names
    assert "k_group_step<0, 1, false, false, false>" in names and "k_group_slot_ids" in names
